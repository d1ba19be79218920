"""Driver for tests/test_reference_self_divergence.py: decodes a tiny model token by token on ONE build of the compiled reference
CPU backend (PB200_REF_VARIANT = v3: AVX2 / v4: AVX-512) and saves the logits.  One build per process (two ggml cores cannot share one)."""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))
import oracle_lib as O          # noqa: E402
from golden.make_reference_golden import divergence_model  # noqa: E402

arch, n_tok, out = sys.argv[1], int(sys.argv[2]), sys.argv[3]
tm, toks = divergence_model(arch)
toks = toks[:n_tok]
ref = O.Ref(4)
logits, _ = tm.ref_decode(ref, toks)
np.save(out, logits)
print(O.ref_variant())
