"""Generates tests/golden/legacy_types_golden.npz: the reference CPU ggml compiled into oracle/_ref on the legacy 32-element weight types
Q4_0, Q4_1 and Q5_0 (python tests/golden/make_legacy_types_golden.py, where the reference tree is present), so that the port and the
CUDA kernels are checked against real reference arithmetic on machines without the reference.

Per type: ggml_quantize_chunk blocks of seeded f32 weights, their dequantize_row_* rows, the q8_0 (Q4_0, Q5_0) or q8_1 (Q4_1) activation
the CPU quantizes for that type, and gref_mul_mat at T = 1 and T > 1 (K = 512 and K = 7 392 = 231 x 32, a row that is not a multiple of
256).  Per model: 40 tokens of gref_decode logits of tiny_model.legacy_golden_models() (weights regenerated from seeds):
a Qwen2 Q4_K_M with n_ff % 256 != 0 (ffn_down Q5_0 in layer 0, Q8_0 in layer 1) and a llama Q4_0 (Q6_K head, Q4_0 everywhere else)."""
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
import oracle_lib as O  # noqa: E402
from tiny_model import legacy_golden_models  # noqa: E402

MULMAT_CASES = [(16, 512, 1), (12, 7392, 3)]   # N, K, T


def mulmat_inputs(t, i, N, K, T):
    rng = np.random.default_rng(1000 * t + i)
    w = (rng.standard_normal((N, K)) * 0.05).astype(np.float32)
    x = rng.standard_normal((T, K)).astype(np.float32)
    return w, x


def main():
    assert O.build_ref(), "the reference tree is needed to record the golden file"
    r = O.Ref()
    out = {}
    for t in (O.Q4_0, O.Q4_1, O.Q5_0):
        n = O.TYPE_NAME[t]
        for i, (N, K, T) in enumerate(MULMAT_CASES):
            w, x = mulmat_inputs(t, i, N, K, T)
            blocks = r.quantize(t, w)
            out[f"{n}_{i}_blocks"] = blocks
            out[f"{n}_{i}_dequant"] = r.dequantize(t, blocks, K)
            out[f"{n}_{i}_act"] = np.stack([r.quantize_act(t, x[j]) for j in range(T)])
            out[f"{n}_{i}_mulmat"] = r.mul_mat(t, blocks, N, K, x)
    for name, (tm, toks) in legacy_golden_models().items():
        logits, hidden = tm.ref_decode(r, toks)
        out[f"{name}_tokens"] = np.asarray(toks, np.int32)
        out[f"{name}_logits"] = logits
        out[f"{name}_hidden"] = hidden
        out[f"{name}_types"] = np.array([f"{k}|{v[0]}" for k, v in tm.tensors.items()])
    np.savez_compressed(HERE / "legacy_types_golden.npz", **out)
    print(f"wrote {HERE / 'legacy_types_golden.npz'}: {len(out)} arrays")


if __name__ == "__main__":
    main()
