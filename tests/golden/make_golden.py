"""Generates tests/golden/*.npz from the UNMODIFIED reference compiled into oracle/_ref (run where the reference source tree is
readable:  python tests/golden/make_golden.py).  The fixtures are committed; the tests never need the reference tree."""
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
import oracle_lib as O  # noqa: E402
from tiny_model import TinyModel  # noqa: E402


def main():
    assert O.build_ref(), "needs the reference source tree to build oracle/_ref"
    r = O.Ref(4)
    # 1) per-type kernels on the analytic input of tests/test-quantize-fns.cpp:30-34 (0.1 + 2 cos(i + off))
    N, K = 6, 1024
    i = np.arange(N * K, dtype=np.float32)
    w = (0.1 + 2.0 * np.cos(i + 0.0)).reshape(N, K).astype(np.float32) * 0.05
    x = (0.1 + 2.0 * np.cos(np.arange(K, dtype=np.float32) + 1.0)).astype(np.float32)
    out = {"w": w, "x": x}
    for t in O.GOLDEN_TYPES:
        n = O.TYPE_NAME[t]
        blocks = r.quantize(t, w)
        out[f"{n}_blocks"] = blocks
        out[f"{n}_dequant"] = r.dequantize(t, blocks, K)
        out[f"{n}_act"] = r.quantize_act(t, x)
        out[f"{n}_mulmat"] = r.mul_mat(t, blocks, N, K, x, n_threads=1)
        sb = O.synth_blocks(t, N, K, 42)
        out[f"{n}_synth_blocks"] = sb
        out[f"{n}_synth_dequant"] = r.dequantize(t, sb, K)
        out[f"{n}_synth_mulmat"] = r.mul_mat(t, sb, N, K, x, n_threads=1)
    np.savez_compressed(HERE / "kquants_golden.npz", **out)
    # 2) whole-graph decode of tiny llama / qwen2 models on the reference CPU backend
    for arch in ("llama", "qwen2"):
        tm = TinyModel(n_layer=2, n_embd=256, n_head=2, n_head_kv=1, n_ff=512, n_vocab=160, n_ctx=32, arch=arch, quantizer=r.quantize,
                       freq_factors=(arch == "llama"), seed=7)
        toks = np.array([(j * 7919 + 13) % 160 for j in range(5)], dtype=np.int32)
        logits, hidden = tm.ref_decode(r, toks)
        d = {"tokens": toks, "logits": logits, "hidden": hidden, "hp_keys": np.array(list(tm.hp.keys())),
             "hp_vals": np.array([float(v) for v in tm.hp.values()], dtype=np.float64)}
        for name, (t, a) in tm.tensors.items():
            d["T|" + name + "|" + str(t)] = a
        np.savez_compressed(HERE / f"tiny_{arch}_golden.npz", **d)
    print("golden written")


if __name__ == "__main__":
    main()
