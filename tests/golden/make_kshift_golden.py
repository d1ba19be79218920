"""Generates tests/golden/kshift_golden.npz: GGML_OP_ROPE on f16 rows computed by the reference CPU backend (ggml_compute_forward_rope_f16,
ggml.c:14269-14380), the arithmetic of the K-shift graph build_k_shift runs on the f16 K cache (src/llama.cpp:10665-10719).  Recorded from
the reference compiled into oracle/_ref (python tests/golden/make_kshift_golden.py, where the reference tree is present), so that
pb200_rope_f16 is checked against real reference arithmetic on machines without the reference.

Cases: NORM / NEOX, n_dims < head_dim, llama-3 style freq factors, YaRN (ext_factor, freq_scale), negative positions (a shift rotates by
delta < 0) and in place (ggml_rope_ext_inplace, as build_k_shift does)."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
import oracle_lib as O  # noqa: E402

# head_dim, n_head, n_rows, n_dims, mode, n_ctx_orig, in_place, freq factors | freq_base, freq_scale, ext_factor, attn_factor, beta_fast, beta_slow
CASES = [
    ((128, 8, 12, 128, 0, 8192, 1, 1), (500000.0, 1.0, 0.0, 1.0, 32.0, 1.0)),     # Llama-3.1 K cache, in place
    ((128, 4, 10, 128, 2, 32768, 1, 0), (1000000.0, 1.0, 0.0, 1.0, 32.0, 1.0)),   # Qwen2 K cache, in place
    ((128, 2, 9, 64, 0, 4096, 0, 0), (10000.0, 0.25, 1.0, 1.0, 32.0, 1.0)),       # YaRN, n_dims < head_dim
    ((80, 3, 7, 32, 2, 2048, 1, 1), (10000.0, 0.5, 0.5, 0.9, 32.0, 1.0)),         # NEOX, partial rotation, YaRN + factors, in place
]


def positions(n, rng):
    base = np.array([-4096, -1, 0, 1, 7, -17, 4095, -2048, 100, -333, 8191, -8190], np.int32)
    return np.concatenate([base, rng.integers(-8192, 8192, max(0, n - base.size), dtype=np.int32)])[:n]


class _IP(C.Structure):
    _fields_ = [("mem_size", C.c_size_t), ("mem_buffer", C.c_void_p), ("no_alloc", C.c_bool)]


def main():
    O.build_ref()
    g = C.CDLL(str(O.ref_dir() / "libggml_ref.so"))
    vp = C.c_void_p
    g.ggml_init.restype = vp
    g.ggml_init.argtypes = [_IP]
    g.ggml_free.argtypes = [vp]
    for n in ("ggml_new_tensor_1d", "ggml_new_tensor_3d", "ggml_rope_ext", "ggml_rope_ext_inplace", "ggml_new_graph", "ggml_get_data"):
        getattr(g, n).restype = vp
    g.ggml_new_tensor_1d.argtypes = [vp, C.c_int, C.c_int64]
    g.ggml_new_tensor_3d.argtypes = [vp, C.c_int, C.c_int64, C.c_int64, C.c_int64]
    g.ggml_rope_ext.argtypes = g.ggml_rope_ext_inplace.argtypes = [vp, vp, vp, vp, C.c_int, C.c_int, C.c_int] + [C.c_float] * 6
    g.ggml_new_graph.argtypes = [vp]
    g.ggml_build_forward_expand.argtypes = [vp, vp]
    g.ggml_graph_compute_with_ctx.argtypes = [vp, vp, C.c_int]
    g.ggml_get_data.argtypes = [vp]
    rng = np.random.default_rng(7)
    out = {}
    for i, (ints, floats) in enumerate(CASES):
        D, H, T, n_dims, mode, n_ctx_orig, in_place, with_ff = ints
        x = (rng.standard_normal((T, H, D)) * 2.0).astype(np.float16).view(np.uint16)
        pos = positions(T, rng)
        ff = (1.0 + rng.uniform(0, 7, n_dims // 2)).astype(np.float32) if with_ff else np.zeros(0, np.float32)
        ctx = g.ggml_init(_IP(64 << 20, None, False))
        a = g.ggml_new_tensor_3d(ctx, O.F16, D, H, T)
        p = g.ggml_new_tensor_1d(ctx, 26, T)   # GGML_TYPE_I32
        f = g.ggml_new_tensor_1d(ctx, O.F32, n_dims // 2) if with_ff else None
        C.memmove(g.ggml_get_data(a), x.ctypes.data, x.nbytes)
        C.memmove(g.ggml_get_data(p), pos.ctypes.data, pos.nbytes)
        if with_ff:
            C.memmove(g.ggml_get_data(f), ff.ctypes.data, ff.nbytes)
        fn = g.ggml_rope_ext_inplace if in_place else g.ggml_rope_ext
        y = fn(ctx, a, p, f, n_dims, mode, n_ctx_orig, *floats)
        gf = g.ggml_new_graph(ctx)
        g.ggml_build_forward_expand(gf, y)
        assert g.ggml_graph_compute_with_ctx(ctx, gf, 4) == 0
        res = np.empty_like(x)
        C.memmove(res.ctypes.data, g.ggml_get_data(y), res.nbytes)
        g.ggml_free(ctx)
        out[f"c{i}_ints"] = np.array(ints, np.int32)
        out[f"c{i}_floats"] = np.array(floats, np.float32)
        out[f"c{i}_x"], out[f"c{i}_pos"], out[f"c{i}_ff"], out[f"c{i}_y"] = x, pos, ff, res
    out["n_cases"] = np.array(len(CASES), np.int32)
    np.savez_compressed(HERE / "kshift_golden.npz", **out)
    print(f"wrote {HERE / 'kshift_golden.npz'}: {len(CASES)} cases")


if __name__ == "__main__":
    main()
