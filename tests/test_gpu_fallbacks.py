"""-m gpu: the fallback rungs of the decode launchers, each against the oracle: attention past the clustered kernel's context
limit (k_attn_rows<true> + a quantize kernel in front of wo), the fused GEMV's producer kernel in front instead of the distributed
prologue, and the per-matrix GEMV kernels for weights the bulk-copy ring cannot read."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle_lib as O
from gpu_util import act_ws, act_ws_fields, dev_f32, dev_u8, ptr, sync
from test_gpu_engine import check_decode_parity
from tiny_model import TinyModel

pytestmark = pytest.mark.gpu


def rel_tol(ref, r=4e-6):
    return r * max(1.0, float(np.max(np.abs(ref))))


def test_engine_long_context_attention_fallback(cuda, pkg, lib, port):
    """n_ctx 16384: the scores no longer fit k_attn2's shared memory (about 15k positions at head_dim 128), so every layer runs
    k_attn_rows<true> and quantizes wo's input in a kernel of its own: one launch per layer more than the same model at a short context."""
    kw = dict(n_layer=2, n_embd=512, n_head=4, n_head_kv=2, n_ff=1024, n_vocab=320, arch="llama", ftype="q4_K_M", seed=9, branch_scale=0.1)
    toks = [(i * 7919 + 13) % 320 for i in range(8)]
    launches = {}
    for n_ctx in (64, 16384):
        tm = TinyModel(n_ctx=n_ctx, **kw)
        eng = tm.load_engine(pkg)
        got = np.zeros((len(toks), tm.hp["n_vocab"]), np.float32)
        n0 = lib.c.pb200_kernel_launches()
        for i, t in enumerate(toks):
            eng.decode(int(t), i, got[i])
        launches[n_ctx] = (lib.c.pb200_kernel_launches() - n0) // len(toks)
        eng.close()
        if n_ctx == 16384:
            want, _ = tm.port_decode(port, toks)
            check_decode_parity(got, want)
    assert launches[16384] == launches[64] + kw["n_layer"], launches


class GemvMat(C.Structure):
    _fields_ = [("type", C.c_int32), ("_pad", C.c_int32), ("W", C.c_void_p), ("n", C.c_int64), ("y", C.c_void_p), ("add", C.c_void_p)]


@pytest.mark.parametrize("prologue", [1, 2], ids=["rms_norm", "silu_mul"])
def test_gemv_fused_prologue_rungs(cuda, lib, port, prologue):
    """pb200_gemv_fused on a q|k|v group of mixed k-quant types: with barrier words the prologue runs distributed inside the GEMV
    (one launch); without them a producer kernel runs in front (two launches).  Both leave the oracle's q8_K quantization of the
    prologue's output in act_ws and match the oracle's mat-vec to fp32 summation order.  The sizes reach every rung: K = 2048 whole
    rows and k_rmsnorm_q8K<2>; 12 288 split rows, the prologue's strided sum of squares and k_rmsnorm_q8K<4>; 28 672 k_rmsnorm_quant."""
    eps = 1e-5
    types, Ns = [O.Q4_K, O.Q4_K, O.Q6_K], [512, 128, 128]
    fn = lib.c.pb200_gemv_fused
    fn.argtypes = [C.c_int, C.POINTER(GemvMat), C.c_int64, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_int, C.c_void_p]
    for K in (2048, 12288, 28672):
        Ws = [O.synth_blocks(t, n, K, seed=17 + i) for i, (t, n) in enumerate(zip(types, Ns))]
        rng = np.random.default_rng(prologue)
        a = rng.standard_normal(K).astype(np.float32)
        b = (1.0 + 0.1 * rng.standard_normal(K)).astype(np.float32) if prologue == 1 else rng.standard_normal(K).astype(np.float32)
        ad, bd = dev_f32(a), dev_f32(b)
        if prologue == 1:
            x = port.rms_norm(a, eps) * b
        else:
            # silu's expf: the device's, from the plain silu * mul ops (same arithmetic as the fused prologues), next to the oracle's
            xd = torch.zeros(K, device="cuda")
            lib.check(lib.c.pb200_silu_mul(ptr(ad), ptr(bd), ptr(xd), K, None), "silu_mul")
            sync()
            x = xd.cpu().numpy()
            assert np.max(np.abs(x - port.silu_mul(a, b))) <= rel_tol(x, 1e-6)
        want_act = port.quantize_act(O.Q4_K, x)
        wants = [port.mul_mat(t, w, n, K, x)[0] for t, n, w in zip(types, Ns, Ws)]
        Wd = [dev_u8(w) for w in Ws]
        for barrier in (True, False):
            ws = act_ws(lib, K)
            sync_ws = torch.zeros(16, dtype=torch.uint8, device="cuda")
            ys = [torch.full((n,), float("nan"), device="cuda") for n in Ns]
            mats = (GemvMat * 3)(*[GemvMat(t, 0, w.data_ptr(), n, y.data_ptr(), None) for t, w, n, y in zip(types, Wd, Ns, ys)])
            n0 = lib.c.pb200_kernel_launches()
            lib.check(fn(3, mats, K, ws.data_ptr(), prologue, ad.data_ptr(), bd.data_ptr(), eps, sync_ws.data_ptr() if barrier else None, 1, None),
                      "gemv_fused")
            sync()
            assert lib.c.pb200_kernel_launches() - n0 == (1 if barrier else 2), (K, barrier)
            assert np.array_equal(act_ws_fields(ws, K, "q8_K"), want_act), f"activation differs (K={K}, barrier={barrier})"
            for y, want in zip(ys, wants):
                assert np.max(np.abs(y.cpu().numpy() - want)) <= rel_tol(want), (K, barrier)


@pytest.mark.parametrize("t", [O.Q8_0, O.Q5_1], ids=lambda t: O.TYPE_NAME[t])
def test_gemv_fused_small_block_types_each_take_the_ring(cuda, lib, port, t):
    """The ring kernel takes Q8_0 / Q5_1 matrices one at a time: a group of two still runs both on it (two instrumented ring
    launches leave their CTA stamps in the trace buffer), not on the generic kernel."""
    K, Ns = 4096, [64, 48]
    Ws = [O.synth_blocks(t, n, K, seed=31 + i) for i, n in enumerate(Ns)]
    x = np.random.default_rng(5).standard_normal(K).astype(np.float32)
    ws = act_ws(lib, K)
    lib.check(lib.c.pb200_quantize_act(t, ptr(dev_f32(x)), K, ptr(ws), None), "q")
    Wd = [dev_u8(w) for w in Ws]
    ys = [torch.full((n,), float("nan"), device="cuda") for n in Ns]
    slots = 4
    trace = torch.zeros(slots * 4096, dtype=torch.int64, device="cuda")
    lib.c.pb200_debug_set_trace.argtypes = [C.c_void_p, C.c_int]
    lib.check(lib.c.pb200_debug_set_trace(trace.data_ptr(), slots), "trace")
    try:
        lib.check(lib.c.pb200_mul_mat_vec_fused(2, (C.c_int * 2)(t, t), (C.c_void_p * 2)(*[w.data_ptr() for w in Wd]), (C.c_int64 * 2)(*Ns), K,
                                                ptr(ws), (C.c_void_p * 2)(*[y.data_ptr() for y in ys]), None), "fused")
        sync()
    finally:
        lib.c.pb200_debug_set_trace(None, 0)
    rows_stamped = (trace.view(slots, 4096) != 0).any(dim=1).cpu().tolist()
    assert rows_stamped == [True, True, False, False], rows_stamped
    for n, w, y in zip(Ns, Ws, ys):
        want = port.mul_mat(t, w, n, K, x)[0]
        assert np.max(np.abs(y.cpu().numpy() - want)) <= rel_tol(want)


def test_gemv_fused_misaligned_weights_take_per_matrix_kernels(cuda, lib, port):
    """One W 8-byte but not 16-byte aligned: the bulk-copy ring cannot read it, so each matrix runs its own kernel (3 launches)."""
    K = 2048
    types, Ns = [O.Q4_K, O.Q4_K, O.Q6_K], [256, 128, 128]
    Ws = [O.synth_blocks(t, n, K, seed=23 + i) for i, (t, n) in enumerate(zip(types, Ns))]
    x = np.random.default_rng(4).standard_normal(K).astype(np.float32)
    ws = act_ws(lib, K)
    lib.check(lib.c.pb200_quantize_act(O.Q4_K, ptr(dev_f32(x)), K, ptr(ws), None), "q")
    bufs = [dev_u8(w, pad=64) for w in Ws]
    shifted = torch.zeros(Ws[1].size + 64, dtype=torch.uint8, device="cuda")
    shifted[8: 8 + Ws[1].size] = torch.from_numpy(np.ascontiguousarray(Ws[1]).view(np.uint8).reshape(-1))
    addrs = [bufs[0].data_ptr(), shifted.data_ptr() + 8, bufs[2].data_ptr()]
    assert addrs[1] % 16 == 8
    ys = [torch.full((n,), float("nan"), device="cuda") for n in Ns]
    n0 = lib.c.pb200_kernel_launches()
    lib.check(lib.c.pb200_mul_mat_vec_fused(3, (C.c_int * 3)(*types), (C.c_void_p * 3)(*addrs), (C.c_int64 * 3)(*Ns), K, ptr(ws),
                                            (C.c_void_p * 3)(*[y.data_ptr() for y in ys]), None), "fused")
    sync()
    assert lib.c.pb200_kernel_launches() - n0 == 3
    for t, n, w, y in zip(types, Ns, Ws, ys):
        want = port.mul_mat(t, w, n, K, x)[0]
        assert np.max(np.abs(y.cpu().numpy() - want)) <= rel_tol(want)
