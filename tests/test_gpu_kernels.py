"""-m gpu: parity of every CUDA kernel against the oracle, through the C ABI (include/prima_b200.h).
Bars: integer/byte results bit-exact (activation quantization, dequantized rows, f16 KV store);
fp32 results within fp32-summation-order distance of the CPU oracle (tolerances stated per test)."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle_lib as O
from gpu_util import act_ws, act_ws_fields, dev_f32, dev_u8, ptr, sync

pytestmark = pytest.mark.gpu
KQ = [O.Q4_K, O.Q5_K, O.Q6_K]
MODE = {O.Q4_K: "q8_K", O.Q5_K: "q8_K", O.Q6_K: "q8_K", O.Q8_0: "q8_0", O.Q5_1: "q8_1"}


def rel_tol(ref):
    return 4e-6 * max(1.0, float(np.max(np.abs(ref))))


@pytest.mark.parametrize("t", O.QUANT_TYPES, ids=lambda t: O.TYPE_NAME[t])
def test_quantize_act_bit_exact(cuda, lib, port, t):
    rng = np.random.default_rng(t)
    K = 2048 if t in KQ else 2080   # 2080 = 65 * 32: ragged vs 256
    cases = [rng.standard_normal(K).astype(np.float32) * s for s in (1.0, 1e-4, 300.0)]
    cases += [np.zeros(K, np.float32), np.tile(np.array([1.0, -1.0, 0.5, -0.5], np.float32), K // 4),
              np.tile(np.array([-3.0, 3.0, 1.5, 0.0], np.float32), K // 4)]
    z = np.zeros(K, np.float32); z[300] = -2.5; cases.append(z)
    for offset in (0, 1):   # 1: x one float past a 16-byte boundary, so the kernel must not use its 128-bit loads
        for x in cases:
            ws = act_ws(lib, K)
            xd = dev_f32(np.concatenate([np.zeros(offset, np.float32), x]))
            lib.check(lib.c.pb200_quantize_act(t, C.c_void_p(xd.data_ptr() + 4 * offset), K, ptr(ws), None), "quantize_act")
            sync()
            got = act_ws_fields(ws, K, MODE[t])
            want = port.quantize_act(t, x)
            assert np.array_equal(got, want), f"activation quantization differs for {O.TYPE_NAME[t]} (x offset {offset})"


@pytest.mark.parametrize("t", KQ, ids=lambda t: O.TYPE_NAME[t])
@pytest.mark.parametrize("N,K", [(64, 256), (37, 512), (8, 2048), (129, 4096), (24, 8192), (19, 14336), (10, 28672),
                                 (21, 29952), (9, 53248)])   # beyond the ring's 29 696: k_gemv_generic (the ring's dot routines)
def test_gemv_kquant_vs_oracle(cuda, lib, port, t, N, K):
    W = O.synth_blocks(t, N, K, seed=N * 31 + K)
    rng = np.random.default_rng(K + N)
    x = rng.standard_normal(K).astype(np.float32)
    want = port.mul_mat(t, W, N, K, x)[0]
    Wd, xd, ws = dev_u8(W), dev_f32(x), act_ws(lib, K)
    y = torch.full((N,), float("nan"), device="cuda")
    lib.check(lib.c.pb200_mul_mat_vec(t, ptr(Wd), N, K, ptr(xd), ptr(y), ptr(ws), None), "mul_mat_vec")
    sync()
    got = y.cpu().numpy()
    assert np.max(np.abs(got - want)) <= rel_tol(want), (np.max(np.abs(got - want)), rel_tol(want))


@pytest.mark.parametrize("t", [O.Q8_0, O.Q5_1], ids=lambda t: O.TYPE_NAME[t])
@pytest.mark.parametrize("N,K", [(16, 64), (33, 7392), (5, 29568), (301, 29568), (64, 1280), (40, 4096), (7, 8192), (130, 14336)])   # K % 128 == 0: the bulk-copy ring (columns of 8 blocks; 29 568 = 115.5 columns, split rows), else k_gemv_generic
def test_gemv_small_block_types_vs_oracle(cuda, lib, port, t, N, K):
    W = O.synth_blocks(t, N, K, seed=N + K)
    x = np.random.default_rng(K).standard_normal(K).astype(np.float32)
    want = port.mul_mat(t, W, N, K, x)[0]
    Wd, xd, ws = dev_u8(W), dev_f32(x), act_ws(lib, K)
    y = torch.zeros(N, device="cuda")
    lib.check(lib.c.pb200_mul_mat_vec(t, ptr(Wd), N, K, ptr(xd), ptr(y), ptr(ws), None), "mul_mat_vec")
    sync()
    got = y.cpu().numpy()
    assert np.max(np.abs(got - want)) <= rel_tol(want)


@pytest.mark.parametrize("t", O.QUANT_TYPES, ids=lambda t: O.TYPE_NAME[t])
def test_gemv_weight_bit_patterns_vs_oracle(cuda, lib, port, t):
    """The weight blocks of oracle_lib.edge_blocks (quant bytes all 0x00 / 0xFF, Q8_0 q = -128, Q6_K scale -128 with q = -32, scales and
    mins of 63, d = 0) through the GEMV families above: k-quant ring; Q8_0 / Q5_1 on the ring (K % 128 == 0) and on k_gemv_generic."""
    for K in ([2048] if t in KQ else [2048, 1984]):
        N = 96
        W = O.edge_blocks(t, N, K, seed=K + t)
        x = np.random.default_rng(K + t).standard_normal(K).astype(np.float32)
        want = port.mul_mat(t, W, N, K, x)[0]
        Wd, xd, ws = dev_u8(W), dev_f32(x), act_ws(lib, K)
        y = torch.full((N,), float("nan"), device="cuda")
        lib.check(lib.c.pb200_mul_mat_vec(t, ptr(Wd), N, K, ptr(xd), ptr(y), ptr(ws), None), "mul_mat_vec")
        sync()
        got = y.cpu().numpy()
        assert np.max(np.abs(got - want)) <= rel_tol(want), (K, np.max(np.abs(got - want)), rel_tol(want))


def test_gemv_golden_reference_quantized_weights(cuda, lib):
    """Weights quantized by the reference's own ggml_quantize_chunk (committed fixture), outputs of its CPU mul_mat."""
    from pathlib import Path
    z = np.load(Path(__file__).resolve().parent / "golden" / "kquants_golden.npz")
    x = z["x"]; K = x.size; N = z["w"].shape[0]
    for t in O.QUANT_TYPES:
        n = O.TYPE_NAME[t]
        for tag in ("", "synth_"):
            Wd, xd, ws = dev_u8(z[f"{n}_{tag}blocks"]), dev_f32(x), act_ws(lib, K)
            y = torch.zeros(N, device="cuda")
            lib.check(lib.c.pb200_mul_mat_vec(t, ptr(Wd), N, K, ptr(xd), ptr(y), ptr(ws), None), "mul_mat_vec")
            sync()
            want = z[f"{n}_{tag}mulmat"][0]
            assert np.max(np.abs(y.cpu().numpy() - want)) <= rel_tol(want), n


def test_gemv_fused_bias_resid_and_host_path(cuda, lib, port):
    K = 2048
    types = [O.Q4_K, O.Q4_K, O.Q6_K]; Ns = [512, 128, 128]
    Ws = [O.synth_blocks(t, n, K, seed=7 + i) for i, (t, n) in enumerate(zip(types, Ns))]
    x = np.random.default_rng(1).standard_normal(K).astype(np.float32)
    ws = act_ws(lib, K)
    xd = dev_f32(x)
    lib.check(lib.c.pb200_quantize_act(O.Q4_K, ptr(xd), K, ptr(ws), None), "q")
    Wd = [dev_u8(w) for w in Ws]
    ys = [torch.zeros(n, device="cuda") for n in Ns]
    lib.check(lib.c.pb200_mul_mat_vec_fused(3, (C.c_int * 3)(*types), (C.c_void_p * 3)(*[w.data_ptr() for w in Wd]), (C.c_int64 * 3)(*Ns), K,
                                            ptr(ws), (C.c_void_p * 3)(*[y.data_ptr() for y in ys]), None), "fused")
    sync()
    for t, n, w, y in zip(types, Ns, Ws, ys):
        want = port.mul_mat(t, w, n, K, x)[0]
        assert np.max(np.abs(y.cpu().numpy() - want)) <= rel_tol(want)
    # bias + residual epilogue
    b = np.random.default_rng(2).standard_normal(Ns[0]).astype(np.float32); r = np.random.default_rng(3).standard_normal(Ns[0]).astype(np.float32)
    y = torch.zeros(Ns[0], device="cuda")
    bd, rd = dev_f32(b), dev_f32(r)
    lib.check(lib.c.pb200_mul_mat_vec_q(types[0], ptr(Wd[0]), Ns[0], K, ptr(ws), ptr(y), ptr(bd), ptr(rd), None), "epi")
    sync()
    want = port.mul_mat(types[0], Ws[0], Ns[0], K, x)[0] + b + r
    assert np.max(np.abs(y.cpu().numpy() - want)) <= rel_tol(want)
    # host-buffer entry point (H2D + quantize + GEMV + D2H)
    yh = np.zeros(Ns[0], np.float32)
    lib.check(lib.c.pb200_mul_mat_vec_host(types[0], ptr(Wd[0]), Ns[0], K, x.ctypes.data_as(C.c_void_p), yh.ctypes.data_as(C.c_void_p)), "host")
    want = port.mul_mat(types[0], Ws[0], Ns[0], K, x)[0]
    assert np.max(np.abs(yh - want)) <= rel_tol(want)


@pytest.mark.parametrize("t", O.QUANT_TYPES + [O.F16, O.F32], ids=lambda t: O.TYPE_NAME[t])
def test_get_rows_dequant_bit_exact(cuda, lib, port, t):
    K, N = 1024, 9
    if t == O.F32:
        tab = np.random.default_rng(0).standard_normal((N, K)).astype(np.float32); want_all = tab
    elif t == O.F16:
        tab = np.random.default_rng(0).standard_normal((N, K)).astype(np.float16); want_all = tab.astype(np.float32)
    else:
        tab = O.synth_blocks(t, N, K, seed=3); want_all = port.dequantize(t, tab, K)
    ids = np.array([8, 0, 3, 3], dtype=np.int32)
    y = torch.zeros(len(ids) * K, device="cuda")
    idd = torch.from_numpy(ids).cuda()
    tabd = dev_u8(tab)
    lib.check(lib.c.pb200_get_rows(t, ptr(tabd), K, ptr(idd), len(ids), ptr(y), None), "get_rows")
    sync()
    assert np.array_equal(y.cpu().numpy().reshape(len(ids), K), want_all[ids])


def test_rms_norm(cuda, lib, port):
    rng = np.random.default_rng(0)
    for n, rows, eps in ((8192, 3, 1e-5), (4096, 1, 1e-6), (64, 5, 1e-5), (29568, 2, 1e-6)):
        x = rng.standard_normal((rows, n)).astype(np.float32) * 3
        y = torch.zeros(rows * n, device="cuda")
        xd = dev_f32(x)
        lib.check(lib.c.pb200_rms_norm(ptr(xd), ptr(y), n, rows, eps, None), "rms_norm")
        sync()
        want = np.stack([port.rms_norm(x[i], eps) for i in range(rows)])
        got = y.cpu().numpy().reshape(rows, n)
        # double-precision sum on both sides: identical scale except for 1-ulp effects of the summation order
        assert np.max(np.abs(got - want) / np.maximum(np.abs(want), 1e-6)) < 3e-7


@pytest.mark.parametrize("mode", [0, 2])
@pytest.mark.parametrize("ff", [False, True])
def test_rope(cuda, lib, port, mode, ff):
    rng = np.random.default_rng(mode)
    H, D, T = 6, 128, 4
    x = rng.standard_normal((T, H, D)).astype(np.float32)
    pos = np.array([0, 1, 77, 4095], dtype=np.int32)
    freq = (1.0 + rng.uniform(0, 7, 64)).astype(np.float32) if ff else None
    y = torch.zeros(T * H * D, device="cuda")
    xd, pd, fd = dev_f32(x), torch.from_numpy(pos).cuda(), (dev_f32(freq) if ff else None)
    lib.check(lib.c.pb200_rope(ptr(xd), ptr(y), T, H, D, D, mode, ptr(pd), 500000.0, 1.0, 0.0, 1.0, 32.0, 1.0, 8192,
                               ptr(fd) if ff else None, None), "rope")
    sync()
    got = y.cpu().numpy().reshape(T, H, D)
    want = np.stack([port.rope(x[i], H, D, mode, int(pos[i]), freq_factors=freq) for i in range(T)])
    # theta is bit-identical (same running product); cosf/sinf differ by <= 2 ulp between CUDA and glibc
    assert np.max(np.abs(got - want)) < 2e-6 * np.max(np.abs(x)) * 2


def test_rope_yarn_and_partial_dims(cuda, lib, port):
    rng = np.random.default_rng(5)
    H, D, T = 2, 128, 2
    x = rng.standard_normal((T, H, D)).astype(np.float32)
    pos = np.array([3, 900], dtype=np.int32)
    y = torch.zeros(T * H * D, device="cuda")
    xd, pd = dev_f32(x), torch.from_numpy(pos).cuda()
    lib.check(lib.c.pb200_rope(ptr(xd), ptr(y), T, H, D, 64, 0, ptr(pd), 10000.0, 0.25, 1.0, 1.0, 32.0, 1.0, 4096, None, None), "rope")
    sync()
    want = np.stack([port.rope(x[i], H, D, 0, int(pos[i]), freq_base=10000.0, freq_scale=0.25, n_ctx_orig=4096, ext_factor=1.0, n_dims=64) for i in range(T)])
    assert np.max(np.abs(y.cpu().numpy().reshape(T, H, D) - want)) < 1e-5


def test_soft_max(cuda, lib, port):
    rng = np.random.default_rng(0)
    ncols, rows = 96, 6
    x = rng.standard_normal((rows, ncols)).astype(np.float32) * 4
    mask = np.zeros((2, ncols), np.float32); mask[0, 50:] = -np.inf; mask[1, 70:] = -np.inf
    y = torch.zeros(rows * ncols, device="cuda")
    xd, md = dev_f32(x), dev_f32(mask)
    lib.check(lib.c.pb200_soft_max(ptr(xd), ptr(md), ptr(y), ncols, rows, 2, 0.088, None), "soft_max")
    sync()
    got = y.cpu().numpy().reshape(rows, ncols)
    want = np.stack([port.soft_max(x[i], mask[i % 2], 0.088) for i in range(rows)])
    assert np.max(np.abs(got - want)) < 3e-7      # reference bar for SOFT_MAX is NMSE 1e-6 (test-backend-ops.cpp:2077)


@pytest.mark.parametrize("n_kv", [1, 5, 32, 200, 1023])
def test_attn_decode(cuda, lib, port, n_kv):
    rng = np.random.default_rng(n_kv)
    H, HK, D, n_ctx = 8, 2, 128, 1024
    q = rng.standard_normal(H * D).astype(np.float32)
    Kc = (rng.standard_normal((n_ctx, HK * D)) * 0.5).astype(np.float16)
    Vc = rng.standard_normal((n_ctx, HK * D)).astype(np.float16)
    out = torch.zeros(H * D, device="cuda")
    pos = torch.tensor([n_kv - 1], dtype=torch.int32, device="cuda")
    qd, kd, vd = dev_f32(q), torch.from_numpy(Kc).cuda(), torch.from_numpy(Vc).cuda()
    lib.check(lib.c.pb200_attn_decode(ptr(qd), ptr(kd), ptr(vd), ptr(out), H, HK, D, ptr(pos), n_ctx, 1.0 / np.sqrt(D), None), "attn")
    sync()
    want = port.attention_decode(q, Kc.view(np.uint16), Vc.view(np.uint16), H, HK, D, n_kv, 1.0 / np.sqrt(D))
    # same f16 roundings of q and of the probabilities as the CPU graph; only fp32 summation order and expf ulp differ.
    # (an f16 probability can flip by one f16 ulp when expf differs in the last bit: bound 2e-4 relative of |V| ~ 1)
    assert np.max(np.abs(out.cpu().numpy() - want)) < 3e-4
    assert np.mean(np.abs(out.cpu().numpy() - want)) < 2e-5


@pytest.mark.parametrize("H,HK,n_tok,pos0", [(8, 2, 21, 5), (64, 8, 9, 120), (16, 2, 6, 1790), (16, 2, 3, 6390)],
                         ids=["tiled-gqa4-ragged", "tiled-gqa8-70B-heads", "tiled-2-tokens-per-cta-long-context", "per-head-fallback-very-long"])
def test_attn_prefill_vs_oracle(cuda, lib, port, H, HK, n_tok, pos0):
    """Prompt-processing attention: every (token, head) row against the oracle's decode attention at that token's causal length.
    Covers the tiled kernel (K/V tiles shared by the GQA group x 4 / 2 tokens) and the per-(head, token) fallback."""
    rng = np.random.default_rng(H + n_tok)
    D = 128
    n_ctx = pos0 + n_tok
    q = rng.standard_normal((n_tok, H * D)).astype(np.float32)
    Kc = (rng.standard_normal((n_ctx, HK * D)) * 0.5).astype(np.float16)
    Vc = rng.standard_normal((n_ctx, HK * D)).astype(np.float16)
    pos_h = (pos0 + np.arange(n_tok)).astype(np.int32)
    out = torch.full((n_tok, H * D), float("nan"), device="cuda")
    pos = torch.from_numpy(pos_h).cuda()
    qd, kd, vd = dev_f32(q), torch.from_numpy(Kc).cuda(), torch.from_numpy(Vc).cuda()
    scale = 1.0 / np.sqrt(D)
    lib.check(lib.c.pb200_attn_prefill(ptr(qd), ptr(kd), ptr(vd), ptr(out), H, HK, D, ptr(pos), n_tok, n_ctx, scale, None), "attn_prefill")
    sync()
    got = out.cpu().numpy()
    assert np.isfinite(got).all()
    for t in range(n_tok):
        want = port.attention_decode(q[t], Kc.view(np.uint16), Vc.view(np.uint16), H, HK, D, int(pos_h[t]) + 1, scale)
        assert np.max(np.abs(got[t] - want)) < 3e-4, (t, np.max(np.abs(got[t] - want)))
        assert np.mean(np.abs(got[t] - want)) < 2e-5


def test_full_size_gemv_properties(cuda, lib):
    """BASELINE sizes (Llama-3-70B shapes): the fused TMA kernel must agree with an independent evaluation —
    dequantized weights (get_rows kernel, bit-exact vs the oracle above) times the dequantized q8_K activation in fp64."""
    import gpu_util
    # N large enough that every CTA streams > 4 tiles: exercises the mbarrier ring wrap-around and both parities
    for t, N, K in ((O.Q4_K, 8192, 8192), (O.Q6_K, 6000, 8192), (O.Q5_K, 6100, 8192), (O.Q4_K, 2500, 28672), (O.Q6_K, 2200, 28672),
                    (O.Q6_K, 8192, 28672)):   # 28 tiles per CTA with split rows: caught an mbarrier parity ABA of the 3-stage ring
        W = O.synth_blocks(t, N, K, seed=K + N + t)
        x = np.random.default_rng(t).standard_normal(K).astype(np.float32)
        Wd, xd, ws = dev_u8(W), dev_f32(x), act_ws(lib, K)
        y = torch.zeros(N, device="cuda")
        lib.check(lib.c.pb200_mul_mat_vec(t, ptr(Wd), N, K, ptr(xd), ptr(y), ptr(ws), None), "mul_mat_vec")
        ids = torch.arange(N, dtype=torch.int32, device="cuda")
        deq = torch.zeros(N * K, device="cuda")
        lib.check(lib.c.pb200_get_rows(t, ptr(Wd), K, ptr(ids), N, ptr(deq), None), "get_rows")
        sync()
        raw = ws.cpu().numpy(); qs = raw[:K].view(np.int8).astype(np.float64); d = raw[K:K + K // 32 * 4].view(np.float32)[: K // 256].astype(np.float64)
        xq = torch.from_numpy(qs * np.repeat(d, 256)).cuda()
        want = (deq.view(N, K).double() @ xq).cpu().numpy()
        got = y.cpu().numpy().astype(np.float64)
        assert np.max(np.abs(got - want)) < 2e-5 * max(1.0, np.max(np.abs(want))), (O.TYPE_NAME[t], N, K)
        # linearity in the rows: duplicated rows give identical results (tile/warp assignment independence)
        W2 = np.concatenate([W.reshape(N, -1)[:64], W.reshape(N, -1)[:64]]).reshape(-1)
        y2 = torch.zeros(128, device="cuda")
        W2d = dev_u8(W2)
        lib.check(lib.c.pb200_mul_mat_vec_q(t, ptr(W2d), 128, K, ptr(ws), ptr(y2), None, None, None), "dup")
        sync()
        assert torch.equal(y2[:64], y2[64:]) and torch.equal(y2[:64], y[:64])
