"""-m gpu: the batched (prefill) k-quant product pb200_mul_mat_q — wgmma tensor cores — against the CPU oracle.

Numerics bar (floating point, stated here): the kernel quantizes every activation row to q8_K exactly as the CPU backend
does and expands the weights with the reference's dequantization formulas evaluated in fp16: the integer q is exact, the
sub-block scale d*sc and offset dmin*m are rounded to fp16, one fused multiply-add, fp16 result; activations d*q8 are
rounded to fp16; products accumulate in fp32 on the tensor pipe.  Versus the oracle's integer dot products that is at most
four fp16 roundings (2^-11 each) on terms no larger than the sub-block's largest weight:
    |err[t,n]| <= 2^-9 * sum_k (|W[n,k]| + max_{32-sub-block}|W[n,.]|) * |x[t,k]|      (checked element-wise)
    NMSE <= 4e-6                              (the reference's own MUL_MAT bar is 5e-4, test-backend-ops.cpp:1639)
Integer-valued inputs with exactly representable scales must come out bit-exact (test_mmq_integer_exact).
"""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle_lib as O
from gpu_util import dev_f32, dev_u8, ptr, sync

pytestmark = pytest.mark.gpu
KQ = [O.Q4_K, O.Q5_K, O.Q6_K]


def run_mmq(lib, t, W, N, K, X, bias=None, ldx=None, resid=None):
    T = X.shape[0]
    ldx = ldx or K
    Xp = np.zeros((T, ldx), np.float32)
    Xp[:, :K] = X
    Wd, xd = dev_u8(W), dev_f32(Xp)
    y = torch.full((T, N), float("nan"), dtype=torch.float32, device="cuda")
    ws = torch.zeros(lib.c.pb200_mul_mat_q_workspace_bytes(K, T) + 64, dtype=torch.uint8, device="cuda")
    bd = dev_f32(bias) if bias is not None else None
    rd = dev_f32(resid) if resid is not None else None
    lib.check(lib.c.pb200_mul_mat_q(t, ptr(Wd), N, K, ptr(xd), ldx, T, ptr(y), ptr(bd) if bd is not None else None,
                                    ptr(rd) if rd is not None else None, ptr(ws), None), "mul_mat_q")
    sync()
    assert lib.c.pb200_aborted() == 0, "tensor-core pipeline gave up (watchdog)"
    return y.cpu().numpy()


def oracle(port, t, W, N, K, X):
    return np.stack([port.mul_mat(t, W, N, K, X[i]).reshape(-1) for i in range(X.shape[0])])


def check(got, want, Wf, X):
    assert np.isfinite(got).all()
    err = np.abs(got - want)
    N, K = Wf.shape
    sub = np.repeat(np.abs(Wf).reshape(N, K // 32, 32).max(axis=2), 32, axis=1)
    bound = 2.0 ** -9 * (np.abs(X) @ (np.abs(Wf) + sub).T) + 1e-6
    assert (err <= bound).all(), f"max err {err.max():.3e} exceeds the fp16-roundings bound (worst ratio {(err / bound).max():.2f})"
    nmse = float(np.sum((got - want) ** 2) / max(np.sum(want ** 2), 1e-30))
    assert nmse <= 4e-6, f"NMSE {nmse:.3e}"


@pytest.mark.parametrize("t", KQ, ids=lambda t: O.TYPE_NAME[t])
@pytest.mark.parametrize("N,K,T", [(128, 256, 16), (256, 512, 33), (384, 1024, 128), (200, 768, 7), (128, 2048, 300)])
def test_mmq_vs_oracle(cuda, lib, port, t, N, K, T):
    rng = np.random.default_rng(1000 * t + N + K + T)
    W = O.synth_blocks(t, N, K, seed=17 * t + N)
    X = rng.standard_normal((T, K)).astype(np.float32)
    X[0] = 0.0                      # an all-zero row quantizes to d = 0
    if T > 2:
        X[2] *= 1e-3
    got = run_mmq(lib, t, W, N, K, X)
    want = oracle(port, t, W, N, K, X)
    Wf = port.dequantize(t, W, N * K).reshape(N, K)
    check(got, want, Wf, X)
    assert np.all(got[0] == 0.0)


@pytest.mark.parametrize("t", [O.Q8_0, O.Q5_1], ids=lambda t: O.TYPE_NAME[t])
@pytest.mark.parametrize("N,K,T", [(256, 448, 33), (128, 1984, 64), (200, 512, 9), (128, 29568, 24)])
def test_mmq_small_block_types_vs_oracle(cuda, lib, port, t, N, K, T):
    """Q8_0 / Q5_1 (32-element blocks; the CPU dot quantizes the activation per 32 values): K % 64 == 0 is enough, so rows that are
    not 16-byte aligned and a short last 256-K group are the norm here; the last case is Qwen2.5-72B's ffn_down K."""
    rng = np.random.default_rng(100 * t + N + K + T)
    W = O.synth_blocks(t, N, K, seed=5 * t + N)
    X = rng.standard_normal((T, K)).astype(np.float32)
    X[0] = 0.0
    got = run_mmq(lib, t, W, N, K, X)
    want = oracle(port, t, W, N, K, X)
    Wf = port.dequantize(t, W, N * K).reshape(N, K)
    check(got, want, Wf, X)
    assert np.all(got[0] == 0.0)


def test_mmq_integer_exact(cuda, lib, port):
    """Small-integer activations and Q4_K blocks whose scales make every weight an exact fp16 integer: the tensor-core
    result must then equal the oracle bit for bit (a layout / swizzle / descriptor error cannot hide behind a tolerance)."""
    N, K, T = 256, 1024, 64
    rng = np.random.default_rng(5)
    nb = N * K // 256
    blk = np.zeros((nb, 144), np.uint8)
    blk[:, 0:2] = np.array([1.0], np.float16).view(np.uint8)        # d = 1
    blk[:, 2:4] = np.array([1.0], np.float16).view(np.uint8)        # dmin = 1
    sc = rng.integers(1, 4, size=(nb, 8)).astype(np.uint8)          # 6-bit scales 1..3, mins 0..7 (j < 4 and j >= 4 packing)
    mn = rng.integers(0, 8, size=(nb, 8)).astype(np.uint8)
    s12 = np.zeros((nb, 12), np.uint8)
    s12[:, 0:4] = sc[:, 0:4]
    s12[:, 4:8] = mn[:, 0:4]
    s12[:, 8:12] = (sc[:, 4:8] & 0xF) | ((mn[:, 4:8] & 0xF) << 4)
    blk[:, 4:16] = s12
    blk[:, 16:] = rng.integers(0, 256, size=(nb, 128)).astype(np.uint8)
    W = blk.reshape(-1)
    # activations: integers in [-127, 127] with the extreme present in every 256-block, so q8_K reproduces them exactly
    X = rng.integers(-20, 21, size=(T, K)).astype(np.float32)
    X[:, ::256] = -127.0
    got = run_mmq(lib, O.Q4_K, W, N, K, X)
    want = oracle(port, O.Q4_K, W, N, K, X)
    assert np.array_equal(got, want)


def test_mmq_bias_residual_ragged_rows_and_strided_input(cuda, lib, port):
    t, N, K, T = O.Q6_K, 200, 2048, 40       # N not a multiple of the 128-row tile, ldx > K, split-K (bias added once)
    rng = np.random.default_rng(9)
    W = O.synth_blocks(t, N, K, seed=3)
    X = rng.standard_normal((T, K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    resid = rng.standard_normal((T, N)).astype(np.float32)
    got = run_mmq(lib, t, W, N, K, X, bias=bias, ldx=K + 64, resid=resid)
    want = (oracle(port, t, W, N, K, X) + bias[None, :]) + resid
    Wf = port.dequantize(t, W, N * K).reshape(N, K)
    check(got, want, Wf, X)


@pytest.mark.parametrize("T", [700, 512])   # 700: two accumulators per tile + a ragged third token tile; 512: two accumulators; both stream-K split
def test_mmq_matches_gemv_columnwise_full_width(cuda, lib, T):
    """Size-independent property at a 70B shape (also the dual-accumulator configuration): every column of the batched product agrees with the decode GEMV (which is
    bit-exact with the oracle) to NMSE <= 4e-6."""
    t, N, K = O.Q4_K, 8192, 8192
    g = torch.Generator(device="cuda").manual_seed(1)
    W = O.synth_blocks(t, 256, K, seed=11)                  # 256 distinct rows, tiled to N
    Wfull = np.tile(W.reshape(256, -1), (N // 256, 1)).reshape(-1)
    X = torch.randn((T, K), generator=g, device="cuda", dtype=torch.float32).cpu().numpy()
    got = run_mmq(lib, t, Wfull, N, K, X)
    # identical weight rows -> identical outputs up to the order of fp32 adds: the stream-K decomposition cuts different output tiles at
    # different K groups, and the two or three partial accumulators of a cut tile meet in dst by fp32 atomic adds
    assert np.max(np.abs(got[:, :256] - got[:, 256:512])) <= 2e-5 * np.max(np.abs(got))
    Wd = dev_u8(Wfull)
    ws = torch.zeros(lib.c.pb200_act_workspace_bytes(K) + 64, dtype=torch.uint8, device="cuda")
    for col in (0, 1, 255, 256, 511, 512, 600, 699):
        if col >= T:
            continue
        xd = dev_f32(X[col])
        y = torch.zeros(N, dtype=torch.float32, device="cuda")
        lib.check(lib.c.pb200_mul_mat_vec(t, ptr(Wd), N, K, ptr(xd), ptr(y), ptr(ws), None), "mul_mat_vec")
        sync()
        ref = y.cpu().numpy()
        nmse = float(np.sum((got[col] - ref) ** 2) / np.sum(ref ** 2))
        assert nmse <= 4e-6, f"column {col}: NMSE {nmse:.3e}"
