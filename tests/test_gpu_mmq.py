"""-m gpu: the batched (prefill) k-quant product pb200_mul_mat_q — wgmma tensor cores — against the CPU oracle.

Numerics bar (floating point, stated here): the kernel quantizes every activation row to q8_K exactly as the CPU backend
does and expands the weights with the reference's dequantization formulas evaluated in fp16: the integer q is exact, the
sub-block scale d*sc and offset dmin*m are rounded to fp16, one fused multiply-add, fp16 result; activations d*q8 are
rounded to fp16 after a power-of-two row scale that puts the row's largest |d*q8| into [2^14, 2^15); products accumulate in
fp32 on the tensor pipe and the epilogue undoes the row scale exactly.  Versus the oracle's integer dot products that is at
most four fp16 roundings (2^-11 each) on terms no larger than the sub-block's largest weight, plus, for activation values
2^24 or more below their row's largest one, the fp16 subnormal spacing 2^-24 at a normalised row maximum >= 2^14:
    |err[t,n]| <= 2^-9 * sum_k (|W[n,k]| + max_{32-sub-block}|W[n,.]|) * |x[t,k]| + 2^-38 * amax_t * sum_k |W[n,k]|
    NMSE <= 4e-6                              (the reference's own MUL_MAT bar is 5e-4, test-backend-ops.cpp:1639)
Both terms scale with the row, so the bar holds at every activation magnitude the CPU backend represents.
Integer-valued inputs with exactly representable scales must come out bit-exact (test_mmq_integer_exact).
"""
import ctypes as C
from collections import namedtuple

import numpy as np
import pytest
import torch

import oracle_lib as O
from gpu_util import dev_f32, dev_u8, ptr, sync
from tiny_model import TinyModel

pytestmark = pytest.mark.gpu
KQ, BLK32 = O.KQ, O.BLK32
FP16_MAX = 65504.0

MmqPlan = namedtuple("MmqPlan", "bn tpad ttiles rtiles ngrp total upc split ctas_per_tile short_group_split")


def mmq_plan(lib, N, K, T):
    """launch_mmq's work decomposition (mmq.cu), restated: BN token columns per tile, 128 weight rows per tile, one unit = one 256-K
    group of one tile, contiguous shares of upc units per CTA (at most one CTA per SM, a share at least MMQ_MIN_UNITS = 8 groups).
    ctas_per_tile: the most CTAs that add into one tile; short_group_split: some tile's last (short, K % 256 != 0) group is in a CTA
    that does not hold the whole tile."""
    bn = 16
    while bn < T and bn < 128:
        bn *= 2
    tpad = -(-T // bn) * bn
    ttiles, rtiles, ngrp = tpad // bn, -(-N // 128), (K // 64 + 3) // 4
    total = rtiles * ttiles * ngrp
    upc = max(-(-total // lib.c.pb200_sm_count()), min(8, ngrp))
    ctas, short_split = 0, False
    for tile in range(total // ngrp):
        u0, u1 = tile * ngrp, (tile + 1) * ngrp - 1
        ctas = max(ctas, u1 // upc - u0 // upc + 1)
        c = u1 // upc
        short_split |= K % 256 != 0 and not (c * upc <= u0 and (c + 1) * upc > u1)
    return MmqPlan(bn, tpad, ttiles, rtiles, ngrp, total, upc, upc % ngrp != 0, ctas, short_split)


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


def bound(Wf, X):
    """The module docstring's element-wise bound, [T, N]."""
    N, K = Wf.shape
    aW = np.abs(Wf).astype(np.float64)
    sub = np.repeat(aW.reshape(N, K // 32, 32).max(axis=2), 32, axis=1)
    aX = np.abs(X).astype(np.float64)
    return 2.0 ** -9 * (aX @ (aW + sub).T) + 2.0 ** -38 * aX.max(axis=1)[:, None] * aW.sum(axis=1)[None, :]


def check(got, want, Wf, X):
    assert np.isfinite(got).all()
    err = np.abs(got.astype(np.float64) - want)
    b = bound(Wf, X)
    assert (err <= b).all(), f"max err {err.max():.3e} exceeds the fp16-roundings bound (worst ratio {(err / np.maximum(b, 1e-300)).max():.2f})"
    nmse = float(np.sum((got - want) ** 2) / max(np.sum(want ** 2), 1e-30))
    assert nmse <= 4e-6, f"NMSE {nmse:.3e}"


# T one below / at / one past each tile width of mmq_pick_bn (16, 32, 64, 128), several 128-column token tiles, and T < 8 (the engine
# takes the GEMV there, the ABI does not): T -> (BN, token tiles)
T_RUNGS = {1: (16, 1), 7: (16, 1), 8: (16, 1), 15: (16, 1), 17: (32, 1), 31: (32, 1), 33: (64, 1), 63: (64, 1), 65: (128, 1),
           127: (128, 1), 129: (128, 2), 257: (128, 3), 512: (128, 4)}
# N <= 64: the second consumer warpgroup has no rows; N = 1: every expansion thread reads (clamped) row 0
N_RUNGS = [1, 16, 64, 65, 127, 129]
# the K widths of the models served (hidden / ffn sizes of Llama 3 8B / 70B, Qwen2.5 7B / 14B / 32B / 72B, Mistral 7B / Nemo)
K_MODEL = [3584, 4096, 5120, 8192, 13824, 14336, 18944, 27648, 28672]
KQ_CASES = ([(128, 256, 16), (256, 512, 33), (384, 1024, 128), (200, 768, 7), (128, 2048, 300)]
            + [(136, 512, T) for T in T_RUNGS] + [(N, 512, 24) for N in N_RUNGS] + [(136, K, 24) for K in K_MODEL])
BLK32_CASES = ([(256, 448, 33), (128, 1984, 64), (200, 512, 9), (128, 29568, 24), (136, 448, 24), (136, 448, 100), (200, 4096, 33)]
               + [(136, 448, T) for T in T_RUNGS] + [(N, 448, 24) for N in N_RUNGS] + [(136, K, 24) for K in K_MODEL + [29568]])


def rung_inputs(lib, N, K, T, seed):
    """Standard-normal rows with row 0 zero; on the rung shapes every row also gets its own power-of-two scale (2^-4 .. 2^4), so a row
    scale read for the wrong token column shows.  Asserts the tile plan the T rung is there for."""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((T, K)).astype(np.float32)
    if T > 1:
        X[0] = 0.0                  # an all-zero row quantizes to d = 0
    if T in T_RUNGS and N == 136:
        X *= (2.0 ** (np.arange(T) % 9 - 4)).astype(np.float32)[:, None]
        p = mmq_plan(lib, N, K, T)
        assert (p.bn, p.ttiles) == T_RUNGS[T], p
    return X


@pytest.mark.parametrize("t", KQ, ids=lambda t: O.TYPE_NAME[t])
@pytest.mark.parametrize("N,K,T", KQ_CASES)
def test_mmq_vs_oracle(cuda, lib, port, t, N, K, T):
    X = rung_inputs(lib, N, K, T, 1000 * t + N + K + T)
    if T > 2:
        X[2] *= 1e-3
    W = O.synth_blocks(t, N, K, seed=17 * t + N)
    got = run_mmq(lib, t, W, N, K, X)
    want = oracle(port, t, W, N, K, X)
    Wf = port.dequantize(t, W, N * K).reshape(N, K)
    check(got, want, Wf, X)
    if T > 1:
        assert np.all(got[0] == 0.0)


@pytest.mark.parametrize("t", BLK32, ids=lambda t: O.TYPE_NAME[t])
@pytest.mark.parametrize("N,K,T", BLK32_CASES)
def test_mmq_small_block_types_vs_oracle(cuda, lib, port, t, N, K, T):
    """The 32-element block types (the CPU dot quantizes the activation per 32 values): K % 64 == 0 is enough, so rows that are not
    16-byte aligned and a short last 256-K group are the norm here; K = 29 568 is Qwen2.5-72B's ffn_down K (Q5_0 in its Q4_K_M)."""
    X = rung_inputs(lib, N, K, T, 100 * t + N + K + T)
    W = O.synth_blocks(t, N, K, seed=5 * t + N)
    got = run_mmq(lib, t, W, N, K, X)
    want = oracle(port, t, W, N, K, X)
    Wf = port.dequantize(t, W, N * K).reshape(N, K)
    check(got, want, Wf, X)
    if T > 1:
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
    t, N, K, T = O.Q6_K, 200, 2048, 40       # N not a multiple of the 128-row tile, ldx > K; every tile in one CTA (stored, not added)
    rng = np.random.default_rng(9)
    W = O.synth_blocks(t, N, K, seed=3)
    X = rng.standard_normal((T, K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    resid = rng.standard_normal((T, N)).astype(np.float32)
    got = run_mmq(lib, t, W, N, K, X, bias=bias, ldx=K + 64, resid=resid)
    want = (oracle(port, t, W, N, K, X) + bias[None, :]) + resid
    Wf = port.dequantize(t, W, N * K).reshape(N, K)
    check(got, want, Wf, X)


@pytest.mark.parametrize("t", KQ + BLK32, ids=lambda t: O.TYPE_NAME[t])
def test_mmq_split_tiles_add_bias_and_residual_once(cuda, lib, port, t):
    """Stream-K tiles shared by several CTAs: the K group 0 segment adds bias and residual, every other segment adds only its partial
    sum into the pre-zeroed output.  Two token tiles, a ragged row tile, >= 3 CTAs per tile; for the 32-element types K = 4160 = 65 steps of
    64, so the short last 256-K group is a partial segment.  Bias and residual together, and each alone."""
    N, T = 200, 150
    K = 8192 if t in KQ else 4160
    p = mmq_plan(lib, N, K, T)
    assert p.split and p.ttiles >= 2 and p.ctas_per_tile >= 3, p
    assert t in KQ or p.short_group_split, p
    rng = np.random.default_rng(40 + t)
    W = O.synth_blocks(t, N, K, seed=21 + t)
    X = rng.standard_normal((T, K)).astype(np.float32)
    X *= (2.0 ** (np.arange(T) % 5 - 2)).astype(np.float32)[:, None]
    bias = rng.standard_normal(N).astype(np.float32)
    resid = rng.standard_normal((T, N)).astype(np.float32)
    base = oracle(port, t, W, N, K, X)
    Wf = port.dequantize(t, W, N * K).reshape(N, K)
    for b, r in ((bias, resid), (bias, None), (None, resid)):
        got = run_mmq(lib, t, W, N, K, X, bias=b, resid=r)
        want = base.copy()
        if b is not None:
            want = want + b[None, :]
        if r is not None:
            want = want + r
        check(got, want, Wf, X)


def range_rows(t, K, rng):
    """Rows 2^s * N(0, 1) over the exponent range the CPU backend's activation quantizer represents, and the edge rows."""
    smax = 60 if t in KQ else 20               # q8_0 / q8_1: the CPU's own f16 d overflows above amax = 127 * 65504 ~ 8.3e6
    base = rng.standard_normal((1, K)).astype(np.float32)
    rows = [rng.standard_normal(K).astype(np.float32) * np.float32(2.0 ** s) for s in range(-60, smax + 1, 2)]
    unit = base[0] / np.abs(base[0]).max()
    rows += [unit * np.float32(65000.0), unit * np.float32(66000.0)]                 # amax just below / just above fp16's largest
    mixed = rng.standard_normal(K).astype(np.float32) * np.float32(1e-3)
    mixed[256:512] *= np.float32(1e8)                                                # one block ~1e5 among ~1e-3 blocks
    one = np.zeros(K, np.float32)
    one[777] = -3.0                                                                   # a single nonzero
    rows += [mixed, one, np.zeros(K, np.float32)]
    if t in BLK32:
        rows.append(unit * np.float32(8.0e6))
    X = np.stack(rows)
    if O.ACT_TYPE[t] == "q8_1":
        # the CPU's q8_1 also stores the block sum s = d * sum(q) as f16, which overflows once |sum of 32 values| > 65 504: rows of
        # (v, -v) pairs keep s = 0 at every magnitude, so the oracle stays finite
        X[:, 1::2] = -X[:, 0::2]
    return X


@pytest.mark.parametrize("t", KQ + BLK32, ids=lambda t: O.TYPE_NAME[t])
def test_mmq_activation_range(cuda, lib, port, t):
    """Activation rows from 2^-60 to 2^60 (k-quants) / 8e6 (32-element types) against the oracle under the module's row-relative bound, and
    per row NMSE <= 4e-6: no overflow to inf at |x| >= 65 520, no precision lost to fp16 subnormals on small rows.  The rows repeat
    in changing order over more than one 128-column token tile, so each token column must find its own row scale."""
    N, K = 136, 1024
    rng = np.random.default_rng(70 + t)
    rows = range_rows(t, K, rng)
    reps = -(-129 // len(rows))
    X = np.concatenate([rows if i % 2 == 0 else rows[::-1] for i in range(reps)])
    T = X.shape[0]
    assert mmq_plan(lib, N, K, T).ttiles >= 2
    W = O.synth_blocks(t, N, K, seed=9 + t)
    got = run_mmq(lib, t, W, N, K, X)
    want = oracle(port, t, W, N, K, X).astype(np.float64)
    assert np.isfinite(want).all()
    Wf = port.dequantize(t, W, N * K).reshape(N, K)
    bad = ~np.isfinite(got)
    err = np.abs(got.astype(np.float64) - want)
    ratio = np.where(bad, np.inf, err / np.maximum(bound(Wf, X), 1e-300))
    amax = np.abs(X).max(axis=1)
    worst = int(np.argmax(np.where(bad, 0, ratio).max(axis=1)))
    assert not bad.any() and (ratio <= 1).all(), (
        f"{int(bad.sum())} non-finite outputs in rows with amax {sorted(set(np.round(amax[bad.any(axis=1)], 1).tolist()))}; "
        f"worst finite bound ratio {np.max(np.where(bad, 0, ratio)):.3g} (row amax {amax[worst]:.3g})")
    zero = amax == 0
    assert np.all(got[zero] == 0.0)
    nmse = np.sum((got - want) ** 2, axis=1) / np.maximum(np.sum(want ** 2, axis=1), 1e-300)
    assert np.all(nmse[~zero] <= 4e-6), f"worst row NMSE {nmse[~zero].max():.3e} (row amax {amax[~zero][np.argmax(nmse[~zero])]:.3g})"


@pytest.mark.parametrize("t", KQ + BLK32, ids=lambda t: O.TYPE_NAME[t])
def test_mmq_weight_bit_patterns(cuda, lib, port, t):
    """Weight blocks synth_blocks never emits (oracle_lib.edge_blocks): quant bytes all 0x00 / all 0xFF, Q8_0 q = -128, Q6_K scale
    -128 with q = -32, 6-bit scales and mins of 63, d = 0 in every or every other block, under the module's bound."""
    N, K, T = (256, 512, 33) if t in KQ else (256, 448, 33)
    W = O.edge_blocks(t, N, K, seed=31 + t)
    X = np.random.default_rng(t).standard_normal((T, K)).astype(np.float32)
    got = run_mmq(lib, t, W, N, K, X)
    want = oracle(port, t, W, N, K, X)
    Wf = port.dequantize(t, W, N * K).reshape(N, K)
    check(got, want, Wf, X)
    if t in (O.Q8_0, O.Q6_K):                # no offset term: d = 0 in every block makes the row's weights zero
        assert np.all(got[:, 4::6] == 0.0)


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
    # different K groups, and the partial accumulators of a cut tile meet in dst by fp32 atomic adds
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


def test_prefill_ffn_down_input_beyond_fp16(cuda, pkg):
    """A one-layer llama whose ffn_norm weight (x300) drives silu(gate) * up, the ffn_down input the prefill builds inside its
    activation pass, past fp16's largest value: the prompt's last-token logits stay finite and within the prefill bar (NMSE 1e-3,
    tests/test_gpu_engine.py) of token-by-token decoding, whose integer-dot GEMV never had an fp16 activation."""
    tm = TinyModel(n_layer=1, n_embd=512, n_head=4, n_head_kv=2, n_ff=1024, n_vocab=256, n_ctx=32, arch="llama", ftype="q4_K_M", seed=11)
    kind, w = tm.tensors["blk.0.ffn_norm.weight"]
    tm.tensors["blk.0.ffn_norm.weight"] = (kind, (w * 300.0).astype(np.float32))
    toks = [(i * 31 + 7) % 256 for i in range(16)]
    eng = tm.load_engine(pkg)
    seq = np.zeros((len(toks), 256), np.float32)
    peak = 0.0
    for i, tok in enumerate(toks):
        eng.decode(int(tok), i, seq[i])
        g = eng.debug_read("g", 1024).astype(np.float64)
        u = eng.debug_read("u", 1024).astype(np.float64)
        with np.errstate(over="ignore"):            # exp(-g) = inf for g << 0: silu -> -0
            peak = max(peak, float(np.max(np.abs(g / (1.0 + np.exp(-g)) * u))))
    assert peak > FP16_MAX, f"max |silu(g) * u| {peak:.3g} does not pass fp16's range"
    eng.kv_clear()
    got = eng.prefill(toks, 0).copy()
    eng.close()
    assert np.isfinite(got).all(), f"{int((~np.isfinite(got)).sum())} non-finite logits"
    nmse = float(np.sum((got - seq[-1]) ** 2) / np.sum(seq[-1] ** 2))
    assert nmse < 1e-3, nmse
