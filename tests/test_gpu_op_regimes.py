"""-m gpu: the plugin's single-op kernels (ops.cu: k_soft_max, k_rope, k_rope_f16, k_get_rows, k_copy_strided, k_rms_norm_rows, k_silu,
k_binary) at the sizes and values where their behaviour changes, through the C ABI, against plain references: float64 numpy where the
op computes, bit-exact numpy / oracle_lib where it only moves, converts or dequantizes.  The shapes of each case are in the tables
below, next to the regime they reach:

* soft_max: a row staged in default shared memory (48 KB for static and dynamic together), staged after raising the kernel's opt-in
  limit (<= L floats, L = the device's opt-in shared memory per block minus the kernel's static shared memory), or computed in place
  in the output row in global memory (> L).  pb200_soft_max_smem reports the dynamic shared memory launch_soft_max gives a row
  length (its own decision, the same function), checked against L computed here from the device's properties.
* rope / rope_f16: angles past 1e5 rad, where sinf / cosf change argument reduction, and negative positions (the K-shift).
* get_rows: more ids than grid.y holds (65 535), and a table whose row offsets pass 4 GiB.
* the f16 store: every rounding tie, overflow to inf, subnormals, -0, inf and NaN, in the three layouts the KV cache uses.
* rms_norm / silu / binary: row lengths off the 256 grid, a long column of rows, squares that overflow or underflow, expf at its
  overflow edge, and broadcast periods."""
import ctypes as C
import ctypes.util
from fractions import Fraction

import numpy as np
import pytest
import torch

import oracle_lib as O
from gpu_util import dev_f32, dev_u8, ptr, sync

pytestmark = pytest.mark.gpu
f32 = np.float32


def nmse(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return float(np.sum((got - want) ** 2) / max(np.sum(want ** 2), 1e-30))


# ================================================================================================ soft_max
SM_H, SM_T, SM_T_PAD = 2, 3, 5      # scores [H][T][n_kv], mask rows T (read) of T_PAD (the rest NaN: never read)
SM_48K = 48 * 1024 // 4             # 12 288 floats: 48 KB, the default shared memory per block (static + dynamic)
SM_GLOBAL = 131072                  # 512 KB: above any per-block opt-in limit, so always the global-memory regime
SM_SCALES = (1.0, 0.088, 2.5, 0.0625)


def sm_cols(static, L):
    """(ncols, regime) at each boundary and one past it.  d48 = the last row length staged within the default 48 KB beside the
    kernel's static shared memory; L = the last one staged after the opt-in."""
    d48 = (SM_48K * 4 - static) // 4
    return ([(n, "default") for n in (1, 255, 256, 257, d48)] + [(n, "optin") for n in (d48 + 1, SM_48K - 1, SM_48K, SM_48K + 1, L - 1, L)]
            + [(L + 1, "global"), (SM_GLOBAL, "global")])


def sm_inputs(n_kv, seed):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((SM_H, SM_T, n_kv)) * 4).astype(np.float32)
    x[0, 0] += 80.0                 # rows whose maximum is far from 0
    x[1, 1] -= 80.0
    mask = np.zeros((SM_T_PAD, n_kv), np.float32)
    for t in range(SM_T):           # causal over n_past = n_kv - T, random holes; column 0 always visible
        mask[t, max(1, n_kv - SM_T + t + 1):] = -np.inf
        mask[t, rng.random(n_kv) < 0.03] = -np.inf
        mask[t, 0] = 0.0
    mask[SM_T:] = np.nan
    return x, mask


def sm_want64(x, mask, scale):
    """float64 softmax of the float32 pre-activation x * scale + mask (the kernel's two float32 roundings)."""
    s = (x * f32(scale)).astype(np.float32) + mask[:SM_T][None]
    s64 = s.astype(np.float64)
    e = np.where(np.isneginf(s64), 0.0, np.exp(s64 - s64.max(axis=-1, keepdims=True)))
    return e / e.sum(axis=-1, keepdims=True)


def sm_check(got, x, mask, scale, port, tag):
    n_kv = x.shape[-1]
    got = got.reshape(SM_H, SM_T, n_kv)
    assert np.isfinite(got).all(), tag
    masked = np.broadcast_to(np.isneginf(mask[:SM_T])[None], got.shape)
    assert np.all(got[masked].view(np.uint32) == 0), f"{tag}: a masked entry is not +0"
    want_port = np.stack([[port.soft_max(x[h, t], mask[t], scale) for t in range(SM_T)] for h in range(SM_H)])
    for name, want in (("port", want_port), ("float64", sm_want64(x, mask, scale))):
        err = float(np.max(np.abs(got - want)))
        assert err < 3e-7, (tag, name, err)
        assert nmse(got, want) < 1e-6, (tag, name, nmse(got, want))


def sm_run(lib, xd, md, y, n_kv, scale):
    lib.check(lib.c.pb200_soft_max(ptr(xd), ptr(md), ptr(y), C.c_int64(n_kv), C.c_int64(SM_H * SM_T), C.c_int64(SM_T), C.c_float(scale), None),
              f"soft_max of {n_kv} columns")


def sm_smem(lib, n_kv):
    """(dynamic, static) shared-memory bytes launch_soft_max gives rows of n_kv columns on the current device."""
    dyn, st = C.c_int64(-1), C.c_int64(-1)
    lib.check(lib.c.pb200_soft_max_smem(n_kv, C.byref(dyn), C.byref(st)), "soft_max_smem")
    return dyn.value, st.value


def test_soft_max_regimes(cuda, lib, port):
    """Every row length at a regime boundary, small to large and back (the kernel's shared-memory attribute only grows), one in-place
    call in the global-memory regime.  The launcher's regime for each length must switch exactly at L."""
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    assert SM_GLOBAL * 4 > optin
    _, static = sm_smem(lib, 1)
    assert 0 < static < 1024, static
    L = (optin - static) // 4
    assert SM_48K + 1 < L - 1
    cols = sm_cols(static, L)
    for n, regime in cols:
        dyn, st = sm_smem(lib, n)
        assert st == static and dyn == (0 if regime == "global" else 4 * n), (n, regime, dyn, st, L)
    x, mask = sm_inputs(SM_GLOBAL, 0)
    xd, md, y = dev_f32(x), dev_f32(mask), torch.full((x.size,), float("nan"), device="cuda")
    sm_run(lib, xd, md, y, SM_GLOBAL, 1.0)                # a long row first: the attribute is not raised for it
    order = cols + cols[::-1]
    data = {n: sm_inputs(n, n) for n, _ in cols}
    dev = {n: (dev_f32(xx), dev_f32(mm)) for n, (xx, mm) in data.items()}
    outs = [torch.full((data[n][0].size,), float("nan"), device="cuda") for n, _ in order]
    inplace = dev_f32(data[L + 1][0])

    for i, (n, _) in enumerate(order):
        sm_run(lib, dev[n][0], dev[n][1], outs[i], n, SM_SCALES[i % len(SM_SCALES)])
    sm_run(lib, inplace, dev[L + 1][1], inplace, L + 1, 0.088)
    sync()
    for i, (n, regime) in enumerate(order):
        sm_check(outs[i].cpu().numpy(), *data[n], SM_SCALES[i % len(SM_SCALES)], port, (n, regime, i))
    sm_check(inplace.cpu().numpy(), *data[L + 1], 0.088, port, (L + 1, "global in place"))
    sm_check(y.cpu().numpy(), x, mask, 1.0, port, (SM_GLOBAL, "global first"))


# ================================================================================================ rope
ROPE_POS = [0, 1, 8191, 8192, 32767, 65535, 105615, 131071]      # 105 615 rad and up: the slow argument reduction of sinf / cosf
ROPE_POS_F16 = ROPE_POS + [-1, -4096, -65536]                    # the K-shift rotates by pos = delta < 0
# name: (head_dim, n_dims, mode, freq_base, freq_scale, ext_factor, freq factors, n_ctx_orig)
ROPE_CASES = {
    "norm-128": (128, 128, 0, 500000.0, 1.0, 0.0, False, 8192),
    "norm-128-ff": (128, 128, 0, 500000.0, 1.0, 0.0, True, 8192),
    "neox-128": (128, 128, 2, 1000000.0, 1.0, 0.0, False, 32768),
    "neox-128-dims64": (128, 64, 2, 10000.0, 1.0, 0.0, False, 4096),
    "neox-80-dims32": (80, 32, 2, 10000.0, 1.0, 0.0, False, 4096),
    "neox-128-ff": (128, 128, 2, 1000000.0, 1.0, 0.0, True, 32768),
    "yarn-norm-128-dims64": (128, 64, 0, 10000.0, 0.25, 1.0, False, 4096),
    "yarn-neox-128-dims64": (128, 64, 2, 10000.0, 0.25, 1.0, False, 4096),
}
ROPE_HEADS = 3
BETA_FAST, BETA_SLOW, ATTN_FACTOR = 32.0, 1.0, 1.0
_libm = C.CDLL(ctypes.util.find_library("m"))
for _fn in ("powf", "logf"):
    getattr(_libm, _fn).restype = C.c_float
_libm.powf.argtypes = [C.c_float, C.c_float]
_libm.logf.argtypes = [C.c_float]


def _round_f32(q: Fraction) -> np.float32:
    """q rounded to the nearest float32, ties to even."""
    r = f32(float(q))
    cands = [r, np.nextafter(r, f32(np.inf)), np.nextafter(r, f32(-np.inf))]
    return min(cands, key=lambda c: (abs(Fraction(float(c)) - q), int(np.array(c).view(np.uint32)) & 1))


def _fma32(a, b, c) -> np.float32:
    return _round_f32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def rope_angles(npos, half, n_dims, base, freq_scale, ext_factor, ff, n_ctx_orig):
    """float32 angles th[pos][pair] as the kernel forms them: the running product of theta_scale (host powf), / freq factor, * freq_scale,
    and YaRN's mix.  With YaRN the mix a * b + c * d may be contracted to a fused multiply-add either way: every candidate is returned.
    Also the float64 attention factor."""
    theta_scale = f32(_libm.powf(f32(base), f32(-2.0) / f32(n_dims)))
    theta = np.array(npos, np.float32)
    th = np.empty((len(npos), half), np.float32)
    for j in range(half):
        th[:, j] = theta
        theta = theta * theta_scale
    extrap = th / (ff[:half] if ff is not None else f32(1.0))
    interp = f32(freq_scale) * extrap
    if ext_factor == 0.0:
        return [interp], float(ATTN_FACTOR)

    def corr_dim(n_rot):
        t = f32(f32(n_ctx_orig) / f32(f32(f32(n_rot) * f32(2)) * f32(np.pi)))
        return f32(f32(f32(n_dims) * f32(_libm.logf(t))) / f32(f32(2) * f32(_libm.logf(f32(base)))))
    lo = max(f32(0), f32(np.floor(corr_dim(BETA_FAST))))
    hi = min(f32(n_dims - 1), f32(np.ceil(corr_dim(BETA_SLOW))))
    y = (np.arange(half, dtype=np.float32) - lo) / max(f32(0.001), f32(hi - lo))
    mix = (f32(1) - np.minimum(f32(1), np.maximum(f32(0), y))) * f32(ext_factor)
    a, b = interp * (f32(1) - mix), extrap * mix
    plain = a + b
    fused = [np.array([[_fma32(interp[p, j], f32(1) - mix[j], b[p, j]) for j in range(half)] for p in range(len(npos))], np.float32),
             np.array([[_fma32(extrap[p, j], mix[j], a[p, j]) for j in range(half)] for p in range(len(npos))], np.float32)]
    return [plain] + fused, float(ATTN_FACTOR) * (1.0 + 0.1 * np.log(1.0 / freq_scale))


def rope_want64(x, th, mscale, n_dims, mode):
    """float64 rotation of float32 x [T][H][D] by the float32 angles th [T][n_dims / 2]; returns (y, tol) with
    tol = 2^-21 (|x0| + |x1|) mscale, the worst case of the kernel's arithmetic: cosf / sinf within 2 ulp on each term (2^-22 |x0| and
    2^-22 |x1|) plus the float32 roundings of mscale, c, s, the two products and the sum.  That is up to 4 float32 ulp of |x0| + |x1|
    rather than 2: a bar of 2 would fail correct kernels whenever the trig errors and the roundings add up.  The fast-math sines and
    cosines miss it by orders of magnitude at these angles."""
    half = n_dims // 2
    x64 = x.astype(np.float64)
    i0 = np.arange(half) if mode & 2 else 2 * np.arange(half)
    i1 = i0 + half if mode & 2 else i0 + 1
    c = (np.cos(th.astype(np.float64)) * mscale)[:, None, :]
    s = (np.sin(th.astype(np.float64)) * mscale)[:, None, :]
    x0, x1 = x64[..., i0], x64[..., i1]
    y = x64.copy()
    y[..., i0], y[..., i1] = x0 * c - x1 * s, x0 * s + x1 * c
    tol = np.zeros_like(y)
    t = 2.0 ** -21 * (np.abs(x0) + np.abs(x1)) * mscale
    tol[..., i0], tol[..., i1] = t, t
    return y, tol


def rope_setup(case, npos, seed):
    D, nd, mode, base, fs, ext, use_ff, n_ctx_orig = ROPE_CASES[case]
    rng = np.random.default_rng(seed)
    ff = (1.0 + rng.uniform(0, 7, nd // 2)).astype(np.float32) if use_ff else None
    ths, mscale = rope_angles(npos, nd // 2, nd, base, fs, ext, ff, n_ctx_orig)
    return D, nd, mode, base, fs, ext, ff, n_ctx_orig, ths, mscale, rng


@pytest.mark.parametrize("case", list(ROPE_CASES))
def test_rope_long_positions(cuda, lib, port, case):
    D, nd, mode, base, fs, ext, ff, n_ctx_orig, ths, mscale, rng = rope_setup(case, ROPE_POS, 1)
    T, H = len(ROPE_POS), ROPE_HEADS
    x = rng.standard_normal((T, H, D)).astype(np.float32)
    pos = np.array(ROPE_POS, np.int32)
    xd, pd, fd = dev_f32(x), torch.from_numpy(pos).cuda(), (dev_f32(ff) if ff is not None else None)
    y = torch.full((x.size,), float("nan"), device="cuda")
    lib.check(lib.c.pb200_rope(ptr(xd), ptr(y), T, H, D, nd, mode, ptr(pd), C.c_float(base), C.c_float(fs), C.c_float(ext), C.c_float(ATTN_FACTOR),
                               C.c_float(BETA_FAST), C.c_float(BETA_SLOW), n_ctx_orig, ptr(fd) if fd is not None else None, None), "rope")
    sync()
    got = y.cpu().numpy().reshape(T, H, D)
    assert np.array_equal(got[..., nd:].view(np.uint32), x[..., nd:].view(np.uint32)), "the dims past n_dims are copied"
    err = None
    for th in ths:                   # within the bar of the float64 rotation by one of the angles the kernel may form
        want, tol = rope_want64(x, th, mscale, nd, mode)
        e = np.abs(got.astype(np.float64) - want) / np.maximum(tol, 1e-300)
        err = e if err is None else np.minimum(err, e)
    worst = np.unravel_index(np.argmax(err), err.shape)
    assert err.max() <= 1.0, (case, "pos", ROPE_POS[worst[0]], "dim", worst[2], float(err.max()))
    # the port (glibc cosf / sinf of the same angle) with the established bar, where the kernel's angle can only be the port's
    same = np.all([ths[0] == t for t in ths], axis=0)
    want = np.stack([port.rope(x[i], H, D, mode, int(pos[i]), freq_base=base, freq_scale=fs, n_ctx_orig=n_ctx_orig, freq_factors=ff,
                               ext_factor=ext, beta_fast=BETA_FAST, beta_slow=BETA_SLOW, n_dims=nd) for i in range(T)])
    half = nd // 2
    i0 = np.arange(half) if mode & 2 else 2 * np.arange(half)
    i1 = i0 + half if mode & 2 else i0 + 1
    for ii in (i0, i1):
        d = np.abs(got[..., ii] - want[..., ii])[np.broadcast_to(same[:, None, :], (T, H, half))]
        assert d.max() < 4e-6 * np.max(np.abs(x)), (case, float(d.max()))
    if len(ths) == 1:
        assert np.max(np.abs(got - want)) < 4e-6 * np.max(np.abs(x))


@pytest.mark.parametrize("case", list(ROPE_CASES))
def test_rope_f16_long_and_negative_positions(cuda, lib, case):
    """f16 rows in place (the K-shift): each output is the f16 rounding of a value within the float32 bar of the float64 rotation.  So
    it equals numpy's f16 rounding of the float64 result, or a neighbour of it where that result lies within the float32 bar (up to 4
    float32 ulp, see rope_want64) of an f16 rounding tie."""
    D, nd, mode, base, fs, ext, ff, n_ctx_orig, ths, mscale, rng = rope_setup(case, ROPE_POS_F16, 2)
    T, H = len(ROPE_POS_F16), ROPE_HEADS
    x16 = rng.standard_normal((T, H, D)).astype(np.float16)
    pos = np.array(ROPE_POS_F16, np.int32)
    yd, pd, fd = torch.from_numpy(x16.copy()).cuda(), torch.from_numpy(pos).cuda(), (dev_f32(ff) if ff is not None else None)
    lib.check(lib.c.pb200_rope_f16(ptr(yd), ptr(yd), T, H, D, nd, mode, ptr(pd), C.c_float(base), C.c_float(fs), C.c_float(ext),
                                   C.c_float(ATTN_FACTOR), C.c_float(BETA_FAST), C.c_float(BETA_SLOW), n_ctx_orig,
                                   ptr(fd) if fd is not None else None, None), "rope_f16")
    sync()
    got = yd.cpu().numpy().reshape(T, H, D)
    assert np.array_equal(got[..., nd:].view(np.uint16), x16[..., nd:].view(np.uint16))
    g = got[..., :nd].astype(np.float64)
    ok = np.zeros(g.shape, bool)
    for th in ths:
        want, tol = rope_want64(x16.astype(np.float32), th, mscale, nd, mode)
        want, tol = want[..., :nd], tol[..., :nd]
        # f16 rounding is monotone: the f16 values of the whole interval want +- tol lie between the roundings of its ends
        lo, hi = (want - tol).astype(np.float16).astype(np.float64), (want + tol).astype(np.float16).astype(np.float64)
        ok |= (lo <= g) & (g <= hi)
    assert ok.all(), (case, np.argwhere(~ok)[:5].tolist())   # so off the f16 rounding of the float64 value only within the bar of a tie


# ================================================================================================ get_rows
GET_ROWS_N_IDS = [65535, 65536, 200003]   # gridDim.y holds at most 65 535 ids
GET_ROWS_TABLE = 37                       # table rows
BIG_TABLE = (132000, 8192)                # f32: rows past 131 072 start beyond 4 GiB


def get_rows_ids(n, n_rows, seed):
    ids = np.random.default_rng(seed).integers(0, n_rows, n).astype(np.int32)
    ids[:4] = [0, n_rows - 1, 0, n_rows - 1]
    ids[-2:] = [n_rows - 1, 0]
    return ids


@pytest.mark.parametrize("n_ids", GET_ROWS_N_IDS)
@pytest.mark.parametrize("t", O.QUANT_TYPES + [O.F16, O.F32], ids=lambda t: O.TYPE_NAME[t])
def test_get_rows_many_ids(cuda, lib, port, t, n_ids):
    K = 256 if t in O.KQ else 288            # 288: a row that is not a multiple of the CTA's 256 elements
    N = GET_ROWS_TABLE
    rng = np.random.default_rng(t)
    if t == O.F32:
        tab = rng.standard_normal((N, K)).astype(np.float32); want_tab = tab
    elif t == O.F16:
        tab = rng.standard_normal((N, K)).astype(np.float16); want_tab = tab.astype(np.float32)
    else:
        tab = O.synth_blocks(t, N, K, seed=t); want_tab = port.dequantize(t, tab, K)
    ids = get_rows_ids(n_ids, N, n_ids + t)
    idd, tabd = torch.from_numpy(ids).cuda(), dev_u8(tab)
    y = torch.full((n_ids, K), float("nan"), device="cuda")
    lib.check(lib.c.pb200_get_rows(t, ptr(tabd), K, ptr(idd), n_ids, ptr(y), None), "get_rows")
    sync()
    want = torch.from_numpy(want_tab).cuda()[idd.long()]
    assert torch.equal(y.view(torch.int32), want.view(torch.int32)), (O.TYPE_NAME[t], n_ids)


def test_get_rows_table_past_4gib(cuda, lib):
    N, K = BIG_TABLE
    g = torch.Generator(device="cuda").manual_seed(0)
    tab = torch.randn((N, K), device="cuda", generator=g)
    ids = np.concatenate([[0, N - 1, 131071, 131072, 65535, 65536, N - 1], np.random.default_rng(3).integers(0, N, 250)]).astype(np.int32)
    assert (int(ids.max()) * K * 4) >> 32 > 0
    idd = torch.from_numpy(ids).cuda()
    y = torch.full((len(ids), K), float("nan"), device="cuda")
    lib.check(lib.c.pb200_get_rows(O.F32, ptr(tab), K, ptr(idd), len(ids), ptr(y), None), "get_rows")
    sync()
    assert torch.equal(y.view(torch.int32), tab[idd.long()].view(torch.int32))
    del tab
    torch.cuda.empty_cache()


# ================================================================================================ the f16 store
def f16_store_values():
    """float32 values whose f16 rounding is an edge: every tie between adjacent f16 values (normals and subnormals) and one float32 ulp on
    either side, the overflow threshold, subnormals down to 2^-24 and the 2^-25 tie, -0, +-inf, NaN."""
    h = np.arange(0, 0x7C00, dtype=np.uint16).view(np.float16).astype(np.float32)          # +0 .. 65 504
    ties = (h[:-1] + (h[1:] - h[:-1]) / 2).astype(np.float32)                             # exact in float32
    near = np.concatenate([np.nextafter(ties, f32(np.inf)), np.nextafter(ties, f32(-np.inf))])
    sub = (np.arange(1, 1024, dtype=np.float32) * f32(2.0 ** -24))
    special = np.array([65504.0, 65519.99, 65520.0, 1e5, 3.4e38, 2.0 ** -24, 2.0 ** -25, 1.5 * 2.0 ** -25, 2.0 ** -26, 1e-30, 0.0,
                        np.inf, np.nan], np.float32)
    special = np.concatenate([special, np.nextafter(f32(2.0 ** -25), f32(1)).reshape(1), np.nextafter(f32(65520.0), f32(0)).reshape(1)])
    v = np.concatenate([h, ties, near, sub, special])
    v = np.concatenate([v, -v])                                                           # -0, -inf, every negative tie
    return v.astype(np.float32)


def f16_check(got, src, tag):
    want = src.astype(np.float16)
    nan = np.isnan(src)
    assert np.array_equal(np.isnan(got), nan), tag
    assert np.array_equal(got[~nan].view(np.uint16), want[~nan].view(np.uint16)), (tag, src[~nan][got[~nan].view(np.uint16)
                                                                                               != want[~nan].view(np.uint16)][:8])


def test_f16_store_rounding(cuda, lib):
    v = f16_store_values()
    E = 256
    v = np.concatenate([v, np.zeros(-v.size % (2 * E), np.float32)])
    R = v.size // E
    arr = lambda a: (C.c_int64 * 4)(*a)  # noqa: E731
    src = v.reshape(R, E)
    xd = dev_f32(src)
    sentinel = 0x7E55                                                                    # a NaN pattern no store writes
    # flat K-cache store: rows [c0, c0 + R) of an [n_ctx][E] f16 cache
    n_ctx, c0 = R + 7, 3
    kc = torch.full((n_ctx * E,), sentinel, dtype=torch.int16, device="cuda")
    lib.check(lib.c.pb200_copy_strided(ptr(xd), C.c_void_p(kc.data_ptr() + c0 * E * 2), 1, arr([E, R, 1, 1]), arr([4, 4 * E, 4 * E * R, 4 * E * R]),
                                       arr([2, 2 * E, 2 * E * n_ctx, 2 * E * n_ctx]), None), "K store")
    # transposed V-cache store: element (token r, feature e) to [e][c0 + r] of an [E][n_ctx] f16 cache
    n_ctx_v, cv = R + 5, 2
    vc = torch.full((E * n_ctx_v,), sentinel, dtype=torch.int16, device="cuda")
    lib.check(lib.c.pb200_copy_strided(ptr(xd), C.c_void_p(vc.data_ptr() + cv * 2), 1, arr([R, E, 1, 1]), arr([4 * E, 4, 4 * E * R, 4 * E * R]),
                                       arr([2, 2 * n_ctx_v, 2 * E * n_ctx_v, 2 * E * n_ctx_v]), None), "V store")
    # cont of a permuted (0, 2, 1, 3) view: x [D2][D1][D0] read as [D1][D2][D0]
    D0, D1 = 64, 8
    D2 = v.size // (D0 * D1)
    x3 = v.reshape(D2, D1, D0)
    pc = torch.full((v.size,), sentinel, dtype=torch.int16, device="cuda")
    lib.check(lib.c.pb200_copy_strided(ptr(xd), ptr(pc), 1, arr([D0, D2, D1, 1]), arr([4, 4 * D0 * D1, 4 * D0, 4 * v.size]),
                                       arr([2, 2 * D0, 2 * D0 * D2, 2 * v.size]), None), "cont")
    sync()
    k = kc.cpu().numpy().reshape(n_ctx, E)
    assert np.all(k[:c0] == sentinel) and np.all(k[c0 + R:] == sentinel)
    f16_check(k[c0:c0 + R].view(np.float16), src, "K store")
    vv = vc.cpu().numpy().reshape(E, n_ctx_v)
    assert np.all(vv[:, :cv] == sentinel) and np.all(vv[:, cv + R:] == sentinel)
    f16_check(vv[:, cv:cv + R].view(np.float16).T, src, "V store")
    f16_check(pc.cpu().numpy().view(np.float16).reshape(D1, D2, D0), x3.transpose(1, 0, 2), "cont of a permuted view")


# ================================================================================================ rms_norm, silu, binary
RMS_ROWS = [(1, 3), (255, 3), (257, 3), (3584, 2), (5120, 2), (18944, 2), (8192, 4096)]   # (columns, rows); 4 096 rows: a long grid.x
RMS_EPS = 1e-5


@pytest.mark.parametrize("n,rows", RMS_ROWS)
def test_rms_norm_row_shapes(cuda, lib, port, n, rows):
    x = (np.random.default_rng(n + rows).standard_normal((rows, n)) * 3).astype(np.float32)
    xd, y = dev_f32(x), torch.full((rows * n,), float("nan"), device="cuda")
    lib.check(lib.c.pb200_rms_norm(ptr(xd), ptr(y), n, rows, C.c_float(RMS_EPS), None), "rms_norm")
    sync()
    got = y.cpu().numpy().reshape(rows, n)
    want = np.stack([port.rms_norm(x[i], RMS_EPS) for i in range(rows)])
    assert np.isfinite(got).all()
    assert np.max(np.abs(got - want) / np.maximum(np.abs(want), 1e-6)) < 3e-7


def test_rms_norm_extreme_magnitudes(cuda, lib, port):
    """|x| ~ 1e19: squares up to 1e38 stay finite; one square past FLT_MAX makes the sum inf and the CPU backend's row +-0.  |x| ~ 1e-30:
    every square underflows to 0 and eps alone sets the scale."""
    n = 4096
    rng = np.random.default_rng(9)
    sign = np.where(rng.random(n) < 0.5, -1.0, 1.0)
    big = (sign * rng.uniform(0.5, 1.0, n) * 1e19).astype(np.float32)
    over = big.copy(); over[100] = 2e19
    tiny = (sign * rng.uniform(0.5, 1.0, n) * 1e-30).astype(np.float32)
    x = np.stack([big, over, tiny])
    xd, y = dev_f32(x), torch.full((x.size,), float("nan"), device="cuda")
    lib.check(lib.c.pb200_rms_norm(ptr(xd), ptr(y), n, 3, C.c_float(RMS_EPS), None), "rms_norm")
    sync()
    got = y.cpu().numpy().reshape(3, n)
    want = np.stack([port.rms_norm(r, RMS_EPS) for r in x])
    assert np.isfinite(got).all() and np.isfinite(want).all()
    assert np.max(np.abs(got[0] - want[0]) / np.abs(want[0])) < 3e-7
    assert np.all(got[1] == 0) and np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32))   # signed zeros, as the CPU gives
    assert np.array_equal(got[2].view(np.uint32), want[2].view(np.uint32))


# bit-exact: exp(-x) vanishes against 1 (x >= 20), overflows to inf (x <= -89: the result is -0), or x is 0, inf or subnormal
SILU_EXACT = [88.7, 89.0, 88.72, 20.0, 1e4, -89.0, -100.0, -1e4, np.inf, -np.inf, -0.0, 0.0, 1e-40, -1e-40]
# the result is x / expf(-x) with expf just below its overflow: within expf's 2 ulp of the correctly rounded exp
SILU_EXPF = [-88.7, -88.72, -20.0]


def test_silu_edges(cuda, lib):
    x = np.array(SILU_EXACT + SILU_EXPF, np.float32)
    xd, y = dev_f32(x), torch.full((x.size,), float("nan"), device="cuda")
    lib.check(lib.c.pb200_silu(ptr(xd), ptr(y), C.c_int64(x.size), None), "silu")
    sync()
    got = y.cpu().numpy()
    with np.errstate(over="ignore", invalid="ignore"):
        e = np.exp(-x.astype(np.float64)).astype(np.float32)           # exp of the float32 x, correctly rounded to float32
        want = x / (f32(1) + e)
    n = len(SILU_EXACT)
    ok = ~np.isnan(want[:n])
    assert np.array_equal(np.isnan(got[:n]), ~ok) and np.sum(~ok) == 1                  # x = -inf: -inf / inf
    assert np.array_equal(got[:n][ok].view(np.uint32), want[:n][ok].view(np.uint32)), list(zip(x[:n][ok], got[:n][ok], want[:n][ok]))
    ulps = np.abs(got[n:].view(np.int32).astype(np.int64) - want[n:].view(np.int32).astype(np.int64))
    assert np.all(np.sign(got[n:]) == np.sign(want[n:])) and np.all(ulps <= 2), list(zip(x[n:], got[n:], want[n:]))


BIN_N = 3 * 33333                                   # 99 999: not a multiple of 256
BIN_PERIODS = [1, 7, BIN_N // 3, BIN_N]


@pytest.mark.parametrize("nb", BIN_PERIODS)
@pytest.mark.parametrize("op", [0, 1], ids=["add", "mul"])
def test_binary_broadcast_periods(cuda, lib, op, nb):
    rng = np.random.default_rng(nb + op)
    a = rng.standard_normal(BIN_N).astype(np.float32)
    b = rng.standard_normal(nb).astype(np.float32)
    ad, bd, y = dev_f32(a), dev_f32(b), torch.full((BIN_N,), float("nan"), device="cuda")
    lib.check(lib.c.pb200_binary(C.c_int(op), ptr(ad), ptr(bd), ptr(y), C.c_int64(BIN_N), C.c_int64(nb), None), "binary")
    sync()
    bb = b[np.arange(BIN_N) % nb]
    want = a + bb if op == 0 else a * bb
    assert np.array_equal(y.cpu().numpy().view(np.uint32), want.view(np.uint32))
