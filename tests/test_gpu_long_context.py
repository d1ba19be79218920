"""Attention over long rows of visible cells, 16 k to 131 k, where short rows cannot show an error:

  * subnormal probabilities: the FA-off arithmetic rounds every probability to f16 before P.V, and 2^-14 = 1 / 16 384 is the smallest
    normal f16.  1 / n still rounds to 2^-14 up to n = 16 392, so a flat row of 16 393 cells or more puts every probability into f16
    subnormals.  k_attn2 stops below that length (pb200_attn_ggml_max_cells()); every path past it is checked here;
  * a dropped, duplicated or misindexed cell: in a random row of 50 k cells one cell holds about 2e-5 of the mass, far under any
    fp32-order bar, so only a row in which chosen cells carry real mass catches it;
  * summation length: the derived bars of k_flash_attn_ext and k_mul_mat_f16 grow with n_kv.

Every row is one of four designs, named in the test id:
  flat     K = 0: every visible cell has the same score, V = 1 + 0.1 N(0, 1);
  needles  the random background plus planted cells (0, 31, 32 767 / 32 768, 65 535 / 65 536 where the row reaches them, the first
           cell of a final partial 32-group or the last cell of the last full one, and the last visible cell) whose scores give each
           a share of the mass between 0.05 and 0.5, with V rows of +-3: a dropped needle moves the output by >= 0.05 |V|;
  sink     one early cell 30 above every other score: every other p rounds to f16 zero, the output is that cell's V row;
  random   the background of Shard.fill (K ~ 0.5 N, V ~ N), the control.

Ops through the C ABI, each against float64 with the kernel's roundings and, on sampled rows, the oracle port:
  * pb200_attn_decode (k_attn_rows<false>) up to the engine's context limit at 64 / 8 and 8 / 2 heads;
  * pb200_attn_prefill on its per-row rung at gqa 8, tokens of one call seeing rows of different lengths;
  * pb200_flash_attn_ext to 131 072 cells, contiguous and as the FA-on graph's views, causal and multi-sequence masks;
  * the plugin's FA-off chain past the fused limit: pb200_mul_mat_f16 KQ -> pb200_soft_max -> pb200_mul_mat_f16 KQV;
and the engine's decode step (k_attn_rows<true>) at positions to its context limit, every launch through check_step, and its prompt
step at pos0 ~ 40 000 bit-identical to the same layer composed from single ops.

Bars are the suite's: the fp32-order bar (3e-4 max, 2e-5 mean per token) plus f16_flip_slack for the FA-off paths, the derived bar
of test_flash_attn_ext_vs_float64 and of test_mul_mat_f16_vs_float64.  For every needle row the test also shows that the bar it
uses is tighter than the move a single dropped needle causes."""
import numpy as np
import pytest
import torch

from gpu_util import dev_f32, ptr, sync
from test_gpu_attention import U, _bind, _i64, engine_max_ctx  # noqa: F401  (engine_max_ctx: fixture)
from test_gpu_decode_layers import (F16_NAN, case_model, check_launches, check_step, f16_bits, f16_flip_slack, layer_types, load_shard,
                                    rope_dev, step, uses_attn2)
from test_gpu_kv_shift import kv_tensors
from test_gpu_prefill_attention import MAX_ERR, MEAN_ERR, attn_batch_plan, sample_tokens
from test_gpu_prefill_layers import Compose, check_cache, check_logits, engine_hidden, engine_kv
from test_gpu_prefill_layers import check_bits as pf_check_bits
from tiny_model import TinyModel

D = 128
F16_MIN_NORMAL = 2.0 ** -14
DESIGNS = ("flat", "needles", "sink", "random")
SINK_CELL = 3
NEEDLE_V = 3.0
SCALE = float(np.float32(1.0) / np.sqrt(np.float32(D)))


# ---------------------------------------------------------------------------------------------------------------- row designs
def needle_cells(n_first, n_last):
    """Needle cells of a row whose tokens see [0, n_first) up to [0, n_last): cells every token sees (0, 31: the last of warp 7's first
    four-load group, 32 767 / 32 768, 65 535 / 65 536, the first cell of a final partial 32-group, or the last cell of the last full
    group) and the last cell, which only the last token's row holds."""
    c = {0, 31}
    for b in (32767, 32768, 65535, 65536):
        if b < n_first - 1:
            c.add(b)
    c.add(n_first // 32 * 32 if n_first % 32 else n_first - 1)
    c.add(n_last - 1)
    return sorted(c)


_BACKGROUND = {}


def background(n, HK):
    """K (0.5 N(0, 1)) and V (N(0, 1)) rows [n][HK][D] in f16, the background of Shard.fill.  Drawn once per HK at the longest n asked
    for so far and sliced: drawing 100 M normals per case would dominate the file's time."""
    if HK not in _BACKGROUND or _BACKGROUND[HK][0].shape[0] < n:
        rng = np.random.default_rng(1000 + HK)
        _BACKGROUND[HK] = tuple((rng.standard_normal((n, HK, D), dtype=np.float32) * a).astype(np.float16) for a in (0.5, 1.0))
    K, V = _BACKGROUND[HK]
    return K[:n].copy(), V[:n].copy()


def make_row(design, n, H, HK, T, n_first, seed):
    """q [T][H][D] f32, K / V [n][HK][D] f16 and the planted cells of one design; tokens see [0, n_first) up to [0, n).  For needles
    and sink the q heads of a kv group are one direction u plus 0.05 N(0, 1) noise, and the planted K rows lie along u: their scores
    are the same to within a few hundredths for every head and token of the group."""
    rng = np.random.default_rng(seed)
    g = H // HK
    K, V = background(n, HK)
    q = rng.standard_normal((T, HK, g, D), dtype=np.float32)
    cells = []
    if design == "flat":
        K[:] = 0
        V = (1 + 0.1 * V.astype(np.float32)).astype(np.float16)
    elif design in ("needles", "sink"):
        u = rng.standard_normal((HK, D))
        q = (u[None, :, None, :] + 0.05 * rng.standard_normal((T, HK, g, D))).astype(np.float32)
        cells = needle_cells(n_first, n) if design == "needles" else [SINK_CELL]
        for hk in range(HK):
            s_bg = SCALE * (K[:, hk].astype(np.float64) @ u[hk])
            bg = np.ones(n, bool)
            bg[cells] = False
            if design == "needles":     # share w each, 0.3 of the mass left to the background of the shortest row
                w = 0.7 / len(cells)
                s_bg = s_bg[:n_first][bg[:n_first]]
                lse = s_bg.max() + np.log(np.sum(np.exp(s_bg - s_bg.max())))
                s = lse + np.log(w / 0.3)
            else:
                s = s_bg[bg].max() + 30.0
            for c in cells:
                K[c, hk] = s / SCALE * u[hk] / (u[hk] @ u[hk])
                V[c, hk] = NEEDLE_V * np.sign(rng.standard_normal(D))
    return q.reshape(T, H, D), K, V, cells


# ---------------------------------------------------------------------------------------------------------------- references
def check_heads(H, HK):
    """Heads checked on the host where all of them would cost too much: the first and last of group 0, one in a middle group, the last."""
    g = H // HK
    return sorted({0, g - 1, g * (HK // 2) + g // 2, H - 1})


def attn64(q, K64, V64, vis, f16_p):
    """float64 attention of heads q [g][D] (f32, rounded to f16 as every kernel does) over one kv head's cells [n][D] (float64 of the
    f16 values) where vis (bool [n]) holds.  f16_p: the FA-off roundings, p = f16(e float32(1 / sum e)).  Returns the output [g][D]
    and the exact probabilities [g][n]."""
    qh = q.astype(np.float16).astype(np.float64)
    s = np.where(vis[None, :], (qh @ K64.T) * SCALE, -np.inf)
    e = np.exp(s - s.max(axis=1, keepdims=True))
    tot = e.sum(axis=1, keepdims=True)
    p = e / tot
    if f16_p:
        pr = (e * (1.0 / tot).astype(np.float32).astype(np.float64)).astype(np.float16).astype(np.float64)
    else:
        pr = p
    return pv(pr, V64), p


def pv(p, V):
    """p [g][n] . V [n][D], as V^T p^T: OpenBLAS takes the other order of this long-K product about a hundred times slower."""
    return (V.T @ p.T).T


def check_design(what, design, got, want, p, V64, cells, tol):
    """Design-specific claims on one group of heads (got / want [g][D], p [g][n] exact): planted shares in [0.05, 0.5] and a bar tighter
    than the move of one dropped needle; the sink's output is its V row to within the f16 rounding of p ~ 1."""
    if design == "needles":
        vis = [c for c in cells if p[:, c].min() > 0]
        assert vis, what
        share = p[:, vis]
        assert share.min() >= 0.05 and share.max() <= 0.5, (what, share.min(), share.max())
        # dropping needle c leaves (out - p_c V_c) / (1 - p_c): it moves the output by p_c |V_c - out| / (1 - p_c)
        move = min(np.max(np.abs(p[:, c:c + 1] * (V64[c][None, :] - want)) / (1 - p[:, c:c + 1])) for c in vis)
        assert move > tol, (what, move, tol)
    elif design == "sink":
        v = V64[SINK_CELL][None, :]
        assert np.all(p[:, SINK_CELL] > 1 - 1e-6), what
        assert np.max(np.abs(got - v) - 2.0 ** -11 * np.abs(v)) < MAX_ERR, (what, np.max(np.abs(got - v)))


def check_fa_off(what, got, want, q, K16, V16, g):
    """One token's heads of one kv group [g][D]: the fp32-order bar, plus f16_flip_slack where a probability sits at an f16 rounding
    boundary (computed only when the plain bar is exceeded: it costs a pass over every cell and dimension).  Returns the largest
    per-element bar it applied."""
    assert np.isfinite(got).all(), what
    err = np.abs(got.astype(np.float64) - want)
    if err.max() < MAX_ERR and err.mean() < MEAN_ERR:
        return MAX_ERR
    slack = f16_flip_slack(q.reshape(-1), K16.view(np.uint16), V16.view(np.uint16), g, 1, SCALE).reshape(g, D)
    assert np.all(err < MAX_ERR + slack) and err.mean() < MEAN_ERR + slack.mean(), \
        (what, err.max(), err.mean(), slack.max(), slack.mean())
    return MAX_ERR + float(slack.max())


def check_port(port, what, got, q, K16, V16, g):
    """The oracle port's attention_decode over the visible cells of one kv group, under the same bar."""
    want = port.attention_decode(q.reshape(-1), K16.view(np.uint16), V16.view(np.uint16), g, 1, D, K16.shape[0], SCALE).reshape(g, D)
    check_fa_off(what + " vs port", got, want.astype(np.float64), q, K16, V16, g)


# ---------------------------------------------------------------------------------------------------------------- 1. pb200_attn_decode
DECODE_NKV = (16383, 16385, 32769, 40000, "max")
DECODE_HEADS = ((64, 8), (8, 2))
DECODE_CASES = [(n, DECODE_HEADS[(i + j) % 2], d) for j, n in enumerate(DECODE_NKV) for i, d in enumerate(DESIGNS)]   # both geometries at every n_kv


def _nkv(n, engine_max):
    return engine_max if n == "max" else n


@pytest.mark.gpu
@pytest.mark.parametrize("n_kv,heads,design", DECODE_CASES, ids=[f"kv{n}-h{h[0]}x{h[1]}-{d}" for n, h, d in DECODE_CASES])
def test_attn_decode_long_rows(cuda, lib, port, engine_max_ctx, n_kv, heads, design):
    """k_attn_rows<false> with n_ctx = n_kv, so the score row fills the shared memory it was sized for: the heads of three kv groups
    against float64 with the kernel's roundings, two against the port, and every case past k_attn2's cell limit."""
    n = _nkv(n_kv, engine_max_ctx)
    H, HK = heads
    g = H // HK
    assert n > lib.c.pb200_attn_ggml_max_cells(), (n, lib.c.pb200_attn_ggml_max_cells())
    q, K, V, cells = make_row(design, n, H, HK, 1, n, seed=n * 10 + H + DESIGNS.index(design))
    out = torch.full((H * D,), float("nan"), device="cuda")
    qd, kd, vd = dev_f32(q), torch.from_numpy(K.reshape(n, HK * D)).cuda(), torch.from_numpy(V.reshape(n, HK * D)).cuda()
    pos = torch.tensor([n - 1], dtype=torch.int32, device="cuda")
    lib.check(lib.c.pb200_attn_decode(ptr(qd), ptr(kd), ptr(vd), ptr(out), H, HK, D, ptr(pos), n, SCALE, None), "attn_decode")
    sync()
    got = out.cpu().numpy().reshape(HK, g, D)
    vis = np.ones(n, bool)
    for hk in sorted({0, HK // 2, HK - 1}):       # kv groups sampled: the kernel's indexing is the same for every head
        K64, V64 = K[:, hk].astype(np.float64), V[:, hk].astype(np.float64)
        qg = q[0, hk * g:(hk + 1) * g]
        want, p = attn64(qg, K64, V64, vis, True)
        what = f"kv head {hk}"
        bar = check_fa_off(what, got[hk], want, qg, K[:, hk], V[:, hk], g)
        check_design(what, design, got[hk], want, p, V64, cells, bar)
        if hk == 0:
            check_port(port, what, got[hk], qg, np.ascontiguousarray(K[:, hk]), np.ascontiguousarray(V[:, hk]), g)


# ---------------------------------------------------------------------------------------------------------------- 2. pb200_attn_prefill
PREFILL_ENDS = (6017, 20000, "max")          # pos0 + T
PREFILL_CASES = [(e, t, d) for e in PREFILL_ENDS for t in (1, 37) for d in DESIGNS] + \
                [(6017, 512, "needles"), (20000, 512, "flat"), ("max", 512, "random")]
PREFILL_G = 8                                # gqa 8, one kv head


@pytest.mark.gpu
@pytest.mark.parametrize("end,n_tok,design", PREFILL_CASES, ids=[f"end{e}-t{t}-{d}" for e, t, d in PREFILL_CASES])
def test_attn_prefill_long_rows(cuda, lib, port, engine_max_ctx, end, n_tok, design):
    """The per-row rung (k_attn_rows<false>, one CTA per (head, token)) with token t at pos0 + t and n_kv_max = pos0 + T: every token
    against float64 (every head up to 37 tokens, the first and last head at 512), the sampled tokens against the port.  Rows past the
    last position are f16 NaN."""
    end = _nkv(end, engine_max_ctx)
    H, HK, g = PREFILL_G, 1, PREFILL_G
    pos0 = end - n_tok
    assert attn_batch_plan(H, HK, end) == "rows"
    q, K, V, cells = make_row(design, end, H, HK, n_tok, pos0 + 1, seed=end + n_tok * 7 + DESIGNS.index(design))
    n_buf = (end + 31) // 32 * 32 + 32
    Kc = np.full((n_buf, D), np.nan, np.float16)
    Vc = np.full((n_buf, D), np.nan, np.float16)
    Kc[:end], Vc[:end] = K[:, 0], V[:, 0]
    pos = (pos0 + np.arange(n_tok)).astype(np.int32)
    out = torch.full((n_tok, H * D), float("nan"), device="cuda")
    qd, kd, vd = dev_f32(q), torch.from_numpy(Kc).cuda(), torch.from_numpy(Vc).cuda()
    pd = torch.from_numpy(pos).cuda()
    lib.check(lib.c.pb200_attn_prefill(ptr(qd), ptr(kd), ptr(vd), ptr(out), H, HK, D, ptr(pd), n_tok, end, SCALE, None), "attn_prefill")
    sync()
    got = out.cpu().numpy().reshape(n_tok, g, D)
    K64, V64 = K[:, 0].astype(np.float64), V[:, 0].astype(np.float64)
    hs = list(range(g)) if n_tok <= 64 else [0, g - 1]        # heads sampled at 512 tokens: the float64 rows dominate the file's time
    for t in range(n_tok):
        n = int(pos[t]) + 1
        want, p = attn64(q[t, hs], K64[:n], V64[:n], np.ones(n, bool), True)
        what = f"token {t} (row of {n} cells)"
        bar = check_fa_off(what, got[t, hs], want, q[t, hs], K[:n, 0], V[:n, 0], len(hs))
        if t == n_tok - 1:
            check_design(what, design, got[t, hs], want, p, V64[:n], cells, bar)
    for t in sample_tokens(n_tok, "rows"):
        n = int(pos[t]) + 1
        check_port(port, f"token {t}", got[t], q[t], np.ascontiguousarray(K[:n, 0]), np.ascontiguousarray(V[:n, 0]), g)


# ---------------------------------------------------------------------------------------------------------------- 3. FLASH_ATTN_EXT and the FA-off chain
FA_NKV = (16384, 32768 + 17, 65536, 131072)
FA_CASES = []
for j, n in enumerate(FA_NKV):
    for i, d in enumerate(DESIGNS):
        FA_CASES.append((n, ((64, 8), (32, 8))[i % 2], (1, 32)[i // 2], ("contig", "views")[(i + j) % 2], ("causal", "holes")[(i // 2 + j) % 2], d))


def fa_case_id(c):
    n, h, t, lay, mk, d = c
    return f"kv{n}-h{h[0]}x{h[1]}-t{t}-{lay}-{mk}-{d}"


def long_mask(kind, n_kv, T, cells, seed):
    """Visible cells [T][n_kv] (bool): causal, the visible region of token t ending at n_kv - T + t; "holes" adds the -inf runs a
    multi-sequence cache leaves (runs of 1 000 and 4 096 cells, a run across 32 768 when the row reaches it) and masks every cell of
    one residue mod 8, so one of k_flash_attn_ext's warps finds its whole stride empty.  The planted cells stay visible."""
    vis = np.ones((T, n_kv), bool)
    for t in range(T):
        vis[t, n_kv - T + t + 1:] = False
    if kind == "holes":
        rng = np.random.default_rng(seed)
        hole = np.zeros(n_kv, bool)
        for start, ln in ((1000, 1000), (n_kv // 2 - 2048, 4096), (int(rng.integers(6000, 9000)), 333)):
            hole[start:start + ln] = True
        if n_kv > 40000:
            hole[32768 - 700: 32768 + 700] = True
        r = next(r for r in range(1, 8) if r not in {c % 8 for c in cells} and r != (n_kv - 1) % 8)
        hole[r::8] = True
        hole[cells] = False
        for t in range(T):
            vis[t, :n_kv - T + t] &= ~hole[:n_kv - T + t]
    return vis


def fa_inputs(case):
    n_kv, (H, HK), T, layout, mask_kind, design = case
    seed = n_kv + H * 3 + T * 5 + DESIGNS.index(design)
    q, K, V, cells = make_row(design, n_kv, H, HK, T, n_kv - T + 1, seed)
    vis = long_mask(mask_kind, n_kv, T, cells, seed)
    return q, K, V, cells, vis


@pytest.mark.gpu
@pytest.mark.parametrize("case", FA_CASES, ids=[fa_case_id(c) for c in FA_CASES])
def test_flash_attn_ext_long_rows(cuda, lib, case):
    """k_flash_attn_ext against float64 on the sampled heads of every token, under the bar derived in test_flash_attn_ext_vs_float64
    (no soft-cap, no ALiBi): |out - ref| <= 2 max|V| (2 delta + (5 ceil(n_kv / 8) + 16) u).  At 131 072 cells and |V| = 3 that is
    about 0.03, and the needle rows show it is below the move of one dropped needle."""
    c = _bind(lib)
    n_kv, (H, HK), T, layout, mask_kind, design = case
    g = H // HK
    q, K, V, cells, vis = fa_inputs(case)
    m = np.where(vis, np.float16(0), np.float16(-np.inf)).astype(np.float16)
    if layout == "contig":                       # q [H][T][D], K / V [HK][n_kv][D], mask rows n_kv
        q_mem, q_nb = np.ascontiguousarray(q.transpose(1, 0, 2)), (D * 4, T * D * 4)
        k_mem, v_mem = np.ascontiguousarray(K.transpose(1, 0, 2)), np.ascontiguousarray(V.transpose(1, 0, 2))
        kv_nb, mpad = (D * 2, n_kv * D * 2), n_kv
    else:                                        # the FA-on graph: q [T][H][D], views of a [n_ctx][HK][D] cache, padded mask rows
        q_mem, q_nb = q, (H * D * 4, D * 4)
        n_ctx = n_kv + 40
        k_mem = np.full((n_ctx, HK, D), np.float16(3e4), np.float16); k_mem[:n_kv] = K
        v_mem = np.full((n_ctx, HK, D), np.float16(3e4), np.float16); v_mem[:n_kv] = V
        kv_nb, mpad = (HK * D * 2, D * 2), (n_kv + 31) // 32 * 32 + 32
    mask_mem = np.full((T, mpad), np.float16(-3e4), np.float16)
    mask_mem[:, :n_kv] = m
    qd, kd, vd, md = dev_f32(q_mem), torch.from_numpy(k_mem).cuda(), torch.from_numpy(v_mem).cuda(), torch.from_numpy(mask_mem).cuda()
    dst = torch.full((T * H * D,), float("nan"), device="cuda")
    lib.check(c.pb200_flash_attn_ext(ptr(qd), ptr(kd), ptr(vd), ptr(md), ptr(dst), D, T, H, HK, n_kv, _i64(q_nb), _i64(kv_nb), _i64(kv_nb),
                                     mpad * 2, SCALE, 0.0, 0.0, None), "flash_attn_ext")
    sync()
    del kd, vd
    got = dst.cpu().numpy().reshape(T, H, D)
    assert np.isfinite(got).all()
    kv64 = {}
    for h in check_heads(H, HK):
        hk = h // g
        if hk not in kv64:
            kv64[hk] = K[:, hk].astype(np.float64), V[:, hk].astype(np.float64)
        K64, V64 = kv64[hk]
        vmax = np.max(np.abs(V64))
        dabs = np.abs(K64) @ np.abs(q[:, h].astype(np.float16).astype(np.float64)).T            # [n][T]
        for t in range(T):
            want, p = attn64(q[t, h:h + 1], K64, V64, vis[t], False)
            s_abs = np.abs(SCALE * (K64 @ q[t, h].astype(np.float16).astype(np.float64)))
            delta = np.max(np.where(vis[t], (D / 32 + 6) * U * SCALE * dabs[:, t] + U * s_abs, 0))
            tol = 2 * vmax * (2 * delta + (5 * np.ceil(n_kv / 8) + 16) * U)
            err = np.max(np.abs(got[t, h] - want[0]))
            assert err <= tol, (f"head {h} token {t}", err, tol)
            if t == T - 1:
                check_design(f"head {h} token {t}", design, got[t, h:h + 1], want, p, V64, cells, tol)


def _mm(c, lib, A, ab, B, bb, ne, r2, K):
    dd = torch.full((ne[0] * ne[1] * ne[2],), float("nan"), device="cuda")
    db = (4, ne[0] * 4, ne[0] * ne[1] * 4, ne[0] * ne[1] * ne[2] * 4)
    lib.check(c.pb200_mul_mat_f16(ptr(A), ptr(B), ptr(dd), K, _i64(ne), r2, 1, _i64(ab), _i64(bb), _i64(db), None), "mul_mat_f16")
    return dd


@pytest.mark.gpu
@pytest.mark.parametrize("case", FA_CASES, ids=[fa_case_id(c) for c in FA_CASES])
def test_fa_off_chain_long_rows(cuda, lib, port, case):
    """The plugin's FA-off attention past the fused limit: KQ = pb200_mul_mat_f16 on the K-cache view, pb200_soft_max with the causal
    f32 mask and the scale, KQV = pb200_mul_mat_f16 on the transposed-V view (rows n_ctx apart).  On the sampled heads, each op against
    float64 on its own device input:
      * KQ and KQV: test_mul_mat_f16_vs_float64's bar, 2 (ceil(K / 32) + 5) u sum |A B| per element (K = 128, then n_kv);
      * soft_max: y = fl(expf(fl(s - max)) float32(1 / sum)) with s = fl(fl(x scale) + mask) restated in float32.  expf is within
        2 ulp (4 u relative) and the subtraction's rounding u |s - max| grows through exp, so each e is within r = u |s - max| + 4 u
        of exp(s - max); the double sum is off by the p-weighted mean of r, and 1 / sum and the product add u each: |y - ref| <=
        2 (r + p . r + 2 u) ref (doubled), plus the smallest normal float for values the device may flush;
    and the composed output of the first and last token against the port's attention_decode over each token's visible cells, under
    the fp32-order bar plus f16_flip_slack."""
    c = _bind(lib)
    n_kv, (H, HK), T, _, mask_kind, design = case
    g = H // HK
    q, K, V, cells, vis = fa_inputs(case)
    n_ctx = n_kv + 40
    Kc = np.full((n_ctx, HK, D), np.float16(3e4), np.float16); Kc[:n_kv] = K
    VT = np.full((HK, D, n_ctx), np.float16(3e4), np.float16); VT[:, :, :n_kv] = V.transpose(1, 2, 0)
    mask = np.where(vis, np.float32(0), np.float32(-np.inf)).astype(np.float32)
    Kd, VTd, qd, md = torch.from_numpy(Kc).cuda(), torch.from_numpy(VT).cuda(), dev_f32(q), dev_f32(mask)
    kq = _mm(c, lib, Kd, (2, HK * D * 2, D * 2, Kc.nbytes), qd, (4, H * D * 4, D * 4, q.nbytes), (n_kv, T, H, 1), g, D)
    pr = torch.full_like(kq, float("nan"))
    lib.check(lib.c.pb200_soft_max(ptr(kq), ptr(md), ptr(pr), n_kv, T * H, T, SCALE, None), "soft_max")
    kqv = _mm(c, lib, VTd, (2, n_ctx * 2, D * n_ctx * 2, VT.nbytes), pr, (4, n_kv * 4, T * n_kv * 4, pr.numel() * 4), (D, T, H, 1), g, n_kv)
    sync()
    del Kd, VTd
    out = kqv.cpu().numpy().reshape(H, T, D)
    assert np.isfinite(out).all()
    heads = check_heads(H, HK) if T == 1 else [0, H - 1]
    kq_h = kq.view(H, T, n_kv)[heads].cpu().numpy()
    pr_h = pr.view(H, T, n_kv)[heads].cpu().numpy()
    del kq, pr
    kv64 = {}
    for i, h in enumerate(heads):
        hk = h // g
        if hk not in kv64:
            kv64[hk] = K[:, hk].astype(np.float64), V[:, hk].astype(np.float64)
        K64, V64 = kv64[hk]
        q16 = q[:, h].astype(np.float16).astype(np.float64)                                    # [T][D]
        # KQ
        want = q16 @ K64.T
        bound = 2 * (np.ceil(D / 32) + 5) * U * (np.abs(q16) @ np.abs(K64).T)
        assert np.all(np.abs(kq_h[i] - want) <= bound), (f"KQ head {h}", np.max(np.abs(kq_h[i] - want) - bound))
        for t in range(T):
            # soft_max on the device's KQ row
            s = (kq_h[i, t] * np.float32(SCALE)).astype(np.float32) + mask[t]
            mx = s.max()
            d = (s - mx).astype(np.float32).astype(np.float64)
            e = np.exp(d)
            p = e / e.sum()
            r = np.where(vis[t], U * np.abs(d) + 4 * U, 0)
            tol = 2 * (r + p @ r + 2 * U) * p + 2.0 ** -126
            y = pr_h[i, t].astype(np.float64)
            assert np.all(y[~vis[t]] == 0), f"soft_max head {h} token {t}: a masked cell's probability is not 0"
            assert np.all(np.abs(y - p) <= tol), (f"soft_max head {h} token {t}", np.max(np.abs(y - p) - tol))
            # KQV on the device's probabilities
            p16 = pr_h[i, t].astype(np.float16).astype(np.float64)
            want = V64.T @ p16
            bound = 2 * (np.ceil(n_kv / 32) + 5) * U * (np.abs(V64).T @ p16)
            assert np.all(np.abs(out[h, t] - want) <= bound), (f"KQV head {h} token {t}", np.max(np.abs(out[h, t] - want) - bound))
            if t == T - 1:
                ref, pe = attn64(q[t, h:h + 1], K64, V64, vis[t], True)
                bar = check_fa_off(f"chain head {h} token {t}", out[h, t:t + 1], ref, q[t, h:h + 1], K[vis[t], hk], V[vis[t], hk], 1)
                check_design(f"chain head {h} token {t}", design, out[h, t:t + 1], ref, pe, V64, cells, bar)
    for t in sorted({0, T - 1}):
        for hk in {t * (HK - 1) // max(T - 1, 1)}:          # the first and last q head of one kv group: the port is a serial loop
            idx = np.nonzero(vis[t])[0]
            hh = [hk * g, hk * g + g - 1]
            check_port(port, f"chain token {t} kv head {hk}", out[hh, t], q[t, hh], np.ascontiguousarray(K[idx, hk]),
                       np.ascontiguousarray(V[idx, hk]), 2)


# ---------------------------------------------------------------------------------------------------------------- 4. the engine's decode step
ENGINE_POS = (16383, 16384, 32767, 32768, 40000, "last")
ENGINE_CASES = [("llama_q4_K_M", "needles"), ("llama_q4_K_M", "flat"), ("llama_q4_0", "needles"), ("llama_q4_0", "random")]


def push(s, slot=0):
    """Write the shard's expected cache of a slot (exp_k / exp_v) into the engine's cache through its views, as Shard.fill does."""
    k, v = kv_tensors(s.eng, None, s.n_seq, 1, s.hp)
    k[slot, 0] = torch.from_numpy(s.exp_k[slot].view(np.int16)).cuda()
    v[slot, 0] = torch.from_numpy(s.exp_v[slot].view(np.int16)).cuda()
    sync()


def plant_needles(s, q_rot, pos, rng):
    """Needle K rows along the device's own rotated q: needle j of kv head hk lies along q head hk * gqa + (j mod gqa), with the score
    that gives it a share of 0.7 / (number of needles) against that head's background; V rows of +-3.  Returns [(cell, head)].
    The step's row has pos + 1 cells, and its last one, the fresh cell pos, holds the step's own k: the needles are those of a row of
    pos + 1 cells that lie below pos, plus pos - 1.  Where the final partial 32-group is the fresh cell alone (pos = 16 384, 32 768)
    no needle sits in it; the single-op tests plant that cell."""
    H, HK = s.hp["n_head"], s.hp["n_head_kv"]
    g = H // HK
    cells = sorted({c for c in needle_cells(pos + 1, pos + 1) if c < pos} | {pos - 1})
    K = s.exp_k[0, :pos].view(np.float16).astype(np.float64).reshape(pos, HK, D)
    qh = q_rot.astype(np.float16).astype(np.float64).reshape(H, D)
    planted = []
    for hk in range(HK):
        for j, c in enumerate(cells):
            h = hk * g + j % g
            s_bg = SCALE * (K[:, hk] @ qh[h])
            lse = s_bg.max() + np.log(np.sum(np.exp(s_bg - s_bg.max())))
            sc = lse + np.log(0.7 / len(cells) / 0.3)
            krow = sc / SCALE * qh[h] / (qh[h] @ qh[h])
            s.exp_k[0, c, hk * D:(hk + 1) * D] = f16_bits(krow)
            s.exp_v[0, c, hk * D:(hk + 1) * D] = f16_bits(NEEDLE_V * np.sign(rng.standard_normal(D)))
            planted.append((c, h))
    return planted


@pytest.mark.gpu
@pytest.mark.parametrize("name,design", ENGINE_CASES, ids=[f"{m}-{d}" for m, d in ENGINE_CASES])
def test_engine_decode_long_positions(cuda, lib, pkg, port, engine_max_ctx, name, design):
    """A one-layer shard at n_ctx = the engine's limit, so every step runs k_attn_rows<true>.  Cells [0, pos) are written through the
    cache views; each step passes check_step (every launch on the device's own inputs, the cache bit for bit) and check_launches.
    needles: a probe step at pos gives the device's rotated q; needle K rows are planted along it and the same token and input are
    run again at the same pos, which gives the same q."""
    tm = case_model(name)
    n_ctx = engine_max_ctx
    hp = dict(tm.hp, n_ctx=n_ctx)
    H, HK = hp["n_head"], hp["n_head_kv"]
    assert not uses_attn2(layer_types(tm.tensors, 1), hp, lib.c.pb200_attn_ggml_max_cells())
    s = load_shard(pkg, tm, 1, False, False, hp=hp)
    ff = tm.tensors["rope_freqs.weight"][1] if "rope_freqs.weight" in tm.tensors else None
    try:
        for pos in ENGINE_POS:
            pos = n_ctx - 1 if pos == "last" else pos
            rng = np.random.default_rng(pos + len(name))
            s.fill(0, pos, rng)
            x = rng.standard_normal(hp["n_embd"]).astype(np.float32)
            if design == "flat":
                s.exp_k[0, :pos] = 0
                s.exp_v[0, :pos] = f16_bits(1 + 0.1 * rng.standard_normal((pos, HK * D)))
                push(s)
            elif design == "needles":
                step(lib, s, 5, pos, x)
                q_rot = rope_dev(lib, hp, s.read("q", H * D), H, pos, ff)
                planted = plant_needles(s, q_rot, pos, rng)
                s.exp_k[0, pos:] = F16_NAN
                s.exp_v[0, pos:] = F16_NAN
                push(s)
            n = step(lib, s, 5, pos, x)
            check_launches(lib, s, n, f"{name} {design}", pos, None)
            check_step(lib, port, s, f"{name} {design} n_ctx {n_ctx}", pos)
            if design == "needles":     # the planted cells carry the mass they were planted for, on the device's own q
                q2 = rope_dev(lib, hp, s.read("q", H * D), H, pos, ff)
                assert np.array_equal(q2.view(np.uint32), q_rot.view(np.uint32)), "the re-run step's q differs from the probe's"
                K = s.exp_k[0, :pos + 1].view(np.float16).astype(np.float64).reshape(pos + 1, HK, D)
                qh = q2.astype(np.float16).astype(np.float64).reshape(H, D)
                for c, h in planted:
                    sc = SCALE * (K[:, h // (H // HK)] @ qh[h])
                    p = np.exp(sc - sc.max())
                    p /= p.sum()
                    assert 0.05 <= p[c] <= 0.5, (pos, c, h, p[c])
    finally:
        s.eng.close()


# ---------------------------------------------------------------------------------------------------------------- 5. the engine's prompt step
PF_CALLS = [(39997, 37), (40000, 512)]       # (pos0, T): n_kv_max = pos0 + T, the per-row rung at gqa 4
PF_NCTX = 40960


def fill_prefill_caches(eng, tm, comp, pos0, seed):
    """Cells [0, pos0) of the engine's and the composition's layer-0 caches: the same seeded f16 rows (K ~ 0.5 N, V ~ N); every cell
    from pos0 on f16 NaN.  Views onto the engine's memory live only in here (see test_gpu_prefill_layers.nan_past)."""
    rng = np.random.default_rng(seed)
    EK = tm.hp["n_head_kv"] * D
    for (ev, cv), a in zip(zip(kv_tensors(eng, tm, 1, 1), (comp.kc[0], comp.vc[0])), (0.5, 1.0)):
        rows = torch.from_numpy(f16_bits(rng.standard_normal((pos0, EK), dtype=np.float32) * a).view(np.int16)).cuda()
        for c in (ev[0, 0], cv):
            c[:pos0] = rows
            c[pos0:] = F16_NAN
    sync()


@pytest.mark.gpu
def test_engine_prefill_long_positions(cuda, lib, pkg):
    """A one-layer model's prompt step (pb200_prefill_stage) at pos0 ~ 40 000 with T = 37 and 512, after cells [0, pos0) were written
    through the cache views, against the same layer built from single ops (test_gpu_prefill_layers.Compose) on identical caches: the K /
    V rows bit-identical, the rows past pos0 + T still f16 NaN, and the output hidden state bit-identical.  The engine must pass the
    attention n_kv_max = pos0 + T and each token's position; the attention's arithmetic itself is pb200_attn_prefill's, checked above."""
    tm = TinyModel(n_layer=1, n_embd=1024, n_head=8, n_head_kv=2, n_ff=2048, n_vocab=512, n_ctx=PF_NCTX, arch="llama", ftype="q4_K_M",
                   freq_factors=True, seed=41, branch_scale=0.1)
    E, V = tm.hp["n_embd"], tm.hp["n_vocab"]
    eng = tm.load_engine(pkg)
    try:
        comp = Compose(lib, tm, [eng])
        for pos0, T in PF_CALLS:
            assert attn_batch_plan(tm.hp["n_head"], tm.hp["n_head_kv"], pos0 + T) == "rows"
            toks = [(i * 7919 + 13 * pos0 + 5) % V for i in range(T)]
            fill_prefill_caches(eng, tm, comp, pos0, seed=pos0 + T)
            lg = np.full(V, np.nan, np.float32)
            hid = eng.prefill_stage(toks, None, T, pos0, lg, synchronize=True)
            assert lib.c.pb200_aborted() == 0
            eng_out, (ek, ev) = engine_hidden(hid, T, E), engine_kv(eng, tm, 1)
            y = comp.layer(0, comp.embed(toks), pos0, T)
            sync()
            where = f"p{pos0}t{T}"
            check_cache(f"{where} K", ek[0], comp.kc[0].cpu().numpy(), pos0, T)
            check_cache(f"{where} V", ev[0], comp.vc[0].cpu().numpy(), pos0, T)
            pf_check_bits(f"{where} hidden out", eng_out, y.cpu().numpy())
            check_logits(f"{where} head", lg, comp.head(y[T - 1]).cpu().numpy())
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------------------------- case checks (no GPU)
def test_long_context_cases():
    """No GPU: flat rows of 16 393 cells and more (their probabilities are f16 subnormals); needles sit at 0, at the last cell, at
    32 767 / 32 768 and 65 535 / 65 536 where the row reaches them, and in a final partial 32-group; every prefill case runs the per-row
    rung at gqa 8.  (That every decode case lies past k_attn2's cell limit is asserted on the GPU, where the limit is known.)"""
    flat = [n for n, _, d in DECODE_CASES if d == "flat" and n != "max"] + [n for n, *_, d in FA_CASES if d == "flat"]
    assert np.float16(np.float32(1.0) / np.float32(16392)) == F16_MIN_NORMAL > np.float16(np.float32(1.0) / np.float32(16393))
    assert sum(np.float16(np.float32(1.0) / np.float32(n)) < F16_MIN_NORMAL for n in flat) >= 3, flat
    rows = [(n, n) for n in DECODE_NKV if n != "max"] + [(n - t + 1, n) for n, _, t, *_ in FA_CASES] + \
           [(e - t + 1, e) for e, t, _ in PREFILL_CASES if e != "max"]
    partial = False
    for n_first, n in rows:
        c = set(needle_cells(n_first, n))
        assert {0, n - 1} <= c, (n_first, n, c)
        for b in (32767, 32768, 65535, 65536):
            assert b in c or b >= n_first - 1, (n_first, n, b)
        if n_first % 32:
            assert n_first // 32 * 32 in c
            partial = True
        assert 0.7 / len(c) >= 0.05, c
    assert partial
    assert any(65536 in needle_cells(a, b) for a, b in rows) and any(32768 in needle_cells(a, b) for a, b in rows)
    for e, t, _ in PREFILL_CASES:
        if e != "max":
            assert attn_batch_plan(PREFILL_G, 1, e) == "rows", (e, t)        # the launcher plans by n_kv_max = pos0 + T
    assert {n for n, *_ in FA_CASES} == set(FA_NKV) and {t for _, _, t, *_ in FA_CASES} == {1, 32}
    for n in FA_NKV:
        mine = [c for c in FA_CASES if c[0] == n]
        assert {c[5] for c in mine} == set(DESIGNS) and {c[3] for c in mine} == {"contig", "views"} and {c[4] for c in mine} == {"causal", "holes"}
    for n in FA_NKV:                          # the holes mask empties one warp's stride and keeps every needle visible
        for T in (1, 32):
            cells = needle_cells(n - T + 1, n)
            vis = long_mask("holes", n, T, cells, 0)
            for t in range(T):
                assert np.array_equal(vis[t, cells], np.array(cells) <= n - T + t), (n, T, t)
            # k_flash_attn_ext's warp r visits cells r, r + 8, ...: one warp finds nothing visible in the last token's whole row
            assert any(not vis[T - 1, r::8].any() for r in range(8)), (n, T)
