"""-m gpu: attention where it goes wrong — long score rows, K/V chunk refills, masks, GQA, head sizes and strided views — each
kernel through the C ABI against a plain reference of the same operation:
  * pb200_attn_ggml (k_attn2<true>, the plugin's fused FA-off chain) against the oracle's decode attention, its cache bytes and its
    q8_K output bit for bit, including the cluster pair's arg-max on ties;
  * the engine's k_attn2<false> over 520 tokens (four 128-cell chunks, three buffer refills) against the oracle decode;
  * pb200_flash_attn_ext and pb200_mul_mat_f16 against float64;
  * soft_max rows longer than shared memory, and the context limit of the attention that keeps its score row there."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle_lib as O
from gpu_util import act_ws, act_ws_fields, dev_f32, ptr, sync
from test_gpu_engine import check_decode_parity
from tiny_model import TinyModel

pytestmark = pytest.mark.gpu
D = 128
U = 2.0 ** -24          # unit roundoff of fp32
ENOTSUP = -3
ROPE = dict(freq_base=500000.0, freq_scale=1.0, ext_factor=0.0, attn_factor=1.0, beta_fast=32.0, beta_slow=1.0, n_ctx_orig=8192)


def _bind(lib):
    c = lib.c
    vp, i64, f32, ci = C.c_void_p, C.c_int64, C.c_float, C.c_int
    c.pb200_attn_ggml.argtypes = [vp, vp, vp, vp, vp, i64, vp, vp, ci, ci, ci, vp, ci, ci, vp, vp, ci, ci] + [f32] * 6 + [ci, vp, f32, ci, vp]
    c.pb200_flash_attn_ext.argtypes = [vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, vp, vp, vp, i64, f32, f32, f32, vp]
    c.pb200_mul_mat_f16.argtypes = [vp, vp, vp, i64, vp, i64, i64, vp, vp, vp, vp]
    return c


def _i64(v):
    return (C.c_int64 * len(v))(*[int(x) for x in v])


def rope_dev(lib, x, n_head, pos, mode, n_dims, ff):
    """pb200_rope of one token's [n_head][128] vector: the same rope_cos_sin / rope_rotate k_attn2 runs."""
    xd, y = dev_f32(x), torch.zeros(n_head * D, device="cuda")
    pd = torch.tensor([pos], dtype=torch.int32, device="cuda")
    fd = dev_f32(ff) if ff is not None else None
    r = ROPE
    lib.check(lib.c.pb200_rope(ptr(xd), ptr(y), 1, n_head, D, n_dims, mode, ptr(pd), r["freq_base"], r["freq_scale"], r["ext_factor"],
                               r["attn_factor"], r["beta_fast"], r["beta_slow"], r["n_ctx_orig"], ptr(fd) if fd is not None else None, None), "rope")
    sync()
    return y.cpu().numpy()


# ------------------------------------------------------------------------------------------------ pb200_attn_ggml (k_attn2<true>)
class AttnGgmlCase:
    """One token of the FA-off chain on the reference graph's tensors: K cache [n_ctx][HK*128], V cache transposed [HK*128][vt_stride]
    with vt_stride > n_cells (and > n_ctx rows of K), a mask row over n_cells cells, this token's K / V stored in cell kv_head."""

    def __init__(self, lib, H, HK, n_cells, kv_head, mode, ff, n_dims, mask_kind, seed, v_override=None):
        rng = np.random.default_rng(seed)
        self.H, self.HK, self.n_cells, self.kv_head, self.mode, self.n_dims = H, HK, n_cells, kv_head, mode, n_dims
        EK = HK * D
        self.n_ctx = n_cells + 24                       # K rows past n_cells must stay untouched too
        self.vt_stride = n_cells + 40                   # columns between n_cells and vt_stride likewise
        self.pos = kv_head + 1009                       # RoPE position != cell
        self.ff = (1.0 + rng.uniform(0, 7, 64)).astype(np.float32) if ff else None
        self.scale = float(1.0 / np.sqrt(D))
        self.q = rng.standard_normal(H * D).astype(np.float32)
        self.k = rng.standard_normal(EK).astype(np.float32)
        self.v = (rng.standard_normal(EK).astype(np.float32) if v_override is None else v_override).astype(np.float32)
        mask = np.zeros(n_cells, np.float32)
        if mask_kind == "causal":                      # cells after the newest visible one masked, like llama.cpp's padded n_kv
            mask[max(kv_head, n_cells - 7) + 1:] = -np.inf
        elif mask_kind in ("holes", "chunk"):
            mask[rng.random(n_cells) < 0.2] = -np.inf
            if mask_kind == "chunk":                   # one whole 128-cell chunk that does not hold the fresh cell
                c = (kv_head // 128 + 1) % ((n_cells + 127) // 128) if n_cells > 128 else None
                if c is not None:
                    mask[c * 128: min(n_cells, c * 128 + 128)] = -np.inf
        elif mask_kind == "only_fresh":
            mask[:] = -np.inf
        mask[kv_head] = 0.0                            # the token always sees itself
        self.mask = mask
        Kc = (rng.standard_normal((self.n_ctx, EK)) * 0.5).astype(np.float16)
        VT = rng.standard_normal((EK, self.vt_stride)).astype(np.float16)
        hidden = np.nonzero(mask == -np.inf)[0]
        # masked cells hold large finite values: attending to one of them by mistake is loud
        Kc[hidden] = (np.sign(rng.standard_normal((hidden.size, EK))) * 3e4).astype(np.float16)
        VT[:, hidden] = (np.sign(rng.standard_normal((EK, hidden.size))) * 3e4).astype(np.float16)
        self.Kc0, self.VT0 = Kc, VT

    def expected(self, lib, port):
        """Out from the oracle over the visible cells in index order (a -inf cell adds exactly 0 to the softmax sum and to P.V),
        and the cache bytes after the store: f16(rope(k)) in row kv_head, f16(v) in column kv_head, nothing else changed."""
        q_rot = rope_dev(lib, self.q, self.H, self.pos, self.mode, self.n_dims, self.ff)
        k_rot = rope_dev(lib, self.k, self.HK, self.pos, self.mode, self.n_dims, self.ff)
        Kc, VT = self.Kc0.copy(), self.VT0.copy()
        Kc[self.kv_head] = k_rot.astype(np.float16)
        VT[:, self.kv_head] = self.v.astype(np.float16)
        vis = np.nonzero(self.mask == 0)[0]
        Kg = np.ascontiguousarray(Kc[vis])
        Vg = np.ascontiguousarray(VT[:, vis].T)
        out = port.attention_decode(q_rot, Kg.view(np.uint16), Vg.view(np.uint16), self.H, self.HK, D, vis.size, self.scale)
        return out, Kc, VT

    def run(self, lib, kv_head=None, kv_head_dev=None, n_cells=None):
        """One pb200_attn_ggml call on fresh copies of the caches: (rc, out, act bytes, K cache, V cache)."""
        c = _bind(lib)
        qd, kd, vd = dev_f32(self.q), dev_f32(self.k), dev_f32(self.v)
        Kd, VTd = torch.from_numpy(self.Kc0.copy()).cuda(), torch.from_numpy(self.VT0.copy()).cuda()
        md = dev_f32(self.mask)
        out = torch.full((self.H * D,), float("nan"), device="cuda")
        ws = act_ws(lib, self.H * D)
        pd = torch.tensor([self.pos], dtype=torch.int32, device="cuda")
        hd = torch.tensor([kv_head_dev], dtype=torch.int32, device="cuda") if kv_head_dev is not None else None
        fd = dev_f32(self.ff) if self.ff is not None else None
        r = ROPE
        rc = c.pb200_attn_ggml(ptr(qd), ptr(kd), ptr(vd), ptr(Kd), ptr(VTd), self.vt_stride, ptr(out), ptr(ws), self.H, self.HK, D, ptr(pd),
                               self.n_cells if n_cells is None else n_cells, self.kv_head if kv_head is None else kv_head,
                               ptr(hd) if hd is not None else None, ptr(md), self.n_dims, self.mode, r["freq_base"], r["freq_scale"],
                               r["ext_factor"], r["attn_factor"], r["beta_fast"], r["beta_slow"], r["n_ctx_orig"],
                               ptr(fd) if fd is not None else None, self.scale, 0, None)
        sync()
        if rc != 0:
            return rc, None, None, None, None
        return rc, out.cpu().numpy(), act_ws_fields(ws, self.H * D, "q8_K"), Kd.cpu().numpy(), VTd.cpu().numpy()


@pytest.fixture(scope="module")
def attn2_max_cells(cuda, lib):
    """The largest n_cells pb200_attn_ggml takes, probed through its return code (the launcher refuses a score row beyond the
    clustered kernel's shared memory before it launches anything)."""
    H, HK = 8, 2
    probe = AttnGgmlCase(lib, H, HK, 32, 0, 0, False, D, "none", seed=1)

    def ok(n):
        case = AttnGgmlCase.__new__(AttnGgmlCase)
        case.__dict__.update(probe.__dict__)
        case.n_cells, case.n_ctx, case.vt_stride = n, n + 8, n + 8
        case.mask = np.zeros(n, np.float32)
        case.Kc0 = np.zeros((n + 8, HK * D), np.float16)
        case.VT0 = np.zeros((HK * D, n + 8), np.float16)
        rc = case.run(lib)[0]
        assert rc in (0, ENOTSUP), rc
        return rc == 0
    lo, hi = 32, 32 * 2048                      # ok(lo), not ok(hi)
    assert ok(lo) and not ok(hi)
    while hi - lo > 32:
        mid = (lo + hi) // 64 * 32
        lo, hi = (mid, hi) if ok(mid) else (lo, mid)
    return lo


# (H, HK), n_cells, kv_head, RoPE mode, freq factors, n_dims, mask.  kv_head covers the first cell, the end of chunk 0 (127), the
# start of chunk 1 (128), the last cell, and the middle of a later chunk; n_cells one chunk, partial second chunks (136, 264) and
# several refills of both buffers (1000, 4096, the maximum).
ATTN_GGML_CASES = [
    ((8, 8), 32, 0, 0, True, 128, "causal"),
    ((8, 2), 128, 127, 2, False, 128, "holes"),
    ((8, 2), 136, 128, 0, True, 128, "causal"),
    ((64, 8), 256, 200, 2, False, 128, "chunk"),
    ((8, 2), 256, 0, 0, True, 128, "chunk"),
    ((8, 2), 264, 263, 0, True, 64, "holes"),
    ((8, 8), 1000, 999, 0, True, 128, "chunk"),
    ((64, 8), 1000, 127, 0, True, 128, "holes"),
    ((64, 8), 4096, 2500, 0, True, 128, "holes"),
    ((8, 8), 4096, 128, 2, False, 64, "causal"),
    ((8, 2), 4096, 4095, 2, False, 128, "chunk"),
    ((8, 2), "max", "last", 2, False, 128, "chunk"),
    ((8, 2), "max", 3333, 0, True, 128, "holes"),
]


@pytest.mark.parametrize("heads,n_cells,kv_head,mode,ff,n_dims,mask_kind", ATTN_GGML_CASES,
                         ids=[f"h{h[0]}x{h[1]}-c{n}-kv{k}-m{m}{'ff' if f else ''}-d{nd}-{mk}" for h, n, k, m, f, nd, mk in ATTN_GGML_CASES])
def test_attn_ggml_vs_oracle(cuda, lib, port, attn2_max_cells, heads, n_cells, kv_head, mode, ff, n_dims, mask_kind):
    H, HK = heads
    if n_cells == "max":
        n_cells = attn2_max_cells
        assert n_cells >= 4096, n_cells
    if kv_head == "last":
        kv_head = n_cells - 1
    check_attn_ggml_case(lib, port, AttnGgmlCase(lib, H, HK, n_cells, kv_head, mode, ff, n_dims, mask_kind, seed=n_cells * 7 + kv_head))


def check_attn_ggml_case(lib, port, case):
    """One AttnGgmlCase against the oracle (fp32-order bar), its cache bytes and q8_K output bit for bit, and the kv_head_dev replay bit
    for bit against the direct launch."""
    want, Kw, VTw = case.expected(lib, port)
    rc, out, act, Kc, VT = case.run(lib)
    assert rc == 0, rc
    # same f16 roundings of q, k, v and of the probabilities as the CPU graph: only fp32 summation order and expf ulps differ (the bar
    # of test_gpu_kernels.py::test_attn_decode)
    err = np.abs(out - want)
    assert np.max(err) < 3e-4 and np.mean(err) < 2e-5, (np.max(err), np.mean(err))
    assert np.array_equal(Kc.view(np.uint16), Kw.view(np.uint16)), "K cache bytes"
    assert np.array_equal(VT.view(np.uint16), VTw.view(np.uint16)), "transposed V cache bytes"
    assert np.array_equal(act, port.quantize_act(O.Q4_K, out)), "q8_K of the output"
    # a captured graph replays with the cell in device memory: kv_head = 0 plus kv_head_dev must give the same bytes
    rc2, out2, act2, Kc2, VT2 = case.run(lib, kv_head=0, kv_head_dev=case.kv_head)
    assert rc2 == 0
    assert np.array_equal(out2.view(np.uint32), out.view(np.uint32)) and np.array_equal(act2, act)
    assert np.array_equal(Kc2.view(np.uint16), Kc.view(np.uint16)) and np.array_equal(VT2.view(np.uint16), VT.view(np.uint16))


def test_attn_ggml_cell_limit(cuda, lib, attn2_max_cells):
    """The next multiple of 32 past the largest accepted n_cells is refused with PB200_ENOTSUP, not launched, and the library
    reports that largest n_cells itself (the ggml-backend plugin plans with it)."""
    assert lib.c.pb200_attn_ggml_max_cells() == attn2_max_cells
    case = AttnGgmlCase(lib, 8, 2, 32, 0, 0, False, D, "none", seed=2)
    n = attn2_max_cells + 32
    case.n_cells, case.mask = n, np.zeros(n, np.float32)
    case.Kc0, case.VT0, case.vt_stride = np.zeros((n, 2 * D), np.float16), np.zeros((2 * D, n), np.float16), n
    assert case.run(lib)[0] == ENOTSUP


def test_attn_ggml_cluster_argmax_tie(cuda, lib, port):
    """Only the fresh cell is visible, so p = 1 exactly and head h's output is f16(v_h).  Heads 2j and 2j+1 (the two CTAs of a
    cluster, one q8_K super-block) reach the same |max| with opposite signs, and head 0 holds the same |max| twice: the block's
    scale takes the sign of the first occurrence (rank 0, lower index), as quantize_row_q8_K does."""
    H = HK = 8
    rng = np.random.default_rng(77)
    v = (rng.uniform(-1, 1, H * D)).astype(np.float16).astype(np.float32)
    for j in range(H // 2):
        a, b = 2 * j * D + (5 + 17 * j), (2 * j + 1) * D + (3 + 29 * j)
        sgn = 1.0 if j % 2 == 0 else -1.0
        v[a], v[b] = 2.5 * sgn, -2.5 * sgn
    v[100] = 2.5                                   # head 0: a second occurrence of +|max| after index 5, before rank 1's -|max|
    case = AttnGgmlCase(lib, H, HK, 128, 37, 0, False, D, "only_fresh", seed=3, v_override=v)
    rc, out, act, _, _ = case.run(lib)
    assert rc == 0
    assert np.array_equal(out, v), "p = 1 must give out = f16(v) exactly"
    want = port.quantize_act(O.Q4_K, v)
    assert np.array_equal(act, want)
    d = act.reshape(H // 2, 292)[:, :4].copy().view(np.float32).ravel()
    # d = 1 / (-127 / max) with max the signed value of the first |max|: blocks 0 and 2 start with +2.5, blocks 1 and 3 with -2.5
    assert np.array_equal(np.sign(d), np.array([-1.0, 1.0, -1.0, 1.0], np.float32)), d


# ------------------------------------------------------------------------------------------------ engine: k_attn2<false> across chunks
def _window_parity(got, want):
    """check_decode_parity without its first-token-exact clause: a window that starts mid-run inherits earlier flips."""
    e = np.max(np.abs(got - want), axis=1)
    nmse = float(np.sum((got - want) ** 2) / np.sum(want ** 2))
    assert nmse < 2e-3, (nmse, e)
    assert np.max(e) < 0.25, e
    assert np.mean(got.argmax(1) == want.argmax(1)) >= 0.9


@pytest.mark.parametrize("arch", ["llama", "qwen2"])
def test_engine_attn2_across_chunks(cuda, pkg, lib, port, arch):
    """520 decoded tokens: positions 128+ stream K/V in several 128-cell chunks through the two buffers per tensor, so every token
    from 256 on refills a buffer and flips its mbarrier parity.  Checked against the oracle decode over the whole run and over each
    128-position window, so an error confined to later chunks is not averaged away; launches per token equal the n_ctx 64 model's,
    so k_attn2 (not the k_attn_rows fallback) ran."""
    kw = dict(n_layer=2, n_embd=512, n_head=4, n_head_kv=2, n_ff=1024, arch=arch, branch_scale=0.1)
    toks = [(i * 7919 + 13) % 320 for i in range(520)]
    tm = TinyModel(n_ctx=640, **kw)
    want, _ = tm.port_decode(port, toks)
    eng = tm.load_engine(pkg)
    got = np.zeros_like(want)
    n0 = lib.c.pb200_kernel_launches()
    for i, t in enumerate(toks):
        eng.decode(int(t), i, got[i])
    per_tok = (lib.c.pb200_kernel_launches() - n0) / len(toks)
    eng.close()
    check_decode_parity(got, want)
    for w0 in range(128, len(toks), 128):
        _window_parity(got[w0: w0 + 128], want[w0: w0 + 128])
    short = TinyModel(n_ctx=64, **kw).load_engine(pkg)
    n0 = lib.c.pb200_kernel_launches()
    for i, t in enumerate(toks[:8]):
        short.decode(int(t), i, None)
    per_tok_short = (lib.c.pb200_kernel_launches() - n0) / 8
    short.close()
    assert per_tok == per_tok_short, (per_tok, per_tok_short)


# ------------------------------------------------------------------------------------------------ pb200_flash_attn_ext vs float64
def _alibi_slopes(H, max_bias):
    if max_bias <= 0:
        return np.ones(H)
    n2 = 1 << int(np.floor(np.log2(H)))
    m0, m1 = 2.0 ** (-max_bias / n2), 2.0 ** (-(max_bias / 2.0) / n2)
    return np.array([m0 ** (h + 1) if h < n2 else m1 ** (2 * (h - n2) + 1) for h in range(H)])


# D, (H, HK), n_kv, n_tok, mask, softcap, max_bias, layout.  12 heads / 6 heads with max_bias take the m1 slope branch; n_kv < 8 leaves
# warps without cells; "views" is llama.cpp's FA-on graph: permuted q, K/V views into a larger cache, a padded mask row.
FA_CASES = [
    (64, (8, 8), 1, 1, "none", 0.0, 0.0, "contig"),
    (80, (32, 8), 5, 3, "finite", 0.0, 0.0, "views"),
    (96, (12, 4), 7, 35, "causal", 0.0, 8.0, "views"),
    (128, (6, 2), 33, 3, "causal", 10.0, 0.0, "contig"),
    (256, (8, 8), 512, 35, "finite", 10.0, 8.0, "views"),
    (128, (32, 8), 1000, 1, "causal", 0.0, 0.0, "views"),
    (128, (12, 4), 512, 3, "finite", 0.0, 8.0, "contig"),
    (256, (6, 2), 1000, 3, "none", 10.0, 0.0, "contig"),
    (64, (6, 2), 33, 35, "finite", 10.0, 8.0, "views"),
    (80, (8, 8), 1000, 35, "causal", 0.0, 0.0, "contig"),
    (96, (32, 8), 1, 3, "none", 0.0, 0.0, "views"),
    (128, (12, 4), 7, 1, "finite", 0.0, 8.0, "views"),
    (256, (12, 4), 5, 35, "causal", 10.0, 0.0, "contig"),
    (64, (32, 8), 512, 1, "causal", 0.0, 8.0, "views"),
]


@pytest.mark.parametrize("Dh,heads,n_kv,n_tok,mask_kind,softcap,max_bias,layout", FA_CASES,
                         ids=[f"d{d}-h{h[0]}x{h[1]}-kv{n}-t{t}-{m}-cap{int(c)}-alibi{int(b)}-{lay}" for d, h, n, t, m, c, b, lay in FA_CASES])
def test_flash_attn_ext_vs_float64(cuda, lib, Dh, heads, n_kv, n_tok, mask_kind, softcap, max_bias, layout):
    """softmax(softcap(scale * K . f16(q)) + slope * mask) . V against float64 of the same f16 inputs.

    Tolerance, from fp32 arithmetic with unit roundoff u = 2^-24 (first order, then doubled):
      * score s of cell c: the dot is Dh/32 fmas per lane and a 5-level warp tree, error <= (Dh/32 + 6) u sum_d |k_d q_d| scaled by
        |scale|; the scale product, the tanhf of the soft-cap (<= 2 ulp of softcap), slope * mask (powf and the product, 4 ulp) and the
        add contribute u |s| + 4 u softcap + 4 u |slope mask|.  delta = the largest of these over the row;
      * a shift delta of the scores moves each softmax weight by a relative 2 delta (numerator and sum);
      * the online softmax rescales its f32 sum and accumulator once per cell of a warp (expf 2 ulp, two products, the fma): about
        5 u per step over ceil(n_kv / 8) steps, then the 8-warp merge and the final 1/S: 16 u;
    so |out - ref| <= max|V| (2 delta + (5 ceil(n_kv / 8) + 16) u), since the output is a convex combination of V rows."""
    c = _bind(lib)
    H, HK = heads
    rng = np.random.default_rng(Dh * 1000 + n_kv * 10 + n_tok + H)
    gqa = H // HK
    scale = float(1.0 / np.sqrt(Dh))
    q = rng.standard_normal((n_tok, H, Dh)).astype(np.float32)                # logical [token][head][d]
    k = rng.standard_normal((n_kv, HK, Dh)).astype(np.float16)                # logical [cell][kv head][d]
    v = rng.standard_normal((n_kv, HK, Dh)).astype(np.float16)
    m = None
    if mask_kind == "finite":
        m = rng.uniform(-2, 2, (n_tok, n_kv)).astype(np.float16)
    elif mask_kind == "causal":                                             # the last n_tok cells are the batch, plus 20 % holes
        m = np.zeros((n_tok, n_kv), np.float16)
        for t in range(n_tok):
            last = max(0, n_kv - n_tok + t)
            m[t, last + 1:] = -np.inf
            m[t, rng.random(n_kv) < 0.2] = -np.inf
            m[t, min(last, n_kv - 1)] = 0.0
    # device layouts
    if layout == "contig":                     # test-backend-ops: q [H][T][D], K/V [HK][n_kv][D], mask rows n_kv
        q_mem = np.ascontiguousarray(q.transpose(1, 0, 2))
        q_nb = (Dh * 4, n_tok * Dh * 4)
        k_mem, v_mem = np.ascontiguousarray(k.transpose(1, 0, 2)), np.ascontiguousarray(v.transpose(1, 0, 2))
        kv_nb = (Dh * 2, n_kv * Dh * 2)
        mpad = n_kv
    else:                                      # FA-on graph: q permuted [T][H][D], K/V views of a cache [n_ctx][HK][D], padded mask rows
        q_mem = np.ascontiguousarray(q)
        q_nb = (H * Dh * 4, Dh * 4)
        n_ctx = n_kv + 40
        k_mem = np.zeros((n_ctx, HK, Dh), np.float16); k_mem[:n_kv] = k; k_mem[n_kv:] = np.float16(3e4)
        v_mem = np.zeros((n_ctx, HK, Dh), np.float16); v_mem[:n_kv] = v; v_mem[n_kv:] = np.float16(3e4)
        kv_nb = (HK * Dh * 2, Dh * 2)
        mpad = (n_kv + 31) // 32 * 32 + 32
    mask_mem = None
    if m is not None:
        mask_mem = np.full((n_tok, mpad), np.float16(-3e4), np.float16)
        mask_mem[:, :n_kv] = m
    qd = dev_f32(q_mem)
    kd, vd = torch.from_numpy(k_mem).cuda(), torch.from_numpy(v_mem).cuda()
    md = torch.from_numpy(mask_mem).cuda() if mask_mem is not None else None
    dst = torch.full((n_tok * H * Dh,), float("nan"), device="cuda")
    lib.check(c.pb200_flash_attn_ext(ptr(qd), ptr(kd), ptr(vd), ptr(md) if md is not None else None, ptr(dst), Dh, n_tok, H, HK, n_kv,
                                     _i64(q_nb), _i64(kv_nb), _i64(kv_nb), mpad * 2, scale, max_bias, softcap, None), "flash_attn_ext")
    sync()
    got = dst.cpu().numpy().reshape(n_tok, H, Dh)
    # float64 reference
    q64 = q.astype(np.float16).astype(np.float64)
    k64, v64 = k.astype(np.float64), v.astype(np.float64)
    kf = np.repeat(k64, gqa, axis=1)                                   # [cell][head][d]
    vf = np.repeat(v64, gqa, axis=1)
    dot = np.einsum("thd,chd->thc", q64, kf)
    dabs = np.einsum("thd,chd->thc", np.abs(q64), np.abs(kf))
    s = dot * scale
    if softcap:
        s = softcap * np.tanh(s / softcap)
    slope = _alibi_slopes(H, max_bias)[None, :, None]
    mm = m.astype(np.float64)[:, None, :] if m is not None else np.zeros((n_tok, 1, n_kv))
    with np.errstate(invalid="ignore"):
        bias = np.where(np.isneginf(mm), -np.inf, slope * mm)
    s = s + bias
    mx = np.max(s, axis=2, keepdims=True)
    e = np.exp(s - mx)
    p = e / np.sum(e, axis=2, keepdims=True)
    want = np.einsum("thc,chd->thd", p, vf)
    fin = np.isfinite(bias)
    delta = np.where(fin, (Dh / 32 + 6) * U * scale * dabs + U * np.abs(np.where(fin, s, 0)) + 4 * U * softcap
                     + 4 * U * np.abs(np.where(fin, bias, 0)), 0).max()
    tol = 2 * np.max(np.abs(v64)) * (2 * delta + (5 * np.ceil(n_kv / 8) + 16) * U)
    err = np.max(np.abs(got - want))
    assert np.isfinite(got).all()
    assert err <= tol, (err, tol)


# ------------------------------------------------------------------------------------------------ pb200_mul_mat_f16 vs float64
def _mm_case(name):
    """(A memory f16, A byte strides, B memory f32, B byte strides, ne of dst, r2, r3, K)"""
    rng = np.random.default_rng(len(name))
    if name == "kq":                  # K-cache view [D, n_kv, HK] times permuted q [D, T, H]: dst [n_kv, T, H], r2 = H / HK
        H, HK, n_kv, T, n_ctx = 8, 2, 200, 5, 256
        Kc = (rng.standard_normal((n_ctx, HK, D)) * 0.5).astype(np.float16)
        q = rng.standard_normal((T, H, D)).astype(np.float32)
        return Kc, (2, HK * D * 2, D * 2, Kc.nbytes), q, (4, H * D * 4, D * 4, q.nbytes), (n_kv, T, H, 1), H // HK, 1, D
    if name == "kqv":                 # transposed-V view [n_kv, D, HK] (rows n_ctx apart) times probabilities [n_kv, T, H]: dst [D, T, H]
        H, HK, n_kv, T, n_ctx = 8, 2, 200, 5, 256
        VT = rng.standard_normal((HK, D, n_ctx)).astype(np.float16)
        p = rng.random((H, T, n_kv)).astype(np.float32) / n_kv
        return VT, (2, n_ctx * 2, D * n_ctx * 2, VT.nbytes), p, (4, n_kv * 4, T * n_kv * 4, p.nbytes), (D, T, H, 1), H // HK, 1, n_kv
    if name == "ragged":              # K = 100: the lanes' last round is partial
        A = rng.standard_normal((3, 7, 100)).astype(np.float16)
        B = rng.standard_normal((3, 5, 100)).astype(np.float32)
        return A, (2, 200, 1400, A.nbytes), B, (4, 400, 2000, B.nbytes), (7, 5, 3, 1), 1, 1, 100
    if name == "r3":                  # A broadcast over dims 2 and 3: r2 = 2, r3 = 2
        A = rng.standard_normal((1, 2, 9, 64)).astype(np.float16)
        B = rng.standard_normal((2, 4, 6, 64)).astype(np.float32)
        return A, (2, 128, 9 * 128, 2 * 9 * 128), B, (4, 256, 6 * 256, 4 * 6 * 256), (9, 6, 4, 2), 2, 2, 64
    raise KeyError(name)


@pytest.mark.parametrize("name", ["kq", "kqv", "ragged", "r3"])
def test_mul_mat_f16_vs_float64(cuda, lib, name):
    """d[i0,i1,i2,i3] = sum_k A[k,i0,i2/r2,i3/r3] * f16(B[k,i1,i2,i3]) against float64 of the same f16 operands.  Each f16 x f16
    product is exact in fp32; a lane sums ceil(K/32) of them by fma and the warp adds 32 partial sums in 5 levels, so
    |d - ref| <= (ceil(K/32) + 5) u sum_k |A B| (first order, u = 2^-24), here with a factor 2."""
    c = _bind(lib)
    A, ab, B, bb, ne, r2, r3, K = _mm_case(name)
    ne0, ne1, ne2, ne3 = ne
    db = (4, ne0 * 4, ne0 * ne1 * 4, ne0 * ne1 * ne2 * 4)
    Ad, Bd = torch.from_numpy(np.ascontiguousarray(A)).cuda(), dev_f32(B)
    dd = torch.full((ne0 * ne1 * ne2 * ne3,), float("nan"), device="cuda")
    lib.check(c.pb200_mul_mat_f16(ptr(Ad), ptr(Bd), ptr(dd), K, _i64(ne), r2, r3, _i64(ab), _i64(bb), _i64(db), None), "mul_mat_f16")
    sync()
    got = dd.cpu().numpy().reshape(ne3, ne2, ne1, ne0)
    st = np.lib.stride_tricks.as_strided
    Av = st(A, shape=(ne3 // r3, ne2 // r2, ne0, K), strides=(ab[3], ab[2], ab[1], ab[0])).astype(np.float64)
    Bv = st(B, shape=(ne3, ne2, ne1, K), strides=(bb[3], bb[2], bb[1], bb[0])).astype(np.float16).astype(np.float64)
    Ar = Av[np.arange(ne3) // r3][:, np.arange(ne2) // r2]
    want = np.einsum("abik,abjk->abji", Ar, Bv)
    bound = np.einsum("abik,abjk->abji", np.abs(Ar), np.abs(Bv)) * (np.ceil(K / 32) + 5) * U * 2
    assert np.all(np.abs(got - want) <= bound), np.max(np.abs(got - want) - bound)


# ------------------------------------------------------------------------------------------------ long rows
@pytest.mark.parametrize("ncols", [60000, 131072])
def test_soft_max_row_longer_than_shared_memory(cuda, lib, port, ncols):
    """A row of more than 58 k floats does not fit the 227 KB of shared memory a block may have: the softmax then runs in place on
    the output row.  Same arithmetic as the staged rows: against the oracle to a few ulp of each value (expf <= 2 ulp apart, the
    double sum's order, float(1 / sum))."""
    rng = np.random.default_rng(ncols)
    rows = 3
    x = (rng.standard_normal((rows, ncols)) * 4).astype(np.float32)
    mask = np.zeros((2, ncols), np.float32)
    mask[0, ncols // 2:] = -np.inf
    mask[1, rng.random(ncols) < 0.3] = -np.inf
    y = torch.full((rows * ncols,), float("nan"), device="cuda")
    xd, md = dev_f32(x), dev_f32(mask)
    lib.check(lib.c.pb200_soft_max(ptr(xd), ptr(md), ptr(y), ncols, rows, 2, 0.088, None), "soft_max")
    sync()
    got = y.cpu().numpy().reshape(rows, ncols)
    want = np.stack([port.soft_max(x[i], mask[i % 2], 0.088) for i in range(rows)])
    assert np.array_equal(got == 0, want == 0)
    assert np.max(np.abs(got - want) / np.maximum(want, 1e-30)) < 1e-6
    assert np.allclose(got.sum(axis=1), 1.0, atol=1e-4)


def _create(lib, pkg, n_ctx):
    hp = pkg.HParams(n_layer=1, n_embd=256, n_head=2, n_head_kv=1, head_dim=128, n_ff=512, n_vocab=64, n_ctx=n_ctx, rope_mode=0,
                     n_ctx_orig=8192, rope_freq_base=500000.0, rope_freq_scale=1.0, rms_eps=1e-5)
    h = lib.c.pb200_model_create(C.byref(hp), 0, 0, 1, 1, 1)
    if h:
        lib.c.pb200_model_free(h)
    return bool(h)


@pytest.fixture(scope="module")
def engine_max_ctx(cuda, pkg, lib):
    lo, hi = 64, 1 << 20
    assert _create(lib, pkg, lo)
    assert not _create(lib, pkg, hi), "pb200_model_create accepts a context whose attention cannot run"
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if _create(lib, pkg, mid) else (lo, mid)
    return lo


def test_attn_single_op_context_limit(cuda, lib, port, engine_max_ctx):
    """pb200_attn_decode / pb200_attn_prefill size k_attn_rows<false>'s score row by n_ctx (n_kv_max): its longest row, probed through
    the return code, is at least the engine's limit (which also covers k_attn_rows<true>, with more static shared memory).  At that
    row length the kernel runs and matches the oracle; one step of 32 above it both entry points return PB200_ENOTSUP, not a CUDA
    error.  Only rows [0, pos] are read, so the probe needs no cache of n_ctx rows."""
    H, HK, n_kv = 8, 2, 300
    rng = np.random.default_rng(4)
    q = rng.standard_normal(H * D).astype(np.float32)
    Kc = (rng.standard_normal((n_kv, HK * D)) * 0.5).astype(np.float16)
    Vc = rng.standard_normal((n_kv, HK * D)).astype(np.float16)
    qd, kd, vd = dev_f32(q), torch.from_numpy(Kc).cuda(), torch.from_numpy(Vc).cuda()
    pos = torch.tensor([n_kv - 1], dtype=torch.int32, device="cuda")
    out = torch.full((H * D,), float("nan"), device="cuda")
    scale = 1.0 / np.sqrt(D)

    def decode(n_ctx):
        rc = lib.c.pb200_attn_decode(ptr(qd), ptr(kd), ptr(vd), ptr(out), H, HK, D, ptr(pos), n_ctx, scale, None)
        sync()
        assert rc in (0, ENOTSUP), rc
        return rc == 0
    lo, hi = engine_max_ctx, 1 << 17
    assert decode(lo) and not decode(hi)
    while hi - lo > 32:
        mid = (lo + hi) // 64 * 32
        lo, hi = (mid, hi) if decode(mid) else (lo, mid)
    assert lo % 32 == 0 and lo > 16384, lo
    out.fill_(float("nan"))
    lib.check(lib.c.pb200_attn_decode(ptr(qd), ptr(kd), ptr(vd), ptr(out), H, HK, D, ptr(pos), lo, scale, None), "attn_decode at the limit")
    sync()
    want = port.attention_decode(q, Kc.view(np.uint16), Vc.view(np.uint16), H, HK, D, n_kv, scale)
    assert np.max(np.abs(out.cpu().numpy() - want)) < 3e-4
    assert lib.c.pb200_attn_decode(ptr(qd), ptr(kd), ptr(vd), ptr(out), H, HK, D, ptr(pos), lo + 32, scale, None) == ENOTSUP
    assert lib.c.pb200_attn_prefill(ptr(qd), ptr(kd), ptr(vd), ptr(out), H, HK, D, ptr(pos), 1, lo + 32, scale, None) == ENOTSUP
    # the refusal leaves no CUDA error behind for the next launcher that reads cudaGetLastError()
    y = torch.zeros(64, device="cuda")
    lib.check(lib.c.pb200_soft_max(ptr(qd), None, ptr(y), 64, 1, 0, 1.0, None), "soft_max after the refusal")
    sync()


def test_engine_context_limit(cuda, pkg, lib, port, engine_max_ctx):
    """pb200_model_create refuses a context the attention fallback cannot hold (one more cell fails), and a model at the largest
    context it accepts decodes within the multi-token parity bar (k_attn_rows<true> with the longest score row)."""
    n_ctx = engine_max_ctx
    assert not _create(lib, pkg, n_ctx + 1)
    tm = TinyModel(n_layer=2, n_embd=512, n_head=4, n_head_kv=2, n_ff=1024, n_ctx=n_ctx, arch="llama", seed=9, branch_scale=0.1)
    toks = [(i * 7919 + 13) % 320 for i in range(4)]
    want, _ = tm.port_decode(port, toks)
    eng = tm.load_engine(pkg)
    got = np.zeros_like(want)
    for i, t in enumerate(toks):
        eng.decode(int(t), i, got[i])
    eng.close()
    check_decode_parity(got, want)
