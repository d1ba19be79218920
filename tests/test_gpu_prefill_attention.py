"""Prompt-processing attention (pb200_attn_prefill, the engine's pb200_prefill) at every launch rung, odd GQA ratios and multi-thousand-token
prompts, plus the decode attention's cluster pairs at odd GQA.

launch_attn_batch (ops.cu) keeps the scores of gqa x TQ query rows in shared memory and takes the first TQ in {4, 2, 1} whose
k_attn_prefill_tiled<TQ> fits 200 KB; beyond that it runs k_attn_rows<false>, one CTA per (head, token).  attn_batch_plan() restates
that arithmetic and every case is named after the rung it reaches; test_cases_reach_every_rung checks without a GPU that the case list
reaches every rung at every GQA ratio, including the last n_kv_pad of each rung and the first of the next.

Checks:
  * every (token, head) row of pb200_attn_prefill against float64 with the kernel's roundings (f16 q, p = f16(e * float32(1 / sum)),
    scores and sums in float64), and sampled tokens against the oracle's decode attention as well, under the fp32-order bar of
    test_gpu_kernels.py::test_attn_decode (3e-4 max, 2e-5 mean per token).  The output starts as NaN and the cache rows past the
    last position are f16 NaN, so a row left unwritten or a read past a token's causal bound shows up;
  * the three tiled rungs on identical data are bit-identical (a row's arithmetic does not depend on TQ or on the tokens that share
    its CTA), and the per-row fallback is within twice the fp32-order bar of them;
  * pb200_attn_ggml (k_attn2<true>) at odd GQA, where one cluster pair of q heads spans two KV heads;
  * the engine at odd-GQA geometries against the oracle port, token by token and after a prefill;
  * 6144-token prompts at the 70B head geometry, whose ubatches pass through all four rungs, prefilled whole and in two chunkings:
    the last-token logits and every position's layer-1 K row, plus a sequential decode of the same prompt."""
import numpy as np
import pytest
import torch

from gpu_util import dev_f32, ptr, sync
from test_gpu_attention import AttnGgmlCase, check_attn_ggml_case
from test_gpu_engine import check_decode_parity, check_prefill_parity, nmse
from test_gpu_kv_shift import kv_tensors
from tiny_model import TinyModel

D = 128
TILED_SMEM = 200 * 1024            # launch_attn_batch's budget for the tiled kernel's dynamic shared memory
ATT_TK, ATT_KSTRIDE = 32, 130      # K / V tile: 32 positions, K rows of 130 halves
RUNGS = (4, 2, 1, "rows")
PLAN_GQAS = (1, 3, 4, 5, 6, 7, 8, 16)
N_UBATCH = 512                     # pb200_prefill's slice length
MAX_ERR, MEAN_ERR = 3e-4, 2e-5     # fp32-order bar of test_gpu_kernels.py::test_attn_decode


def pad32(n):
    return (n + 31) // 32 * 32


def attn_batch_plan(n_head, n_head_kv, n_kv_max):
    """The kernel launch_attn_batch runs: TQ 4, 2 or 1 of k_attn_prefill_tiled, or "rows" (k_attn_rows<false>)."""
    if n_head % n_head_kv:
        return "rows"
    gqa = n_head // n_head_kv
    n_kv_pad = pad32(n_kv_max)
    for tq in (4, 2, 1):
        if gqa * tq * n_kv_pad * 4 + gqa * tq * D * 4 + ATT_TK * ATT_KSTRIDE * 2 <= TILED_SMEM:
            return tq
    return "rows"


def rung_tag(rung):
    return f"tq{rung}" if rung != "rows" else "rows"


def rung_edges(gqa):
    """[(rung, its last n_kv_pad, the next rung)] walking n_kv_pad up in steps of 32 until the per-row fallback."""
    edges, n = [], 32
    cur = attn_batch_plan(gqa, 1, n)
    while cur != "rows":
        nxt = attn_batch_plan(gqa, 1, n + 32)
        if nxt != cur:
            edges.append((cur, n, nxt))
        cur, n = nxt, n + 32
    return edges


# ---- pb200_attn_prefill cases: (gqa, n_head_kv, n_tok, pos0, n_kv_max); token t sits at position pos0 + t ----
CASES = []
for g in sorted(set(PLAN_GQAS) | {2}):
    for _, last, _ in rung_edges(g):          # the last n_kv_max of a rung and the first of the next, the newest token at n_kv_max - 1
        for n_kv_max in (last, last + 1):
            CASES.append((g, 2, 5, n_kv_max - 5, n_kv_max))
for n_kv_max in (700, 2000, 4000, 6100):      # gqa 8 inside each rung: ntq < TQ tails of every size
    for n_tok in (1, 2, 3, 5, 511):
        CASES.append((8, 1, n_tok, n_kv_max - n_tok, n_kv_max))
for j in range(12):                           # the ubatches pb200_prefill makes of a 6144-token prompt: n_kv_max = pos0 + T
    CASES.append((8, 1, N_UBATCH, N_UBATCH * j, N_UBATCH * (j + 1)))
CASES += [(5, 2, 77, 1001, 1200), (3, 3, 130, 2001, 2900), (7, 1, 64, 45, 3000), (16, 1, 200, 333, 700)]   # pos0 not a multiple of 32


def case_id(c):
    g, hk, n_tok, pos0, n_kv_max = c
    return f"{rung_tag(attn_batch_plan(g * hk, hk, n_kv_max))}-gqa{g}-hk{hk}-t{n_tok}-pos{pos0}-kv{n_kv_max}"


def test_cases_reach_every_rung():
    """No GPU: the restated plan has the rungs the launcher's arithmetic gives for gqa 8 (Llama-3-8B / 70B, Qwen2.5-72B), and the case
    list reaches every rung at every listed GQA ratio, with the last n_kv_pad of each rung and the first n_kv_pad of the next."""
    assert rung_edges(8) == [(4, 1376, 2), (2, 2912, 1), (1, 5984, "rows")]
    assert [attn_batch_plan(64, 8, n) for n in (1, 1376, 1377, 2912, 2913, 5984, 5985, 6016)] == [4, 4, 2, 2, 1, 1, "rows", "rows"]
    assert attn_batch_plan(10, 4, 32) == "rows"          # n_head not a multiple of n_head_kv: per-row kernel at any length
    for g in PLAN_GQAS:
        mine = [c for c in CASES if c[0] == g]
        plans = {(attn_batch_plan(g * c[1], c[1], c[4]), pad32(c[4])) for c in mine}
        assert {r for r, _ in plans} == set(RUNGS), (g, plans)
        edges = rung_edges(g)
        assert [e[0] for e in edges] == [4, 2, 1], (g, edges)
        for cur, last, nxt in edges:
            assert (cur, last) in plans and (nxt, last + 32) in plans, (g, cur, last, nxt)
    for c in CASES:
        g, hk, n_tok, pos0, n_kv_max = c
        assert pos0 >= 0 and pos0 + n_tok <= n_kv_max and n_tok <= 65535, c
    assert any(c[3] % 32 for c in CASES if c[2] > 64)


# ---- data and references ----
def make_inputs(g, hk, pos, n_buf, seed):
    """q [n_tok][H*128]; K (x 0.5) / V caches [n_buf][HK*128] f16 whose rows from max(pos) + 1 to the buffer's end are f16 NaN."""
    rng = np.random.default_rng(seed)
    H, n_kv = g * hk, int(pos.max()) + 1
    q = rng.standard_normal((len(pos), H * D)).astype(np.float32)
    Kc = np.full((n_buf, hk * D), np.nan, np.float16)
    Vc = np.full((n_buf, hk * D), np.nan, np.float16)
    Kc[:n_kv] = rng.standard_normal((n_kv, hk * D)) * 0.5
    Vc[:n_kv] = rng.standard_normal((n_kv, hk * D))
    return q, Kc, Vc


def attn_prefill(lib, q, Kc, Vc, pos, H, HK, n_kv_max):
    out = torch.full((len(pos), H * D), float("nan"), device="cuda")
    qd, kd, vd = dev_f32(q), torch.from_numpy(Kc).cuda(), torch.from_numpy(Vc).cuda()
    pd = torch.from_numpy(np.ascontiguousarray(pos, np.int32)).cuda()
    lib.check(lib.c.pb200_attn_prefill(ptr(qd), ptr(kd), ptr(vd), ptr(out), H, HK, D, ptr(pd), len(pos), n_kv_max, 1.0 / np.sqrt(D), None),
              "attn_prefill")
    sync()
    return out.cpu().numpy()


def reference(q, Kc, Vc, pos, H, HK):
    """float64 with the kernel's roundings: s = float32(scale) * K . f16(q), e = exp(s - max), p = f16(e * float32(1 / sum e)),
    out = sum_p p V over cache rows [0, pos]."""
    g, n_kv = H // HK, int(pos.max()) + 1
    scale = np.float64(np.float32(1.0 / np.sqrt(D)))
    q16 = q.reshape(len(pos), HK, g, D).astype(np.float16).astype(np.float64)
    K64 = np.ascontiguousarray(Kc[:n_kv].reshape(n_kv, HK, D).transpose(1, 0, 2)).astype(np.float64)
    V64 = np.ascontiguousarray(Vc[:n_kv].reshape(n_kv, HK, D).transpose(1, 0, 2)).astype(np.float64)
    out = np.empty((len(pos), HK, g, D))
    for t, p in enumerate(pos):
        n = int(p) + 1
        for hk in range(HK):
            s = (q16[t, hk] @ K64[hk, :n].T) * scale
            e = np.exp(s - s.max(axis=1, keepdims=True))
            inv = (1.0 / e.sum(axis=1)).astype(np.float32).astype(np.float64)
            pr = (e * inv[:, None]).astype(np.float16).astype(np.float64)
            out[t, hk] = pr @ V64[hk, :n]
    return out.reshape(len(pos), H * D)


def check_rows(got, want, tol=1.0, what=""):
    """Every token's row within tol x the fp32-order bar: max over the row and mean per token."""
    assert np.isfinite(got).all(), f"{what}: non-finite output at tokens {np.nonzero(~np.isfinite(got).all(axis=1))[0][:16]}"
    err = np.abs(got - want)
    mx, mean = err.max(axis=1), err.mean(axis=1)
    bad = np.nonzero((mx >= tol * MAX_ERR) | (mean >= tol * MEAN_ERR))[0]
    assert bad.size == 0, (what, bad[:16], mx[bad[:16]], mean[bad[:16]])


def sample_tokens(n_tok, rung):
    """First and last token of the first CTA, first token of the last CTA and the last (ragged) token."""
    tq = rung if rung != "rows" else 1
    return sorted({0, min(tq, n_tok) - 1, (n_tok - 1) // tq * tq, n_tok - 1})


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_attn_prefill_every_row(cuda, lib, port, case):
    g, HK, n_tok, pos0, n_kv_max = case
    H = g * HK
    rung = attn_batch_plan(H, HK, n_kv_max)
    pos = (pos0 + np.arange(n_tok)).astype(np.int32)
    q, Kc, Vc = make_inputs(g, HK, pos, pad32(n_kv_max) + 32, seed=g * 1000003 + n_tok * 1009 + pos0)
    got = attn_prefill(lib, q, Kc, Vc, pos, H, HK, n_kv_max)
    check_rows(got, reference(q, Kc, Vc, pos, H, HK), what=case_id(case))
    for t in sample_tokens(n_tok, rung):
        n = int(pos[t]) + 1
        want = port.attention_decode(q[t], Kc[:n].view(np.uint16), Vc[:n].view(np.uint16), H, HK, D, n, 1.0 / np.sqrt(D))
        err = np.abs(got[t] - want)
        assert err.max() < MAX_ERR and err.mean() < MEAN_ERR, (t, err.max(), err.mean())


# ---- the same rows through every rung ----
INDEP = [(8, 1, 37), (3, 2, 23), (16, 1, 29)]


@pytest.mark.gpu
@pytest.mark.parametrize("g,HK,n_tok", INDEP, ids=[f"gqa{g}-hk{hk}-t{n}" for g, hk, n in INDEP])
def test_rungs_bit_identical(cuda, lib, g, HK, n_tok):
    """Same q / K / V / positions, n_kv_max raised so that the launcher takes TQ 4, then 2, then 1, then the per-row kernel.  Inside the
    tiled kernel a row's score, softmax and P.V chain do not depend on TQ or on its CTA's other tokens (past the row's causal length it
    only adds exact zeros), so the three tiled outputs must be bit-identical; k_attn_rows sums in another order and must be within
    twice the fp32-order bar of them, and not bit-identical (evidence that the last n_kv_max did leave the tiled kernel).  Positions are
    shuffled and of different lengths within each CTA."""
    H = g * HK
    edges = rung_edges(g)
    first = {4: 1, **{nxt: last + 1 for _, last, nxt in edges}}          # the smallest n_kv_max of each rung
    rng = np.random.default_rng(g * 100 + n_tok)
    n_kv = edges[0][1]                                                  # every row fits TQ 4
    pos = rng.permutation(n_kv)[:n_tok].astype(np.int32)
    pos[rng.integers(n_tok)] = n_kv - 1
    q, Kc, Vc = make_inputs(g, HK, pos, pad32(first["rows"]) + 32, seed=g + n_tok)
    outs = {}
    for rung in RUNGS:
        n_kv_max = max(first[rung], n_kv)
        assert attn_batch_plan(H, HK, n_kv_max) == rung
        outs[rung] = attn_prefill(lib, q, Kc, Vc, pos, H, HK, n_kv_max)
    check_rows(outs[4], reference(q, Kc, Vc, pos, H, HK), what="tq4")
    for rung in (2, 1):
        assert np.array_equal(outs[rung].view(np.uint32), outs[4].view(np.uint32)), (rung, np.nonzero(outs[rung] != outs[4]))
    check_rows(outs["rows"], outs[4], tol=2.0, what="rows vs tiled")
    assert not np.array_equal(outs["rows"].view(np.uint32), outs[4].view(np.uint32))


# ---- decode attention: cluster pairs across two KV heads ----
# (H, HK), n_cells, kv_head, RoPE mode, freq factors, n_dims, mask: gqa 3, 5 and 7, so heads 2j and 2j + 1 of some cluster read different
# KV heads
ODD_GGML = [((6, 2), 304, 303, 0, True, 128, "causal"), ((10, 2), 1000, 128, 2, False, 128, "holes"),
            ((14, 2), 264, 263, 0, False, 64, "chunk"), ((24, 8), 4096, 2500, 2, True, 128, "holes")]


@pytest.mark.gpu
@pytest.mark.parametrize("heads,n_cells,kv_head,mode,ff,n_dims,mask_kind", ODD_GGML,
                         ids=[f"h{h[0]}x{h[1]}-c{n}-kv{k}-m{m}{'ff' if f else ''}-d{nd}-{mk}" for h, n, k, m, f, nd, mk in ODD_GGML])
def test_attn_ggml_odd_gqa(cuda, lib, port, heads, n_cells, kv_head, mode, ff, n_dims, mask_kind):
    H, HK = heads
    check_attn_ggml_case(lib, port, AttnGgmlCase(lib, H, HK, n_cells, kv_head, mode, ff, n_dims, mask_kind, seed=H * 1000 + n_cells))


# ---- the engine at odd GQA ----
ODD_ENGINE = [(6, 2), (10, 2), (14, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("arch", ["llama", "qwen2"])
@pytest.mark.parametrize("H,HK", ODD_ENGINE, ids=[f"h{h}x{hk}" for h, hk in ODD_ENGINE])
def test_engine_odd_gqa_vs_port(cuda, pkg, port, H, HK, arch):
    """n_embd = H * 128 at gqa 3, 5, 7: 44 tokens decoded against the oracle port (the multi-token bar), then a 36-token prefill and
    8 decode steps under the bars of test_prefill_matches_sequential_decode_and_oracle."""
    tm = TinyModel(n_layer=2, n_embd=H * 128, n_head=H, n_head_kv=HK, n_ff=1024, n_vocab=384, n_ctx=64, arch=arch,
                   ftype="q4_K_M" if arch == "llama" else "q5_K_M", freq_factors=arch == "llama", seed=H, branch_scale=0.1)
    toks = [(i * 7919 + 13) % 384 for i in range(44)]
    T = 36
    want, _ = tm.port_decode(port, toks)
    eng = tm.load_engine(pkg)
    seq = np.zeros_like(want)
    for i, t in enumerate(toks):
        eng.decode(int(t), i, seq[i])
    eng.kv_clear()
    got = np.zeros_like(want)
    eng.prefill(toks[:T], 0, got[T - 1])
    for i in range(T, len(toks)):
        eng.decode(int(toks[i]), i, got[i])
    eng.close()
    check_decode_parity(seq, want)
    check_prefill_parity(got, seq, want, T)


# ---- long prompts at the 70B head geometry ----
LONG_N = 6144
LONG_SPLITS = {"whole": [LONG_N], "700s": [700] * 8 + [544], "3000+3144": [3000, 3144]}
K_ROW_BAR = 2.0 ** -6         # 32 f16 ulps of a row's largest |K|; see test_long_prompt_70b_heads


def ubatch_rungs(sizes, n_head=64, n_head_kv=8):
    """The rung of every ubatch pb200_prefill runs for consecutive calls of these sizes."""
    out, p0 = [], 0
    for T in sizes:
        for done in range(0, T, N_UBATCH):
            out.append(attn_batch_plan(n_head, n_head_kv, p0 + done + min(N_UBATCH, T - done)))
        p0 += T
    return out


def test_long_prompt_splits_cover_the_rungs():
    """No GPU: one 6144-token call passes through all four rungs, and the chunkings put some of the same tokens into other rungs."""
    assert set(ubatch_rungs(LONG_SPLITS["whole"])) == set(RUNGS)
    assert ubatch_rungs(LONG_SPLITS["700s"]) != ubatch_rungs(LONG_SPLITS["whole"])
    assert all(sum(s) == LONG_N for s in LONG_SPLITS.values())


@pytest.mark.gpu
def test_long_prompt_70b_heads(cuda, pkg):
    """2 layers of 64 q heads over 8 KV heads (n_embd 8192), a 6144-token prompt decoded token by token (k_attn2, independent of the
    prompt kernels) and prefilled in one call (ubatches at TQ 4, 2, 1 and the per-row kernel), in calls of 700 and in 3000 + 3144.

    Layer-1 K rows: the K row of every position depends on that token's layer-0 attention row.  Each prefill's rows are checked
    against the sequential decode's rows and against the one-call prefill's rows: max |dK| <= K_ROW_BAR x max |K| of the row.  What
    moves a correct row is the order of fp32 additions (the stream-K cuts of the mat-muls, <= 3 atomic adds per element whose order
    varies from run to run, test_gpu_mmq.py; the per-row kernel against the tiled one), against decode also the prefill mat-mul's fp16
    operand roundings (test_gpu_mmq.py's bound).  Those flip a q8_K code of the layer-1 activation now and then (a 1/127-of-amax step
    on one input of the K product) and the final f16 rounding of K.  Measured on an H100 SXM (700 W): rows move by <= 6.7e-3 between
    chunkings, <= 5.4e-3 between two runs of the same call, <= 8.6e-3 against decode (median 4e-3, about 8 ulps), so the bar is
    32 ulps.  A prompt kernel one cell short for one TQ slot (n_kv - 1) moves rows by 2.4e-2 to 7e-2 against decode.

    Last-token logits: NMSE 1e-3 and a greedy token within 0.1 of the best (test_prefill_matches_sequential_decode_and_oracle's
    prefill-vs-decode bar), against decode and between the prefills.  test_prefill_chunked_equals_whole's 1e-6 does not hold at this
    size: its small matrices have no stream-K cuts, these do, and two runs of the same one-call prefill are already 1.1e-4 apart on
    an H100 (chunkings 1.2e-4 to 1.4e-4, decode 1.8e-4)."""
    tm = TinyModel(n_layer=2, n_embd=8192, n_head=64, n_head_kv=8, n_ff=512, n_vocab=256, n_ctx=LONG_N + 64, arch="llama",
                   ftype="q4_K_M", seed=61, branch_scale=0.1)
    toks = [(i * 7919 + 13) % 256 for i in range(LONG_N)]
    eng = tm.load_engine(pkg)

    def layer1_k():
        kc, _ = kv_tensors(eng, tm, 1, 2)
        return kc[0, 1, :LONG_N].cpu().numpy().view(np.float16).astype(np.float32)
    logits, k1 = {"decode": np.zeros(tm.hp["n_vocab"], np.float32)}, {}
    for i, t in enumerate(toks):
        eng.decode(int(t), i, logits["decode"] if i == LONG_N - 1 else None)
    k1["decode"] = layer1_k()
    for name, sizes in LONG_SPLITS.items():
        eng.kv_clear()
        p0 = 0
        for T in sizes:
            logits[name] = eng.prefill(toks[p0:p0 + T], p0).copy()
            p0 += T
        k1[name] = layer1_k()
    eng.close()
    for name in LONG_SPLITS:
        assert np.isfinite(logits[name]).all() and np.isfinite(k1[name]).all(), name
        for ref in ("decode", "whole"):
            a, b = logits[ref], logits[name]
            rel = np.abs(k1[name] - k1[ref]).max(axis=1) / np.abs(k1[ref]).max(axis=1)
            print(f"{name} vs {ref}: logits NMSE {nmse(b, a):.3e}; layer-1 K rows max {rel.max():.3e} at {rel.argmax()}")
            bad = np.nonzero(rel > K_ROW_BAR)[0]
            assert bad.size == 0, (name, ref, bad[:16], rel[bad[:16]])
            assert nmse(b, a) < 1e-3, (name, ref, nmse(b, a))
            assert a[b.argmax()] >= a.max() - 0.1, (name, ref)
