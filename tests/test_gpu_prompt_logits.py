"""-m gpu: logits at every prompt position (pb200_prompt_head), their scoring on the device (pb200_token_scores) and llama-perplexity's
chunk loop on the engine (prima.cpp_b200/perplexity.py).

1. k_token_scores against a float64 numpy restatement of the reference's log_softmax (f32 expf of the f32 difference, double sum) at
   vocabularies from 160 to 262 144, with exact ties at the maximum, -inf entries, a -inf target and unscored targets (-1, n_vocab).
2. The head rows bit for bit against the same head built from single ops on pb200_prefill_hidden_device's rows: pb200_rms_norm ->
   pb200_binary mul -> pb200_mul_mat_q, or pb200_mul_mat_vec per row below 8 rows.  Bit identity holds where every output tile of the
   mat-mul is computed by one CTA; every shape here is asserted unsplit (mmq_plan), as in test_gpu_prefill_layers.py.  The last row is
   also held against the prefill's own last-token logits (the decode GEMV head): to the GEMV bar (4e-6 of the largest |logit|) where the
   range takes the row-by-row GEMV (each T has such a range), to test_gpu_mmq.py's NMSE 4e-6 where it takes the fp16 tensor cores.
3. All rows of a 36-token prompt against the engine's sequential decode, the port oracle token by token and the reference CPU backend's
   batched prompt, with test_gpu_engine.py's prefill bars.
4. A prompt_head call changes nothing that prefill left: K / V cache, pb200_logits_device, the slot's words, the hidden rows; a decode
   step afterwards gives identical logits.
5. Two pipeline shards, head per micro-batch on the head shard, against the whole model.
6. Every argument error.
7. Perplexity end to end on a tiny llama: the mean nll equals the scores of the loop's own head calls and the restatement on their
   logits, and ppl agrees with the port oracle decoding every chunk token by token."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from gpu_util import act_ws, dev_f32, ptr, sync
from test_gpu_kv_shift import _dev, kv_tensors
from test_gpu_mmq import mmq_plan
from test_gpu_prefill_layers import pf_tc
from tiny_model import TinyModel

pytestmark = pytest.mark.gpu
EINVAL, ESTATE = -1, -4


def nmse(a, b):
    return float(np.sum((a.astype(np.float64) - b) ** 2) / np.sum(b.astype(np.float64) ** 2))


def restate_scores(logits, targets):
    """perplexity.cpp log_softmax per row: (nll f8, logit f4, prob f4, top i4); unscored rows (target outside [0, n_vocab)) zero."""
    n, V = logits.shape
    mx = logits.max(axis=1)
    top = logits.argmax(axis=1)
    out = []
    for r in range(n):
        e = np.exp((logits[r] - mx[r]).astype(np.float32)).astype(np.float64)
        s = float(np.sum(e))
        t = int(targets[r])
        if 0 <= t < V:
            l = logits[r, t]
            out.append((float(mx[r]) + math.log(s) - float(l), float(l), float(np.float32(np.exp(np.float32(l - mx[r]))) / np.float32(s)), int(top[r])))
        else:
            out.append((0.0, 0.0, 0.0, int(top[r])))
    return out


# ---- 1. the scoring kernel ----
SCORE_CASES = [(V, n) for V in (160, 384, 32000) for n in (1, 37, 512)] + [(128256, 64), (152064, 512), (262144, 130)]


@pytest.mark.parametrize("V,n", SCORE_CASES, ids=[f"V{V}-rows{n}" for V, n in SCORE_CASES])
def test_token_scores_kernel(cuda, lib, pkg, V, n):
    rng = np.random.default_rng(V + n)
    scale = np.exp(rng.uniform(np.log(0.05), np.log(40.0), n)).astype(np.float32)
    x = (rng.standard_normal((n, V)).astype(np.float32) * scale[:, None]).astype(np.float32)
    tg = rng.integers(0, V, n).astype(np.int32)
    for r in range(n):
        kind = r % 6
        if kind == 1:                                         # exact ties at the maximum: the first index wins
            m = x[r].max()
            idx = rng.choice(V, size=min(4, V), replace=False)
            x[r, idx] = m + 1.0
        elif kind == 2:                                       # -inf entries, target among them: nll +inf, prob 0
            idx = rng.choice(V, size=V // 10, replace=False)
            x[r, idx] = -np.inf
            tg[r] = idx[0]
        elif kind == 3:
            tg[r] = -1                                        # unscored
        elif kind == 4:
            tg[r] = V                                         # unscored
        elif kind == 5:
            x[r, rng.choice(V, size=V // 3, replace=False)] = -np.inf
    if n == 1:
        tg[0] = int(np.argmax(x[0]))
    xd, td = dev_f32(x), torch.from_numpy(tg).cuda()
    out = torch.full((n * 24,), 0xA5, dtype=torch.uint8, device="cuda")
    before = lib.c.pb200_kernel_launches()
    lib.token_scores(xd.data_ptr(), n, V, td.data_ptr(), out.data_ptr())
    sync()
    assert lib.c.pb200_kernel_launches() - before == 1
    got = out.cpu().numpy().view(np.dtype(pkg.TokenScore))
    want = restate_scores(x, tg)
    for r, (nll, logit, prob, top) in enumerate(want):
        g = got[r]
        assert int(g["top"]) == top, (r, int(g["top"]), top)
        assert np.float32(g["logit"]).view(np.uint32) == np.float32(logit).view(np.uint32), (r, g["logit"], logit)
        if math.isinf(nll):
            assert math.isinf(g["nll"]) and g["nll"] > 0 and g["prob"] == 0.0, (r, g)
            continue
        assert abs(g["nll"] - nll) <= 1e-6 * max(1.0, abs(nll)), (r, g["nll"], nll)
        assert abs(g["prob"] - prob) <= 1e-6 * max(1.0, abs(prob)), (r, g["prob"], prob)
        if not 0 <= tg[r] < V:
            assert g["nll"] == 0.0 and g["logit"] == 0.0 and g["prob"] == 0.0, (r, g)


# ---- 2. head rows bit for bit against single ops ----
def tiny(arch, V=384, n_ctx=640, **kw):
    ftype = "q4_K_M" if arch == "llama" else "q5_K_M"
    return TinyModel(n_layer=2, n_embd=1024, n_head=8, n_head_kv=2, n_ff=2048, n_vocab=V, n_ctx=n_ctx, arch=arch, ftype=ftype, seed=31,
                     branch_scale=0.1, **kw)


def compose_head(lib, eng, tm, hid, row0, n):
    """output_norm and the head from single ops on the hidden rows hid [T][E] (device): rms_norm -> mul -> mul_mat_q (pf_tc), else
    quantize + mul_mat_vec per row."""
    c, hp = lib.c, tm.hp
    E, V = hp["n_embd"], hp["n_vocab"]
    x = hid[row0:row0 + n].contiguous()
    y = torch.full_like(x, float("nan"))
    lib.check(c.pb200_rms_norm(ptr(x), ptr(y), E, n, hp["rms_eps"], None), "rms_norm")
    w, _, _ = eng.tensor_device("output_norm.weight")
    xn = torch.full_like(x, float("nan"))
    lib.check(c.pb200_binary(C.c_int(1), ptr(y), C.c_void_p(w), ptr(xn), C.c_int64(n * E), C.c_int64(E), None), "binary mul")
    W, _, t = eng.tensor_device("output.weight")
    out = torch.full((n, V), float("nan"), dtype=torch.float32, device="cuda")
    if pf_tc(t, E, n):
        assert not mmq_plan(lib, V, E, n).split, (V, E, n, mmq_plan(lib, V, E, n))
        ws = torch.empty(c.pb200_mul_mat_q_workspace_bytes(E, n), dtype=torch.uint8, device="cuda")
        lib.check(c.pb200_mul_mat_q(t, C.c_void_p(W), V, E, ptr(xn), E, n, ptr(out), None, None, ptr(ws), None), "mul_mat_q")
    else:
        aws = act_ws(lib, E)
        for i in range(n):
            lib.check(c.pb200_mul_mat_vec(t, C.c_void_p(W), V, E, C.c_void_p(xn.data_ptr() + i * E * 4), C.c_void_p(out.data_ptr() + i * V * 4),
                                          ptr(aws), None), "mul_mat_vec")
    sync()
    return out.cpu().numpy()


HEAD_CASES = {5: [(0, 5), (2, 3), (4, 1)], 36: [(0, 36), (3, 8), (30, 6), (35, 1)], 512: [(0, 512), (256, 200), (100, 7), (511, 1)]}


@pytest.mark.parametrize("arch", ["llama", "qwen2"])
def test_head_rows_bit_identical_to_single_ops(cuda, lib, pkg, arch):
    tm = tiny(arch)
    E, V = tm.hp["n_embd"], tm.hp["n_vocab"]
    eng = tm.load_engine(pkg)
    try:
        for T, ranges in HEAD_CASES.items():
            toks = [(i * 7919 + 13 * T) % V for i in range(T)]
            last = eng.prefill(toks, 0).copy()
            hid = _dev(lib.c.pb200_prefill_hidden_device(eng.h), (T, E), "<f4").clone()
            for row0, n in ranges:
                before = lib.c.pb200_kernel_launches()
                got, _ = eng.prompt_head(row0, n)
                assert lib.c.pb200_aborted() == 0
                launches = lib.c.pb200_kernel_launches() - before
                assert launches == (2 if pf_tc(tm.tensors["output.weight"][0], E, n) else 1 + 2 * n), (T, row0, n, launches)
                want = compose_head(lib, eng, tm, hid, row0, n)
                bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
                assert bad.size == 0, f"T {T} rows [{row0}, {row0 + n}): {len(bad)} logits differ, first {tuple(bad[0])}"
                if row0 + n == T and not pf_tc(tm.tensors["output.weight"][0], E, n):
                    # the same integer-dot GEMV as the prefill's last-token head: only the rms scale's summation order differs
                    err = float(np.max(np.abs(got[-1].astype(np.float64) - last)))
                    assert err <= 4e-6 * float(np.max(np.abs(last))), (T, err)
                elif row0 + n == T:
                    assert nmse(got[-1], last) < 4e-6, (T, nmse(got[-1], last))     # fp16 tensor-core operands: test_gpu_mmq.py's bar
    finally:
        eng.close()


# ---- 3. every row against the oracles ----
ORACLE_CASES = [("llama", "q4_K_M", True, 384), ("qwen2", "q5_K_M", False, 384), ("llama", "q4_K_M", True, 330)]


def oracle_model(arch, ftype, ff, V):
    """test_prefill_matches_sequential_decode_and_oracle's models (V 330: a vocabulary that is not a multiple of 128)."""
    return TinyModel(n_layer=3, n_embd=1024, n_head=8, n_head_kv=2, n_ff=2816 if arch == "llama" else 3104, n_vocab=V, n_ctx=96, arch=arch,
                     ftype=ftype, freq_factors=ff, seed=23, branch_scale=0.1)


def all_rows(pkg, tm, toks):
    eng = tm.load_engine(pkg)
    seq = np.zeros((len(toks), tm.hp["n_vocab"]), np.float32)
    for i, t in enumerate(toks):
        eng.decode(int(t), i, seq[i])
    eng.kv_clear()
    eng.prefill(toks, 0)
    got, _ = eng.prompt_head(0, len(toks))
    eng.close()
    return got, seq


@pytest.mark.parametrize("arch,ftype,ff,V", ORACLE_CASES, ids=[f"{a}-{f}-V{v}" for a, f, _, v in ORACLE_CASES])
def test_all_rows_match_sequential_decode_and_port(cuda, pkg, port, arch, ftype, ff, V):
    tm = oracle_model(arch, ftype, ff, V)
    toks = [(i * 7919 + 13) % V for i in range(36)]
    got, seq = all_rows(pkg, tm, toks)
    want, _ = tm.port_decode(port, toks)
    assert nmse(got, seq) < 1e-3, nmse(got, seq)
    assert nmse(got, want) < 2e-3, nmse(got, want)
    assert np.mean(got.argmax(1) == want.argmax(1)) >= 0.85
    assert np.mean(got.argmax(1) == seq.argmax(1)) >= 0.85


@pytest.mark.parametrize("arch,ftype,ff,V", ORACLE_CASES, ids=[f"{a}-{f}-V{v}" for a, f, _, v in ORACLE_CASES])
def test_all_rows_match_reference_batched_prompt(cuda, pkg, ref, arch, ftype, ff, V):
    tm = oracle_model(arch, ftype, ff, V)
    toks = [(i * 7919 + 13) % V for i in range(36)]
    got, _ = all_rows(pkg, tm, toks)
    want, _ = tm.ref_decode(ref, toks, batch_prefill=len(toks))
    assert nmse(got, want) < 2e-3, nmse(got, want)
    assert np.mean(got.argmax(1) == want.argmax(1)) >= 0.85


# ---- 4. nothing else changes ----
@pytest.mark.parametrize("T", [36, 5])
def test_prompt_head_changes_nothing_else(cuda, lib, pkg, T):
    tm = tiny("llama", n_ctx=96)
    E, V = tm.hp["n_embd"], tm.hp["n_vocab"]
    toks = [(i * 31 + 7) % V for i in range(T)]
    eng = tm.load_engine(pkg)
    try:
        eng.prefill(toks, 0)
        eng.decode(3, T, None)                               # the step after the prompt, without a head call
        want_next = eng.debug_read("logits", V)
        eng.prefill(toks, 0)
        eng.set_tokpos_seq(0, 11, T)

        def state():
            k, v = kv_tensors(eng, tm, 1, tm.hp["n_layer"])
            return (k.cpu().numpy(), v.cpu().numpy(), _dev(eng.logits_ptr, (V,), "<f4").cpu().numpy(),
                    _dev(eng.token_ptr(0), (4,), "<i4").cpu().numpy(), _dev(eng.hidden_out_ptr, (E,), "<f4").cpu().numpy(),
                    _dev(lib.c.pb200_prefill_hidden_device(eng.h), (T, E), "<f4").cpu().numpy())
        sync()
        before = state()
        eng.prompt_head(0, T, targets=np.arange(T) % V)
        eng.prompt_head(T - 3, 3, targets=[-1, 2, 5], logits=False)
        after = state()
        for name, a, b in zip(("K", "V", "logits", "slot words", "hidden out", "hidden rows"), before, after):
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), name
        eng.decode(3, T, None)
        assert np.array_equal(eng.debug_read("logits", V).view(np.uint32), want_next.view(np.uint32))
    finally:
        eng.close()


# ---- 5. pipeline shards ----
def test_pipeline_shards_head_per_micro_batch(cuda, pkg):
    """test_prefill_stage_pipeline_matches_single_model's model and micro-batches; the head shard scores each micro-batch's rows."""
    tm = TinyModel(n_layer=4, n_embd=512, n_head=4, n_head_kv=2, n_ff=1024, n_vocab=256, n_ctx=96, arch="llama", ftype="q4_K_M",
                   freq_factors=False, seed=8, branch_scale=0.1)
    toks = [(i * 31 + 7) % 256 for i in range(72)]
    one = tm.load_engine(pkg)
    one.prefill(toks, 0)
    want, want_s = one.prompt_head(0, 72, targets=toks[1:] + [-1])
    one.close()
    a = tm.load_engine(pkg, layers=(0, 2), with_embd=True, with_head=False)
    b = tm.load_engine(pkg, layers=(2, 4), with_embd=False, with_head=True)
    rows, scores = [], []
    for p0, n in ((0, 40), (40, 32)):
        h = a.prefill_stage(toks[p0:p0 + n], None, n, p0, synchronize=True)   # b reads a's rows from another stream
        b.prefill_stage(None, h, n, p0)
        lg, s = b.prompt_head(0, n, targets=(toks[1:] + [-1])[p0:p0 + n])
        rows.append(lg)
        scores.append(s)
    a.close(); b.close()
    got = np.concatenate(rows)
    assert nmse(got, want) < 1e-6, nmse(got, want)
    got_s = np.concatenate(scores)
    assert np.allclose(got_s["nll"][:-1], want_s["nll"][:-1], rtol=1e-3, atol=1e-3) and got_s["nll"][-1] == 0.0


# ---- 6. argument errors ----
def test_argument_errors(cuda, lib, pkg):
    tm = tiny("llama", n_ctx=64)
    V = tm.hp["n_vocab"]
    c = lib.c
    out = np.zeros((16, V), np.float32)
    sc = np.zeros(16, np.dtype(pkg.TokenScore))
    tg = np.zeros(16, np.int32)

    def call(m, row0, n, t=tg, lg=out, s=None):
        p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
        return c.pb200_prompt_head(m, row0, n, p(t), p(lg), p(s))
    assert call(None, 0, 1) == ESTATE
    raw = pkg.Model(pkg.HParams(**tm.hp), 0)
    assert call(raw.h, 0, 1) == ESTATE                                            # not finalized
    raw.close()
    eng = tm.load_engine(pkg)
    noh = tm.load_engine(pkg, layers=(0, 1), with_embd=True, with_head=False)
    try:
        assert call(noh.h, 0, 1) == ESTATE
        assert call(eng.h, 0, 1) == EINVAL                                        # no prefill yet
        eng.prefill(list(range(12)), 0)
        assert call(eng.h, 0, 12) == 0 and call(eng.h, 11, 1, s=sc) == 0
        assert call(eng.h, -1, 2) == EINVAL
        assert call(eng.h, 0, 0) == EINVAL and call(eng.h, 0, -3) == EINVAL
        assert call(eng.h, 5, 8) == EINVAL and call(eng.h, 12, 1) == EINVAL and call(eng.h, 0, 13) == EINVAL
        assert call(eng.h, 0, 4, lg=None) == EINVAL                               # both outputs NULL
        assert call(eng.h, 0, 4, t=None, lg=None, s=sc) == EINVAL                 # scores without targets
        bad = tg.copy(); bad[2] = V
        assert call(eng.h, 0, 4, t=bad) == EINVAL
        neg = tg.copy(); neg[1] = -7
        assert call(eng.h, 0, 4, t=neg, lg=None, s=sc) == 0 and sc["nll"][1] == 0.0
        assert call(eng.h, 0, 4, t=None) == 0                                     # logits only
        d = dev_f32(np.zeros((2, V), np.float32))
        t = torch.zeros(2, dtype=torch.int32, device="cuda")
        o = torch.zeros(48, dtype=torch.uint8, device="cuda")
        for args in ((None, 2, V, ptr(t), ptr(o)), (ptr(d), 2, V, None, ptr(o)), (ptr(d), 2, V, ptr(t), None), (ptr(d), 0, V, ptr(t), ptr(o)),
                     (ptr(d), 2, 0, ptr(t), ptr(o)), (ptr(d), 1 << 31, V, ptr(t), ptr(o))):
            assert c.pb200_token_scores(*args, None) == EINVAL, args
    finally:
        eng.close(); noh.close()


# ---- 7. perplexity end to end ----
@pytest.mark.parametrize("n_ctx,n_chunks", [(64, 3), (1000, 1)])
def test_perplexity_end_to_end(cuda, pkg, port, n_ctx, n_chunks):
    """The chunk loop's mean nll equals the mean of the scores its prompt_head calls returned to 1e-12 (the loop's accumulation), and the
    restatement on those calls' own logits to 1e-8: the restatement's numpy f32 exp and the device's expf differ by an ulp or two per
    term, which moves each nll by about 1e-8, within the kernel's 1e-6 bar.  The perplexity agrees with the port oracle decoding every
    chunk token by token (with the same BOS substitution) to 1 %.  n_ctx 1000 spans two ubatches, both with scored rows (from 500 on)."""
    tm = TinyModel(n_layer=2, n_embd=512, n_head=4, n_head_kv=2, n_ff=1024, n_vocab=320, n_ctx=1024, arch="llama", ftype="q4_K_M",
                   freq_factors=True, seed=41, branch_scale=0.1)
    V, bos = 320, 1
    toks = ((np.arange(max(n_chunks, 2) * n_ctx) * 7919 + 13) % V).astype(np.int32)
    eng = tm.load_engine(pkg)
    seen = []
    head = eng.prompt_head

    def spy(row0, n, targets=None, logits=True):
        lg, s = head(row0, n, targets=targets, logits=True)
        seen.append((lg, np.asarray(targets), s["nll"].copy()))
        return lg, s
    eng.prompt_head = spy
    import io
    res = pkg.perplexity.perplexity(toks, n_ctx, pkg.perplexity.model_run_chunk(eng), n_chunks, bos, out=io.StringIO())
    eng.close()
    first = n_ctx // 2
    assert res.count == n_chunks * (n_ctx - 1 - first)
    assert len(seen) == n_chunks * (2 if n_ctx > 512 else 1)                    # one head call per ubatch with scored rows
    own = np.concatenate([v for _, _, v in seen])
    assert own.size == res.count and abs(float(np.mean(own)) / res.nll - 1) < 1e-12, (float(np.mean(own)), res.nll)
    nll = [s[0] for lg, tg, _ in seen for s in restate_scores(lg, tg)]
    assert abs(float(np.mean(nll)) / res.nll - 1) < 1e-8, (float(np.mean(nll)), res.nll)
    onll = []
    for i in range(n_chunks):
        ch = toks[i * n_ctx:(i + 1) * n_ctx].copy()
        ch[0] = bos
        lg, _ = tm.port_decode(port, ch)
        onll += [s[0] for s in restate_scores(lg[first:n_ctx - 1], ch[first + 1:])]
    ppl_port = math.exp(float(np.mean(onll)))
    print(f"n_ctx {n_ctx}: ppl {res.ppl:.6f} (engine) vs {ppl_port:.6f} (port oracle, token by token)")
    assert abs(res.ppl / ppl_port - 1) < 1e-2, (res.ppl, ppl_port)
