"""-m gpu: llama-perplexity's KL-divergence modes on the device: the log-probability writer (pb200_logprobs_u16), the KLD function
(pb200_kld_scores), both on prompt rows (pb200_prompt_head_kld) and end to end (prima.cpp_b200/perplexity.py).

1. pb200_logprobs_u16 against the reference's records in tests/golden/kld_golden.npz at vocabularies 160 to 262 144 (ties at the
   maximum, -inf entries and a -inf target, ranges under and far over 16, constant rows): scale and every entry bit for bit, pad
   included; min_log_prob and nll within 2 ulp.
2. pb200_kld_scores against the golden outputs: same_top exact, nll and nll_base within 2 ulp, p_diff to the ulps of its two expf,
   kld within kld_ref.kld_bound (5e-7 of the sum of the terms' magnitudes, plus 2 ulp of max + lse times the base mass included).
3. pb200_prompt_head_kld bit for bit against the two kernels on pb200_prompt_head's logits of the same rows, in writer mode, compare
   mode and both, with the tensor-core head (>= 8 rows) and the row-by-row one; nothing else changes; every argument error.
4. Two pipeline shards: the head shard's records and KLD per micro-batch against the whole model.
5. End to end on a tiny llama, 3 chunks: (a) the engine against its own base file; (b) against a base file of the port oracle's
   token-by-token logits written by the reference's writer, per position equal to the reference's KLD function on the engine's logits."""
import ctypes as C
import hashlib
import io
import math

import numpy as np
import pytest
import torch

import kld_ref as K
from gpu_util import dev_f32, ptr, sync
from test_gpu_kv_shift import _dev, kv_tensors
from test_gpu_prefill_layers import pf_tc
from test_gpu_prompt_logits import nmse, tiny
from tiny_model import TinyModel

pytestmark = pytest.mark.gpu
EINVAL, ESTATE = -1, -4
VOCABS = (160, 1001, 32000, 128256, 152064, 262144)
f4, f8 = np.float32, np.float64


def ulps(a, b):
    a, b = f4(a), f4(b)
    if a == b:
        return 0
    return abs(int(np.array(a).view(np.int32)) - int(np.array(b).view(np.int32)))


def golden(V):
    with np.load(K.GOLDEN) as z:
        g = {k[len(f"V{V}_"):]: z[k] for k in z.files if k.startswith(f"V{V}_")}
    xs, ys, toks = [], [], []
    for k, s in zip(g["kinds"], g["seeds"]):
        x, y, t = K.make_rows(V, int(s), K.KINDS[int(k)])
        xs.append(x); ys.append(y); toks.append(t)
    return g, np.stack(xs), np.stack(ys), np.array(toks, np.int32)


def device_records(lib, rows, toks, V):
    n, nv = len(rows), K.record_u16s(V)
    x, t = dev_f32(rows), torch.from_numpy(np.ascontiguousarray(toks, np.int32)).cuda()
    rec = torch.full((n * nv,), 0xA5A5 - 65536, dtype=torch.int16, device="cuda")        # poisoned: every entry must be written
    nll = torch.full((n,), float("nan"), dtype=torch.float32, device="cuda")
    before = lib.c.pb200_kernel_launches()
    lib.logprobs_u16(x.data_ptr(), n, V, t.data_ptr(), rec.data_ptr(), nll.data_ptr())
    sync()
    assert lib.c.pb200_kernel_launches() - before == 1
    return rec.cpu().numpy().view(np.uint16).reshape(n, nv), nll.cpu().numpy()


# ---- 1. the writer ----
@pytest.mark.parametrize("V", VOCABS)
def test_logprobs_u16_matches_reference(cuda, lib, V):
    g, xs, ys, toks = golden(V)
    rows, tg = np.concatenate([xs, ys]), np.concatenate([toks, toks])
    rec, nll = device_records(lib, rows, tg, V)
    sc, mlp = K.header(rec)
    assert np.array_equal(sc.view(np.uint32), g["scale"].view(np.uint32)), (sc, g["scale"])
    for r in range(len(rows)):
        assert ulps(mlp[r], g["min_log_prob"][r]) <= 2, (r, mlp[r], g["min_log_prob"][r])
        assert ulps(nll[r], g["nll"][r]) <= 2, (r, nll[r], g["nll"][r])
        if "records" in g:
            assert np.array_equal(rec[r, 4:], g["records"][r, 4:]), (r, np.flatnonzero(rec[r, 4:] != g["records"][r, 4:])[:8])
        else:
            assert hashlib.sha256(rec[r, 4:].astype("<u2").tobytes()).digest() == g["sha"][r].tobytes(), r
    # an unscored target: nll 0, the record unchanged
    rec2, nll2 = device_records(lib, rows[:2], np.array([-1, V], np.int32), V)
    assert np.array_equal(rec2, rec[:2]) and not nll2.any()


# ---- 2. the KLD function ----
def golden_base(lib, g, ys, toks, V):
    """The base rows' records: entries from the device (held bit for bit to the reference by test 1), header from the reference."""
    rec, _ = device_records(lib, ys, toks, V)
    n = len(ys)
    rec[:, :4] = np.stack([g["scale"][n:], g["min_log_prob"][n:]], axis=1).astype(f4).view(np.uint16)
    return rec


def device_kld(lib, pkg, xs, base, toks, V):
    n = len(xs)
    x, b = dev_f32(xs), torch.from_numpy(base.view(np.int16).copy()).cuda()
    t = torch.from_numpy(np.ascontiguousarray(toks, np.int32)).cuda()
    out = torch.full((n * 24,), 0xA5, dtype=torch.uint8, device="cuda")
    before = lib.c.pb200_kernel_launches()
    lib.kld_scores(x.data_ptr(), n, V, b.data_ptr(), t.data_ptr(), out.data_ptr())
    sync()
    assert lib.c.pb200_kernel_launches() - before == 1
    return out.cpu().numpy().view(np.dtype(pkg.KldScore))


def check_kld(got, xs, base, toks, want):
    """want[r] = (kld, nll, nll_base, p_diff, same_top) of the reference's function."""
    for r in range(len(xs)):
        kld, nll, nll_base, p_diff, top = want[r]
        g = got[r]
        assert bool(g["same_top"]) == bool(top), r
        assert ulps(g["nll"], nll) <= 2 and ulps(g["nll_base"], nll_base) <= 2, (r, g, want[r])
        p, pb = f8(np.exp(-f8(nll))), f8(np.exp(-f8(nll_base)))
        tol = (p * 3 * f8(np.spacing(abs(f4(nll)))) if np.isfinite(nll) else 0.0) + 4 * f8(np.spacing(f4(p))) + 4 * f8(np.spacing(f4(pb)))
        assert abs(f8(g["p_diff"]) - f8(p_diff)) <= tol, (r, g["p_diff"], p_diff, tol)
        bound = K.kld_bound(xs[r], base[r])
        assert abs(g["kld"] - kld) <= bound, (r, g["kld"], kld, bound)


@pytest.mark.parametrize("V", VOCABS)
def test_kld_scores_match_reference(cuda, lib, pkg, V):
    g, xs, ys, toks = golden(V)
    base = golden_base(lib, g, ys, toks, V)
    got = device_kld(lib, pkg, xs, base, toks, V)
    want = list(zip(g["kld"], g["kld_nll"], g["kld_nll_base"], g["p_diff"], g["same_top"]))
    check_kld(got, xs, base, toks, want)
    # unscored targets zero what depends on them
    un = device_kld(lib, pkg, xs[:2], base[:2], np.array([-1, V], np.int32), V)
    assert not un["nll"].any() and not un["nll_base"].any() and not un["p_diff"].any()
    assert np.array_equal(un["kld"], got["kld"][:2]) and np.array_equal(un["same_top"], got["same_top"][:2])


def test_kernel_argument_errors(cuda, lib):
    c, V = lib.c, 160
    d = dev_f32(np.zeros((2, V), np.float32))
    t = torch.zeros(2, dtype=torch.int32, device="cuda")
    r = torch.zeros(2 * K.record_u16s(V) + 2, dtype=torch.int16, device="cuda")
    o = torch.zeros(48, dtype=torch.uint8, device="cuda")
    nl = torch.zeros(2, dtype=torch.float32, device="cuda")
    assert c.pb200_logprob_record_u16s(V) == 164 and c.pb200_logprob_record_u16s(1001) == 1006 and c.pb200_logprob_record_u16s(0) == 0
    rp = ptr(r)
    odd = C.c_void_p(r.data_ptr() + 2)
    for args in ((None, 2, V, ptr(t), rp, None), (ptr(d), 2, V, ptr(t), None, None), (ptr(d), 2, V, None, rp, ptr(nl)),
                 (ptr(d), 0, V, ptr(t), rp, None), (ptr(d), 2, 0, ptr(t), rp, None), (ptr(d), 1 << 31, V, ptr(t), rp, None),
                 (ptr(d), 2, V, ptr(t), odd, None)):
        assert c.pb200_logprobs_u16(*args, None) == EINVAL, args
    for args in ((None, 2, V, rp, ptr(t), ptr(o)), (ptr(d), 2, V, None, ptr(t), ptr(o)), (ptr(d), 2, V, rp, None, ptr(o)),
                 (ptr(d), 2, V, rp, ptr(t), None), (ptr(d), 0, V, rp, ptr(t), ptr(o)), (ptr(d), 2, -1, rp, ptr(t), ptr(o)),
                 (ptr(d), 2, V, odd, ptr(t), ptr(o))):
        assert c.pb200_kld_scores(*args, None) == EINVAL, args


# ---- 3. prompt rows ----
def kernels_on(lib, pkg, lg, toks, base):
    V = lg.shape[1]
    rec, nll = device_records(lib, lg, toks, V)
    kld = device_kld(lib, pkg, lg, base, toks, V) if base is not None else None
    return rec, nll, kld


@pytest.mark.parametrize("arch", ["llama", "qwen2"])
def test_prompt_head_kld_bit_identical_to_kernels(cuda, lib, pkg, arch):
    tm = tiny(arch, n_ctx=96)
    E, V = tm.hp["n_embd"], tm.hp["n_vocab"]
    T = 36
    toks = [(i * 7919 + 13) % V for i in range(T)]
    eng = tm.load_engine(pkg)
    try:
        eng.prefill(toks, 0)
        eng.set_tokpos_seq(0, 11, T)

        def state():
            k, v = kv_tensors(eng, tm, 1, tm.hp["n_layer"])
            return (k.cpu().numpy(), v.cpu().numpy(), _dev(eng.logits_ptr, (V,), "<f4").cpu().numpy(),
                    _dev(eng.token_ptr(0), (4,), "<i4").cpu().numpy(), _dev(eng.hidden_out_ptr, (E,), "<f4").cpu().numpy(),
                    _dev(lib.c.pb200_prefill_hidden_device(eng.h), (T, E), "<f4").cpu().numpy())
        sync()
        before = state()
        rng = np.random.default_rng(3)
        for row0, n in ((0, 36), (3, 8), (30, 5), (35, 1)):
            tg = np.array([(toks + [1])[row0 + i + 1] for i in range(n)], np.int32)
            lg, _ = eng.prompt_head(row0, n)
            fused = pf_tc(tm.tensors["output.weight"][0], E, n)
            other = (lg + rng.standard_normal(lg.shape).astype(f4) * f4(0.2)).astype(f4)
            base, _ = device_records(lib, other, tg, V)
            want_rec, want_nll, want_kld = kernels_on(lib, pkg, lg, tg, base)
            head_launches = 2 if fused else 1 + 2 * n                      # test_gpu_prompt_logits.py's count of the head
            for records, with_base in ((True, False), (False, True), (True, True)):
                b0 = lib.c.pb200_kernel_launches()
                rec, nll, kld = eng.prompt_head_kld(row0, n, tg, records=records, base=base if with_base else None)
                assert lib.c.pb200_aborted() == 0
                assert lib.c.pb200_kernel_launches() - b0 == head_launches + records + with_base, (row0, n, records, with_base)
                if records:
                    assert np.array_equal(rec, want_rec) and np.array_equal(nll.view(np.uint32), want_nll.view(np.uint32)), (row0, n)
                else:
                    assert rec is None and nll is None
                if with_base:
                    assert np.array_equal(kld.view(np.uint8), want_kld.view(np.uint8)), (row0, n)
                else:
                    assert kld is None
        after = state()
        for name, a, b in zip(("K", "V", "logits", "slot words", "hidden out", "hidden rows"), before, after):
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), name
    finally:
        eng.close()


def test_prompt_head_kld_argument_errors(cuda, lib, pkg):
    tm = tiny("llama", n_ctx=64)
    V = tm.hp["n_vocab"]
    nv = K.record_u16s(V)
    c = lib.c
    tg = np.zeros(16, np.int32)
    rec = np.zeros((16, nv), np.uint16)
    nll = np.zeros(16, np.float32)
    base = np.zeros((16, nv), np.uint16)
    kld = np.zeros(16, np.dtype(pkg.KldScore))

    def call(m, row0, n, t=tg, r=rec, nl=None, b=None, k=None):
        p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
        return c.pb200_prompt_head_kld(m, row0, n, p(t), p(r), p(nl), p(b), p(k))
    assert call(None, 0, 1) == ESTATE
    raw = pkg.Model(pkg.HParams(**tm.hp), 0)
    assert call(raw.h, 0, 1) == ESTATE
    raw.close()
    eng = tm.load_engine(pkg)
    noh = tm.load_engine(pkg, layers=(0, 1), with_embd=True, with_head=False)
    try:
        assert call(noh.h, 0, 1) == ESTATE
        assert call(eng.h, 0, 1) == EINVAL                                        # no prefill yet
        eng.prefill(list(range(12)), 0)
        assert call(eng.h, 0, 12) == 0 and call(eng.h, 0, 12, nl=nll, b=base, k=kld) == 0 and call(eng.h, 11, 1, r=None, b=base, k=kld) == 0
        assert call(eng.h, -1, 2) == EINVAL and call(eng.h, 0, 0) == EINVAL and call(eng.h, 5, 8) == EINVAL and call(eng.h, 0, 13) == EINVAL
        assert call(eng.h, 0, 4, r=None) == EINVAL                                # no output
        assert call(eng.h, 0, 4, r=None, nl=nll, b=base, k=kld) == EINVAL         # nll without records
        assert call(eng.h, 0, 4, b=base) == EINVAL and call(eng.h, 0, 4, k=kld) == EINVAL
        assert call(eng.h, 0, 4, t=None) == EINVAL
        for v in (-1, V):
            bad = tg.copy(); bad[2] = v
            assert call(eng.h, 0, 4, t=bad) == EINVAL
    finally:
        eng.close(); noh.close()


# ---- 4. pipeline shards ----
def test_pipeline_shards_records_and_kld(cuda, lib, pkg):
    tm = TinyModel(n_layer=4, n_embd=512, n_head=4, n_head_kv=2, n_ff=1024, n_vocab=256, n_ctx=96, arch="llama", ftype="q4_K_M",
                   freq_factors=False, seed=8, branch_scale=0.1)
    toks = [(i * 31 + 7) % 256 for i in range(72)]
    tg = np.array(toks[1:] + [0], np.int32)
    one = tm.load_engine(pkg)
    one.prefill(toks, 0)
    lg, _ = one.prompt_head(0, 72)
    other = (lg + np.random.default_rng(4).standard_normal(lg.shape).astype(f4) * f4(0.2)).astype(f4)
    base, _ = device_records(lib, other, tg, 256)
    want_rec, want_nll, want_kld = one.prompt_head_kld(0, 72, tg, records=True, base=base)
    one.close()
    a = tm.load_engine(pkg, layers=(0, 2), with_embd=True, with_head=False)
    b = tm.load_engine(pkg, layers=(2, 4), with_embd=False, with_head=True)
    recs, nlls, klds, lgs = [], [], [], []
    for p0, n in ((0, 40), (40, 32)):
        h = a.prefill_stage(toks[p0:p0 + n], None, n, p0, synchronize=True)
        b.prefill_stage(None, h, n, p0)
        r, v, k = b.prompt_head_kld(0, n, tg[p0:p0 + n], records=True, base=base[p0:p0 + n])
        lgs.append(b.prompt_head(0, n)[0])
        recs.append(r); nlls.append(v); klds.append(k)
    a.close(); b.close()
    got_lg = np.concatenate(lgs)
    assert nmse(got_lg, lg) < 1e-6
    # the shard's rows are the two kernels on its own logits, and close to the whole model's
    rec, nll, kld = np.concatenate(recs), np.concatenate(nlls), np.concatenate(klds)
    r2, n2, k2 = kernels_on(lib, pkg, got_lg, tg, base)
    assert np.array_equal(rec, r2) and np.array_equal(nll, n2) and np.array_equal(kld.view(np.uint8), k2.view(np.uint8))
    dec = lambda r: (K.header(r)[0][:, None] * r[:, 4:4 + 256].astype(f4) + K.header(r)[1][:, None])
    assert float(np.max(np.abs(dec(rec) - dec(want_rec)))) < 1e-2
    assert np.allclose(nll, want_nll, rtol=1e-3, atol=1e-3) and np.allclose(kld["kld"], want_kld["kld"], rtol=1e-2, atol=1e-4)


# ---- 5. end to end ----
def e2e_model():
    return TinyModel(n_layer=2, n_embd=512, n_head=4, n_head_kv=2, n_ff=1024, n_vocab=320, n_ctx=128, arch="llama", ftype="q4_K_M",
                     freq_factors=True, seed=41, branch_scale=0.1)


def test_engine_against_its_own_base_file(cuda, pkg, tmp_path):
    """(a) The record step is scale = (max - min_logit) / 65535 <= 16 / 65535 in log-probability, and rounding to the nearest step leaves
    every decoded log-probability above -16 within half a step, e_i, of the engine's own.  KLD = sum p_base_i (log p_base_i - log p_i) =
    sum p_base_i e_i is then within half a step of 0 (sum p_base = 1 + O(e)), terms below -16 left out weigh under e^-16 each, and the
    float roundings of the decoded values add about 2^-19 * 16: |mean KLD| <= 8 / 65535 + 1e-5.  ln(PPL(Q)/PPL(base)) is the mean of
    nll_base - nll = e_target: the same bound.  Every row's top keeps its entry 65535, the only one, unless another logit lies within half
    a step of the maximum."""
    tm = e2e_model()
    V, n_ctx, bos = 320, 64, 1
    toks = ((np.arange(3 * n_ctx) * 7919 + 13) % V).astype(np.int32)
    eng = tm.load_engine(pkg)
    path = tmp_path / "self.kld"
    try:
        run = pkg.perplexity.model_run_chunk(eng)
        res = pkg.perplexity.perplexity(toks, n_ctx, run, 3, bos, out=io.StringIO(), logits_file=path)
        out = io.StringIO()
        kl = pkg.perplexity.kl_divergence(path, run, bos, out=out)
    finally:
        eng.close()
    bound = 8 / 65535 + 1e-5
    print(out.getvalue())
    assert kl.sums.count == 3 * (n_ctx - 1 - n_ctx // 2) >= 93
    assert kl.sums.n_same_top == kl.sums.count
    mean_kld = kl.sums.sum_kld / kl.sums.count
    assert abs(mean_kld) <= bound and abs(kl.chunk_rows[-1][2]) <= bound, (mean_kld, kl.chunk_rows[-1])
    assert abs(res.nll - kl.sums.sum_nll / kl.sums.count) < 1e-6                 # the writer's nll and the comparison's: the same head


def test_engine_against_port_oracle_base_file(cuda, pkg, port, tmp_path):
    """(b) The port oracle decodes every chunk token by token; the reference's writer (libppl_ref.so, else the golden-checked
    restatement) turns its rows into a base file.  kl_divergence() on the engine gives, per position, the reference's KLD function on the
    engine's own head logits of that position and the file's record."""
    tm = e2e_model()
    V, n_ctx, bos, n_chunk = 320, 64, 1, 3
    toks = ((np.arange(n_chunk * n_ctx) * 7919 + 13) % V).astype(np.int32)
    first = n_ctx // 2
    ref = K.RefPpl() if K.REF_LIB.exists() else None
    writer = ref.logprobs_u16 if ref else K.logprobs_u16
    kld_fn = ref.kld_row if ref else K.kld_row
    path = tmp_path / "port.kld"
    with open(path, "wb") as f:
        pkg.perplexity.write_base_header(f, n_ctx, V, toks)
        for i in range(n_chunk):
            ch = toks[i * n_ctx:(i + 1) * n_ctx].copy()
            ch[0] = bos
            lp, _ = tm.port_decode(port, ch)
            for q in range(first, n_ctx - 1):
                f.write(writer(lp[q].astype(f4), int(ch[q + 1]))[0].astype("<u2").tobytes())
    eng = tm.load_engine(pkg)
    seen = []
    head_kld = eng.prompt_head_kld

    def spy(row0, n, targets, records=False, base=None):
        r = head_kld(row0, n, targets, records=records, base=base)
        seen.append((eng.prompt_head(row0, n)[0], np.asarray(targets), np.asarray(base), r[2]))
        return r
    eng.prompt_head_kld = spy
    try:
        kl = pkg.perplexity.kl_divergence(path, pkg.perplexity.model_run_chunk(eng), bos, out=io.StringIO())
    finally:
        eng.close()
    assert kl.sums.count == n_chunk * (n_ctx - 1 - first) and len(seen) == n_chunk
    got = np.concatenate([s[3] for s in seen])
    want = [kld_fn(lg[r], bs[r], int(tg[r])) for lg, tg, bs, _ in seen for r in range(len(tg))]
    check_kld(got, [lg[r] for lg, tg, _, _ in seen for r in range(len(tg))], [bs[r] for _, tg, bs, _ in seen for r in range(len(tg))],
              None, want)
    assert np.array_equal(kl.kld_values, got["kld"].astype(f4))
    print(f"engine vs port oracle: mean KLD {kl.sums.sum_kld / kl.sums.count:.3e}, same top {kl.sums.n_same_top}/{kl.sums.count}")
