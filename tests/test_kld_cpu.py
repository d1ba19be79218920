"""CPU: llama-perplexity's KL-divergence modes as host logic (prima.cpp_b200/perplexity.py) and the numpy restatement the GPU tests use.

1. The pb200_kld_score layout of the ctypes binding.
2. The restatement (tests/kld_ref.py) against the reference's own functions recorded in tests/golden/kld_golden.npz: scale and every entry
   exact, min_log_prob and nll within 2 ulp, the KLD outputs to the bounds test_gpu_kld.py holds the device to.
3. KldSums over the golden per-row values equals the reference's accumulated kl_divergence_result exactly (both add serially).
4. The base file: writer and reader round-trip byte for byte against the layout written out here, odd and even vocabularies.
5. perplexity(logits_file=...) and kl_divergence() with a fake run_chunk against a plain serial restatement of the reference's loops,
   sums, statistics and printed lines: fewer than 100 positions, a constant row (scale == 0), BOS replacement.
6. A bad magic, a truncated file, another vocabulary and a larger n_ctx raise ValueError."""
import ctypes as C
import hashlib
import io
import math
import struct

import numpy as np
import pytest

import kld_ref as K
import pkgload

pkg = pkgload.load()
PPL = pkg.perplexity
f4, f8 = np.float32, np.float64


def ulps(a, b):
    return abs(int(np.asarray(a, f4).view(np.int32)) - int(np.asarray(b, f4).view(np.int32)))


# ---- 1 ----
def test_kld_score_layout():
    T = pkg.KldScore
    assert C.sizeof(T) == 24
    assert [(n, getattr(T, n).offset) for n, _ in T._fields_] == [("kld", 0), ("nll", 8), ("nll_base", 12), ("p_diff", 16), ("same_top", 20)]
    d = np.dtype(T)
    assert d.itemsize == 24 and d["kld"] == np.float64 and d["same_top"] == np.int32
    assert [pkg.record_u16s(v) for v in (1, 2, 160, 1001, 152064)] == [6, 6, 164, 1006, 152068]


# ---- 2 ----
def golden_cases(z, V):
    p = f"V{V}_"
    xs, ys, toks = [], [], []
    for k, s in zip(z[p + "kinds"], z[p + "seeds"]):
        x, y, t = K.make_rows(V, int(s), K.KINDS[int(k)])
        xs.append(x); ys.append(y); toks.append(t)
    assert toks == list(z[p + "targets"])
    return xs, ys, toks


@pytest.mark.parametrize("V", [160, 1001, 32000, 128256])
def test_restatement_matches_golden(V):
    with np.load(K.GOLDEN) as z:
        p = f"V{V}_"
        xs, ys, toks = golden_cases(z, V)
        recs = []
        for r, (x, t) in enumerate(zip(xs + ys, toks + toks)):
            rec, nll = K.logprobs_u16(x, t)
            sc, mlp = K.header(rec)
            assert sc.view(np.uint32) == z[p + "scale"][r].view(np.uint32), (r, sc, z[p + "scale"][r])
            assert ulps(mlp, z[p + "min_log_prob"][r]) <= 2 and ulps(nll, z[p + "nll"][r]) <= 2, (r, mlp, nll)
            if p + "records" in z:
                assert np.array_equal(rec[4:], z[p + "records"][r][4:]), r
            else:
                assert hashlib.sha256(rec[4:].astype("<u2").tobytes()).digest() == z[p + "sha"][r].tobytes(), r
            recs.append(rec)
        n = len(xs)
        for r in range(n):
            base = recs[n + r].copy()
            base[:4] = np.array([z[p + "scale"][n + r], z[p + "min_log_prob"][n + r]], f4).view(np.uint16)   # the reference's header
            kld, nll, nll_base, p_diff, top = K.kld_row(xs[r], base, toks[r])
            assert top == bool(z[p + "same_top"][r]), r
            if math.isinf(z[p + "kld_nll"][r]):
                assert math.isinf(nll) and ulps(p_diff, z[p + "p_diff"][r]) <= 2
            else:
                assert ulps(nll, z[p + "kld_nll"][r]) <= 2, (r, nll, z[p + "kld_nll"][r])
            assert nll_base == z[p + "kld_nll_base"][r]                                  # from the record alone: exact
            assert abs(float(p_diff) - float(z[p + "p_diff"][r])) <= 4 * np.spacing(f4(1.0)) * 0.5, (r, p_diff, z[p + "p_diff"][r])
            assert abs(kld - z[p + "kld"][r]) <= K.kld_bound(xs[r], base), (r, kld, z[p + "kld"][r], K.kld_bound(xs[r], base))


# ---- 3 ----
@pytest.mark.parametrize("V", [160, 1001, 32000, 128256, 152064, 262144])
def test_sums_of_golden_rows_equal_reference_sums(V):
    with np.load(K.GOLDEN) as z:
        p = f"V{V}_"
        k = PPL.KldSums()
        k.add(z[p + "kld"], z[p + "kld_nll"], z[p + "kld_nll_base"], z[p + "p_diff"], z[p + "same_top"])
        got = np.array([getattr(k, n) for n in PPL.SUMS])
        want = z[p + "sums"]
        assert np.array_equal(got, want) or all(a == b or (math.isnan(a) and math.isnan(b)) for a, b in zip(got, want)), (got, want)
        assert f4(k.max_p_diff) == z[p + "max_p_diff"] and k.n_same_top == z[p + "n_same_top"] and k.count == z[p + "count"]
        assert np.array_equal(z[p + "kld"].astype(f4), z[p + "kld_values"]) and np.array_equal(z[p + "p_diff"], z[p + "p_diff_values"])


# ---- fakes: a deterministic "model" over token ids ----
def fake_logits(tokens, p, V, shift=0, const=False):
    if const:
        return np.full(V, f4(0.5), f4)
    rng = np.random.default_rng(int(tokens[p]) * 7919 + 131 * p + shift)
    return (rng.standard_normal(V) * f4(2.5)).astype(f4)


def fake_run_chunk(V, shift=0, const_chunk=None, log=None):
    state = {"chunk": 0}

    def run_chunk(tokens, first, records=False, base=None):
        if log is not None:
            log.append(tokens.copy())
        const = state["chunk"] == const_chunk
        state["chunk"] += 1
        n_ctx = len(tokens)
        rows = [fake_logits(tokens, q, V, shift, const) for q in range(first, n_ctx - 1)]
        tg = tokens[first + 1:n_ctx]
        if records:
            out = [K.logprobs_u16(x, t) for x, t in zip(rows, tg)]
            return np.stack([r for r, _ in out]), np.array([v for _, v in out], f4)
        s = np.zeros(len(rows), np.dtype(pkg.KldScore))
        for i, (x, t) in enumerate(zip(rows, tg)):
            s[i] = K.kld_row(x, base[i], t)
        return s
    run_chunk.n_vocab, run_chunk.n_ctx = V, 4096
    return run_chunk


def write_base_by_hand(path, n_ctx, V, toks, records):
    with open(path, "wb") as f:
        f.write(b"_logits_" + struct.pack("<iii", n_ctx, V, len(toks) // n_ctx) + struct.pack(f"<{len(toks)}i", *toks))
        for r in records:
            f.write(struct.pack(f"<{r.size}H", *r.reshape(-1)))


# ---- 4 and 5 (writer) ----
@pytest.mark.parametrize("V,n_ctx,n_chunks,bos", [(33, 16, 3, None), (40, 17, 2, 1), (1001, 64, 2, 3)])
def test_writer_file_and_lines(tmp_path, V, n_ctx, n_chunks, bos):
    toks = ((np.arange(n_chunks * n_ctx + 5) * 37 + 11) % V).astype(np.int32)
    log, out = [], io.StringIO()
    path = tmp_path / "base.kld"
    res = PPL.perplexity(toks, n_ctx, fake_run_chunk(V, log=log, const_chunk=1), n_chunks, bos, out=out, logits_file=path)
    first = n_ctx // 2
    # serial restatement: the chunk's input (BOS in front), the records of its scored rows, the [i]ppl lines from the float nll
    nll = nll2 = 0.0
    count, recs, lines = 0, [], ""
    for i in range(n_chunks):
        ch = toks[i * n_ctx:(i + 1) * n_ctx].copy()
        if bos is not None:
            ch[0] = bos
        assert np.array_equal(log[i], ch)
        for q in range(first, n_ctx - 1):
            rec, v = K.logprobs_u16(fake_logits(ch, q, V, 0, i == 1), ch[q + 1])
            recs.append(rec)
            nll += float(v); nll2 += float(v) * float(v); count += 1
        lines += f"[{i + 1}]{math.exp(nll / count):.4f},"
    assert out.getvalue().startswith(lines + "\n")
    assert res.count == count and res.nll == pytest.approx(nll / count, rel=1e-13)
    want = tmp_path / "want.kld"
    write_base_by_hand(want, n_ctx, V, toks[:n_chunks * n_ctx], recs)          # the original ids, before BOS replacement
    assert path.read_bytes() == want.read_bytes()
    assert all(not r[4:].any() for r in recs[(n_ctx - 1 - first):2 * (n_ctx - 1 - first)])   # the constant chunk: scale 0, entries 0
    bf = PPL.read_base_header(path)
    assert (bf.n_ctx, bf.n_vocab, bf.n_chunk) == (n_ctx, V, n_chunks) and np.array_equal(bf.tokens, toks[:n_chunks * n_ctx])
    with open(path, "rb") as f:
        assert np.array_equal(bf.records(f, 1), np.stack(recs[n_ctx - 1 - first:2 * (n_ctx - 1 - first)]))


# ---- 5 (compare) ----
def restate_kl_divergence(path, V, shift, bos, const_chunk):
    """A plain serial restatement of the reference's kl_divergence(): reads the file with struct, loops row by row with Python floats
    and float32 products, and formats every line with the reference's printf formats."""
    import numpy as np
    b = open(path, "rb").read()
    n_ctx, nv_, n_chunk = struct.unpack_from("<iii", b, 8)
    toks = np.frombuffer(b, "<i4", n_ctx * n_chunk, 20)
    nv = K.record_u16s(V)
    first = n_ctx // 2
    ns = n_ctx - 1 - first
    off = 20 + 4 * n_ctx * n_chunk
    S = dict(nll=0.0, nll2=0.0, nb=0.0, nb2=0.0, nnb=0.0, kld=0.0, kld2=0.0, pd=0.0, pd2=0.0, pd4=0.0)
    same = count = 0
    kv, pv, lines = [], [], []

    def mu(s, s2, c):
        if c < 1:
            return 0.0, 0.0
        f = s / c
        df = s2 / c - f * f
        return f, (math.sqrt(df / (c - 1)) if df > 0 and c > 10 else 0.0)

    def cov(a, b_, ab, c):
        return 0.0 if c < 10 else (ab / c - (a / c) * (b_ / c)) / (c - 1)
    for i in range(n_chunk):
        ch = toks[i * n_ctx:(i + 1) * n_ctx].copy()
        if bos is not None:
            ch[0] = bos
        for j in range(ns):
            rec = np.frombuffer(b, "<u2", nv, off + 2 * nv * (i * ns + j))
            t = int(toks[i * n_ctx + first + j + 1])
            kld, nll, nb, pdiff, top = K.kld_row(fake_logits(ch, first + j, V, shift, i == const_chunk), rec, t)
            S["nll"] += float(nll); S["nll2"] += float(f4(nll * nll)); S["nb"] += float(nb); S["nb2"] += float(f4(nb * nb))
            S["nnb"] += float(f4(nll * nb)); S["kld"] += kld; S["kld2"] += kld * kld; S["pd"] += float(pdiff)
            p2 = float(f4(pdiff * pdiff)); S["pd2"] += p2; S["pd4"] += p2 * p2
            same += top; count += 1
            kv.append(f4(kld)); pv.append(pdiff)
        lp, lb = mu(S["nll"], S["nll2"], count), mu(S["nb"], S["nb2"], count)
        c = cov(S["nll"], S["nb"], S["nnb"], count)
        kl, mse = mu(S["kld"], S["kld2"], count), mu(S["pd2"], S["pd4"], count)
        rms = math.sqrt(mse[0])
        tp = same / count
        lines += ["", "chunk             PPL               ln(PPL(Q)/PPL(base))          KL Divergence              Δp RMS            Same top p",
                  "%4d" % (i + 1) + "    %9.4f ± %9.4f" % (math.exp(lp[0]), math.exp(lp[0]) * lp[1])
                  + "    %10.5f ± %10.5f" % (lp[0] - lb[0], math.sqrt(lp[1] ** 2 + lb[1] ** 2 - 2 * c))
                  + "    %10.5f ± %10.5f" % kl + "    %6.3f ± %6.3f %%" % (100 * rms, 100 * (0.5 / rms * mse[1]))
                  + "    %6.3f ± %6.3f %%" % (100 * tp, 100 * math.sqrt(tp * (1 - tp) / (count - 1)))]
    lines.append("")
    if count >= 100:
        kv, pv = sorted(kv), sorted(pv)

        def pct(v, fr):
            fr = f4(fr)
            q = f4(fr * f4(len(v) - 1)); ip = int(q); q = f4(q - f4(ip))
            return f4(f4((f4(1) - q) * v[ip]) + f4(q * v[min(ip + 1, len(v) - 1)]))

        def med(v):
            return f4(f4(0.5) * f4(v[len(v) // 2] + v[len(v) // 2 - 1])) if len(v) % 2 == 0 else v[len(v) // 2]
        lp, lb = mu(S["nll"], S["nll2"], count), mu(S["nb"], S["nb2"], count)
        c = cov(S["nll"], S["nb"], S["nnb"], count)
        ppl, pb = math.exp(lp[0]), math.exp(lb[0])
        r, ru = lp[0] - lb[0], math.sqrt(lp[1] ** 2 + lb[1] ** 2 - 2 * c)
        lines += ["====== Perplexity statistics ======",
                  "Mean PPL(Q)                   : %10.6f ± %10.6f" % (ppl, ppl * lp[1]),
                  "Mean PPL(base)                : %10.6f ± %10.6f" % (pb, pb * lb[1]),
                  "Cor(ln(PPL(Q)), ln(PPL(base))): %6.2f%%" % (100 * c / (lp[1] * lb[1])),
                  "Mean ln(PPL(Q)/PPL(base))     : %10.6f ± %10.6f" % (r, ru),
                  "Mean PPL(Q)/PPL(base)         : %10.6f ± %10.6f" % (math.exp(r), math.exp(r) * ru),
                  "Mean PPL(Q)-PPL(base)         : %10.6f ± %10.6f" % (ppl - pb, math.sqrt((ppl * lp[1]) ** 2 + (pb * lb[1]) ** 2 - 2 * ppl * pb * c)),
                  "", "====== KL divergence statistics ======",
                  "Mean    KLD: %10.6f ± %10.6f" % mu(S["kld"], S["kld2"], count), "Maximum KLD: %10.6f" % kv[-1],
                  "99.9%%   KLD: %10.6f" % pct(kv, 0.999), "99.0%%   KLD: %10.6f" % pct(kv, 0.99), "99.0%%   KLD: %10.6f" % pct(kv, 0.99),
                  "Median  KLD: %10.6f" % med(kv), "10.0%%   KLD: %10.6f" % pct(kv, 0.1), " 5.0%%   KLD: %10.6f" % pct(kv, 0.05),
                  " 1.0%%   KLD: %10.6f" % pct(kv, 0.01), "Minimum KLD: %10.6f" % kv[0], "", "====== Token probability statistics ======"]
        pd = mu(S["pd"], S["pd2"], count)
        lines.append("Mean    Δp: %6.3f ± %5.3f %%" % (100 * pd[0], 100 * pd[1]))
        lines.append("Maximum Δp: %6.3f%%" % (100.0 * float(pv[-1])))
        for lab, fr in (("99.9%", .999), ("99.0%", .99), ("95.0%", .95), ("90.0%", .9), ("75.0%", .75), ("Median", None), ("25.0%", .25),
                        ("10.0%", .1), (" 5.0%", .05), (" 1.0%", .01), (" 0.1%", .001)):
            v = 100.0 * float(med(pv) if fr is None else pct(pv, fr))
            lines.append(("Median  Δp" if fr is None else lab + "   Δp") + ": %6.3f%%" % v)
        lines.append("Minimum Δp: %6.3f%%" % (100.0 * float(pv[0])))
        mse = mu(S["pd2"], S["pd4"], count)
        rms = math.sqrt(mse[0])
        tp = same / count
        lines += ["RMS Δp    : %6.3f ± %5.3f %%" % (100 * rms, 100 * 0.5 / rms * mse[1]),
                  "Same top p: %6.3f ± %5.3f %%" % (100 * tp, 100 * math.sqrt(tp * (1 - tp) / (count - 1)))]
    return "\n".join(lines) + "\n", S, kv


@pytest.mark.parametrize("V,n_ctx,n_chunks,bos,const_chunk", [(33, 16, 3, None, None), (40, 17, 2, 1, None), (160, 64, 4, 3, 2),
                                                             (1001, 100, 3, None, 1)])
def test_kl_divergence_matches_serial_restatement(tmp_path, V, n_ctx, n_chunks, bos, const_chunk):
    toks = ((np.arange(n_chunks * n_ctx) * 37 + 11) % V).astype(np.int32)
    path = tmp_path / "base.kld"
    PPL.perplexity(toks, n_ctx, fake_run_chunk(V, shift=0, const_chunk=const_chunk), n_chunks, bos, out=io.StringIO(), logits_file=path)
    log, out = [], io.StringIO()
    res = PPL.kl_divergence(path, fake_run_chunk(V, shift=5, const_chunk=const_chunk, log=log), bos, out=out)
    want, S, _ = restate_kl_divergence(path, V, 5, bos, const_chunk)
    first = n_ctx // 2
    for i, t in enumerate(log):
        ch = toks[i * n_ctx:(i + 1) * n_ctx].copy()
        if bos is not None:
            ch[0] = bos
        assert np.array_equal(t, ch)
    assert res.sums.count == n_chunks * (n_ctx - 1 - first)
    got_lines, want_lines = out.getvalue().split("\n"), want.split("\n")
    assert got_lines == want_lines
    assert (res.ppl is None) == (res.sums.count < 100)
    assert res.sums.sum_kld == pytest.approx(S["kld"], rel=1e-13) and res.sums.sum_nll_nll_base == pytest.approx(S["nnb"], rel=1e-13)


def test_kl_divergence_of_a_model_against_itself(tmp_path):
    """The same fake model on both sides: every top agrees, ln(PPL ratio) and KLD are at the record's quantization level."""
    V, n_ctx = 257, 64
    toks = ((np.arange(4 * n_ctx) * 13 + 5) % V).astype(np.int32)
    path = tmp_path / "self.kld"
    PPL.perplexity(toks, n_ctx, fake_run_chunk(V), 4, None, out=io.StringIO(), logits_file=path)
    res = PPL.kl_divergence(path, fake_run_chunk(V), None, out=io.StringIO())
    assert res.same_top == 100.0 and abs(res.ln_ratio) < 1e-3 and abs(res.kld) < 1e-5


# ---- 6 ----
def test_bad_files_raise(tmp_path):
    V, n_ctx = 33, 16
    toks = ((np.arange(2 * n_ctx) * 37 + 11) % V).astype(np.int32)
    good = tmp_path / "good.kld"
    PPL.perplexity(toks, n_ctx, fake_run_chunk(V), 2, None, out=io.StringIO(), logits_file=good)
    b = good.read_bytes()
    bad = tmp_path / "bad.kld"
    bad.write_bytes(b"_logitz_" + b[8:])
    with pytest.raises(ValueError, match="does not look like"):
        PPL.kl_divergence(bad, fake_run_chunk(V), out=io.StringIO())
    for cut in (10, 20 + 4 * n_ctx, len(b) - 1):
        bad.write_bytes(b[:cut])
        with pytest.raises(ValueError):
            PPL.kl_divergence(bad, fake_run_chunk(V), out=io.StringIO())
    with pytest.raises(ValueError, match="inconsistent vocabulary"):
        PPL.kl_divergence(good, fake_run_chunk(V + 1), out=io.StringIO())
    rc = fake_run_chunk(V)
    rc.n_ctx = n_ctx - 1
    with pytest.raises(ValueError, match="computed with 16"):
        PPL.kl_divergence(good, rc, out=io.StringIO())
    assert PPL.kl_divergence(good, lambda t, f, records=False, base=None: None, out=io.StringIO()) is None   # a rank without the head
