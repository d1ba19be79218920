"""llama-perplexity's chunk loop (examples/perplexity/perplexity.cpp:475-687) and its KL-divergence mode (kl_divergence, :1686-1955) as host
logic over a run_chunk callable, and run_chunk for a whole model and for the last rank of a layer pipeline.

The token ids are split into chunks of n_ctx tokens.  Each chunk is evaluated from position 0 (with its first token replaced by BOS when
one is given) and positions [first, n_ctx - 1), first = n_ctx // 2, are scored against the ORIGINAL next token, so every scored position
has at least n_ctx // 2 tokens of context.  run_chunk(tokens, first) gets the chunk's input ids (n_ctx of them) and returns one
TokenScore record per scored position p, scored against tokens[p + 1] (positions >= first >= 1 never read the BOS-replaced token 0), or
None on a pipeline rank that does not hold the head.  The two KL-divergence modes call it with a keyword:
  - run_chunk(tokens, first, records=True) -> (uint16 records [n][record_u16s(n_vocab)], f32 nll [n]): the writer
    (--kl-divergence-base FILE), whose records perplexity(..., logits_file=FILE) stores in the reference's base-file layout;
  - run_chunk(tokens, first, base=records) -> KldScore records [n]: the comparison (--kl-divergence) against one chunk's base records,
    which kl_divergence() reads from such a file, then accumulates and prints as the reference does.
Both run on the device (pb200_prompt_head_kld): only the records and 24 bytes per row cross PCIe, never the logits.

The base file (perplexity.cpp:496-552, little-endian): "_logits_", int32 n_ctx, int32 n_vocab, int32 n_chunk, int32 tokens[n_chunk * n_ctx]
(the original ids, before BOS replacement), then per chunk n_ctx - 1 - n_ctx // 2 records.

Not provided: ppl_stride (perplexity_v2), HellaSwag / Winogrande / multiple choice, several chunks as sequences of one batch, and
tokenization (token ids come from the caller)."""
from __future__ import annotations

import math
import os
import sys
from dataclasses import dataclass, field

import numpy as np


@dataclass
class Result:
    ppl: float                  # exp(mean nll)
    nll: float                  # mean nll over the scored positions
    uncertainty: float | None   # the reference's +/- on ppl (None where its variance estimate is not positive)
    count: int                  # scored positions
    chunk_ppl: list = field(default_factory=list)   # running ppl after each chunk, the numbers of the [i]ppl, lines


MAGIC = b"_logits_"


def record_u16s(n_vocab: int) -> int:
    """uint16 entries of one log-probability record: {f32 scale, f32 min_log_prob}, n_vocab entries, a zero pad when n_vocab is odd."""
    return 2 * ((n_vocab + 1) // 2) + 4


def write_base_header(f, n_ctx: int, n_vocab: int, tokens) -> None:
    """The base file's header as perplexity.cpp:496-552 writes it: magic, int32 n_ctx, n_vocab, n_chunk, int32 tokens[n_chunk * n_ctx]."""
    tokens = np.asarray(tokens, dtype="<i4")
    if tokens.size % n_ctx:
        raise ValueError(f"{tokens.size} tokens are not whole chunks of {n_ctx}")
    f.write(MAGIC)
    f.write(np.array([n_ctx, n_vocab, tokens.size // n_ctx], dtype="<i4").tobytes())
    f.write(tokens.tobytes())


@dataclass
class BaseFile:
    """A base file's header, with where its records start and how many bytes each chunk's records take."""
    path: str
    n_ctx: int
    n_vocab: int
    n_chunk: int
    tokens: np.ndarray          # int32 [n_chunk * n_ctx], the original ids
    offset: int                 # byte offset of chunk 0's records
    chunk_bytes: int

    def records(self, f, i: int) -> np.ndarray:
        """Chunk i's records [n_ctx - 1 - n_ctx // 2][record_u16s(n_vocab)] uint16, read from the open file f."""
        f.seek(self.offset + i * self.chunk_bytes)
        b = f.read(self.chunk_bytes)
        if len(b) != self.chunk_bytes:
            raise ValueError(f"{self.path}: truncated in the log-probabilities of chunk {i}")
        return np.frombuffer(b, dtype="<u2").reshape(self.n_ctx - 1 - self.n_ctx // 2, record_u16s(self.n_vocab))


def read_base_header(path) -> BaseFile:
    """Reads and checks a base file's header.  A bad magic or a file shorter than its header, tokens and every chunk's records says it is
    not such a file: ValueError (the reference logs and returns, or stops at the chunk it cannot read)."""
    size = os.path.getsize(path)
    with open(path, "rb") as f:
        if f.read(8) != MAGIC:
            raise ValueError(f"{path} does not look like a file containing log-probabilities")
        h = f.read(12)
        if len(h) != 12:
            raise ValueError(f"{path}: failed reading n_ctx, n_vocab, n_chunk")
        n_ctx, n_vocab, n_chunk = (int(v) for v in np.frombuffer(h, dtype="<i4"))
        if n_ctx < 3 or n_vocab <= 0 or n_chunk <= 0:
            raise ValueError(f"{path}: n_ctx {n_ctx}, n_vocab {n_vocab}, n_chunk {n_chunk}")
        tb = f.read(4 * n_ctx * n_chunk)
        if len(tb) != 4 * n_ctx * n_chunk:
            raise ValueError(f"{path}: failed reading evaluation tokens")
    chunk_bytes = (n_ctx - 1 - n_ctx // 2) * record_u16s(n_vocab) * 2
    offset = 20 + len(tb)
    if size < offset + n_chunk * chunk_bytes:
        raise ValueError(f"{path}: truncated: {size} bytes, {n_chunk} chunks need {offset + n_chunk * chunk_bytes}")
    return BaseFile(str(path), n_ctx, n_vocab, n_chunk, np.frombuffer(tb, dtype="<i4").astype(np.int32), offset, chunk_bytes)


def perplexity(tokens, n_ctx: int, run_chunk, n_chunks: int = -1, bos: int | None = None, out=None, logits_file=None,
               n_vocab: int | None = None) -> Result | None:
    """The reference's perplexity() over token ids: at least 2 * n_ctx tokens, len // n_ctx chunks (at most n_chunks when n_chunks >= 0).
    nll and nll^2 accumulate in double.  out (default stdout) gets the reference's output: "[i]ppl," after each chunk on one line, then
    "Final estimate: PPL = ... +/- ...".  Returns None when run_chunk returns None (a pipeline rank without the head).
    logits_file: also write llama-perplexity --kl-divergence-base's base file there (n_vocab: the model's, default run_chunk.n_vocab).
    The chunks then run in writer mode, and the [i]ppl lines come from the writer's float nll, as in the reference."""
    out = out or sys.stdout
    if logits_file is not None:
        n_vocab = n_vocab if n_vocab is not None else getattr(run_chunk, "n_vocab", None)
        if n_vocab is None:
            raise ValueError("writing a base file needs n_vocab")
    tokens = np.asarray(tokens, dtype=np.int32)
    if n_ctx < 3:
        raise ValueError(f"n_ctx {n_ctx}: a chunk needs at least 3 tokens to score one")
    if len(tokens) < 2 * n_ctx:
        raise ValueError(f"you need at least {2 * n_ctx} tokens to evaluate perplexity with a context of {n_ctx} (got {len(tokens)})")
    n_chunk_max = len(tokens) // n_ctx
    n_chunk = n_chunk_max if n_chunks < 0 else min(n_chunks, n_chunk_max)
    first = n_ctx // 2
    n_scored = n_ctx - 1 - first
    nll = nll2 = 0.0
    count = 0
    res = Result(0.0, 0.0, None, 0)
    f = None
    try:
        for i in range(n_chunk):
            chunk = tokens[i * n_ctx:(i + 1) * n_ctx].copy()
            if bos is not None:
                chunk[0] = bos
            s = run_chunk(chunk, first) if logits_file is None else run_chunk(chunk, first, records=True)
            if s is None:
                return None
            if logits_file is None:
                v = np.asarray(s["nll"], dtype=np.float64)
            else:
                rec = np.asarray(s[0])
                v = np.asarray(s[1], dtype=np.float32).astype(np.float64)     # the writer's float nll, widened
                if rec.shape != (n_scored, record_u16s(n_vocab)) or rec.dtype != np.uint16:
                    raise ValueError(f"run_chunk returned records {rec.shape} {rec.dtype}, expected {(n_scored, record_u16s(n_vocab))} uint16")
            if v.shape != (n_scored,):
                raise ValueError(f"run_chunk returned {v.shape} scores, expected {n_scored}")
            if logits_file is not None:
                if f is None:
                    f = open(logits_file, "wb")
                    write_base_header(f, n_ctx, n_vocab, tokens[:n_chunk * n_ctx])
                f.write(np.ascontiguousarray(rec, dtype="<u2").tobytes())
            nll += float(v.sum())
            nll2 += float((v * v).sum())
            count += v.size
            res.chunk_ppl.append(math.exp(nll / count))
            out.write(f"[{i + 1}]{res.chunk_ppl[-1]:.4f},")
            out.flush()
    finally:
        if f is not None:
            f.close()
    out.write("\n")
    nll /= count
    nll2 /= count
    res.ppl, res.nll, res.count = math.exp(nll), nll, count
    nll2 -= nll * nll
    if nll2 > 0:
        res.uncertainty = math.sqrt(nll2 / (count - 1)) * res.ppl
        out.write(f"Final estimate: PPL = {res.ppl:.4f} +/- {res.uncertainty:.5f}\n")
    else:
        out.write("Unexpected negative standard deviation of log(prob)\n")
    return res


# ---- KL-divergence: the reference's kl_divergence_result sums and its three statistics blocks ----
SUMS = ("sum_nll", "sum_nll2", "sum_nll_base", "sum_nll_base2", "sum_nll_nll_base", "sum_kld", "sum_kld2", "sum_p_diff", "sum_p_diff2",
        "sum_p_diff4")


@dataclass
class KldSums:
    """kl_divergence_result (perplexity.cpp:221-235).  add() takes rows in order and adds each term as the reference's serial loop does:
    the float fields widened, nll*nll, nll_base*nll_base, nll*nll_base and p_diff*p_diff as float products, kld*kld and p_diff2^2 in
    double."""
    sum_nll: float = 0.0
    sum_nll2: float = 0.0
    sum_nll_base: float = 0.0
    sum_nll_base2: float = 0.0
    sum_nll_nll_base: float = 0.0
    sum_kld: float = 0.0
    sum_kld2: float = 0.0
    sum_p_diff: float = 0.0
    sum_p_diff2: float = 0.0
    sum_p_diff4: float = 0.0
    max_p_diff: float = 0.0
    n_same_top: int = 0
    count: int = 0

    def add(self, kld, nll, nll_base, p_diff, same_top) -> None:
        f4, f8 = np.float32, np.float64
        nll, nll_base, p_diff = (np.asarray(a, dtype=f4) for a in (nll, nll_base, p_diff))
        kld = np.asarray(kld, dtype=f8)
        p_diff2 = (p_diff * p_diff).astype(f8)
        terms = (nll, nll * nll, nll_base, nll_base * nll_base, nll * nll_base, kld, kld * kld, p_diff, p_diff2, p_diff2 * p_diff2)
        for name, t in zip(SUMS, terms):
            # cumsum runs left to right: the serial order of the reference's loop, from the running total on
            setattr(self, name, float(np.cumsum(np.concatenate(([getattr(self, name)], t.astype(f8))))[-1]))
        if p_diff.size:
            self.max_p_diff = float(max(f4(self.max_p_diff), np.max(np.abs(p_diff))))
        self.n_same_top += int(np.count_nonzero(np.asarray(same_top)))
        self.count += int(kld.size)


def _f8(x):
    return np.float64(x)


def mean_and_uncertainty(s, s2, count):
    """The reference's mean_and_uncertainty: (mean, its uncertainty), the latter 0 unless the variance is positive and count > 10."""
    if count < 1:
        return _f8(0.0), _f8(0.0)
    with np.errstate(all="ignore"):
        f = _f8(s) / count
        df = _f8(s2) / count - f * f
        df = np.sqrt(df / (count - 1)) if df > 0 and count > 10 else _f8(0.0)
    return f, df


def covariance(sa, sb, sab, count):
    if count < 10:
        return _f8(0.0)
    with np.errstate(all="ignore"):
        return (_f8(sab) / count - (_f8(sa) / count) * (_f8(sb) / count)) / (count - 1)


def percentile(values, fraction):
    """The reference's percentile over sorted float32 values, in float32 arithmetic."""
    f4 = np.float32
    fraction = f4(fraction)
    if fraction <= 0:
        return values[0]
    if fraction >= 1:
        return values[-1]
    p = f4(fraction * f4(len(values) - 1))
    ip = int(p)
    p = f4(p - f4(ip))
    return f4(f4((f4(1) - p) * values[ip]) + f4(p * values[min(ip + 1, len(values) - 1)]))


def median(values):
    """The reference's median of sorted float32 values: 0.5f * (the two middle values) for an even count."""
    n = len(values)
    return np.float32(np.float32(0.5) * np.float32(values[n // 2] + values[n // 2 - 1])) if n % 2 == 0 else values[n // 2]


KLD_HEADER = "chunk             PPL               ln(PPL(Q)/PPL(base))          KL Divergence              Δp RMS            Same top p\n"
KLD_PERCENTILES = (("99.9%", 0.999), ("99.0%", 0.990), ("99.0%", 0.990), ("Median", None), ("10.0%", 0.100), (" 5.0%", 0.050), (" 1.0%", 0.010))
P_DIFF_PERCENTILES = (("99.9%", 0.999), ("99.0%", 0.990), ("95.0%", 0.950), ("90.0%", 0.900), ("75.0%", 0.750), ("Median", None),
                      ("25.0%", 0.250), ("10.0%", 0.100), (" 5.0%", 0.050), (" 1.0%", 0.010), (" 0.1%", 0.001))


@dataclass
class KldResult:
    """Every number kl_divergence() prints.  The per-chunk rows are (ppl, ±, ln ratio, ±, KLD, ±, Δp RMS %, ±, same top %, ±) after each
    chunk; the statistics (the three final blocks) are None below 100 scored positions, where the reference prints none."""
    sums: KldSums
    kld_values: np.ndarray      # float32 KLD per scored position, in position order
    p_diff_values: np.ndarray   # float32 p - p_base of the target per scored position
    chunk_rows: list = field(default_factory=list)
    ppl: float | None = None
    ppl_unc: float | None = None
    ppl_base: float | None = None
    ppl_base_unc: float | None = None
    cor: float | None = None                 # correlation of ln PPL(Q) and ln PPL(base), in %
    ln_ratio: float | None = None
    ln_ratio_unc: float | None = None
    ratio: float | None = None
    ratio_unc: float | None = None
    diff: float | None = None
    diff_unc: float | None = None
    kld: float | None = None
    kld_unc: float | None = None
    kld_max: float | None = None
    kld_min: float | None = None
    kld_percentiles: dict = field(default_factory=dict)      # label -> value, "Median" included
    p_diff: float | None = None              # mean, in %
    p_diff_unc: float | None = None
    p_diff_max: float | None = None          # in %
    p_diff_min: float | None = None
    p_diff_percentiles: dict = field(default_factory=dict)   # label -> value in %
    rms_p_diff: float | None = None          # in %
    rms_p_diff_unc: float | None = None
    same_top: float | None = None            # in %
    same_top_unc: float | None = None


def _chunk_row(k: KldSums):
    log_ppl = mean_and_uncertainty(k.sum_nll, k.sum_nll2, k.count)
    with np.errstate(all="ignore"):
        ppl = np.exp(log_ppl[0])
        ppl_unc = ppl * log_ppl[1]
        log_ppl_base = mean_and_uncertainty(k.sum_nll_base, k.sum_nll_base2, k.count)
        cov = covariance(k.sum_nll, k.sum_nll_base, k.sum_nll_nll_base, k.count)
        ratio = log_ppl[0] - log_ppl_base[0]
        ratio_unc = np.sqrt(log_ppl[1] * log_ppl[1] + log_ppl_base[1] * log_ppl_base[1] - 2.0 * cov)
        kl = mean_and_uncertainty(k.sum_kld, k.sum_kld2, k.count)
        mse = mean_and_uncertainty(k.sum_p_diff2, k.sum_p_diff4, k.count)
        rms = np.sqrt(mse[0])
        rms_unc = 0.5 / rms * mse[1]
        top = 1.0 * _f8(k.n_same_top) / k.count
        top_unc = np.sqrt(top * (1 - top) / _f8(k.count - 1))
    return tuple(float(v) for v in (ppl, ppl_unc, ratio, ratio_unc, kl[0], kl[1], 100.0 * rms, 100.0 * rms_unc, 100.0 * top, 100.0 * top_unc))


def kl_divergence(path, run_chunk, bos: int | None = None, out=None, n_vocab: int | None = None, n_ctx: int | None = None) -> KldResult | None:
    """llama-perplexity --kl-divergence against the base file at path (perplexity.cpp:1686-1955).  Its n_ctx and chunk count are the
    file's; each chunk's original ids go to run_chunk(tokens, first, base=records), with the first replaced by bos when given, and its
    KldScore rows accumulate in the reference's kl_divergence_result.  out (default stdout) gets the reference's lines: after each chunk a
    blank line, the table header and the chunk's row; then the perplexity, KL-divergence and token-probability statistics, unless fewer
    than 100 positions were scored.  n_vocab / n_ctx: the model's (default run_chunk.n_vocab / .n_ctx); a file whose vocabulary differs,
    or whose n_ctx is larger, raises ValueError, as do a bad magic and a truncated file.  Returns None where run_chunk returns None (a
    pipeline rank without the head, which still runs every chunk)."""
    out = out or sys.stdout
    bf = read_base_header(path)
    n_vocab = n_vocab if n_vocab is not None else getattr(run_chunk, "n_vocab", None)
    n_ctx = n_ctx if n_ctx is not None else getattr(run_chunk, "n_ctx", None)
    if n_vocab is not None and bf.n_vocab != n_vocab:
        raise ValueError(f"{path}: inconsistent vocabulary ({bf.n_vocab} vs {n_vocab})")
    if n_ctx is not None and bf.n_ctx > n_ctx:
        raise ValueError(f"{path} has been computed with {bf.n_ctx}, while the current context is {n_ctx}")
    N, first = bf.n_ctx, bf.n_ctx // 2
    n_scored = N - 1 - first
    k = KldSums()
    kld_values = np.zeros(n_scored * bf.n_chunk, np.float32)
    p_diff_values = np.zeros(n_scored * bf.n_chunk, np.float32)
    res = KldResult(k, kld_values, p_diff_values)
    head = True
    with open(path, "rb") as f:
        for i in range(bf.n_chunk):
            chunk = bf.tokens[i * N:(i + 1) * N].copy()
            if bos is not None:
                chunk[0] = bos
            s = run_chunk(chunk, first, base=bf.records(f, i))
            if s is None:
                head = False
                continue
            s = np.asarray(s)
            if s.shape != (n_scored,):
                raise ValueError(f"run_chunk returned {s.shape} scores, expected {n_scored}")
            k.add(s["kld"], s["nll"], s["nll_base"], s["p_diff"], s["same_top"])
            kld_values[i * n_scored:(i + 1) * n_scored] = s["kld"].astype(np.float32)
            p_diff_values[i * n_scored:(i + 1) * n_scored] = s["p_diff"]
            row = _chunk_row(k)
            res.chunk_rows.append(row)
            out.write("\n")
            out.write(KLD_HEADER)
            out.write(f"{i + 1:4d}")
            out.write("    %9.4f ± %9.4f" % row[0:2])
            out.write("    %10.5f ± %10.5f" % row[2:4])
            out.write("    %10.5f ± %10.5f" % row[4:6])
            out.write("    %6.3f ± %6.3f %%" % row[6:8])
            out.write("    %6.3f ± %6.3f %%" % row[8:10])
            out.write("\n")
            out.flush()
    if not head:
        return None
    out.write("\n")
    if k.count < 100:                       # the reference does no statistics on so few values
        return res
    _statistics(res, out)
    return res


def _statistics(res: KldResult, out) -> None:
    """The reference's three statistics blocks (perplexity.cpp:1862-1954), printed to out and stored in res."""
    k, f8 = res.sums, np.float64
    kv, pv = np.sort(res.kld_values), np.sort(res.p_diff_values)
    w = out.write
    with np.errstate(all="ignore"):
        log_ppl = mean_and_uncertainty(k.sum_nll, k.sum_nll2, k.count)
        ppl = np.exp(log_ppl[0])
        ppl_unc = ppl * log_ppl[1]
        log_ppl_base = mean_and_uncertainty(k.sum_nll_base, k.sum_nll_base2, k.count)
        ppl_base = np.exp(log_ppl_base[0])
        ppl_base_unc = ppl_base * log_ppl_base[1]
        cov = covariance(k.sum_nll, k.sum_nll_base, k.sum_nll_nll_base, k.count)
        cor = cov / (log_ppl[1] * log_ppl_base[1])
        ratio = log_ppl[0] - log_ppl_base[0]
        ratio_unc = np.sqrt(log_ppl[1] * log_ppl[1] + log_ppl_base[1] * log_ppl_base[1] - 2.0 * cov)
        pr = np.exp(ratio)
        pr_unc = pr * ratio_unc
        ppl_cov = ppl * ppl_base * cov
        diff = ppl - ppl_base
        diff_unc = np.sqrt(ppl_unc * ppl_unc + ppl_base_unc * ppl_base_unc - 2.0 * ppl_cov)
        kl = mean_and_uncertainty(k.sum_kld, k.sum_kld2, k.count)
        pd = mean_and_uncertainty(k.sum_p_diff, k.sum_p_diff2, k.count)
        mse = mean_and_uncertainty(k.sum_p_diff2, k.sum_p_diff4, k.count)
        rms = np.sqrt(mse[0])
        rms_unc = 0.5 / rms * mse[1]
        top = 1.0 * f8(k.n_same_top) / k.count
        top_unc = np.sqrt(top * (1.0 - top) / f8(k.count - 1))
    w("====== Perplexity statistics ======\n")
    w("Mean PPL(Q)                   : %10.6f ± %10.6f\n" % (ppl, ppl_unc))
    w("Mean PPL(base)                : %10.6f ± %10.6f\n" % (ppl_base, ppl_base_unc))
    w("Cor(ln(PPL(Q)), ln(PPL(base))): %6.2f%%\n" % (100.0 * cor))
    w("Mean ln(PPL(Q)/PPL(base))     : %10.6f ± %10.6f\n" % (ratio, ratio_unc))
    w("Mean PPL(Q)/PPL(base)         : %10.6f ± %10.6f\n" % (pr, pr_unc))
    w("Mean PPL(Q)-PPL(base)         : %10.6f ± %10.6f\n" % (diff, diff_unc))
    w("\n")
    w("====== KL divergence statistics ======\n")
    w("Mean    KLD: %10.6f ± %10.6f\n" % (kl[0], kl[1]))
    w("Maximum KLD: %10.6f\n" % kv[-1])
    for label, fr in KLD_PERCENTILES:
        v = median(kv) if fr is None else percentile(kv, fr)
        res.kld_percentiles[label] = float(v)
        w(("Median  KLD" if fr is None else f"{label}   KLD") + ": %10.6f\n" % v)
    w("Minimum KLD: %10.6f\n" % kv[0])
    w("\n")
    w("====== Token probability statistics ======\n")
    w("Mean    Δp: %6.3f ± %5.3f %%\n" % (100.0 * pd[0], 100.0 * pd[1]))
    w("Maximum Δp: %6.3f%%\n" % (100.0 * f8(pv[-1])))
    for label, fr in P_DIFF_PERCENTILES:
        v = 100.0 * f8(median(pv) if fr is None else percentile(pv, fr))
        res.p_diff_percentiles[label] = float(v)
        w(("Median  Δp" if fr is None else f"{label}   Δp") + ": %6.3f%%\n" % v)
    w("Minimum Δp: %6.3f%%\n" % (100.0 * f8(pv[0])))
    w("RMS Δp    : %6.3f ± %5.3f %%\n" % (100.0 * rms, 100.0 * rms_unc))
    w("Same top p: %6.3f ± %5.3f %%\n" % (100.0 * top, 100.0 * top_unc))
    out.flush()
    for name, v in (("ppl", ppl), ("ppl_unc", ppl_unc), ("ppl_base", ppl_base), ("ppl_base_unc", ppl_base_unc), ("cor", 100.0 * cor),
                    ("ln_ratio", ratio), ("ln_ratio_unc", ratio_unc), ("ratio", pr), ("ratio_unc", pr_unc), ("diff", diff),
                    ("diff_unc", diff_unc), ("kld", kl[0]), ("kld_unc", kl[1]), ("kld_max", kv[-1]), ("kld_min", kv[0]),
                    ("p_diff", 100.0 * pd[0]), ("p_diff_unc", 100.0 * pd[1]), ("p_diff_max", 100.0 * f8(pv[-1])),
                    ("p_diff_min", 100.0 * f8(pv[0])), ("rms_p_diff", 100.0 * rms), ("rms_p_diff_unc", 100.0 * rms_unc),
                    ("same_top", 100.0 * top), ("same_top_unc", 100.0 * top_unc)):
        setattr(res, name, float(v))


def _scored_rows(j0: int, n: int, first: int, n_ctx: int):
    """Rows [a - j0, b - j0) of the micro-batch [j0, j0 + n) hold the scored positions [a, b), or None."""
    a, b = max(first, j0), min(j0 + n, n_ctx - 1)
    return (a, b) if a < b else None


def _head(model, tokens, first, a, b, j0, records, base):
    """The rows of scored positions [a, b) (micro-batch rows from a - j0) in the mode run_chunk was called in."""
    tg = tokens[a + 1:b + 1]
    if records or base is not None:
        rec, nll, kld = model.prompt_head_kld(a - j0, b - a, tg, records=records, base=None if base is None else base[a - first:b - first])
        return (rec, nll) if records else kld
    return model.prompt_head(a - j0, b - a, targets=tg, logits=False)[1]


def _join(out, records):
    if records:
        return np.concatenate([r for r, _ in out]), np.concatenate([v for _, v in out])
    return np.concatenate(out)


def model_run_chunk(model, ubatch: int = 512):
    """run_chunk for a whole model (Model): the chunk is prefilled in ubatches of at most 512 tokens at positions 0.., each followed by
    prompt_head (or prompt_head_kld in the KL-divergence modes) on its scored rows.  No kv_clear is needed between chunks: the engine
    keeps cell == position, and every cell a chunk reads has been rewritten by that chunk first."""
    def run_chunk(tokens, first, records=False, base=None):
        n_ctx, out = len(tokens), []
        for j0 in range(0, n_ctx, ubatch):
            n = min(ubatch, n_ctx - j0)
            model.prefill(tokens[j0:j0 + n], j0)
            ab = _scored_rows(j0, n, first, n_ctx)
            if ab:
                out.append(_head(model, tokens, first, ab[0], ab[1], j0, records, base))
        return _join(out, records)
    run_chunk.n_vocab, run_chunk.n_ctx = model.hp.n_vocab, model.hp.n_ctx
    return run_chunk


def pipeline_run_chunk(pipe, model=None):
    """run_chunk for one rank of a PrefillPipeline (call it on every rank with the same chunks).  model: this rank's Model on the last
    rank, whose prompt_head (prompt_head_kld) scores each micro-batch from the pipeline's outputs hook; the other ranks pass None and get
    None back."""
    last = pipe.rank == pipe.world - 1

    def run_chunk(tokens, first, records=False, base=None):
        n_ctx, out = len(tokens), []

        def outputs(j0, n):
            ab = _scored_rows(j0, n, first, n_ctx)
            if ab:
                out.append(_head(model, tokens, first, ab[0], ab[1], j0, records, base))

        pipe.run(tokens, n_ctx, 0, outputs=outputs if last else None)
        return _join(out, records) if last else None
    if model is not None:
        run_chunk.n_vocab, run_chunk.n_ctx = model.hp.n_vocab, model.hp.n_ctx
    return run_chunk
