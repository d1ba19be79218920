"""llama-perplexity's log-probability writer and KL-divergence functions (examples/perplexity/perplexity.cpp:118-153, 237-296) restated in
numpy, the seeded rows of tests/golden/kld_golden.npz, and a ctypes binding of the reference's own functions (oracle/_ref/libppl_ref.so,
built by `make -C oracle -f Makefile.perplexity` where the reference tree is present).

The restatement rounds every float operation on its own, as the reference's scalar code does: scale and every entry of a record are
exact; the double sums run in numpy's order, and numpy's float32 exp may differ from glibc's expf in the last bit, so min_log_prob, nll
and the KLD terms agree to a few ulp."""
import ctypes as C
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
REF_LIB = ROOT / "oracle" / "_ref" / "libppl_ref.so"
GOLDEN = ROOT / "tests" / "golden" / "kld_golden.npz"
f4, f8 = np.float32, np.float64

# the golden rows: kinds of logit rows per vocabulary (make_rows)
KINDS = ("normal", "ties", "neg_inf", "narrow", "wide", "constant", "spike", "self")


def record_u16s(n_vocab: int) -> int:
    return 2 * ((n_vocab + 1) // 2) + 4


def make_rows(V: int, seed: int, kind: str):
    """One golden case: (x, y, tok) — the logits row x, the base model's row y whose record x is compared against, and the target."""
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal(V) * f4(3.0)).astype(f4)
    tok = int(rng.integers(0, V))
    if kind == "ties":                                # exact ties at the maximum: the first index wins
        x[rng.choice(V, size=min(4, V), replace=False)] = x.max() + f4(1.0)
    elif kind == "neg_inf":                           # -inf entries, the target among them
        idx = rng.choice(V, size=V // 10, replace=False)
        x[idx] = -np.inf
        tok = int(idx[0])
    elif kind == "narrow":                            # max - min under 16: min_logit is the row's min
        x = rng.uniform(-5.0, 5.0, V).astype(f4)
    elif kind == "wide":                              # far over 16
        x = (rng.standard_normal(V) * f4(40.0)).astype(f4)
    elif kind == "constant":                          # scale == 0: every entry 0
        x = np.full(V, f4(1.25), f4)
    elif kind == "spike":
        x[tok] = x.max() + f4(12.0)
    y = x.copy()
    if kind not in ("self", "constant"):              # the base: the same row moved a little, -inf entries kept
        fin = np.isfinite(y)
        y[fin] = (y[fin] + (rng.standard_normal(int(fin.sum())) * f4(0.3)).astype(f4)).astype(f4)
    return x, y, tok


def nearest_int(v):
    """perplexity.cpp:118-123 on a float32 array: round through the float adder (ties to even)."""
    return ((np.asarray(v, f4) + f4(12582912.0)).astype(f4).view(np.int32) & 0x007FFFFF) - 0x00400000


def logprobs_u16(x, tok):
    """log_softmax(n_vocab, logits, uint16_t *, tok): (record [record_u16s(V)] uint16, float nll)."""
    x = np.asarray(x, f4)
    V = x.size
    mx, mn = x.max(), x.min()
    min_logit = max(mn, f4(mx - f4(16)))
    s = float(np.sum(np.exp((x - mx).astype(f4)).astype(f8)))
    lse = f4(np.log(s))
    min_log_prob = f4(f4(min_logit - mx) - lse)
    scale = f4(f4(mx - min_logit) / f4(65535.0))
    rec = np.zeros(record_u16s(V), np.uint16)
    rec[:4] = np.array([scale, min_log_prob], f4).view(np.uint16)
    if scale != 0:
        inv = f4(f4(1.0) / scale)
        with np.errstate(invalid="ignore"):
            q = nearest_int((inv * (x - min_logit).astype(f4)).astype(f4))
        rec[4:4 + V] = np.where(x > min_logit, q, 0).astype(np.uint16)
    return rec, f4(f4(mx + lse) - x[tok])


def header(rec):
    """(scale, min_log_prob) of a record or of records [..., nv]."""
    h = np.ascontiguousarray(np.asarray(rec)[..., :4]).view(f4)
    return h[..., 0], h[..., 1]


def kld_terms(x, rec):
    """The KLD function's terms expf(p_log_base) * (p_log_base - l + max + lse), float32, 0 where p_log_base <= -16; with the row's
    (max, lse)."""
    x = np.asarray(x, f4)
    V = x.size
    scale, mlp = header(rec)
    mx = x.max()
    lse = f4(np.log(float(np.sum(np.exp((x - mx).astype(f4)).astype(f8)))))
    pl = ((scale * rec[4:4 + V].astype(f4)).astype(f4) + mlp).astype(f4)
    with np.errstate(invalid="ignore", over="ignore"):
        t = (np.exp(pl).astype(f4) * ((pl - x).astype(f4) + f4(mx + lse)).astype(f4)).astype(f4)
    return np.where(pl > f4(-16.0), t, f4(0.0))


def kld_bound(x, rec):
    """How far two correct implementations' KLD of one row may lie apart.  Each term is a float product of expf(p_log_base) and a float
    difference; an expf within 2 ulp of glibc's moves a term by about 2^-22 of its magnitude, hence 5e-7 * sum|term| (with the double
    sums' order, far smaller).  And lse = (float) log(sum) may round to the neighbouring float where the sums differ in their last bits
    (expf's ulps again), which moves max + lse, and with it every term's difference, by up to 2 ulp of max + lse: at most
    2 ulp(max + lse) * sum p_base over the terms included."""
    x = np.asarray(x, f4)
    V = x.size
    scale, mlp = header(rec)
    mx = x.max()
    lse = f4(np.log(float(np.sum(np.exp((x - mx).astype(f4)).astype(f8)))))
    pl = ((scale * rec[4:4 + V].astype(f4)).astype(f4) + mlp).astype(f4)
    p_base = float(np.sum(np.where(pl > f4(-16.0), np.exp(pl.astype(f8)), 0.0)))
    return 5e-7 * float(np.sum(np.abs(kld_terms(x, rec).astype(f8)))) + 2 * float(np.spacing(abs(f4(mx + lse)))) * p_base


def kld_row(x, rec, tok):
    """log_softmax(n_vocab, logits, base_log_prob, tok, kld) for one row: (kld double, nll, nll_base, p_diff float, same_top)."""
    x = np.asarray(x, f4)
    V = x.size
    scale, mlp = header(rec)
    mx = x.max()
    lse = f4(np.log(float(np.sum(np.exp((x - mx).astype(f4)).astype(f8)))))
    nll = f4(f4(mx + lse) - x[tok])
    nll_base = -f4(f4(scale * f4(rec[4 + tok])) + mlp)
    pl = ((scale * rec[4:4 + V].astype(f4)).astype(f4) + mlp).astype(f4)
    kld = float(np.sum(kld_terms(x, rec).astype(f8)))
    with np.errstate(over="ignore"):
        p_diff = f4(np.exp(-nll).astype(f4) - np.exp(-nll_base).astype(f4))
    return kld, nll, nll_base, p_diff, int(np.argmax(x)) == int(np.argmax(pl))


class KldResultC(C.Structure):
    """kl_divergence_result (perplexity.cpp:221-235)."""
    _fields_ = [(n, C.c_double) for n in ("sum_nll", "sum_nll2", "sum_nll_base", "sum_nll_base2", "sum_nll_nll_base", "sum_kld", "sum_kld2",
                                          "sum_p_diff", "sum_p_diff2", "sum_p_diff4")] + \
               [("max_p_diff", C.c_float), ("n_same_top", C.c_size_t), ("count", C.c_size_t)]


class RefPpl:
    """The reference's functions from oracle/_ref/libppl_ref.so."""

    def __init__(self, path=REF_LIB):
        self.c = C.CDLL(str(path))
        vp = C.c_void_p
        self.c.ppl_ref_logprobs_u16.argtypes = [C.c_int, vp, vp, C.c_int]
        self.c.ppl_ref_logprobs_u16.restype = C.c_double
        self.c.ppl_ref_kld.argtypes = [C.c_int, vp, vp, C.c_int, vp, vp]
        self.c.ppl_ref_kld.restype = C.c_double
        self.c.ppl_ref_process_logits_kld.argtypes = [C.c_int, vp, vp, C.c_int, vp, vp, vp, vp]
        assert self.c.ppl_ref_result_bytes() == C.sizeof(KldResultC)

    @staticmethod
    def _p(a):
        return a.ctypes.data_as(C.c_void_p)

    def logprobs_u16(self, x, tok):
        x = np.ascontiguousarray(x, f4)
        rec = np.zeros(record_u16s(x.size), np.uint16)
        nll = self.c.ppl_ref_logprobs_u16(x.size, self._p(x), self._p(rec), int(tok))
        return rec, f4(nll)

    def kld_row(self, x, rec, tok):
        x, rec = np.ascontiguousarray(x, f4), np.ascontiguousarray(rec, np.uint16)
        acc, pd = KldResultC(), np.zeros(1, f4)
        kld = self.c.ppl_ref_kld(x.size, self._p(x), self._p(rec), int(tok), C.byref(acc), self._p(pd))
        return kld, f4(acc.sum_nll), f4(acc.sum_nll_base), pd[0], bool(acc.n_same_top)

    def process_kld(self, xs, recs, toks):
        """process_logits of the compare mode over rows xs [n][V] scored against toks (n ids): (sums, kld_values, p_diff_values)."""
        xs, recs = np.ascontiguousarray(xs, f4), np.ascontiguousarray(recs, np.uint16)
        n, V = xs.shape
        tk = np.zeros(n + 1, np.int32)
        tk[1:] = toks                                 # process_logits scores row i against tokens[i + 1]
        acc = KldResultC()
        kv, pv = np.zeros(n, f4), np.zeros(n, f4)
        self.c.ppl_ref_process_logits_kld(V, self._p(xs), self._p(tk), n, self._p(recs), C.byref(acc), self._p(kv), self._p(pv))
        return acc, kv, pv
