"""numpy restatement of the reference's sampler chain for temp > 0 without mirostat (gpt_sampler_init, common/sampling.cpp:140-224,
default order), the semantics csrc/sample.cu implements.  Line numbers refer to src/llama-sampling.cpp unless another file is named.

  top-k    :91-165   k <= 0: whole vocabulary, clamped to n_vocab; the result is sorted by logit, descending
  top-p    :557-588  skipped for p >= 1; softmax at temperature 1 (:66-89, float: expf(l - l0), running float sum, divide), then
                     the shortest prefix whose running float sum reaches p with i + 1 >= min_keep
  min-p    :624-684  (sorted branch) skipped for p <= 0; keeps index 0, stops at the first i with logit < l0 + logf(p), i >= min_keep
  temp     :913-918  logit / temp (IEEE division; temp_ext with dynatemp_range 0)
  softmax  :66-89
  dist     :18-46, :415-480  std::mt19937(seed) through libstdc++'s std::discrete_distribution (bits/random.tcc:2657-2678, 3349-3381):
                     probabilities normalised in double by their double sum, double running sums with the last one set to 1.0,
                     u = generate_canonical<double, 53> = (g1 + g2 * 2^32) / 2^64 over two 32-bit outputs (u >= 1 -> nextafter(1, 0)),
                     pick = the first index whose running sum is >= u.  One survivor: nothing is drawn, the generator does not advance.

Equal logits are ordered by ascending token id (the reference's std::sort leaves that order unspecified).  expf is taken as the
float rounding of the double exponential.  std::mt19937(seed) and numpy's legacy RandomState(seed) produce the same 32-bit stream.
"""
from __future__ import annotations

import numpy as np

DEFAULTS = dict(top_k=40, top_p=0.95, min_p=0.05, temp=0.8, min_keep=0)   # common/common.h:103-137


def make_logits(seed: int, n: int, scale: float = 3.0, spike: float = 0.0) -> np.ndarray:
    """Seeded float32 logits without ties (so the descending order is the same under any tie rule); spike is added to the maximum."""
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal(n) * scale).astype(np.float32)
    x[int(np.argmax(x))] += np.float32(spike)
    while True:
        o = np.argsort(x, kind="stable")
        dup = x[o][1:] == x[o][:-1]
        if not dup.any():
            return x
        j = o[1:][dup]
        x[j] = np.nextafter(x[j], np.float32(np.inf))


class MT19937:
    """The 32-bit output stream of std::mt19937(seed)."""

    def __init__(self, seed: int):
        self.rs = np.random.RandomState(seed & 0xFFFFFFFF)

    def next(self) -> int:
        return int(self.rs.randint(0, 2 ** 32, dtype=np.uint64))


def _expf(x: np.ndarray) -> np.ndarray:
    return np.exp(x.astype(np.float64)).astype(np.float32)


def descending_order(logits: np.ndarray) -> np.ndarray:
    n = logits.size
    return np.lexsort((np.arange(n), -logits.astype(np.float64)))


def chain(logits, rng: MT19937, top_k=40, top_p=0.95, min_p=0.05, temp=0.8, min_keep=0, exact_top_p=False) -> dict:
    """One draw.  exact_top_p: cut top-p where the double running sum of the float softmax reaches p, as the device does, instead of
    the reference's float running sum (which drifts when it runs over a whole vocabulary of tiny probabilities).  Returns the token,
    the survivor count, the survivors' final p and double running sums, the position of the pick in the descending order, and
    `margin`: the smallest distance of a decision from its threshold, taken where the decision falls (the running sums on either side
    of the top-p cut vs p, the logits on either side of the min-p stop vs the threshold, the running sums on either side of the pick
    vs u), inf where no such decision was taken; `top_p_n`: the top-p survivor count (k where top-p is off)."""
    lg = np.asarray(logits, dtype=np.float32)
    n = lg.size
    order = descending_order(lg)
    k = n if top_k <= 0 else min(top_k, n)
    ids = order[:k]
    l = lg[ids]
    size = k
    margin = np.inf
    if top_p < 1.0:
        e = _expf(l - l[0])
        p = e / np.cumsum(e, dtype=np.float32)[-1]
        cum = np.cumsum(p, dtype=np.float32)
        if exact_top_p:
            cum = np.cumsum(e.astype(np.float64)) / np.sum(e.astype(np.float64))
        tp = float(np.float32(top_p))
        reach = np.nonzero(cum >= np.float32(top_p))[0]
        hit = np.nonzero((cum >= np.float32(top_p)) & (np.arange(1, size + 1) >= min_keep))[0]
        if hit.size:
            size = int(hit[0]) + 1
        if not reach.size:                                   # the running sum never reaches p: decided by the last sum
            margin = min(margin, tp - float(cum[-1]))
        elif int(reach[0]) + 1 >= min_keep:                  # decided by the running sum, not by min_keep
            j = int(reach[0])
            margin = min(margin, float(cum[j]) - tp, tp - float(cum[j - 1]) if j else np.inf)
    top_p_n = size
    if min_p > 0.0 and size:
        min_logit = np.float32(l[0] + np.float32(np.log(np.float64(np.float32(min_p)))))
        ls = l[:size]
        stop = (ls < min_logit) & (np.arange(size) >= min_keep)
        stop[0] = False
        hit = np.nonzero(stop)[0]
        start = max(1, min_keep)                             # the first index the threshold can stop at
        end = int(hit[0]) if hit.size else size
        for j in (end - 1, end):                             # the logits on either side of the stop
            if start <= j < ls.size:
                margin = min(margin, abs(float(ls[j]) - float(min_logit)))
        size = end
    lt = l[:size] / np.float32(temp)
    e = _expf(lt - lt[0])
    p = e / np.cumsum(e, dtype=np.float32)[-1]
    if size == 1:
        return dict(token=int(ids[0]), n_surv=1, p=p, cum=np.ones(1), pos=0, margin=margin, order=order, top_p_n=top_p_n)
    pd = p.astype(np.float64)
    q = pd / np.cumsum(pd)[-1]
    cp = np.cumsum(q)
    cp[-1] = 1.0
    g1, g2 = rng.next(), rng.next()
    u = (float(g1) + float(g2) * 4294967296.0) / 18446744073709551616.0
    if u >= 1.0:
        u = float(np.nextafter(1.0, 0.0))
    sel = int(np.searchsorted(cp, u, side="left"))
    margin = min(margin, float(cp[sel]) - u, u - float(cp[sel - 1]) if sel else np.inf)
    return dict(token=int(ids[sel]), n_surv=size, p=p, cum=cp, pos=sel, margin=margin, order=order, top_p_n=top_p_n)
