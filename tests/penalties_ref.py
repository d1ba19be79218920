"""numpy restatement of the two samplers the reference puts in front of every chain (gpt_sampler_init, common/sampling.cpp:156-172),
the semantics pb200_penalty_apply / pb200_penalty_accept implement.  Line numbers refer to src/llama-sampling.cpp.

  logit bias  :1568-1645  logit[token] += bias per entry in list order (one rounded f32 add each); ids outside [0, n_vocab) ignored
  penalties   :1373-1566  ignore_eos: logit[eos] = -inf; early exit when last_n == 0 or repeat 1 / freq 0 / present 0; otherwise for
                          every id occurring count > 0 times among the last min(last_n, accepted) accepted tokens
                              logit = logit <= 0 ? logit * repeat : logit / repeat
                              logit -= float(count) * freq + float(count > 0) * present
                          each operation rounded to f32 separately (no FMA); with !penalize_nl the newline keeps its logit.
                          last_n < 0 is clamped to 0 (:1549); eos / nl id -1 (LLAMA_TOKEN_NULL) turn ignore_eos off / penalize_nl on
  accept      :1395-1402  the token joins a ring of capacity last_n; nothing when last_n == 0
"""
from __future__ import annotations

from dataclasses import dataclass, field
from fractions import Fraction

import numpy as np

F32 = np.float32


@dataclass
class Penalties:
    last_n: int = 64                     # common/common.h:118-126
    repeat: float = 1.0
    freq: float = 0.0
    present: float = 0.0
    penalize_nl: bool = False
    ignore_eos: bool = False
    nl_token: int = -1
    eos_token: int = -1
    logit_bias: list = field(default_factory=list)    # (token, bias) pairs

    def __post_init__(self):
        self.last_n = int(self.last_n)     # kept as given: < 0 behaves as 0 (History and apply clamp it, like the reference)
        self.repeat, self.freq, self.present = float(F32(self.repeat)), float(F32(self.freq)), float(F32(self.present))


class History:
    """The penalties sampler's ring of accepted tokens (llama_sampler_penalties::prev)."""

    def __init__(self, last_n: int):
        self.cap = max(int(last_n), 0)
        self.toks: list[int] = []

    def accept(self, tokens) -> None:
        if self.cap == 0:
            return
        self.toks.extend(int(t) for t in np.atleast_1d(tokens))
        del self.toks[:-self.cap]


def apply(logits, p: Penalties, hist: History) -> np.ndarray:
    """The penalised copy of a logits row."""
    x = np.array(logits, dtype=F32, copy=True)
    n = x.size
    for t, b in p.logit_bias:
        if 0 <= t < n:
            x[t] = F32(x[t] + F32(b))
    if p.ignore_eos and 0 <= p.eos_token < n:
        x[p.eos_token] = -np.inf
    last_n = max(p.last_n, 0)
    if last_n == 0 or (p.repeat == 1.0 and p.freq == 0.0 and p.present == 0.0):
        return x
    keep_nl = not p.penalize_nl and 0 <= p.nl_token < n
    nl_logit = x[p.nl_token] if keep_nl else None
    ids, counts = np.unique(np.array(hist.toks[-last_n:], dtype=np.int64), return_counts=True)
    ok = (ids >= 0) & (ids < n)
    ids, counts = ids[ok], counts[ok]
    if ids.size:
        l = x[ids]
        l = np.where(l <= 0, l * F32(p.repeat), l / F32(p.repeat)).astype(F32)
        sub = (counts.astype(F32) * F32(p.freq) + F32(1.0) * F32(p.present)).astype(F32)
        x[ids] = (l - sub).astype(F32)
    if keep_nl:
        x[p.nl_token] = nl_logit
    return x


def fma_differs(count: int, freq: float, present: float) -> bool:
    """Whether count * freq + present rounds differently as one fused operation than as a rounded product and a rounded sum."""
    f, pr = Fraction(float(F32(freq))), Fraction(float(F32(present)))
    fused = F32(float(count * f + pr))
    return bool(fused != F32(F32(count) * F32(freq)) + F32(pr)) if np.isfinite(fused) else False


def diff(row, base):
    """Indices and values where row differs from base bit for bit."""
    a, b = np.asarray(row, F32).view(np.uint32), np.asarray(base, F32).view(np.uint32)
    idx = np.nonzero(a != b)[0].astype(np.int32)
    return idx, np.asarray(row, F32)[idx]


def greedy(row) -> int:
    """First index of the maximum (llama_sampler_greedy_apply, the device's k_argmax)."""
    return int(np.argmax(row))


def seq_logits(seed: int, n: int, recent) -> np.ndarray:
    """Step logits of the recorded sequences: seeded noise, with the last 4 distinct tokens of the sequence so far raised by 4 so that,
    without penalties, the sequence would cycle through them.  The penalty decides the token."""
    x = (np.random.default_rng(seed).standard_normal(n)).astype(F32)
    seen = []
    for t in reversed(list(recent)):
        if t not in seen:
            seen.append(t)
        if len(seen) == 4:
            break
    for t in seen:
        if 0 <= t < n:
            x[t] = F32(x[t] + F32(4.0))
    return x
