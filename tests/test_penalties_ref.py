"""The numpy restatement of logit bias and penalties (tests/penalties_ref.py) against the reference's own samplers, recorded in
tests/golden/penalties_golden.npz (make_penalties_golden.py): every penalised row bit for bit, the greedy and default-chain tokens
drawn from it, and the 1000-step sequences that feed every token back into the history."""
from pathlib import Path

import numpy as np
import pytest

import penalties_ref as P
import sampling_ref as S

GOLDEN = Path(__file__).resolve().parent / "golden" / "penalties_golden.npz"


@pytest.fixture(scope="module")
def z():
    return np.load(GOLDEN)


def golden_case(z, i):
    """(n_vocab, input row, Penalties, accepted history, case name) of single-row case i, rebuilt as the generator built it."""
    n = int(z["n_vocab"][i])
    last_n, pnl, ieos, nl, eos = (int(v) for v in z["cfg"][i])
    rep, freq, pres = (float(v) for v in z["cfg_f"][i])
    b0, b1 = z["bias_off"][i], z["bias_off"][i + 1]
    bias = list(zip(z["bias_tok"][b0:b1].tolist(), z["bias_val"][b0:b1].tolist()))
    p = P.Penalties(last_n, rep, freq, pres, bool(pnl), bool(ieos), nl, eos, bias)
    hist = z["hist"][z["hist_off"][i]:z["hist_off"][i + 1]]
    x = S.make_logits(int(z["logit_seed"][i]), n, 3.0)
    hid = hist[(hist >= 0) & (hist < n)]
    x[hid[:6]] = 0.0
    x[hid[6]] = -0.0
    return n, x, p, hist, str(z["case_names"][z["case"][i]])


def golden_row(z, i, x):
    d0, d1 = z["diff_off"][i], z["diff_off"][i + 1]
    row = x.copy()
    row[z["diff_idx"][d0:d1]] = z["diff_val"][d0:d1]
    return row


def seq_case(z, name):
    k = f"seq_{name}_"
    last_n, pnl, ieos, nl, eos = (int(v) for v in z[k + "cfg"])
    rep, freq, pres = (float(v) for v in z[k + "cfg_f"])
    p = P.Penalties(last_n, rep, freq, pres, bool(pnl), bool(ieos), nl, eos, list(zip(z[k + "bias_tok"].tolist(), z[k + "bias_val"].tolist())))
    return int(z[k + "n_vocab"]), p, z[k + "prompt"], z[k + "token"], int(z[k + "logit_base"]), int(z[k + "dist_seed"])


def test_rows_are_bit_identical_to_the_reference(z):
    names = set()
    for i in range(len(z["case"])):
        n, x, p, hist, name = golden_case(z, i)
        h = P.History(p.last_n)
        h.accept(hist)
        got = P.apply(x, p, h)
        want = golden_row(z, i, x)
        assert (got.view(np.uint32) == want.view(np.uint32)).all(), (i, n, name, np.nonzero(got.view(np.uint32) != want.view(np.uint32))[0][:8])
        names.add(name)
        if name == "neutral" or name == "last_n_-1":
            assert z["diff_off"][i + 1] == z["diff_off"][i], name
    assert names == set(str(s) for s in z["case_names"])


def test_cases_cover_the_corners(z):
    """The recorded cases reach what the semantics single out: counts whose count * freq + present rounds differently under FMA,
    history logits of exactly +0, -0, negative and positive, the newline and EOS in the history, duplicate / out-of-range / -inf bias."""
    fma = signs = 0
    for i in range(len(z["case"])):
        n, x, p, hist, name = golden_case(z, i)
        ln = max(p.last_n, 0)
        ids, c = np.unique(hist[-ln:] if ln else hist[:0], return_counts=True)
        fma += any(P.fma_differs(int(k), p.freq, p.present) for k in c) if p.freq else 0
        v = x[hist[(hist >= 0) & (hist < n)]]
        signs += bool((v == 0).any() and np.signbit(v[v == 0]).any() and (v < 0).any() and (v > 0).any())
        assert p.nl_token in hist.tolist() and p.eos_token in hist.tolist()
    assert fma >= 3 and signs == len(z["case"])
    toks = [t for t, _ in zip(z["bias_tok"], z["bias_val"])]
    assert len(toks) != len(set(toks)) and np.isneginf(z["bias_val"]).any() and (z["bias_tok"] < 0).any()


def test_tokens_follow_from_the_rows(z):
    for i in range(len(z["case"])):
        n, x, p, hist, name = golden_case(z, i)
        row = golden_row(z, i, x)
        assert P.greedy(row) == int(z["token_greedy"][i]), (i, name)
        r = S.chain(row, S.MT19937(int(z["dist_seed"][i])), **S.DEFAULTS)
        assert r["token"] == int(z["token_dist"][i]), (i, name)


def test_last_n_below_zero_is_off():
    x = S.make_logits(3, 100)
    h = P.History(-1)
    h.accept([1, 2, 3])
    assert h.toks == []
    assert (P.apply(x, P.Penalties(last_n=-1, repeat=1.5), h) == x).all()


@pytest.mark.parametrize("name", ["greedy", "dist"])
def test_sequences_reproduce_the_reference(z, name):
    n, p, prompt, want, base, dseed = seq_case(z, name)
    h = P.History(p.last_n)
    h.accept(prompt)
    rng = S.MT19937(dseed)
    toks = []
    for i in range(len(want)):
        row = P.apply(P.seq_logits(base + i, n, list(prompt) + toks), p, h)
        t = P.greedy(row) if name == "greedy" else S.chain(row, rng, **S.DEFAULTS)["token"]
        assert t == int(want[i]), (name, i)
        h.accept(t)
        toks.append(t)
    # without the penalties the same logits would cycle through a handful of tokens
    assert len(set(want.tolist())) > 100
