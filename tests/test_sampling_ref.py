"""The numpy restatement of the sampler chain (tests/sampling_ref.py) against the reference's own chain, recorded in
tests/golden/sampling_golden.npz (make_sampling_golden.py): every single draw and every step of the carried-generator sequences."""
from pathlib import Path

import numpy as np
import pytest

import sampling_ref as S

GOLDEN = Path(__file__).resolve().parent / "golden" / "sampling_golden.npz"


@pytest.fixture(scope="module")
def z():
    return np.load(GOLDEN)


def test_mt19937_stream_matches_std():
    m = S.MT19937(1234)
    assert [m.next() for _ in range(3)] == [822569775, 2137449171, 2671936806]   # std::mt19937(1234)


def test_single_draws_reproduce_the_reference(z):
    assert len(z["token"]) >= 200
    for i in range(len(z["token"])):
        logits = S.make_logits(int(z["logit_seed"][i]), int(z["n_vocab"][i]), 3.0, float(z["spike"][i]))
        r = S.chain(logits, S.MT19937(int(z["dist_seed"][i])), int(z["top_k"][i]), float(z["top_p"][i]), float(z["min_p"][i]),
                    float(z["temp"][i]), int(z["min_keep"][i]))
        assert (r["token"], r["n_surv"]) == (int(z["token"][i]), int(z["n_surv"][i])), i
        h = min(r["n_surv"], z["p_head"].shape[1])
        # expf is the float rounding of the double exponential here; glibc's expf can differ from it in the last place
        np.testing.assert_allclose(r["p"][:h], z["p_head"][i][:h], rtol=3e-7, atol=0)
        if r["n_surv"] > 1:
            np.testing.assert_allclose([r["cum"][r["pos"] - 1] if r["pos"] else 0.0, r["cum"][r["pos"]]], z["cum_sel"][i], rtol=1e-9, atol=0)


@pytest.mark.parametrize("j", [0, 1])
def test_sequences_reproduce_the_reference(z, j):
    n = int(z["seq_n_vocab"][j])
    tk, tp, mp, t, mk = z["seq_params"][j]
    rng = S.MT19937(int(z["seq_dist_seed"][j]))
    every = int(z["seq_spike_every"][j])
    singles = 0
    for i, (want, surv) in enumerate(zip(z["seq_token"][j], z["seq_n_surv"][j])):
        logits = S.make_logits(int(z["seq_logit_base"][j]) + i, n, 3.0, 12.0 if i % every == 0 else 0.0)
        r = S.chain(logits, rng, int(tk), float(tp), float(mp), float(t), int(mk))
        assert (r["token"], r["n_surv"]) == (int(want), int(surv)), i
        singles += r["n_surv"] == 1
    assert singles > 0     # steps that must leave the generator where it was
