"""-m gpu: seeded sampling on the device (csrc/sample.cu, pb200_sample / pb200_sample_seq) against the reference's sampler chain.

The device cuts top-p where the exact running mass reaches p; the reference's float running sum drifts when it runs over a whole
vocabulary, so the device is compared with sampling_ref.chain(exact_top_p=True), and that restatement with the reference's tokens.
Where a decision of the chain lies within MARGIN of its threshold (top-p running sum vs p, a logit vs the min-p threshold, u vs the
running sums; sampling_ref.chain's `margin`), the device's fixed-point sums and expf may land on the other side: there the token must
be one of the neighbours of the reference's pick in the descending order.  Everywhere else it must be the reference's token."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import sampling_ref as S

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden" / "sampling_golden.npz"
REF_LIB = ROOT / "oracle" / "_ref" / "libsampling_ref.so"
MARGIN = 1e-5
DRIFT_MASS = 1e-3       # the most softmax mass the reference's float running sum may leave between its top-p cut and the exact one
DRIFT_SHARE = 0.02      # ... and the share of draws in which that moves the reference's token away from the device's
EINVAL, ESTATE = -1, -4


def _params(pkg, top_k, top_p, min_p, temp, min_keep, seed=0):
    return pkg.Sampling(int(top_k), float(top_p), float(min_p), float(temp), int(min_keep), int(seed) & 0xFFFFFFFF)


class Dev:
    """A generator state and a token slot in device memory."""

    def __init__(self, lib, n_tok=1):
        self.lib = lib
        self.state = torch.zeros(lib.sampler_state_bytes(), dtype=torch.uint8, device="cuda")
        self.tok = torch.full((n_tok,), -1, dtype=torch.int32, device="cuda")

    def seed(self, seed):
        self.lib.sampler_seed(self.state.data_ptr(), int(seed))

    def sample(self, logits_t, p, slot=0, stream=0):
        self.lib.sample(logits_t.data_ptr(), logits_t.numel(), p, self.state.data_ptr(), self.tok.data_ptr() + 4 * slot, stream)


def _agrees(got, r):
    """The token rule: equal where every decision clears MARGIN, else a neighbour of the reference's pick."""
    if r["margin"] > MARGIN:
        return got == r["token"], True
    o = r["order"]
    i = int(np.nonzero(o == r["token"])[0][0])
    return got in set(int(t) for t in o[max(0, i - 1): i + 2]), False


def _agrees_with_reference(got, rf, r, logits, args):
    """The device token against the reference's own (rf: sampling_ref.chain with the float running sum, which reproduces it; r: the
    same with the exact top-p sum the device uses).  Returns (ok, drift): drift marks a draw where the two top-p cuts differ and
    the reference's token is therefore not the device's; that is accepted only for top-k 0 with top-p < 1, with the cuts at most 1 %
    of the survivors and DRIFT_MASS of softmax mass apart."""
    ok, _ = _agrees(got, rf)
    if ok:
        return True, False
    top_k, top_p = args[0], args[1]
    if not (top_k <= 0 and top_p < 1.0 and rf["top_p_n"] != r["top_p_n"]):
        return False, False
    lo, hi = sorted((rf["top_p_n"], r["top_p_n"]))
    lg = np.asarray(logits, np.float64)[r["order"]]
    e = np.exp(lg - lg[0])
    ce = np.cumsum(e) / e.sum()
    return hi - lo <= 0.01 * hi and ce[hi - 1] - ce[lo - 1] <= DRIFT_MASS, True


def test_golden_single_draws(cuda, pkg, lib):
    z = np.load(GOLDEN)
    d = Dev(lib)
    same = golden = drift = 0
    for i in range(len(z["token"])):
        n = int(z["n_vocab"][i])
        logits = S.make_logits(int(z["logit_seed"][i]), n, 3.0, float(z["spike"][i]))
        args = (int(z["top_k"][i]), float(z["top_p"][i]), float(z["min_p"][i]), float(z["temp"][i]), int(z["min_keep"][i]))
        rf = S.chain(logits, S.MT19937(int(z["dist_seed"][i])), *args)
        assert rf["token"] == int(z["token"][i])
        r = S.chain(logits, S.MT19937(int(z["dist_seed"][i])), *args, exact_top_p=True)
        d.seed(int(z["dist_seed"][i]))
        d.sample(torch.from_numpy(logits).cuda(), _params(pkg, *args))
        got = int(d.tok.item())
        ok, _ = _agrees(got, r)
        assert ok, (i, n, args, got, r["token"], r["margin"])
        same += got == r["token"]
        golden += got == int(z["token"][i])
        ok, drifted = _agrees_with_reference(got, rf, r, logits, args)
        assert ok, (i, n, args, got, rf["token"], rf["top_p_n"], r["top_p_n"])
        drift += drifted
    print(f"{same} of {len(z['token'])} draws equal to the exact-top-p restatement, {golden} to the reference's token, {drift} top-p drifts")
    assert same >= 0.99 * len(z["token"]) and drift <= DRIFT_SHARE * len(z["token"])


@pytest.mark.parametrize("j", [0, 1])
def test_golden_sequences_carry_the_generator(cuda, pkg, lib, j):
    z = np.load(GOLDEN)
    n = int(z["seq_n_vocab"][j])
    args = tuple(z["seq_params"][j])
    p = _params(pkg, *args)
    rng, rng_f = S.MT19937(int(z["seq_dist_seed"][j])), S.MT19937(int(z["seq_dist_seed"][j]))
    every = int(z["seq_spike_every"][j])
    steps = len(z["seq_token"][j])
    d = Dev(lib, steps)
    d.seed(int(z["seq_dist_seed"][j]))
    refs, frefs = [], []
    ca = (int(args[0]), float(args[1]), float(args[2]), float(args[3]), int(args[4]))
    for i in range(steps):
        logits = S.make_logits(int(z["seq_logit_base"][j]) + i, n, 3.0, 12.0 if i % every == 0 else 0.0)
        refs.append(S.chain(logits, rng, *ca, exact_top_p=True))
        frefs.append(S.chain(logits, rng_f, *ca))
        d.sample(torch.from_numpy(logits).cuda(), p, slot=i)
    got = d.tok.cpu().numpy()
    assert [r["token"] for r in frefs] == list(z["seq_token"][j])
    for i, (r, rf) in enumerate(zip(refs, frefs)):
        ok, _ = _agrees(int(got[i]), r)
        assert ok, (i, int(got[i]), r["token"], r["margin"])
        ok, _ = _agrees(int(got[i]), rf)             # top-k 40: the two top-p sums cut alike, so the reference's own token holds too
        assert ok, (i, int(got[i]), rf["token"], rf["margin"])
    assert sum(int(got[i]) == r["token"] for i, r in enumerate(refs)) >= 0.99 * steps


def test_chi_square_of_200k_draws(cuda, pkg, lib):
    from scipy.stats import chisquare
    logits = S.make_logits(77, 40, 1.0)
    prob = np.exp(logits.astype(np.float64) - logits.max())
    prob /= prob.sum()
    N = 200_000
    d = Dev(lib, N)
    d.seed(2024)
    lt = torch.from_numpy(logits).cuda()
    p = _params(pkg, 0, 1.0, 0.0, 1.0, 0)
    for i in range(N):
        d.sample(lt, p, slot=i)
    counts = np.bincount(d.tok.cpu().numpy(), minlength=40)
    assert counts.sum() == N
    stat, pval = chisquare(counts, prob * N)
    assert pval > 1e-3, (stat, pval)


def test_graph_replay_matches_direct_calls(cuda, pkg, lib):
    logits = torch.from_numpy(S.make_logits(5, 128256)).cuda()
    p = _params(pkg, 40, 0.95, 0.05, 0.8, 0)
    d = Dev(lib)
    d.seed(99)
    want = []
    for _ in range(100):
        d.sample(logits, p)
        want.append(int(d.tok.item()))
    d.seed(99)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            d.sample(logits, p, stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    got = []
    for _ in range(100):
        g.replay()
        got.append(int(d.tok.item()))
    assert got == want
    assert len(set(want)) > 1


def test_invalid_parameters_are_refused(cuda, pkg, lib):
    logits = torch.from_numpy(S.make_logits(3, 1000)).cuda()
    d = Dev(lib)
    d.seed(1)
    nan, inf = float("nan"), float("inf")
    bad = [(40, nan, 0.05, 0.8, 0), (40, 0.95, nan, 0.8, 0), (40, 0.95, 0.05, nan, 0), (40, 0.95, 0.05, inf, 0), (40, inf, 0.05, 0.8, 0),
           (40, 0.0, 0.05, 0.8, 0), (40, -0.1, 0.05, 0.8, 0), (40, 1.01, 0.05, 0.8, 0), (40, 0.95, -0.01, 0.8, 0), (40, 0.95, 1.0, 0.8, 0),
           (40, 0.95, 0.05, 0.8, -1), (40, 0.95, 0.05, -inf, 0)]
    for args in bad:
        rc = lib.c.pb200_sample(C.c_void_p(logits.data_ptr()), 1000, C.byref(_params(pkg, *args)), C.c_void_p(d.state.data_ptr()),
                                C.c_void_p(d.tok.data_ptr()), None)
        assert rc == EINVAL, args
    assert lib.c.pb200_sample(C.c_void_p(logits.data_ptr()), 0, C.byref(_params(pkg, 40, 0.95, 0.05, 0.8, 0)), C.c_void_p(d.state.data_ptr()),
                              C.c_void_p(d.tok.data_ptr()), None) == EINVAL
    torch.cuda.synchronize()        # no CUDA error left behind: the next call and synchronisation succeed
    d.sample(logits, _params(pkg, 40, 0.95, 0.05, 0.8, 0))
    torch.cuda.synchronize()
    assert 0 <= int(d.tok.item()) < 1000


def test_min_p_alone_and_one_entry_leave_one_survivor(cuda, pkg, lib):
    """Paths whose last cluster operation is a reduction (min-p with top-p off leaving one token; a one-entry vocabulary): the
    token is the top one and the generator does not move (the next real draw is the stream's first)."""
    d = Dev(lib)
    for n in (128256, 1000, 1):
        logits = S.make_logits(11 + n, n, 3.0, 12.0)
        d.seed(7)
        for _ in range(20):
            d.sample(torch.from_numpy(logits).cuda(), _params(pkg, 0, 1.0, 0.05, 0.8, 0))
            assert int(d.tok.item()) == int(np.argmax(logits))
        other = S.make_logits(3, 1000)
        d.sample(torch.from_numpy(other).cuda(), _params(pkg, 40, 0.95, 0.05, 0.8, 0))
        r = S.chain(other, S.MT19937(7), **S.DEFAULTS, exact_top_p=True)
        assert _agrees(int(d.tok.item()), r)[0]


def test_vanishing_weights_keep_the_top_token(cuda, pkg, lib):
    """A temperature so small that l0 / temp overflows, or a row of -inf logits: every softmax weight is 0, the token is the top one
    (the greedy limit) and always a valid index."""
    d = Dev(lib)
    d.seed(3)
    logits = S.make_logits(21, 128256)
    for temp in (1e-38, 1e-45):
        for top_k, top_p in ((0, 1.0), (40, 0.95), (0, 0.9)):
            d.sample(torch.from_numpy(logits).cuda(), _params(pkg, top_k, top_p, 0.0, temp, 0))
            assert int(d.tok.item()) == int(np.argmax(logits)), (temp, top_k, top_p)
    ninf = np.full(1000, -np.inf, np.float32)
    for top_k, top_p, min_p in ((0, 1.0, 0.0), (40, 0.95, 0.05), (0, 0.9, 0.0)):
        d.sample(torch.from_numpy(ninf).cuda(), _params(pkg, top_k, top_p, min_p, 0.8, 0))
        assert int(d.tok.item()) == 0, (top_k, top_p, min_p)   # all equal: the lowest id first


def _model():
    from tiny_model import TinyModel
    return TinyModel(n_layer=2, n_embd=512, n_head=4, n_head_kv=2, n_ff=1024, n_vocab=320, n_ctx=48, seed=9, branch_scale=0.3)


def _engine(tm, pkg, n_seq):
    eng = pkg.Model(pkg.HParams(**tm.hp), 0, None, True, True)
    for name, (t, a) in tm.tensors.items():
        eng.set_tensor(name, t, a)
    eng.set_n_seq(n_seq)
    eng.finalize()
    return eng


def _i32(ptr):
    class V:
        __cuda_array_interface__ = {"shape": (1,), "typestr": "<i4", "data": (ptr, False), "version": 2}
    return torch.as_tensor(V(), device="cuda")


def test_greedy_is_the_argmax_kernel(cuda, pkg, lib):
    tm = _model()
    eng = _engine(tm, pkg, 1)
    smp = _i32(eng.sample_ptr(0))
    d = Dev(lib)
    d.seed(0)
    logits = torch.zeros(tm.hp["n_vocab"], dtype=torch.float32, device="cuda")
    with pytest.raises(pkg.Pb200Error):
        eng.sample_seq(0)                        # no parameters set for the slot: PB200_ESTATE
    eng.set_sampling(0, temp=0.0, seed=1)
    for tok, pos in ((5, 0), (17, 1), (300, 2)):
        eng.decode_seq_async(0, tok, pos)
        eng.argmax_seq(0)
        eng.synchronize()
        want = int(smp.item())
        eng.sample_seq(0)
        eng.synchronize()
        assert int(smp.item()) == want
        logits.copy_(torch.from_numpy(eng.debug_read("logits", tm.hp["n_vocab"])))
        for temp in (0.0, -1.0):
            d.sample(logits, _params(pkg, 40, 0.95, 0.05, temp, 0))
            assert int(d.tok.item()) == want
    eng.close()


def test_engine_slots_sample_like_the_host_chain(cuda, pkg, lib):
    tm = _model()
    starts = [(5, 0, 11), (77, 3, 22), (200, 1, 33)]     # token, position, seed
    steps = 16
    nv = tm.hp["n_vocab"]
    want, rows = [], []
    for tok, pos, seed in starts:                      # host-driven: pb200_decode logits through the restated chain
        eng = tm.load_engine(pkg)
        rng = S.MT19937(seed)
        logits = np.zeros(nv, np.float32)
        hist, rr = [], []
        for _ in range(steps):
            eng.decode(tok, pos, logits)
            r = S.chain(logits.copy(), rng, **S.DEFAULTS, exact_top_p=True)
            tok, pos = r["token"], pos + 1
            hist.append(tok); rr.append(r)
        eng.close()
        want.append(hist); rows.append(rr)
    eng = _engine(tm, pkg, len(starts))
    smps = [_i32(eng.sample_ptr(s)) for s in range(len(starts))]
    for s, (tok, pos, seed) in enumerate(starts):
        eng.set_tokpos_seq(s, tok, pos)
        eng.set_sampling(s, seed=seed)
    got = [[] for _ in starts]
    for _ in range(steps):
        for s in range(len(starts)):
            eng.step_seq_dev(s, True)
            eng.sample_seq(s, True)
        eng.synchronize()
        for s in range(len(starts)):
            got[s].append(int(smps[s].item()))
    eng.close()
    for s in range(len(starts)):
        for i in range(steps):
            ok, cleared = _agrees(got[s][i], rows[s][i])
            assert ok, (s, i, got[s], want[s])
            if not cleared:
                break                                  # a boundary pick may legitimately differ; the histories part from here
            assert got[s][i] == want[s][i]


@pytest.mark.skipif(not REF_LIB.exists(), reason="oracle/_ref/libsampling_ref.so not built (make -C oracle -f Makefile.sampling)")
def test_random_parameters_against_the_live_reference(cuda, pkg, lib):
    sys.path.insert(0, str(ROOT / "tests" / "golden"))
    from make_sampling_golden import RefChain
    ref = C.CDLL(str(REF_LIB))
    g = np.random.default_rng(31337)
    d = Dev(lib)
    same = agree_ref = drift = 0
    N = 500
    for i in range(N):
        n = int(g.choice([50, 1000, 5000, 32000, 128256]))
        top_k = int(g.choice([0, 1, 5, 40, 100, 1000]))
        top_p = float(np.float32(g.choice([1.0, 0.99, 0.95, 0.9, 0.5, 0.1])))
        min_p = float(np.float32(g.choice([0.0, 0.01, 0.05, 0.1, 0.5])))
        temp = float(np.float32(g.choice([0.1, 0.5, 0.8, 1.0, 1.5, 3.0])))
        min_keep = int(g.choice([0, 0, 1, 3, 50]))
        seed = int(g.integers(0, 2 ** 32))
        logits = S.make_logits(500000 + i, n, float(g.choice([1.0, 3.0, 8.0])))
        ch = RefChain(ref, top_k, top_p, min_p, temp, min_keep, seed)
        tok_ref, _, _, _ = ch(logits)
        ch.close()
        rf = S.chain(logits, S.MT19937(seed), top_k, top_p, min_p, temp, min_keep)
        agree_ref += rf["token"] == tok_ref
        r = S.chain(logits, S.MT19937(seed), top_k, top_p, min_p, temp, min_keep, exact_top_p=True)
        d.seed(seed)
        d.sample(torch.from_numpy(logits).cuda(), _params(pkg, top_k, top_p, min_p, temp, min_keep))
        got = int(d.tok.item())
        ok, _ = _agrees(got, r)
        assert ok, (i, n, top_k, top_p, min_p, temp, min_keep, got, r["token"], r["margin"])
        same += got == r["token"]
        ok, drifted = _agrees_with_reference(got, dict(rf, token=tok_ref), r, logits, (top_k, top_p))
        assert ok, (i, n, top_k, top_p, min_p, temp, min_keep, got, tok_ref)
        drift += drifted
    print(f"{same} of {N} draws equal to the exact-top-p restatement; the restatement equals the live reference in {agree_ref}; "
          f"{drift} top-p drifts")
    assert agree_ref >= 0.99 * N and same >= 0.99 * N and drift <= DRIFT_SHARE * N
