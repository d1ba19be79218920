"""-m gpu: logit bias and penalties on the device (csrc/sample.cu: k_penalize, k_penalty_accept; pb200_penalty_* and the slot API)
against the reference's samplers, recorded in tests/golden/penalties_golden.npz and restated in tests/penalties_ref.py.

The penalised row is compared bit for bit.  Tokens drawn from it follow test_gpu_sampling's rule: greedy tokens must be equal; a
sampled token must be the restatement's (exact top-p) where every decision of the chain clears MARGIN, else a neighbour of it."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import penalties_ref as P
import sampling_ref as S
from test_gpu_sampling import Dev, _agrees, _engine, _i32, _model, _params
from test_penalties_ref import golden_case, golden_row, seq_case

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden" / "penalties_golden.npz"
REF_LIB = ROOT / "oracle" / "_ref" / "libsampling_ref.so"
EINVAL = -1
DEFAULTS = tuple(S.DEFAULTS.values())


def _struct(pkg, p: P.Penalties):
    return pkg.penalties(p.last_n, p.repeat, p.freq, p.present, p.penalize_nl, p.ignore_eos, p.nl_token, p.eos_token, p.logit_bias)


class Pen:
    """A penalty state in device memory and the output row of its apply."""

    def __init__(self, lib, pkg, n, p: P.Penalties):
        self.lib, self.n = lib, n
        self.pp = _struct(pkg, p)
        self.state = torch.zeros(lib.penalty_state_bytes(n, self.pp), dtype=torch.uint8, device="cuda")
        self.out = torch.full((n,), float("nan"), dtype=torch.float32, device="cuda")
        lib.penalty_init(self.state.data_ptr(), n, self.pp)

    def accept(self, toks_t, n=None, stream=0):
        self.lib.penalty_accept(self.state.data_ptr(), toks_t.data_ptr(), toks_t.numel() if n is None else n, stream)

    def apply(self, logits_t, stream=0):
        self.lib.penalty_apply(logits_t.data_ptr(), self.n, self.state.data_ptr(), self.out.data_ptr(), stream)


def _bits(t):
    return t.cpu().numpy().view(np.uint32)


def test_apply_is_bit_identical_to_every_golden_row(cuda, pkg, lib):
    z = np.load(GOLDEN)
    d = Dev(lib)
    for i in range(len(z["case"])):
        n, x, p, hist, name = golden_case(z, i)
        pen = Pen(lib, pkg, n, p)
        pen.accept(torch.from_numpy(hist.astype(np.int32)).cuda())
        xt = torch.from_numpy(x).cuda()
        pen.apply(xt)
        want = golden_row(z, i, x)
        got = pen.out.cpu().numpy()
        bad = np.nonzero(got.view(np.uint32) != want.view(np.uint32))[0]
        assert bad.size == 0, (i, n, name, bad[:8], got[bad[:8]], want[bad[:8]])
        assert (_bits(xt) == x.view(np.uint32)).all()                 # the input row is not touched
        d.sample(pen.out, _params(pkg, 40, 0.95, 0.05, 0.0, 0))      # greedy on the penalised row
        assert int(d.tok.item()) == int(z["token_greedy"][i]), (i, name)
        d.seed(int(z["dist_seed"][i]))
        d.sample(pen.out, _params(pkg, *DEFAULTS))
        got_t = int(d.tok.item())
        r = S.chain(want, S.MT19937(int(z["dist_seed"][i])), **S.DEFAULTS, exact_top_p=True)
        rf = S.chain(want, S.MT19937(int(z["dist_seed"][i])), **S.DEFAULTS)
        assert rf["token"] == int(z["token_dist"][i])
        assert _agrees(got_t, r)[0] and _agrees(got_t, rf)[0], (i, name, got_t, r["token"], r["margin"])


@pytest.mark.parametrize("name", ["greedy", "dist"])
def test_golden_sequences_with_the_history_on_the_device(cuda, pkg, lib, name):
    z = np.load(GOLDEN)
    n, p, prompt, want, base, dseed = seq_case(z, name)
    pen = Pen(lib, pkg, n, p)
    pen.accept(torch.from_numpy(prompt.astype(np.int32)).cuda())
    d = Dev(lib)
    d.seed(dseed)
    sp = _params(pkg, *DEFAULTS[:3], 0.0 if name == "greedy" else DEFAULTS[3], 0)
    h = P.History(p.last_n)
    h.accept(prompt)
    rng = S.MT19937(dseed)
    toks = []
    for i in range(len(want)):
        x = P.seq_logits(base + i, n, list(prompt) + toks)
        pen.apply(torch.from_numpy(x).cuda())
        d.sample(pen.out, sp)
        pen.accept(d.tok)
        got = int(d.tok.item())
        if name == "greedy":
            assert got == int(want[i]), i
        else:
            r = S.chain(P.apply(x, p, h), rng, **S.DEFAULTS, exact_top_p=True)
            ok, cleared = _agrees(got, r)
            assert ok, (i, got, r["token"], r["margin"])
            if not cleared:
                break                                  # a boundary pick may legitimately differ; the histories part from here
            assert got == int(want[i]), i
        h.accept(got)
        toks.append(got)
    assert len(toks) >= 100, len(toks)


def test_neutral_configuration_changes_nothing(cuda, pkg, lib):
    n = 128256
    x = torch.from_numpy(S.make_logits(41, n)).cuda()
    pen = Pen(lib, pkg, n, P.Penalties(last_n=64, repeat=1.0, nl_token=13, eos_token=2))
    pen.accept(torch.arange(0, 300, dtype=torch.int32, device="cuda"))
    pen.apply(x)
    assert (_bits(pen.out) == _bits(x)).all()
    a, b = Dev(lib, 200), Dev(lib, 200)
    a.seed(5)
    b.seed(5)
    p = _params(pkg, *DEFAULTS)
    for i in range(200):
        pen.apply(x)
        a.sample(pen.out, p, slot=i)
        pen.accept(a.tok[i:i + 1])
        b.sample(x, p, slot=i)
    assert (a.tok.cpu() == b.tok.cpu()).all()
    assert len(set(a.tok.cpu().tolist())) > 1


def test_graph_replay_matches_direct_calls(cuda, pkg, lib):
    n = 152064
    x = torch.from_numpy(S.make_logits(8, n, 1.0)).cuda()
    p = P.Penalties(last_n=16, repeat=1.3, freq=0.4, present=0.4, logit_bias=[(3, 2.0), (3, 0.5), (n + 1, 1.0)])
    sp = _params(pkg, *DEFAULTS)

    def run(replay):
        pen = Pen(lib, pkg, n, p)
        d = Dev(lib)
        d.seed(17)
        out = []
        if replay:
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                with torch.cuda.graph(g, stream=s):
                    cs = torch.cuda.current_stream().cuda_stream
                    pen.apply(x, cs)
                    d.sample(pen.out, sp, stream=cs)
                    pen.accept(d.tok, stream=cs)
            torch.cuda.synchronize()
        for _ in range(60):
            if replay:
                g.replay()
            else:
                pen.apply(x)
                d.sample(pen.out, sp)
                pen.accept(d.tok)
            out.append(int(d.tok.item()))
        return out

    want = run(False)
    assert run(True) == want
    assert len(set(want)) > 8                      # the penalties walk the picks away from repeated tokens


def test_invalid_arguments_are_refused(cuda, pkg, lib):
    n = 1000
    st = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    x = torch.from_numpy(S.make_logits(3, n)).cuda()
    out = torch.zeros(n, dtype=torch.float32, device="cuda")
    nan, inf = float("nan"), float("inf")
    bad = [dict(repeat=nan), dict(repeat=inf), dict(repeat=0.0), dict(repeat=-1.1), dict(freq=nan), dict(freq=-inf), dict(present=nan),
           dict(present=inf), dict(logit_bias=[(1, 0.5), (2, nan)])]
    for kw in bad:
        assert lib.c.pb200_penalty_init(C.c_void_p(st.data_ptr()), n, C.byref(pkg.penalties(**kw)), None) == EINVAL, kw
    p = pkg.penalties(logit_bias=[(1, 0.5)])
    p.n_logit_bias = -1
    assert lib.c.pb200_penalty_init(C.c_void_p(st.data_ptr()), n, C.byref(p), None) == EINVAL
    p = pkg.penalties()
    p.n_logit_bias = 3                              # NULL list
    p.logit_bias = C.cast(None, C.POINTER(pkg.LogitBias))
    assert lib.c.pb200_penalty_init(C.c_void_p(st.data_ptr()), n, C.byref(p), None) == EINVAL
    good = pkg.penalties(repeat=1.1, logit_bias=[(5, -inf)])
    assert lib.c.pb200_penalty_init(None, n, C.byref(good), None) == EINVAL
    assert lib.c.pb200_penalty_init(C.c_void_p(st.data_ptr()), 0, C.byref(good), None) == EINVAL
    assert lib.c.pb200_penalty_init(C.c_void_p(st.data_ptr()), n, None, None) == EINVAL
    lib.penalty_init(st.data_ptr(), n, good)
    assert lib.c.pb200_penalty_apply(C.c_void_p(x.data_ptr()), n, C.c_void_p(st.data_ptr()), C.c_void_p(x.data_ptr()), None) == EINVAL
    assert lib.c.pb200_penalty_apply(C.c_void_p(x.data_ptr()), 0, C.c_void_p(st.data_ptr()), C.c_void_p(out.data_ptr()), None) == EINVAL
    assert lib.c.pb200_penalty_accept(C.c_void_p(st.data_ptr()), None, 2, None) == EINVAL
    assert lib.c.pb200_penalty_accept(C.c_void_p(st.data_ptr()), None, -1, None) == EINVAL
    torch.cuda.synchronize()                         # nothing left behind: the valid state still works
    lib.penalty_apply(x.data_ptr(), n, st.data_ptr(), out.data_ptr())
    o = out.cpu().numpy()
    assert np.isneginf(o[5]) and (np.delete(o, 5) == np.delete(x.cpu().numpy(), 5)).all()


@pytest.mark.skipif(not REF_LIB.exists(), reason="oracle/_ref/libsampling_ref.so not built (make -C oracle -f Makefile.sampling)")
def test_random_parameters_against_the_live_reference(cuda, pkg, lib):
    sys.path.insert(0, str(ROOT / "tests" / "golden"))
    from make_penalties_golden import RefSampler
    ref = C.CDLL(str(REF_LIB))
    g = np.random.default_rng(4242)
    d = Dev(lib)
    N = 150
    same = 0
    for i in range(N):
        n = int(g.choice([50, 1000, 5000, 32000, 128256, 152064]))
        nb = int(g.choice([0, 0, 3, 40, 600]))
        bias = [(int(t), float(v)) for t, v in zip(g.integers(-2, n + 2, nb), (g.standard_normal(nb) * 3).astype(np.float32))]
        if nb and g.random() < 0.3:
            bias[int(g.integers(nb))] = (bias[0][0], float("-inf"))
        p = P.Penalties(int(g.choice([-1, 0, 1, 8, 64, 1024])), float(np.float32(g.choice([1.0, 1.05, 1.1, 1.3, 0.8, 2.0]))),
                        float(np.float32(g.choice([0.0, 0.05, 0.1, 0.33, -0.2]))), float(np.float32(g.choice([0.0, 0.1, 0.7, -0.3]))),
                        bool(g.random() < 0.5), bool(g.random() < 0.5), int(g.choice([-1, 0, 13, n - 1])), int(g.choice([-1, 2, n - 1])), bias)
        hist = g.choice(min(n, int(g.choice([10, 100, n]))), size=int(g.integers(0, 2000))).astype(np.int32)
        x = S.make_logits(700000 + i, n, float(g.choice([1.0, 3.0])))
        x[hist[:3]] = 0.0
        dseed = int(g.integers(0, 2 ** 32))
        pre, grd, dst = RefSampler(ref, n, p), RefSampler(ref, n, p, "greedy"), RefSampler(ref, n, p, dseed)
        for s in (pre, grd, dst):
            s.accept(hist)
        _, row = pre(x)
        tok_g, _ = grd(x)
        tok_d, _ = dst(x)
        for s in (pre, grd, dst):
            s.close()
        pen = Pen(lib, pkg, n, p)
        if hist.size:
            pen.accept(torch.from_numpy(hist).cuda())
        pen.apply(torch.from_numpy(x).cuda())
        got = pen.out.cpu().numpy()
        assert (got.view(np.uint32) == row.view(np.uint32)).all(), (i, n, p, np.nonzero(got.view(np.uint32) != row.view(np.uint32))[0][:8])
        d.sample(pen.out, _params(pkg, 40, 0.95, 0.05, 0.0, 0))
        assert int(d.tok.item()) == tok_g, i
        d.seed(dseed)
        d.sample(pen.out, _params(pkg, *DEFAULTS))
        r = S.chain(row, S.MT19937(dseed), **S.DEFAULTS, exact_top_p=True)
        rf = S.chain(row, S.MT19937(dseed), **S.DEFAULTS)
        assert rf["token"] == tok_d, i
        assert _agrees(int(d.tok.item()), r)[0], (i, int(d.tok.item()), r["token"], r["margin"])
        same += int(d.tok.item()) == tok_d
    assert same >= 0.98 * N


def test_engine_slots_with_penalties(cuda, pkg, lib):
    """Three penalised slots and one without, device-resident (step_seq_dev + sample_seq with feed_back), against pb200_decode on
    one engine per slot with the penalties and the chain restated on the host."""
    tm = _model()
    nv = tm.hp["n_vocab"]
    steps = 24
    starts = [(5, 0), (77, 3), (200, 1), (31, 2)]       # token, position
    prompts = [[9, 9, 40, 5], [11, 77, 77], [3, 200, 150, 150, 200], [31]]
    # the unpenalised argmax after slot 1's first token: the EOS id of the ignore_eos slot
    eng = tm.load_engine(pkg)
    first = np.zeros(nv, np.float32)
    eng.decode(starts[1][0], starts[1][1], first)
    eng.close()
    eos = int(np.argmax(first))
    cfg = [  # (penalties or None, temp, seed)
        (P.Penalties(last_n=64, repeat=1.3, nl_token=9), 0.0, 0),
        (P.Penalties(last_n=16, repeat=1.0, ignore_eos=True, eos_token=eos, nl_token=-1), 0.0, 0),
        (P.Penalties(last_n=64, repeat=1.0, freq=0.4, present=0.6, logit_bias=[(1, 3.0), (1, 0.25), (nv, 5.0)]), DEFAULTS[3], 33),
        (None, DEFAULTS[3], 44),
    ]
    hosts, want, rows = [], [], []
    for (tok, pos), prompt, (p, temp, seed) in zip(starts, prompts, cfg):
        e = tm.load_engine(pkg)
        h = P.History(p.last_n if p else 0)
        h.accept(prompt)
        rng = S.MT19937(seed)
        logits = np.zeros(nv, np.float32)
        hist, rr = [], []
        for _ in range(steps):
            e.decode(tok, pos, logits)
            row = P.apply(logits, p, h) if p else logits.copy()
            r = dict(token=P.greedy(row), margin=np.inf, order=None) if temp <= 0 else S.chain(row, rng, **S.DEFAULTS, exact_top_p=True)
            tok, pos = r["token"], pos + 1
            if p:
                h.accept(tok)
            hist.append(tok); rr.append(r)
        hosts.append((e, h, tok, pos)); want.append(hist); rows.append(rr)
    assert want[1][0] != eos                           # the EOS logit is forced to -inf
    eng = _engine(tm, pkg, len(starts))
    smps = [_i32(eng.sample_ptr(s)) for s in range(len(starts))]
    eng.set_penalties(3, repeat=2.0)                   # set, then removed: the slot must run exactly as if never set
    eng.set_penalties(3, None)
    with pytest.raises(pkg.Pb200Error):
        eng.accept(3, [1, 2])                          # PB200_ESTATE: no penalties on the slot
    for s, ((tok, pos), prompt, (p, temp, seed)) in enumerate(zip(starts, prompts, cfg)):
        eng.set_tokpos_seq(s, tok, pos)
        eng.set_sampling(s, *DEFAULTS[:3], temp, 0, seed)
        if p:
            eng.set_penalties(s, _struct(pkg, p))
            eng.accept(s, prompt)
    got = [[] for _ in starts]
    launches = [[] for _ in starts]
    for _ in range(steps):
        for s in range(len(starts)):
            eng.step_seq_dev(s, True)
            n0 = lib.c.pb200_kernel_launches()
            eng.sample_seq(s, True)
            launches[s].append(lib.c.pb200_kernel_launches() - n0)
        eng.synchronize()
        for s in range(len(starts)):
            got[s].append(int(smps[s].item()))
    assert [set(l) for l in launches] == [{3}, {3}, {3}, {1}]
    for s in range(len(starts)):
        for i in range(steps):
            ok, cleared = _agrees(got[s][i], rows[s][i]) if rows[s][i]["order"] is not None else (got[s][i] == want[s][i], True)
            assert ok, (s, i, got[s], want[s])
            if not cleared:
                break
            assert got[s][i] == want[s][i], (s, i, got[s], want[s])
    # pb200_argmax_seq on the ignore_eos slot stays the plain argmax of the raw logits, which pb200_logits_device keeps
    eng.set_tokpos_seq(1, *starts[1])
    eng.step_seq_dev(1, False)
    eng.argmax_seq(1)
    eng.synchronize()
    assert int(smps[1].item()) == eos == int(np.argmax(eng.debug_read("logits", nv)))
    eng.sample_seq(1)
    eng.synchronize()
    assert int(smps[1].item()) != eos
    # pb200_kv_clear leaves the history: one more greedy step of slot 0 from an empty cache, on both sides
    e, h, tok, pos = hosts[0]
    e.kv_clear()
    eng.kv_clear()
    logits = np.zeros(nv, np.float32)
    e.decode(tok, 0, logits)
    eng.set_tokpos_seq(0, tok, 0)
    eng.step_seq_dev(0, False)
    eng.sample_seq(0)
    eng.synchronize()
    row = P.apply(logits, cfg[0][0], h)
    assert int(smps[0].item()) == P.greedy(row)
    for e, *_ in hosts:
        e.close()
    eng.close()
