"""-m gpu: prompts into any sequence slot (pb200_prefill_seq, pb200_prefill_stage_seq) and the KV copy between slots (pb200_kv_seq_cp).

- A prompt into slot 1 or 2 writes the K / V rows and gives the logits that the slot-0 form gives, bit for bit, on the tensor-core path
  (12 tokens) and the GEMV loop (5), over several ubatches (600 tokens) and for a continued prompt (pos0 > 0); 40 device-resident decode
  steps afterwards give the same tokens and logits.  Slot 0 itself is held to the reference by test_gpu_engine.py.
- Isolation: a prompt into slot 2 between the steps of slots 0 and 1 changes nothing of theirs, and nothing of slot 2 outside its cells.
- Launches: prefill_seq launches what prefill launches; kv_seq_cp launches no kernel.
- kv_seq_cp: the copied cells bit for bit on every layer and nothing else, the reference's bound conventions, shards without head,
  embedding or layers, every error code, and a shared system prompt copied to every slot against prefilling it into each.
- Pipeline shards in one process (2 and 3 shards, hidden states handed over in device memory): prefill_stage_seq into slot 2 and the
  decode after it against the whole model's prefill_seq(2), and kv_seq_cp on every shard.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import legacy_types as L
from tiny_model import TinyModel

pytestmark = pytest.mark.gpu

EINVAL, ENOTSUP, ESTATE = -1, -3, -4
N_SEQ = 3
SHAPE = dict(n_layer=2, n_embd=512, n_head=4, n_head_kv=2, n_ff=1024, n_vocab=320, n_ctx=64)
MODELS = ["q4_K_M", "q4_0"]


def tiny(name, **kw):
    """The tiny models of test_gpu_engine_slots.py, with their shape changed by kw."""
    shape = {**SHAPE, **kw}
    return TinyModel(**shape, seed=21, branch_scale=0.3) if name == "q4_K_M" else L.q4_0_model(22, **shape)


def load(tm, pkg, layers=None, with_embd=True, with_head=True):
    eng = pkg.Model(pkg.HParams(**tm.hp), 0, layers, with_embd, with_head)
    for name, (t, a) in tm.tensors.items():
        eng.set_tensor(name, t, a)
    eng.set_n_seq(N_SEQ)
    eng.finalize()
    return eng


def _dev(ptr, shape, typestr):
    class V:
        __cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (ptr, False), "version": 2}
    return torch.as_tensor(V(), device="cuda")


def kv(eng, tm, n_layer=None):
    """The f16 caches as int16 [n_seq][layer][n_ctx][n_head_kv * 128] (pb200_kv_device)."""
    nl = tm.hp["n_layer"] if n_layer is None else n_layer
    shape = (N_SEQ, nl, tm.hp["n_ctx"], tm.hp["n_head_kv"] * 128)
    return _dev(eng.kv_ptr(False), shape, "<i2"), _dev(eng.kv_ptr(True), shape, "<i2")


def words(eng):
    """{token, pos} words [n_seq][4] and sample words [n_seq] of the slots."""
    return _dev(eng.token_ptr(0), (N_SEQ, 4), "<i4"), _dev(eng.sample_ptr(0), (N_SEQ,), "<i4")


def snap(*ts):
    """Clones taken on torch's stream, finished before the engine's stream runs on."""
    out = [t.clone() for t in ts]
    torch.cuda.synchronize()
    return out


def same(a, b):
    return np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


def prompt(n, mul, add, nv):
    return [(mul * i + add) % nv for i in range(n)]


def decode_from_prompt(eng, seq, pos, steps):
    """After a prompt that ends at pos - 1: set the slot's position, pick the first token on the device from the prompt's logits, then
    `steps` device-resident steps (step_seq_dev + argmax_seq with feed-back).  Returns (tokens, logits per step)."""
    nv = eng.hp.n_vocab
    _, smp = words(eng)
    eng.set_tokpos_seq(seq, 0, pos)
    eng.argmax_seq(seq, True)
    eng.synchronize()
    toks, logits = [int(smp[seq])], []
    for _ in range(steps):
        eng.step_seq_dev(seq, True)
        eng.argmax_seq(seq, True)
        logits.append(eng.debug_read("logits", nv))       # synchronises the engine stream
        toks.append(int(smp[seq]))
    return toks, logits


def assert_same_run(a, b):
    assert a[0] == b[0]
    assert all(same(x, y) for x, y in zip(a[1], b[1]))


# ---- 1. the same result in any slot ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n_tokens", [12, 5])
@pytest.mark.parametrize("model", MODELS)
def test_prompt_into_any_slot_is_bit_identical(cuda, pkg, model, n_tokens):
    tm = tiny(model)
    eng = load(tm, pkg)
    c = eng.lib.c
    nv = tm.hp["n_vocab"]
    K, V = kv(eng, tm)
    toks = np.array(prompt(n_tokens, 7, 1, nv), np.int32)
    lg0 = np.zeros(nv, np.float32)
    assert c.pb200_prefill(eng.h, toks.ctypes.data, n_tokens, 0, lg0.ctypes.data) == 0   # the slot-0 form
    run0 = decode_from_prompt(eng, 0, n_tokens, 40)
    for s in (1, 2):
        lg = eng.prefill(toks, 0, seq=s).copy()
        assert same(lg, lg0)
        for X in (K, V):
            assert torch.equal(X[s, :, :n_tokens], X[0, :, :n_tokens])
        assert_same_run(decode_from_prompt(eng, s, n_tokens, 40), run0)
    for X in (K, V):                                       # prompt rows and the 40 decoded rows of every layer
        assert torch.equal(X[1], X[0]) and torch.equal(X[2], X[0])
    eng.close()


@pytest.mark.parametrize("model", MODELS)
def test_long_and_continued_prompt_in_slot_2(cuda, pkg, model):
    """600 tokens (two ubatches: 512 + 88), then 9 more at pos0 = 600 (a continued prompt), into slot 0 and slot 2."""
    tm = tiny(model, n_ctx=640)
    eng = load(tm, pkg)
    nv = tm.hp["n_vocab"]
    K, V = kv(eng, tm)
    first, more = prompt(600, 13, 5, nv), prompt(9, 3, 2, nv)
    got = {}
    for s in (0, 2):
        a = eng.prefill(first, 0, seq=s).copy()
        b = eng.prefill(more, 600, seq=s).copy()
        got[s] = (a, b, decode_from_prompt(eng, s, 609, 10))
    assert same(got[2][0], got[0][0]) and same(got[2][1], got[0][1])
    assert_same_run(got[2][2], got[0][2])
    for X in (K, V):
        assert torch.equal(X[2], X[0])
        assert bool((X[1] == 0).all())                     # slot 1 never written
    eng.close()


# ---- 2. isolation ---------------------------------------------------------------------------------------------------------------

def test_prompt_into_slot_2_between_steps_changes_nothing_else(cuda, pkg):
    tm = tiny("q4_K_M")
    nv = tm.hp["n_vocab"]
    p2, at = prompt(12, 5, 4, nv), 3                       # slot 2's prompt: cells [3, 15)

    def run(with_prompt):
        eng = load(tm, pkg)
        K, V = kv(eng, tm)
        W, S = words(eng)
        for pos in range(30):                              # slot 2 has 30 cells before the prompt comes
            eng.decode_seq_async(2, (3 * pos + 5) % nv, pos)
        starts = {0: prompt(10, 7, 1, nv), 1: prompt(7, 11, 3, nv)}
        for s, p in starts.items():
            eng.prefill(p, 0, seq=s)
            eng.set_tokpos_seq(s, 0, len(p))
            eng.argmax_seq(s, True)
        out = {0: ([], []), 1: ([], [])}
        for step in range(16):
            if with_prompt and step == 6:
                eng.synchronize()
                k0, v0, w0, s0 = snap(K, V, W, S)
                eng.prefill(p2, at, seq=2)                 # synchronises
                for X, X0 in ((K, k0), (V, v0)):
                    assert torch.equal(X[:2], X0[:2])
                    assert torch.equal(X[2, :, :at], X0[2, :, :at]) and torch.equal(X[2, :, at + 12:], X0[2, :, at + 12:])
                    assert bool((X[2, :, at:at + 12] != X0[2, :, at:at + 12]).any(dim=-1).all())
                assert torch.equal(W, w0) and torch.equal(S, s0)   # every slot's words, slot 2's own included
            for s in (0, 1):
                eng.step_seq_dev(s, True)
                eng.argmax_seq(s, True)
                out[s][1].append(eng.debug_read("logits", nv))
                out[s][0].append(int(S[s]))
        eng.close()
        return out

    a, b = run(True), run(False)
    for s in (0, 1):
        assert_same_run(a[s], b[s])


# ---- 3. launches ----------------------------------------------------------------------------------------------------------------

WANT_PREFILL = {"q4_K_M": {12: 36, 5: 160}, "q4_0": {12: 42, 5: 160}}   # test_gpu_engine_slots.py's table


@pytest.mark.parametrize("model", MODELS)
def test_launches(cuda, pkg, model):
    tm = tiny(model)
    eng = load(tm, pkg)
    c = eng.lib.c
    nv = tm.hp["n_vocab"]

    def count(f):
        eng.synchronize()
        n0 = c.pb200_kernel_launches()
        f()
        eng.synchronize()
        return int(c.pb200_kernel_launches() - n0)

    for n in (12, 5):
        toks = np.array(prompt(n, 7, 1, nv), np.int32)
        want = count(lambda: c.pb200_prefill(eng.h, toks.ctypes.data, n, 0, None))
        assert want == WANT_PREFILL[model][n]
        for s in (0, 1, 2):
            assert count(lambda: eng.prefill(toks, 0, seq=s)) == want
            assert count(lambda: eng.prefill_stage(toks, None, n, 0, synchronize=True, seq=s)) == want
    assert count(lambda: eng.kv_copy(0, 2)) == 0
    assert count(lambda: eng.kv_copy(1, 0, 3, 9)) == 0
    eng.close()


# ---- 4. kv_seq_cp ---------------------------------------------------------------------------------------------------------------

def fill_random(K, V, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    for X in (K, V):
        X.copy_(torch.randint(-30000, 30000, X.shape, dtype=torch.int16, device="cuda", generator=g))
    torch.cuda.synchronize()


SHARDS = {   # name -> (layers, with_embd, with_head)
    "whole": (None, True, True),
    "no_head": ((0, 1), True, False),
    "no_embd": ((1, 2), False, True),
}


@pytest.mark.parametrize("shard", list(SHARDS))
def test_kv_copy_cells_and_bounds(cuda, pkg, shard):
    """Every copy against the same copy done on a clone: the copied cells bit for bit on every layer, nothing else changed; the
    negative-bound and clamping conventions; src == dst and empty ranges are no-ops."""
    layers, we, wh = SHARDS[shard]
    tm = tiny("q4_K_M")
    eng = load(tm, pkg, layers, we, wh)
    nl = tm.hp["n_layer"] if layers is None else layers[1] - layers[0]
    n_ctx = tm.hp["n_ctx"]
    K, V = kv(eng, tm, nl)
    W, S = words(eng)
    fill_random(K, V, 5)
    for s in range(N_SEQ):
        eng.set_tokpos_seq(s, 10 + s, 20 + s)
    eng.synchronize()
    wk, wv, w0, s0 = snap(K, V, W, S)
    cases = [
        ((0, 2, 4, 13), (4, 13)),
        ((1, 2, -1, 7), (0, 7)),
        ((0, 1, 30, -1), (30, n_ctx)),
        ((2, 0, 50, 1000), (50, n_ctx)),
        ((1, 0, -5, -5), (0, n_ctx)),
        ((1, 1, -1, -1), None),
        ((0, 1, 5, 5), None),
        ((0, 1, 9, 3), None),
        ((0, 1, n_ctx, -1), None),
        ((0, 2, 70, 80), None),
    ]
    for (src, dst, p0, p1), rng in cases:
        if rng is not None:
            a, b = rng
            assert not torch.equal(wk[dst, :, a:b], wk[src, :, a:b])   # the copy is visible
            wk[dst, :, a:b] = wk[src, :, a:b]
            wv[dst, :, a:b] = wv[src, :, a:b]
            torch.cuda.synchronize()
        eng.kv_copy(src, dst, p0, p1)
        eng.synchronize()
        assert torch.equal(K, wk) and torch.equal(V, wv), (src, dst, p0, p1)
    assert torch.equal(W, w0) and torch.equal(S, s0)
    eng.close()


def test_kv_copy_on_a_shard_without_layers(cuda, pkg):
    tm = tiny("q4_K_M")
    eng = load(tm, pkg, (2, 2), False, True)
    c = eng.lib.c
    assert eng.kv_ptr(False) == 0
    for src, dst, p0, p1 in ((0, 1, -1, -1), (2, 0, 3, 9), (1, 1, 0, 4)):
        assert c.pb200_kv_seq_cp(eng.h, src, dst, p0, p1) == 0
    assert c.pb200_kv_seq_cp(eng.h, 0, N_SEQ, -1, -1) == EINVAL
    eng.close()


def test_error_codes(cuda, pkg):
    """pb200_kv_seq_cp's codes, and those of the two prefill _seq forms: seq outside [0, n_seq) is EINVAL right after the model check,
    every other argument gives the code of the slot-0 form for the same arguments."""
    lib = pkg.Lib.get()
    c = lib.c
    tm = tiny("q4_K_M")
    E, nv, n_ctx = tm.hp["n_embd"], tm.hp["n_vocab"], tm.hp["n_ctx"]
    full = load(tm, pkg)
    shard = load(tm, pkg, (1, 2), False, False)
    hp = pkg.HParams(**tm.hp)
    unf = c.pb200_model_create(C.byref(hp), 0, 0, 2, 1, 1)
    assert unf and c.pb200_model_set_n_seq(unf, N_SEQ) == 0
    toks = np.arange(1, 9, dtype=np.int32)
    bad = toks.copy()
    bad[3] = nv
    host = np.zeros(nv, np.float32)
    hid = torch.zeros(8 * E, device="cuda")
    torch.cuda.synchronize()
    tp, bp, lp, hp_ = toks.ctypes.data, bad.ctypes.data, host.ctypes.data, hid.data_ptr()

    # kv_seq_cp
    assert c.pb200_kv_seq_cp(None, 0, 1, -1, -1) == ESTATE
    assert c.pb200_kv_seq_cp(unf, 0, 1, -1, -1) == ESTATE
    for h in (full.h, shard.h):
        for src, dst in ((-1, 0), (0, -1), (N_SEQ, 0), (0, N_SEQ), (N_SEQ, N_SEQ), (-1, -1)):
            assert c.pb200_kv_seq_cp(h, src, dst, -1, -1) == EINVAL
            assert c.pb200_kv_seq_cp(h, src, dst, 5, 5) == EINVAL        # the slots are checked before the range
        assert c.pb200_kv_seq_cp(h, 0, 1, -1, -1) == 0
    assert c.pb200_synchronize(full.h) == 0 and c.pb200_synchronize(shard.h) == 0

    # prefill_seq: (tokens, n, pos0, logits) variants against pb200_prefill
    pf = [(tp, 8, 0, lp), (tp, 8, 0, None), (None, 8, 0, None), (tp, 0, 0, None), (tp, -2, 0, None), (tp, 8, -1, None),
          (tp, 8, n_ctx - 4, None), (bp, 8, 0, None), (tp, 8, n_ctx - 8, None)]
    for h in (None, unf):
        for s in (0, 1, -1, N_SEQ):
            assert c.pb200_prefill_seq(h, s, tp, 8, 0, None) == ESTATE
            assert c.pb200_prefill_stage_seq(h, s, tp, None, 8, 0, None, 1) == ESTATE
    for h in (full.h, shard.h):
        for s in (-1, N_SEQ):
            for args in pf:
                assert c.pb200_prefill_seq(h, s, *args) == EINVAL
        for args in pf:
            want = c.pb200_prefill(h, *args)
            for s in (1, 2):
                assert c.pb200_prefill_seq(h, s, *args) == want, (args, s)
    assert c.pb200_prefill_seq(shard.h, 1, tp, 8, 0, None) == ENOTSUP       # whole prompts start at the embedding

    # prefill_stage_seq: (tokens, hidden, n, pos0, logits, synchronize) variants against pb200_prefill_stage
    st = [(tp, hp_, 8, 0, None, 1), (tp, None, 8, 0, lp, 1), (None, hp_, 8, 0, None, 1), (tp, None, 8, 0, None, 0), (tp, hp_, 0, 0, None, 1),
          (tp, hp_, 513, 0, None, 1), (tp, hp_, 8, -1, None, 1), (tp, hp_, 8, n_ctx - 4, None, 1), (tp, hp_, 8, 0, lp, 0),
          (bp, hp_, 8, 0, None, 1), (None, None, 8, 0, None, 1)]
    for h in (full.h, shard.h):
        for s in (-1, N_SEQ):
            for args in st:
                assert c.pb200_prefill_stage_seq(h, s, *args) == EINVAL
        for args in st:
            want = c.pb200_prefill_stage(h, *args)
            assert c.pb200_synchronize(h) == 0
            for s in (1, 2):
                assert c.pb200_prefill_stage_seq(h, s, *args) == want, (args, s)
                assert c.pb200_synchronize(h) == 0
    c.pb200_model_free(unf)
    full.close()
    shard.close()


@pytest.mark.parametrize("model", MODELS)
def test_system_prompt_copied_to_every_slot(cuda, pkg, model):
    """The server's pattern: a prefix prefilled into slot 0 and copied to slots 1 and 2, then a different suffix prefilled into each slot,
    against prefilling the same prefix and then the same suffix straight into that slot (the same two calls, so the same ubatches)."""
    tm = tiny(model, n_ctx=96)
    nv = tm.hp["n_vocab"]
    pre = prompt(20, 7, 3, nv)
    suf = [prompt(12, 5, 1, nv), prompt(9, 11, 2, nv), prompt(5, 3, 7, nv)]

    a = load(tm, pkg)
    a.prefill(pre, 0, seq=0)
    a.kv_copy(0, 1, 0, len(pre))
    a.kv_copy(0, 2)                                        # the whole slot: what lies past the prefix is rewritten before it is read
    got = {}
    for s in range(N_SEQ):
        lg = a.prefill(suf[s], len(pre), seq=s).copy()
        got[s] = (lg, decode_from_prompt(a, s, len(pre) + len(suf[s]), 20))

    b = load(tm, pkg)
    want = {}
    for s in range(N_SEQ):
        b.prefill(pre, 0, seq=s)
        lg = b.prefill(suf[s], len(pre), seq=s).copy()
        want[s] = (lg, decode_from_prompt(b, s, len(pre) + len(suf[s]), 20))

    for s in range(N_SEQ):
        assert same(got[s][0], want[s][0]), s
        assert_same_run(got[s][1], want[s][1])
    n_used = [len(pre) + len(x) + 20 for x in suf]
    for X, Y in zip(kv(a, tm), kv(b, tm)):
        for s in range(N_SEQ):
            assert torch.equal(X[s, :, :n_used[s]], Y[s, :, :n_used[s]])
    a.close()
    b.close()


# ---- 5. pipeline shards in one process ------------------------------------------------------------------------------------------

def decode_host(engs, seq, tok, pos, steps):
    """Host-driven steps of slot seq through a chain of shards (hidden state handed over with get_hidden / set_hidden), greedy on the
    last shard's device argmax.  Returns (tokens, logits per step)."""
    last = engs[-1]
    nv = last.hp.n_vocab
    _, smp = words(last)
    toks, logits = [], []
    for i in range(steps):
        for j, e in enumerate(engs):
            if j:
                e.set_hidden(engs[j - 1].hidden())
            e.decode_seq_async(seq, tok, pos + i)
        last.argmax_seq(seq, False)
        logits.append(last.debug_read("logits", nv))
        tok = int(smp[seq])
        toks.append(tok)
    return toks, logits


@pytest.mark.parametrize("model", MODELS)
def test_prefill_stage_seq_on_pipeline_shards(cuda, pkg, model):
    tm = tiny(model, n_layer=3)
    nv, nl = tm.hp["n_vocab"], 3
    toks = prompt(40, 31, 7, nv)
    ubs = ((0, 24), (24, 16))                              # the same micro-batches on the whole model and on the shards
    whole = load(tm, pkg)
    for p0, n in ubs:
        lw = whole.prefill(toks[p0:p0 + n], p0, seq=2).copy()
    t0 = int(np.argmax(lw))
    want = decode_host([whole], 2, t0, 40, 10)
    whole.kv_copy(2, 0)
    whole.synchronize()
    KW, VW = snap(*kv(whole, tm))
    want0 = decode_host([whole], 0, 17, 50, 5)             # slot 0 continues from slot 2's copied cells
    for bounds in ([0, 2, 3], [0, 1, 2, 3]):
        shards = [load(tm, pkg, (a, b), a == 0, b == nl) for a, b in zip(bounds, bounds[1:])]
        lg = np.zeros(nv, np.float32)
        for p0, n in ubs:
            h = None
            for i, e in enumerate(shards):
                out = lg if i == len(shards) - 1 and p0 + n == len(toks) else None
                h = e.prefill_stage(toks[p0:p0 + n] if i == 0 else None, h, n, p0, out, synchronize=True, seq=2)
        assert same(lg, lw), bounds
        assert_same_run(decode_host(shards, 2, t0, 40, 10), want)
        for e in shards:
            e.kv_copy(2, 0)
            e.synchronize()
        for e, a, b in zip(shards, bounds, bounds[1:]):
            K, V = kv(e, tm, b - a)
            assert torch.equal(K, KW[:, a:b]) and torch.equal(V, VW[:, a:b]), (bounds, a)   # slot 1 untouched (zero) on both sides
        assert_same_run(decode_host(shards, 0, 17, 50, 5), want0)
        for e in shards:
            e.close()
    whole.close()
