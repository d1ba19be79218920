"""-m gpu: the engine's sequence slots as the C ABI shows them.

- The code every engine entry point returns for a NULL model, an unfinalized model, seq = -1 and seq = n_seq, a shard without the
  embedding and the head, and a slot without sampling parameters or penalties.  The codes documented in include/prima_b200.h are
  asserted by name; the table pins the rest, including which check comes first.
- The kernel launches each slot call enqueues (pb200_kernel_launches), for a Q4_K_M and a Q4_0 model with three slots.
- That a slot's calls write only that slot: its K / V cache block, its {token, pos} words at pb200_token_device(m, seq), its sample word.
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
SHAPE = dict(n_layer=2, n_embd=512, n_head=4, n_head_kv=2, n_ff=1024, n_vocab=320, n_ctx=48)


def q4_k_m():
    return TinyModel(**SHAPE, seed=21, branch_scale=0.3)


def q4_0():
    return L.q4_0_model(22, **SHAPE)


def load(tm, pkg, n_seq=N_SEQ, layers=None, with_embd=True, with_head=True):
    eng = pkg.Model(pkg.HParams(**tm.hp), 0, layers, with_embd, with_head)
    for name, (t, a) in tm.tensors.items():
        eng.set_tensor(name, t, a)
    eng.set_n_seq(n_seq)
    eng.finalize()
    return eng


def unfinalized(pkg, tm, layers=(0, SHAPE["n_layer"]), with_embd=True, with_head=True):
    lib = pkg.Lib.get()
    hp = pkg.HParams(**tm.hp)
    h = lib.c.pb200_model_create(C.byref(hp), 0, layers[0], layers[1], int(with_embd), int(with_head))
    assert h
    assert lib.c.pb200_model_set_n_seq(h, N_SEQ) == 0
    return h


def _dev(ptr, shape, typestr):
    class V:
        __cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (ptr, False), "version": 2}
    return torch.as_tensor(V(), device="cuda")


def kv_views(eng, hp, n_layer):
    """The f16 caches as int16 [n_seq][layer][n_ctx][n_head_kv * 128], the layout pb200_kv_device documents."""
    shape = (N_SEQ, n_layer, hp["n_ctx"], hp["n_head_kv"] * 128)
    return _dev(eng.kv_ptr(False), shape, "<i2"), _dev(eng.kv_ptr(True), shape, "<i2")


# ---- 1. error codes -------------------------------------------------------------------------------------------------------------

def entry_points(pkg, hp):
    """name -> call(c, h, seq) of every engine entry point with otherwise valid arguments (plus a few invalid variants).  Pointer getters
    give 1 for an address and 0 for NULL.  Calls that give a slot sampling parameters or penalties come last, so that the other calls
    see a bare slot."""
    E, nv, n_ctx = hp["n_embd"], hp["n_vocab"], hp["n_ctx"]
    vp = C.c_void_p
    toks = np.arange(1, 9, dtype=np.int32)
    host = np.zeros(max(E, nv), np.float32)
    smp, smp_bad = pkg.sampling(seed=1), pkg.sampling(top_p=2.0, seed=1)
    pen, pen_bad = pkg.penalties(repeat=1.1), pkg.penalties(repeat=0.0)
    keep = (toks, host, smp, smp_bad, pen, pen_bad)

    def ptr(a):
        return a.ctypes.data_as(vp)

    def nn(v):
        return int(bool(v))

    def tensor_device(name):
        return lambda c, h, s: c.pb200_model_tensor_device(h, name, C.byref(vp()), C.byref(C.c_size_t()), None)

    calls = {
        "token_device": lambda c, h, s: nn(c.pb200_token_device(h, s)),
        "sample_device": lambda c, h, s: nn(c.pb200_sample_device(h, s)),
        "kv_device": lambda c, h, s: nn(c.pb200_kv_device(h, 0)),
        "logits_device": lambda c, h, s: nn(c.pb200_logits_device(h)),
        "hidden_in_device": lambda c, h, s: nn(c.pb200_hidden_in_device(h)),
        "hidden_out_device": lambda c, h, s: nn(c.pb200_hidden_out_device(h)),
        "stream": lambda c, h, s: nn(c.pb200_stream(h)),
        "prefill_hidden_device": lambda c, h, s: nn(c.pb200_prefill_hidden_device(h)),
        "weight_bytes": lambda c, h, s: nn(c.pb200_model_weight_bytes(h) > 0),
        "set_n_seq": lambda c, h, s: c.pb200_model_set_n_seq(h, N_SEQ),
        "tensor_alloc": lambda c, h, s: c.pb200_model_tensor_alloc(h, b"output_norm.weight", 0, E * 4, C.byref(vp())),
        "set_tensor": lambda c, h, s: c.pb200_model_set_tensor(h, b"output_norm.weight", 0, ptr(host), E * 4),
        "synth": lambda c, h, s: c.pb200_model_synth(h, 0, 1),
        "finalize": lambda c, h, s: c.pb200_model_finalize(h),
        "tensor_device": tensor_device(b"output.weight"),
        "tensor_device_layer": tensor_device(b"blk.0.attn_q.weight"),
        "decode": lambda c, h, s: c.pb200_decode(h, 1, 0, ptr(host)),
        "decode_bad_pos": lambda c, h, s: c.pb200_decode(h, 1, n_ctx, None),
        "decode_async": lambda c, h, s: c.pb200_decode_async(h, 1, 0),
        "decode_async_bad_token": lambda c, h, s: c.pb200_decode_async(h, nv, 0),
        "synchronize": lambda c, h, s: c.pb200_synchronize(h),
        "profile_step": lambda c, h, s: c.pb200_profile_step(h, 1, 0, None, None, None, None),
        "profile_step_bad_token": lambda c, h, s: c.pb200_profile_step(h, nv, 0, None, None, None, None),
        "prefill": lambda c, h, s: c.pb200_prefill(h, ptr(toks), 8, 0, None),
        "prefill_over_ctx": lambda c, h, s: c.pb200_prefill(h, ptr(toks), 8, n_ctx - 4, None),
        "prefill_stage": lambda c, h, s: c.pb200_prefill_stage(h, ptr(toks), None, 8, 0, None, 1),
        "prefill_stage_async_logits": lambda c, h, s: c.pb200_prefill_stage(h, ptr(toks), None, 8, 0, ptr(host), 0),
        "kv_clear": lambda c, h, s: c.pb200_kv_clear(h),
        "get_hidden": lambda c, h, s: c.pb200_get_hidden(h, ptr(host)),
        "set_hidden": lambda c, h, s: c.pb200_set_hidden(h, ptr(host)),
        "debug_read": lambda c, h, s: c.pb200_debug_read(h, b"q", ptr(host), 8),
        "set_use_graph": lambda c, h, s: c.pb200_set_use_graph(h, 1),
        "decode_seq_async": lambda c, h, s: c.pb200_decode_seq_async(h, s, 1, 0),
        "decode_seq_async_bad_pos": lambda c, h, s: c.pb200_decode_seq_async(h, s, 1, -1),
        "step_seq_dev": lambda c, h, s: c.pb200_step_seq_dev(h, s, 0),
        "set_tokpos_seq": lambda c, h, s: c.pb200_set_tokpos_seq(h, s, 1, 0),
        "argmax_seq": lambda c, h, s: c.pb200_argmax_seq(h, s, 1),
        "kv_seq_shift": lambda c, h, s: c.pb200_kv_seq_shift(h, s, 4, 8, -2),
        "kv_seq_shift_bad_delta": lambda c, h, s: c.pb200_kv_seq_shift(h, s, 4, 8, 1),
        "kv_seq_shift_past_ctx": lambda c, h, s: c.pb200_kv_seq_shift(h, s, 4, n_ctx + 1, -2),
        "sample_seq": lambda c, h, s: c.pb200_sample_seq(h, s, 1),
        "sampler_accept_seq": lambda c, h, s: c.pb200_sampler_accept_seq(h, s, ptr(toks), 8),
        "sampling_set_seq_bad": lambda c, h, s: c.pb200_sampling_set_seq(h, s, C.byref(smp_bad)),
        "penalties_set_seq_bad": lambda c, h, s: c.pb200_penalties_set_seq(h, s, C.byref(pen_bad)),
        "penalties_clear": lambda c, h, s: c.pb200_penalties_set_seq(h, s, None),
        "sampling_set_seq": lambda c, h, s: c.pb200_sampling_set_seq(h, s, C.byref(smp)),
        "penalties_set_seq": lambda c, h, s: c.pb200_penalties_set_seq(h, s, C.byref(pen)),
    }
    return calls, keep


CONDITIONS = ("null", "unfinalized", "seq_neg", "seq_n", "shard", "bare_slot")

# entry point -> code per CONDITIONS, recorded from the engine
WANT = {
    "token_device":               (0, 0, 0, 0, 1, 1),
    "sample_device":              (0, 0, 0, 0, 1, 1),
    "kv_device":                  (0, 0, 1, 1, 1, 1),
    "logits_device":              (0, 0, 1, 1, 0, 1),
    "hidden_in_device":           (0, 0, 1, 1, 1, 1),
    "hidden_out_device":          (0, 0, 1, 1, 1, 1),
    "stream":                     (0, 1, 1, 1, 1, 1),
    "prefill_hidden_device":      (0, 0, 0, 0, 0, 0),
    "weight_bytes":               (0, 0, 1, 1, 1, 1),
    "set_n_seq":                  (EINVAL, 0, ESTATE, ESTATE, ESTATE, ESTATE),
    "tensor_alloc":               (EINVAL, 0, ESTATE, ESTATE, ESTATE, ESTATE),
    "set_tensor":                 (EINVAL, 0, ESTATE, ESTATE, ESTATE, ESTATE),
    "synth":                      (EINVAL, 0, ESTATE, ESTATE, ESTATE, ESTATE),
    "finalize":                   (EINVAL, ESTATE, 0, 0, 0, 0),
    "tensor_device":              (EINVAL, ESTATE, 0, 0, ESTATE, 0),
    "tensor_device_layer":        (EINVAL, ESTATE, 0, 0, ESTATE, 0),
    "decode":                     (ESTATE, ESTATE, 0, 0, 0, 0),
    "decode_bad_pos":             (ESTATE, ESTATE, EINVAL, EINVAL, EINVAL, EINVAL),
    "decode_async":               (ESTATE, ESTATE, 0, 0, 0, 0),
    "decode_async_bad_token":     (ESTATE, ESTATE, EINVAL, EINVAL, EINVAL, EINVAL),
    "synchronize":                (EINVAL, 0, 0, 0, 0, 0),
    "profile_step":               (ESTATE, ESTATE, 0, 0, 0, 0),
    "profile_step_bad_token":     (ESTATE, ESTATE, EINVAL, EINVAL, EINVAL, EINVAL),
    "prefill":                    (ESTATE, ESTATE, 0, 0, ENOTSUP, 0),
    "prefill_over_ctx":           (ESTATE, ESTATE, EINVAL, EINVAL, EINVAL, EINVAL),
    "prefill_stage":              (ESTATE, ESTATE, 0, 0, EINVAL, 0),
    "prefill_stage_async_logits": (ESTATE, ESTATE, EINVAL, EINVAL, EINVAL, EINVAL),
    "kv_clear":                   (ESTATE, ESTATE, 0, 0, 0, 0),
    "get_hidden":                 (EINVAL, EINVAL, 0, 0, 0, 0),
    "set_hidden":                 (EINVAL, EINVAL, 0, 0, 0, 0),
    "debug_read":                 (EINVAL, EINVAL, 0, 0, 0, 0),
    "set_use_graph":              (EINVAL, 0, 0, 0, 0, 0),
    "decode_seq_async":           (ESTATE, ESTATE, EINVAL, EINVAL, 0, 0),
    "decode_seq_async_bad_pos":   (ESTATE, ESTATE, EINVAL, EINVAL, EINVAL, EINVAL),
    "step_seq_dev":               (ESTATE, ESTATE, EINVAL, EINVAL, 0, 0),
    "set_tokpos_seq":             (ESTATE, ESTATE, EINVAL, EINVAL, 0, 0),
    "argmax_seq":                 (ESTATE, ESTATE, EINVAL, EINVAL, ESTATE, 0),
    "kv_seq_shift":               (ESTATE, ESTATE, EINVAL, EINVAL, 0, 0),
    "kv_seq_shift_bad_delta":     (EINVAL, EINVAL, EINVAL, EINVAL, EINVAL, EINVAL),
    "kv_seq_shift_past_ctx":      (ESTATE, ESTATE, EINVAL, EINVAL, EINVAL, EINVAL),
    "sample_seq":                 (ESTATE, ESTATE, EINVAL, EINVAL, ESTATE, ESTATE),
    "sampler_accept_seq":         (ESTATE, ESTATE, EINVAL, EINVAL, ESTATE, ESTATE),
    "sampling_set_seq_bad":       (ESTATE, ESTATE, EINVAL, EINVAL, ESTATE, EINVAL),
    "penalties_set_seq_bad":      (ESTATE, ESTATE, EINVAL, EINVAL, ESTATE, EINVAL),
    "penalties_clear":            (ESTATE, ESTATE, EINVAL, EINVAL, ESTATE, 0),
    "sampling_set_seq":           (ESTATE, ESTATE, EINVAL, EINVAL, ESTATE, 0),
    "penalties_set_seq":          (ESTATE, ESTATE, EINVAL, EINVAL, ESTATE, 0),
}


def error_table(pkg):
    """entry point -> the code of each CONDITIONS column.  Every unfinalized call gets a fresh model, so that synth or finalize on one
    cannot change what the next call sees."""
    c = pkg.Lib.get().c
    tm = q4_k_m()
    full = load(tm, pkg)
    shard = load(tm, pkg, layers=(1, 2), with_embd=False, with_head=False)
    calls, keep = entry_points(pkg, tm.hp)
    got = {}
    for name, f in calls.items():
        row = []
        for cond in CONDITIONS:
            if cond == "unfinalized":
                h = unfinalized(pkg, tm)
                row.append(f(c, h, 0))
                c.pb200_model_free(h)
                continue
            h = {"null": None, "shard": shard.h}.get(cond, full.h)
            seq = {"seq_neg": -1, "seq_n": N_SEQ, "bare_slot": 1}.get(cond, 0)
            row.append(f(c, h, seq))
        assert c.pb200_synchronize(full.h) == 0 and c.pb200_synchronize(shard.h) == 0, name
        got[name] = tuple(row)
    full.close()
    shard.close()
    del keep
    return got


def test_error_codes_of_every_entry_point(cuda, pkg):
    got = error_table(pkg)
    assert got == WANT, "\n".join(f"{k!r}: {v}," for k, v in got.items() if WANT.get(k) != v)
    col = {c: i for i, c in enumerate(CONDITIONS)}
    # documented in include/prima_b200.h
    assert got["kv_seq_shift_bad_delta"][col["null"]] == EINVAL           # delta, p0, p1 are checked before the model
    for cond in ("null", "unfinalized"):
        assert got["kv_seq_shift"][col[cond]] == ESTATE
    for cond in ("seq_neg", "seq_n"):
        assert got["kv_seq_shift"][col[cond]] == EINVAL
    assert got["kv_seq_shift_past_ctx"][col["bare_slot"]] == EINVAL
    for f in ("sample_seq", "sampler_accept_seq"):                          # a slot without parameters / penalties
        assert got[f][col["bare_slot"]] == ESTATE
    for f in ("penalties_set_seq", "sampler_accept_seq"):                   # a shard without the head
        assert got[f][col["shard"]] == ESTATE
    assert got["prefill"][col["shard"]] == ENOTSUP                          # whole prompts start at the embedding


def tensor_lookup(pkg):
    """(code, address or NULL) of pb200_model_tensor_alloc for names of this shard, of other stages, unknown names and wrong sizes, then
    pb200_model_tensor_device for a few of them; on a two-layer model's shard [1, 2) without embedding / head and on the whole model."""
    lib = pkg.Lib.get()
    c = lib.c
    tm = q4_k_m()
    E, nv = tm.hp["n_embd"], tm.hp["n_vocab"]
    q4k = lambda n, k: int(c.pb200_row_bytes(12, k)) * n
    names = [
        ("token_embd.weight", 12, q4k(nv, E)),
        ("output.weight", 14, int(c.pb200_row_bytes(14, E)) * nv),
        ("output_norm.weight", 0, E * 4),
        ("rope_freqs.weight", 0, 64 * 4),
        ("rope_freqs.weight#size", 0, 63 * 4),
        ("blk.0.attn_q.weight", 12, q4k(512, E)),
        ("blk.1.attn_q.weight#type", 0, q4k(512, E)),
        ("blk.1.attn_q.weight#size", 12, q4k(512, E) - 144),
        ("blk.1.attn_k.weight", 12, q4k(256, E)),
        ("blk.1.attn_norm.weight", 0, E * 4),
        ("blk.1.attn_norm.weight#size", 0, E * 4 + 4),
        ("blk.1.attn_q.bias", 0, 512 * 4),
        ("blk.1.attn_rot.weight", 0, 16),
        ("blk.x", 0, 16),
        ("blk.7.ffn_up.weight", 12, q4k(1024, E)),
        ("nonsense.weight", 0, 16),
    ]
    got = {}
    for which, kw in (("shard", dict(layers=(1, 2), with_embd=False, with_head=False)), ("full", {})):
        h = unfinalized(pkg, tm, **kw)
        for name, t, nb in names:
            p = C.c_void_p()
            rc = c.pb200_model_tensor_alloc(h, name.split("#")[0].encode(), t, nb, C.byref(p))
            got[(which, "alloc", name)] = (rc, int(bool(p.value)))
        for name in ("output.weight", "rope_freqs.weight", "blk.0.attn_q.weight", "blk.1.attn_k.weight", "blk.1.ffn_up.weight", "blk.x",
                     "nonsense.weight"):
            rc = c.pb200_model_tensor_device(h, name.encode(), C.byref(C.c_void_p()), C.byref(C.c_size_t()), None)
            got[(which, "device", name)] = (rc,)
        c.pb200_model_free(h)
    return got


WANT_LOOKUP = {
    ("shard", "alloc", "token_embd.weight"): (0, 0),
    ("shard", "alloc", "output.weight"): (0, 0),
    ("shard", "alloc", "output_norm.weight"): (0, 0),
    ("shard", "alloc", "rope_freqs.weight"): (0, 1),
    ("shard", "alloc", "rope_freqs.weight#size"): (EINVAL, 0),
    ("shard", "alloc", "blk.0.attn_q.weight"): (0, 0),
    ("shard", "alloc", "blk.1.attn_q.weight#type"): (ENOTSUP, 0),
    ("shard", "alloc", "blk.1.attn_q.weight#size"): (EINVAL, 0),
    ("shard", "alloc", "blk.1.attn_k.weight"): (0, 1),
    ("shard", "alloc", "blk.1.attn_norm.weight"): (0, 1),
    ("shard", "alloc", "blk.1.attn_norm.weight#size"): (EINVAL, 0),
    ("shard", "alloc", "blk.1.attn_q.bias"): (0, 1),
    ("shard", "alloc", "blk.1.attn_rot.weight"): (0, 0),
    ("shard", "alloc", "blk.x"): (0, 0),
    ("shard", "alloc", "blk.7.ffn_up.weight"): (0, 0),
    ("shard", "alloc", "nonsense.weight"): (EINVAL, 0),
    ("shard", "device", "output.weight"): (ESTATE,),
    ("shard", "device", "rope_freqs.weight"): (0,),
    ("shard", "device", "blk.0.attn_q.weight"): (ESTATE,),
    ("shard", "device", "blk.1.attn_k.weight"): (0,),
    ("shard", "device", "blk.1.ffn_up.weight"): (ESTATE,),
    ("shard", "device", "blk.x"): (ESTATE,),
    ("shard", "device", "nonsense.weight"): (ESTATE,),
    ("full", "alloc", "token_embd.weight"): (0, 1),
    ("full", "alloc", "output.weight"): (0, 1),
    ("full", "alloc", "output_norm.weight"): (0, 1),
    ("full", "alloc", "rope_freqs.weight"): (0, 1),
    ("full", "alloc", "rope_freqs.weight#size"): (EINVAL, 0),
    ("full", "alloc", "blk.0.attn_q.weight"): (0, 1),
    ("full", "alloc", "blk.1.attn_q.weight#type"): (ENOTSUP, 0),
    ("full", "alloc", "blk.1.attn_q.weight#size"): (EINVAL, 0),
    ("full", "alloc", "blk.1.attn_k.weight"): (0, 1),
    ("full", "alloc", "blk.1.attn_norm.weight"): (0, 1),
    ("full", "alloc", "blk.1.attn_norm.weight#size"): (EINVAL, 0),
    ("full", "alloc", "blk.1.attn_q.bias"): (0, 1),
    ("full", "alloc", "blk.1.attn_rot.weight"): (0, 0),
    ("full", "alloc", "blk.x"): (0, 0),
    ("full", "alloc", "blk.7.ffn_up.weight"): (0, 0),
    ("full", "alloc", "nonsense.weight"): (EINVAL, 0),
    ("full", "device", "output.weight"): (0,),
    ("full", "device", "rope_freqs.weight"): (0,),
    ("full", "device", "blk.0.attn_q.weight"): (0,),
    ("full", "device", "blk.1.attn_k.weight"): (0,),
    ("full", "device", "blk.1.ffn_up.weight"): (ESTATE,),
    ("full", "device", "blk.x"): (ESTATE,),
    ("full", "device", "nonsense.weight"): (ESTATE,),
}


def test_tensor_lookup_codes(cuda, pkg):
    got = tensor_lookup(pkg)
    assert got == WANT_LOOKUP, "\n".join(f"{k!r}: {v}," for k, v in got.items() if WANT_LOOKUP.get(k) != v)


# ---- 2. launch counts ----------------------------------------------------------------------------------------------------------

def launch_counts(pkg, tm):
    """pb200_kernel_launches() added by each call, on one model with three slots (calls in this order)."""
    c = pkg.Lib.get().c
    eng = load(tm, pkg)
    nv = tm.hp["n_vocab"]
    logits = np.zeros(nv, np.float32)
    got = {}

    def count(name, f):
        eng.synchronize()
        n0 = c.pb200_kernel_launches()
        f()
        eng.synchronize()
        got[name] = int(c.pb200_kernel_launches() - n0)

    count("decode_graph", lambda: eng.decode(3, 0, logits))
    eng.set_use_graph(False)
    count("decode_direct", lambda: eng.decode(4, 1, logits))
    eng.set_use_graph(True)
    count("decode_async", lambda: eng.decode_async(5, 2))
    count("decode_seq_async", lambda: eng.decode_seq_async(1, 5, 0))
    count("step_seq_dev_advance", lambda: eng.step_seq_dev(1, True))
    count("step_seq_dev", lambda: eng.step_seq_dev(2, False))
    count("argmax_seq", lambda: eng.argmax_seq(1, True))
    count("sampling_set_seq", lambda: eng.set_sampling(2, seed=7))
    count("sample_seq", lambda: eng.sample_seq(2, False))
    count("penalties_set_seq_0_bias", lambda: eng.set_penalties(2, repeat=1.1, last_n=64))
    count("sampler_accept_seq", lambda: eng.accept(2, [1, 2, 3]))
    count("sample_seq_penalties", lambda: eng.sample_seq(2, False))
    count("penalties_set_seq_last_n_0", lambda: eng.set_penalties(2, repeat=1.1, last_n=0))
    count("sample_seq_penalties_last_n_0", lambda: eng.sample_seq(2, False))
    count("penalties_set_seq_300_bias", lambda: eng.set_penalties(2, repeat=1.1, logit_bias=[(i % nv, 0.5) for i in range(300)]))
    count("kv_seq_shift", lambda: eng.kv_shift(1, 1, 2, -1))
    count("prefill_12", lambda: eng.prefill([(7 * i + 1) % nv for i in range(12)], 0))
    count("prefill_5", lambda: eng.prefill([(5 * i + 2) % nv for i in range(5)], 0))
    count("profile_step", lambda: eng.profile_step(1, 0))
    eng.close()
    return got


WANT_LAUNCHES = {   # recorded from the engine
    "q4_K_M": {
        "decode_graph": 12, "decode_direct": 12, "decode_async": 12, "decode_seq_async": 12, "step_seq_dev_advance": 13,
        "step_seq_dev": 12, "argmax_seq": 1, "sampling_set_seq": 0, "sample_seq": 1, "penalties_set_seq_0_bias": 1,
        "sampler_accept_seq": 1, "sample_seq_penalties": 3, "penalties_set_seq_last_n_0": 1, "sample_seq_penalties_last_n_0": 2,
        "penalties_set_seq_300_bias": 2, "kv_seq_shift": 1, "prefill_12": 36, "prefill_5": 160, "profile_step": 12,
    },
    "q4_0": {
        "decode_graph": 26, "decode_direct": 26, "decode_async": 26, "decode_seq_async": 26, "step_seq_dev_advance": 27,
        "step_seq_dev": 26, "argmax_seq": 1, "sampling_set_seq": 0, "sample_seq": 1, "penalties_set_seq_0_bias": 1,
        "sampler_accept_seq": 1, "sample_seq_penalties": 3, "penalties_set_seq_last_n_0": 1, "sample_seq_penalties_last_n_0": 2,
        "penalties_set_seq_300_bias": 2, "kv_seq_shift": 1, "prefill_12": 42, "prefill_5": 160, "profile_step": 26,
    },
}


@pytest.mark.parametrize("model", ["q4_K_M", "q4_0"])
def test_launch_counts(cuda, pkg, model):
    got = launch_counts(pkg, {"q4_K_M": q4_k_m, "q4_0": q4_0}[model]())
    step = got["decode_graph"]
    assert got["decode_direct"] == got["decode_async"] == got["decode_seq_async"] == got["step_seq_dev"] == step
    assert got["step_seq_dev_advance"] == step + 1
    assert got["argmax_seq"] == got["sample_seq"] == got["sampler_accept_seq"] == got["kv_seq_shift"] == 1
    assert got["sample_seq_penalties"] == 3 and got["sample_seq_penalties_last_n_0"] == 2
    assert got["penalties_set_seq_0_bias"] == 1 and got["penalties_set_seq_300_bias"] == 2   # 256 bias entries per init launch
    assert got == WANT_LAUNCHES[model], got


# ---- 3. slot isolation ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("graph", [True, False])
def test_decoding_one_slot_leaves_the_other_slots_alone(cuda, pkg, graph):
    tm = q4_k_m()
    eng = load(tm, pkg)
    eng.set_use_graph(graph)
    K, V = kv_views(eng, tm.hp, SHAPE["n_layer"])
    for s in (0, 2):
        for pos in range(5):
            eng.decode_seq_async(s, 10 + pos + s, pos)
    eng.synchronize()
    k0, v0 = K.clone(), V.clone()
    words = _dev(eng.token_ptr(0), (N_SEQ, 4), "<i4")
    w0 = words.clone()
    for pos in range(7):
        eng.decode_seq_async(1, 20 + pos, pos)
    eng.synchronize()
    for s in (0, 2):
        assert torch.equal(K[s], k0[s]) and torch.equal(V[s], v0[s])
        assert torch.equal(words[s], w0[s])
    for X, X0 in ((K, k0), (V, v0)):
        assert bool((X[1, :, :7] != X0[1, :, :7]).any(dim=-1).all())     # every layer's row at every decoded position
        assert torch.equal(X[1, :, 7:], X0[1, :, 7:])
    assert words[1, :2].tolist() == [26, 6]
    eng.close()


def test_prefill_writes_slot_0_only(cuda, pkg):
    tm = q4_k_m()
    eng = load(tm, pkg)
    K, V = kv_views(eng, tm.hp, SHAPE["n_layer"])
    for s in (1, 2):
        for pos in range(4):
            eng.decode_seq_async(s, 30 + pos + s, pos)
    eng.synchronize()
    k0, v0 = K.clone(), V.clone()
    eng.prefill([(3 * i + 1) % tm.hp["n_vocab"] for i in range(12)], 0)
    for X, X0 in ((K, k0), (V, v0)):
        assert torch.equal(X[1:], X0[1:])
        assert bool((X[0, :, :12] != 0).any(dim=-1).all())
        assert torch.equal(X[0, :, 12:], X0[0, :, 12:])
    eng.close()


def test_token_and_sample_words_are_where_the_header_says(cuda, pkg):
    tm = q4_k_m()
    eng = load(tm, pkg)
    base, sbase = eng.token_ptr(0), eng.sample_ptr(0)
    assert [eng.token_ptr(s) - base for s in range(N_SEQ)] == [0, 16, 32]     # int32 {token, pos}, 16 bytes apart
    assert [eng.sample_ptr(s) - sbase for s in range(N_SEQ)] == [0, 4, 8]
    assert eng.token_ptr(N_SEQ) is None and eng.sample_ptr(-1) is None
    words = _dev(base, (N_SEQ, 4), "<i4")
    samples = _dev(sbase, (N_SEQ,), "<i4")
    for s in range(N_SEQ):
        eng.set_tokpos_seq(s, 100 + s, 10 + s)
    eng.synchronize()
    assert words[:, :2].tolist() == [[100, 10], [101, 11], [102, 12]]
    eng.decode(5, 2, np.zeros(tm.hp["n_vocab"], np.float32))                  # pb200_decode is slot 0
    eng.decode_seq_async(1, 7, 3)
    eng.step_seq_dev(2, True)
    eng.argmax_seq(2, True)
    eng.synchronize()
    assert words[:2, :2].tolist() == [[5, 2], [7, 3]]
    assert words[2, :2].tolist() == [int(samples[2]), 13]
    eng.close()
