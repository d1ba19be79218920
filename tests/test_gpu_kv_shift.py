"""-m gpu: prima's context shift on the device (pb200_kv_seq_shift, pb200_rope_f16).

When llama-cli's context fills it drops half of the cells after n_keep and moves the rest down (llama_kv_cache_seq_rm + seq_add,
examples/main/main.cpp:578-608); the next decode re-rotates the moved K rows in place on the f16 cache (build_k_shift,
src/llama.cpp:10665-10719).  A shifted K row is f16(rope(f32(K_old), delta)): it is rounded twice, so it is NOT the row the engine
would store for the new position directly.  The restatement below does the same on the port model's caller-owned cache."""
import ctypes as C
import json
import os
import re
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from tiny_model import TinyModel

pytestmark = pytest.mark.gpu
G = Path(__file__).resolve().parent / "golden"
ROOT = Path(__file__).resolve().parent.parent


def check_decode_parity(got, want):
    """The multi-token bar of the engine's parity tests: first token exact, NMSE over the run below the reference's whole-block bar
    (2e-3), max-abs bounded, greedy tokens agree on >= 90 % of the steps."""
    e = np.max(np.abs(got - want), axis=1)
    assert e[0] < 1e-5, e[0]
    nmse = float(np.sum((got - want) ** 2) / np.sum(want ** 2))
    assert nmse < 2e-3, (nmse, e)
    assert np.max(e) < 0.25, e
    assert np.mean(got.argmax(1) == want.argmax(1)) >= 0.9


def llama_cli_shift(n_past, n_keep):
    """(p0, p1, delta) of llama-cli's context shift: n_discard = (n_past - n_keep) / 2 cells after n_keep go, the rest moves down."""
    n_discard = (n_past - n_keep) // 2
    return n_keep + n_discard, n_past, -n_discard


def port_kv_shift(port, hp, ff, kc, vc, p0, p1, delta):
    """The compacted shift on the port model's cache ([n_layer][n_ctx][n_head_kv * 128] f16 bits): K rows of cells [p0, p1) ->
    f16(port_rope(f32(K), pos = delta)) in cell c + delta (ggml_compute_forward_rope_f16, ggml.c:14269-14380), V rows copied."""
    HK = hp["n_head_kv"]
    for l in range(kc.shape[0]):
        src = kc[l, p0:p1].view(np.float16).astype(np.float32).reshape(-1)
        y = port.rope(src, (p1 - p0) * HK, 128, hp["rope_mode"], delta, freq_base=hp["rope_freq_base"], freq_scale=hp["rope_freq_scale"],
                      n_ctx_orig=hp["n_ctx_orig"], freq_factors=ff)
        kc[l, p0 + delta:p1 + delta] = y.astype(np.float16).view(np.uint16).reshape(p1 - p0, -1)
        vc[l, p0 + delta:p1 + delta] = vc[l, p0:p1].copy()


def _dev(ptr, shape, typestr):
    class V:
        __cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (ptr, False), "version": 2}
    return torch.as_tensor(V(), device="cuda")


def kv_tensors(eng, tm, n_seq, n_layer):
    shape = (n_seq, n_layer, tm.hp["n_ctx"], tm.hp["n_head_kv"] * 128)
    return _dev(eng.kv_ptr(False), shape, "<i2"), _dev(eng.kv_ptr(True), shape, "<i2")


def load(tm, pkg, n_seq=1, layers=None, with_embd=True, with_head=True):
    eng = pkg.Model(pkg.HParams(**tm.hp), 0, layers, with_embd, with_head)
    for name, (t, a) in tm.tensors.items():
        eng.set_tensor(name, t, a)
    eng.set_n_seq(n_seq)
    eng.finalize()
    return eng


def rope_f16(lib, x, pos, n_head, head_dim, n_dims, mode, ff=None, floats=(500000.0, 1.0, 0.0, 1.0, 32.0, 1.0), n_ctx_orig=8192, out=None):
    """pb200_rope_f16 on a device f16 tensor (as int16) [n_rows][n_head][head_dim]; out=None: a new tensor, out=x: in place."""
    y = torch.empty_like(x) if out is None else out
    pos_d = torch.as_tensor(np.ascontiguousarray(pos, np.int32)).cuda()
    ff_d = None if ff is None or len(ff) == 0 else torch.as_tensor(np.ascontiguousarray(ff, np.float32)).cuda()
    rc = lib.c.pb200_rope_f16(C.c_void_p(x.data_ptr()), C.c_void_p(y.data_ptr()), x.shape[0], n_head, head_dim, n_dims, mode, C.c_void_p(pos_d.data_ptr()),
                              *[float(f) for f in floats], n_ctx_orig, None if ff_d is None else C.c_void_p(ff_d.data_ptr()), None)
    assert rc == 0, rc
    torch.cuda.synchronize()
    return y


# ---------------------------------------------------------------------------------------------------------------------------------
def test_rope_f16_matches_reference_cpu_backend(cuda, lib):
    """pb200_rope_f16 against GGML_OP_ROPE on f16 computed by the reference CPU backend (golden/make_kshift_golden.py): NORM / NEOX,
    n_dims < head_dim, freq factors, YaRN, negative positions, out of place and in place."""
    z = np.load(G / "kshift_golden.npz")
    for i in range(int(z["n_cases"])):
        D, H, T, n_dims, mode, n_ctx_orig, in_place, _ = [int(v) for v in z[f"c{i}_ints"]]
        x, want = z[f"c{i}_x"], z[f"c{i}_y"]
        xd = torch.as_tensor(x.view(np.int16).copy()).cuda()
        for inplace in (False, True):
            src = xd.clone()
            got = rope_f16(lib, src, z[f"c{i}_pos"], H, D, n_dims, mode, z[f"c{i}_ff"], z[f"c{i}_floats"], n_ctx_orig, out=src if inplace else None)
            g = got.cpu().numpy().view(np.uint16)
            ulp = np.abs(g.astype(np.int32) - want.astype(np.int32))
            if z[f"c{i}_floats"][2] == 0.0:
                assert ulp.max() <= 1, (i, inplace, int(ulp.max()))
                assert np.mean(ulp == 0) > 0.99, (i, inplace, float(np.mean(ulp == 0)))
            else:
                # YaRN: the ramp mix of two angles is rounded differently (the reference's CPU build contracts it into an FMA), and at
                # positions of several thousand one f32 ulp of the angle is ~5e-4 rad: bounded by the row's magnitude, not by one f16 ulp
                gf, wf = g.view(np.float16).astype(np.float32), want.view(np.float16).astype(np.float32)
                xf = np.abs(x.view(np.float16).astype(np.float32)).max(axis=-1, keepdims=True)
                assert np.all(np.abs(gf - wf) <= np.abs(wf) * 2.0 ** -10 + 2e-3 * xf), (i, inplace)
                assert np.mean(ulp == 0) > 0.9, (i, inplace, float(np.mean(ulp == 0)))
            if n_dims < D:   # the un-rotated tail is copied bit for bit
                assert np.array_equal(g.reshape(T, H, D)[..., n_dims:], x[..., n_dims:])


SHIFTS = [  # (n_past, n_keep) of llama-cli's rule, and explicit (p0, p1, delta)
    llama_cli_shift(63, 0),    # overlapping: the moved block is longer than |delta|
    llama_cli_shift(63, 4),
    (40, 50, -30),             # disjoint
    (5, 60, -1),               # one cell down: every destination was a source
]


@pytest.mark.parametrize("arch,n_head,n_head_kv,ff", [("llama", 8, 1, True), ("llama", 8, 2, False), ("qwen2", 4, 4, False), ("qwen2", 8, 2, False),
                                                        ("qwen2", 8, 1, True)])
def test_shift_kernel_moves_and_rotates(cuda, pkg, lib, port, arch, n_head, n_head_kv, ff):
    tm = TinyModel(n_layer=3, n_embd=512, n_head=n_head, n_head_kv=n_head_kv, n_ff=512, n_vocab=256, n_ctx=64, arch=arch, freq_factors=ff, seed=4)
    hp = tm.hp
    ffv = tm.tensors["rope_freqs.weight"][1] if ff else None
    eng = load(tm, pkg, n_seq=2)
    K, V = kv_tensors(eng, tm, 2, 3)
    tokpos = [_dev(eng.token_ptr(s), (2,), "<i4") for s in range(2)]
    g = torch.Generator(device="cuda").manual_seed(1)
    for seq in (0, 1):
        for p0, p1, delta in SHIFTS:
            K.copy_(torch.randn(K.shape, generator=g, device="cuda").half().view(torch.int16))
            V.copy_(torch.randn(V.shape, generator=g, device="cuda").half().view(torch.int16))
            eng.set_tokpos_seq(seq, 17, p1)
            eng.set_tokpos_seq(1 - seq, 23, p1)
            torch.cuda.synchronize()
            k0, v0 = K.cpu().numpy().view(np.uint16), V.cpu().numpy().view(np.uint16)
            # the same rows through pb200_rope_f16, in place on a copy: the shift must reproduce it bit for bit
            rows = K[seq, :, p0:p1].clone().reshape(3 * (p1 - p0), n_head_kv, 128)
            rope_f16(lib, rows, np.full(rows.shape[0], delta, np.int32), n_head_kv, 128, 128, hp["rope_mode"], ffv,
                     (hp["rope_freq_base"], hp["rope_freq_scale"], 0.0, 1.0, 32.0, 1.0), hp["n_ctx_orig"], out=rows)
            eng.kv_shift(seq, p0, p1, delta)
            eng.synchronize()
            k1, v1 = K.cpu().numpy().view(np.uint16), V.cpu().numpy().view(np.uint16)
            d0, d1 = p0 + delta, p1 + delta
            assert np.array_equal(v1[seq, :, d0:d1], v0[seq, :, p0:p1])
            assert np.array_equal(k1[seq, :, d0:d1], rows.cpu().numpy().view(np.uint16).reshape(3, p1 - p0, -1))
            kp, vp = k0[seq].copy(), v0[seq].copy()
            port_kv_shift(port, hp, ffv, kp, vp, p0, p1, delta)
            ulp = np.abs(k1[seq, :, d0:d1].astype(np.int32) - kp[:, d0:d1].astype(np.int32))
            assert ulp.max() <= 1, int(ulp.max())
            assert np.array_equal(k1[seq, :, :d0], k0[seq, :, :d0]) and np.array_equal(v1[seq, :, :d0], v0[seq, :, :d0])
            assert np.array_equal(k1[1 - seq], k0[1 - seq]) and np.array_equal(v1[1 - seq], v0[1 - seq])
            assert tokpos[seq].tolist() == [17, p1 + delta]        # position moved, token kept
            assert tokpos[1 - seq].tolist() == [23, p1]
    # a position below p0 stays where it is
    eng.set_tokpos_seq(0, 5, 10)
    eng.kv_shift(0, 20, 30, -5)
    eng.synchronize()
    assert tokpos[0].tolist() == [5, 10]
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------------------
def run_with_shifts(n_ctx, n_keep, toks, decode, shift):
    """Teacher-forced token stream through llama-cli's context-shift rule: shift when n_past + 1 >= n_ctx, then decode at n_past."""
    n_past = 0
    for i, t in enumerate(toks):
        if n_past + 1 >= n_ctx:
            p0, p1, delta = llama_cli_shift(n_past, n_keep)
            shift(p0, p1, delta)
            n_past += delta
        decode(i, t, n_past)
        n_past += 1


@pytest.mark.parametrize("arch,ff,n_keep", [("llama", True, 0), ("qwen2", False, 5)])
def test_engine_vs_port_across_shifts(cuda, pkg, port, arch, ff, n_keep):
    """About 3 x n_ctx tokens with several context shifts: the engine's logits against the port model whose cache is shifted by
    the restatement above, step by step, under the engine's multi-token bar."""
    n_ctx = 64
    tm = TinyModel(n_layer=3, n_embd=1024, n_head=8, n_head_kv=2, n_ff=2816 if arch == "llama" else 3104, n_vocab=384, n_ctx=n_ctx, arch=arch,
                   ftype="q4_K_M" if arch == "llama" else "q5_K_M", freq_factors=ff, seed=11, branch_scale=0.1)
    toks = [(i * 7919 + 13) % 384 for i in range(3 * n_ctx)]
    m = tm.oracle_struct()
    kc = m._keep[-2].reshape(3, n_ctx, -1)
    vc = m._keep[-1].reshape(3, n_ctx, -1)
    ffv = tm.tensors["rope_freqs.weight"][1] if ff else None
    want = np.zeros((len(toks), 384), np.float32)
    hid = np.zeros(1024, np.float32)
    shifts = []

    def port_decode(i, t, pos):
        port.lib.port_llama_decode(C.byref(m), int(t), pos, want[i].ctypes.data_as(C.c_void_p), hid.ctypes.data_as(C.c_void_p))

    def port_shift(p0, p1, delta):
        shifts.append((p0, p1, delta))
        port_kv_shift(port, tm.hp, ffv, kc, vc, p0, p1, delta)

    run_with_shifts(n_ctx, n_keep, toks, port_decode, port_shift)
    assert len(shifts) >= 4
    eng = tm.load_engine(pkg)
    got = np.zeros_like(want)
    run_with_shifts(n_ctx, n_keep, toks, lambda i, t, pos: eng.decode(int(t), pos, got[i]), lambda *a: eng.kv_shift(0, *a))
    eng.close()
    check_decode_parity(got, want)
    first = n_ctx - 1   # the first step after the first shift
    e = np.max(np.abs(got[first:] - want[first:]), axis=1)
    assert np.mean(got[first:].argmax(1) == want[first:].argmax(1)) >= 0.9, e


# ---------------------------------------------------------------------------------------------------------------------------------
def _ring_model(n_ctx=40):
    return TinyModel(n_layer=4, n_embd=512, n_head=4, n_head_kv=2, n_ff=1024, n_vocab=320, n_ctx=n_ctx, seed=9, branch_scale=0.3, freq_factors=True)


def host_greedy_with_shifts(tm, pkg, tok, steps, n_keep):
    """Host-driven greedy decoding (pb200_decode + host argmax) through llama-cli's shifts: logits per step."""
    eng = tm.load_engine(pkg)
    out = np.zeros((steps, tm.hp["n_vocab"]), np.float32)
    cur = [tok]

    def dec(i, _t, pos):
        eng.decode(cur[0], pos, out[i])
        cur[0] = int(out[i].argmax())
    run_with_shifts(tm.hp["n_ctx"], n_keep, [0] * steps, dec, lambda *a: eng.kv_shift(0, *a))
    eng.close()
    return out


def device_loop(tm, pkg, steps, seeds, shifted, n_keep, graph=True):
    """pb200_step_seq_dev + pb200_argmax_seq(feed_back) on a two-slot model; slot s is shifted by llama-cli's rule when `shifted[s]`
    (and otherwise runs only while it fits the context).  Returns each slot's logits per step, copied on the model stream."""
    eng = load(tm, pkg, n_seq=2)
    eng.set_use_graph(graph)
    n_ctx = tm.hp["n_ctx"]
    lg = _dev(eng.logits_ptr, (tm.hp["n_vocab"],), "<f4")
    ext = torch.cuda.ExternalStream(eng.stream)
    hist = [[] for _ in seeds]
    n_past = [0, 0]
    for s, tok in enumerate(seeds):
        eng.set_tokpos_seq(s, tok, 0)
    for _ in range(steps):
        for s in range(2):
            if n_past[s] + 1 >= n_ctx:
                if not shifted[s]:
                    continue
                p0, p1, delta = llama_cli_shift(n_past[s], n_keep)
                eng.kv_shift(s, p0, p1, delta)    # moves the slot's device position too: nothing crosses the host
                n_past[s] += delta
            eng.step_seq_dev(s, True)
            eng.argmax_seq(s, True)
            with torch.cuda.stream(ext):
                hist[s].append(lg.clone())
            n_past[s] += 1
    eng.synchronize()
    eng.close()
    return [torch.stack(h).cpu().numpy() if h else None for h in hist]


def test_device_resident_loop_with_shifts(cuda, pkg):
    tm = _ring_model()
    steps, n_keep = 100, 3
    want1 = host_greedy_with_shifts(tm, pkg, 77, steps, n_keep)
    want0 = host_greedy_with_shifts(tm, pkg, 5, tm.hp["n_ctx"] - 1, n_keep)   # slot 0 never needs a shift
    got = device_loop(tm, pkg, steps, [5, 77], [False, True], n_keep)
    assert np.array_equal(got[1], want1)              # device loop == host loop, bit for bit, through two shifts
    assert np.array_equal(got[0], want0)              # shifting slot 1 leaves slot 0 untouched
    got_direct = device_loop(tm, pkg, steps, [5, 77], [False, True], n_keep, graph=False)
    assert np.array_equal(got_direct[1], got[1]) and np.array_equal(got_direct[0], got[0])   # graph replay == direct launches


def test_two_shards_shifted_match_one_model(cuda, pkg):
    """Two layer-window shards on one device (one without the head, one without the embedding), both shifted, against one model."""
    tm = _ring_model()
    toks = [(i * 31 + 7) % 320 for i in range(90)]
    want = np.zeros((len(toks), 320), np.float32)
    eng = tm.load_engine(pkg)
    run_with_shifts(tm.hp["n_ctx"], 2, toks, lambda i, t, pos: eng.decode(int(t), pos, want[i]), lambda *a: eng.kv_shift(0, *a))
    eng.close()
    s0 = tm.load_engine(pkg, layers=(0, 3), with_embd=True, with_head=False)
    s1 = tm.load_engine(pkg, layers=(3, 4), with_embd=False, with_head=True)
    got = np.zeros_like(want)

    def dec(i, t, pos):
        s0.decode(int(t), pos, None)
        s1.set_hidden(s0.hidden())
        s1.decode(int(t), pos, got[i])

    def shift(*a):
        s0.kv_shift(0, *a)
        s1.kv_shift(0, *a)
    run_with_shifts(tm.hp["n_ctx"], 2, toks, dec, shift)
    s0.close(); s1.close()
    assert np.array_equal(got, want)


# ---------------------------------------------------------------------------------------------------------------------------------
# The plugin: llama-cli on the "B200" ggml backend reaching a full context.
def test_backend_ops_rope_f16_cases_run(cuda):
    """test-backend-ops -o ROPE (the reference's own harness, unmodified) on B200_0: the type=f16 cases are claimed and pass."""
    import oracle_lib as O
    exe, plugin = O.ORACLE / "_ref" / "v3" / "test-backend-ops", ROOT / "prima.cpp_b200" / "libggml-b200.so"
    if not exe.exists() or not plugin.exists():
        pytest.skip("oracle/_ref/v3/test-backend-ops or libggml-b200.so not built (build() builds them only where the reference source tree is readable)")
    p = subprocess.run([str(exe), "test", "-b", "B200_0", "-o", "ROPE"], env=dict(os.environ, LD_PRELOAD=str(plugin)), capture_output=True, text=True,
                       timeout=900)
    out = re.sub(r"\x1b\[[0-9;]*m", "", p.stdout + p.stderr)
    f16 = [l for l in out.splitlines() if "ROPE(type=f16" in l]
    ok = [l for l in f16 if ": OK" in l]
    assert p.returncode == 0, out[-2000:]
    assert ok and len(ok) == len([l for l in f16 if "v=0" in l]), (len(ok), len(f16), f16[:5])   # every contiguous f16 case ran and passed
    assert not [l for l in f16 if "FAIL" in l], f16


def run_kshift_host(arch, n_head_kv, n_keep, n_shifts):
    if not (ROOT / "host" / "_ggml" / "libllama_graph_host.so").exists() or not (ROOT / "prima.cpp_b200" / "libggml-b200.so").exists():
        pytest.skip("host/_ggml or the plugin is not built (build() builds them only where the reference source tree is readable)")
    cmd = [sys.executable, str(ROOT / "tests" / "ggml_kshift_parity.py"), arch, str(n_head_kv), str(n_keep), str(n_shifts)]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-4000:]
    return json.loads(p.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("arch,n_head_kv,n_keep", [("llama", 1, 0), ("qwen2", 2, 3)])
def test_plugin_context_shift_matches_cpu_backend(cuda, arch, n_head_kv, n_keep):
    """An 8-token prompt, then decode steps through two of llama-cli's context shifts, on B200_0 and on the reference CPU backend with
    the host stand-in's cell bookkeeping (holes, the K-shift graph, new tokens in freed cells below live shifted ones), under the
    whole-graph bar of tests/test_gpu_ggml_graph.py.  n_head_kv = 1: the K-shift view [128, 1, n_ctx] has the shape of a one-token q."""
    r = run_kshift_host(arch, n_head_kv, n_keep, 2)
    L, steps = r["n_layer"], r["steps"]
    assert r["shifts"] == 2 and r["k_shifts"] == {"CPU": 2, "B200_0": 2}, r["k_shifts"]
    assert r["kshift_nodes"] > 0 and r["kshift_unsupported"] == 0, r     # the scheduler would find B200_0 for every K-shift node
    assert all(s["cells_equal"] and s["unsupported_nodes"] == 0 for s in steps)
    sq_err, sq_ref = sum(s["sq_err"] for s in steps), sum(s["sq_ref"] for s in steps)
    agree = [a for s in steps for a in s["argmax_agree_per_row"]]
    worst = max(max(s["max_abs_per_row"]) for s in steps)
    assert sq_err / sq_ref < 2e-3 and worst < 0.25 and sum(agree) >= 0.9 * len(agree), (sq_err / sq_ref, worst, sum(agree), len(agree))
    shifted = [i for i, s in enumerate(steps) if s["shift"]]
    assert len(shifted) == 2
    for i in shifted:
        assert steps[i]["kv_max_abs"] < 0.25, steps[i]                  # the K caches after both backends' K-shift graphs
    # after the first shift the freed cells lie below the moved ones: the new token goes into a hole below live shifted cells (after
    # the second, the reference's slot search may find the cells compacted again, as with n_keep > 0)
    assert steps[shifted[0]]["live_above"] > 0, steps[shifted[0]]
    decode = [s for s in steps if s["n"] == 1]
    plain = [s for s in decode if not s["shift"]]
    assert all(s["fused_steps"] >= 5 * L for s in decode), [s["fused_steps"] for s in decode]   # the decode plan stays fused
    for i in shifted:   # the K-shift graph itself ran 1:1: one more node per layer than a plain step, no extra fused step
        assert steps[i]["fused_steps"] == plain[-1]["fused_steps"], (steps[i], plain[-1])
        assert steps[i]["nodes"] == plain[-1]["nodes"] + L, (steps[i]["nodes"], plain[-1]["nodes"])
    assert sum(s["graph_replays"] for s in steps[shifted[-1] + 1:]) >= 10, [s["graph_replays"] for s in steps]   # replays resume
