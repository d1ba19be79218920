"""-m gpu: the ggml-backend plugin at the served models' layer shapes.  tests/test_gpu_ggml_graph.py runs the plugin on n_embd 1024 with
8 / 2 heads; this file runs full-size Llama-3-70B, Llama-3-8B and Qwen2.5-72B layers through graph_compute (the host stand-in of
tests/ggml_graph_parity.py) against the reference's CPU backend, the engine (pb200_decode) on the same bytes and the reference's
recorded logits.  What the fusion planner composes depends on the dimensions: which MUL_MATs the fused GEMV takes (k-quants with
K % 256 == 0 up to 29 696), whether gate / up may stay private (not when ffn_down is a 32-element type, as at Qwen2.5-72B's n_ff 29 568),
the attention step at 64 / 8 heads, the grow-only workspace sizes and the head group at full vocabulary.  So every decode step's launch
count and fused-step count are checked against the plan restated below, exactly.

Each test prints the measured value and the limit of every bar it asserts."""
import numpy as np
import pytest

import oracle_lib as O
from ggml_parity_util import Layer0, check_logits, decodes, prompt, prompt_steps, run_script, sessions
from golden import make_reference_golden as RG
from tiny_model import TinyModel
from test_gpu_engine import check_decode_parity, check_tie_split_parity

pytestmark = pytest.mark.gpu
G = RG.HERE


def bar(name, value, limit):
    """Prints one bar's measured value against its limit, then asserts value < limit."""
    print(f"  {name}: {value:.3e} (limit {limit:.0e}, margin x{limit / max(value, 1e-30):.1f})")
    assert value < limit, (name, value, limit)


def floor_bar(name, value, limit):
    """Prints one lower bar (argmax agreement) against its limit, then asserts value >= limit."""
    print(f"  {name}: {value:.3f} (limit {limit})")
    assert value >= limit, (name, value, limit)


# ------------------------------------------------------------------------------------------------------------------ the launch plan
# What the planner (prima.cpp_b200/ggml_backend/ggml_b200.cpp) must choose for one decode token, per weight mixture.  A fused GEMV
# step with the rms-norm or silu·mul prologue is one launch (the ring kernel quantizes its own activation behind one grid barrier);
# after the fused attention, wo's activation is already quantized (one launch); with a separate quantize prologue it is two.  Nodes that
# are not fused run 1:1: one launch each, two for a one-column MUL_MAT (quantize + GEMV).
#   (kind, prologue or op, what it computes)
HEAD_IN = [("node", "GET_ROWS", "token_embd")]
LLAMA_LAYER = [("gemv", "rms_norm", "attn_q|attn_k|attn_v (+ q / k / v biases for qwen2), outputs private"),
               ("attn", "-", "rope q / k, K / V cache store, KQ, soft_max, KQV, cont; output quantized for wo"),
               ("gemv", "from_attn", "attn_output + residual"),
               ("gemv", "rms_norm", "ffn_gate|ffn_up, outputs private"),
               ("gemv", "silu_mul", "ffn_down + residual")]
# Qwen2.5-72B: n_ff 29 568 is not a multiple of 256, so ffn_down is Q5_1 / Q8_0 (q5_K_M) or Q5_0 / Q8_0 (q4_K_M), which the fused GEMV
# does not take.  Gate and up then cannot stay private (assign_private_slots): each is a one-matrix group behind its own quantize
# launch, and the norm, silu, mul, ffn_down and residual add run 1:1 with the activation materialised.
QWEN_LAYER = LLAMA_LAYER[:3] + [("node", "RMS_NORM", "ffn_norm"), ("node", "MUL", "ffn_norm weight"),
                                ("gemv", "quantize", "ffn_up"), ("gemv", "quantize", "ffn_gate"),
                                ("node", "UNARY", "silu(gate)"), ("node", "MUL", "silu(gate) * up"),
                                ("node", "MUL_MAT", "ffn_down, one column"), ("node", "ADD", "residual")]
HEAD_OUT = [("gemv", "rms_norm", "output (the head), output_norm as prologue")]


def plan(arch, n_layer):
    return HEAD_IN + (LLAMA_LAYER if arch == "llama" else QWEN_LAYER) * n_layer + HEAD_OUT


def plan_counts(arch, n_layer):
    """(kernel launches, fused steps) of one decode token under plan(arch, n_layer)."""
    launches = fused = 0
    for kind, what, _ in plan(arch, n_layer):
        fused += kind != "node"
        launches += 2 if (kind == "gemv" and what == "quantize") or (kind == "node" and what == "MUL_MAT") else 1
    return launches, fused


def check_plan(r, arch):
    """Every decode step of run r ran plan(arch, n_layer) exactly and no node was left to the CPU."""
    want = plan_counts(arch, r["n_layer"])
    got = sorted({(s["launches"], s["fused_steps"]) for s in r["steps"] if "clear" not in s and s["n"] == 1})
    print(f"  plan: (launches, fused steps) per decode token {got}, restated {want}")
    assert got == [want], (got, want)
    assert all(s["unsupported_nodes"] == 0 for s in r["steps"] if "clear" not in s)


def test_plan_restatement():
    """The restated plan's own arithmetic: 5 launches and 5 fused steps per Llama layer, 14 launches and 5 fused steps per Qwen2.5-72B
    layer, the embedding rows and the head group around them."""
    assert plan_counts("llama", 2) == (12, 11)
    assert plan_counts("qwen2", 2) == (30, 11)
    assert plan_counts("llama", 80) == (402, 401)


# ------------------------------------------------------------------------------------------------------------------------ the cases
# dims: [n_layer, n_embd, n_head, n_head_kv, n_ff, n_vocab, n_ctx]
DECODE_STEPS = 72          # n_kv buckets 32, 64 and 96
CASES = {
    "llama3-70b": dict(arch="llama", dims=[2, 8192, 64, 8, 28672, 512, 96], ftype="q4_K_M", freq_factors=True),
    "llama3-8b": dict(arch="llama", dims=[2, 4096, 32, 8, 14336, 512, 96], ftype="q4_K_M", freq_factors=False),
    "qwen25-72b-q5_K_M": dict(arch="qwen2", dims=[2, 8192, 64, 8, 29568, 512, 96], ftype="q5_K_M", freq_factors=False),
    "qwen25-72b-q4_K_M": dict(arch="qwen2", dims=[2, 8192, 64, 8, 29568, 512, 96], ftype="q4_K_M", freq_factors=False),
}
# with the engine beside the plugin on the same bytes
ENGINE_CASES = ("llama3-70b", "qwen25-72b-q5_K_M", "qwen25-72b-q4_K_M")
# Bars against the CPU backend.  A full-size layer quantizes ~10^5 activation codes per token (q8_K of n_embd three times, of n_ff once,
# per layer), so a code whose x * 127 / amax lies within an fp32 ulp of a rounding tie already at token 0 can happen, and then the CPU
# backend's token 0 is a few 1e-2 away from the device's.  Measured on an H100 80GB HBM3 (token 0, max-abs on the logits vs the CPU
# backend): llama3-70b 4.2e-3, qwen25-72b-q5_K_M 2.9e-2, qwen25-72b-q4_K_M 3.1e-2, llama3-8b 4.8e-7.  Where token 0 is split, a second
# CPU reference says whether a split is what happened: the oracle port (tests/oracle_lib.py, the reference's scalar loops restated in
# C) decoding token 0 of the same TinyModel.
#   "exact": the CPU backend agrees to fp32 order; test_gpu_ggml_graph's multi-token bar applies unchanged (first token < 1e-4).
#   "port":  the device's token 0 agrees with the port to fp32 order (< 1e-4): it is the CPU backend that rounds a code the other way;
#            against the CPU backend the multi-token bar without first-token exactness.
#   "split": the port is itself more than 1e-3 from the CPU backend at token 0 and from the device: the three round codes differently.
#            Token 0 must then be bit-identical to the engine on the same bytes (ENGINE_CASES), whose decode the engine's tests check
#            against the port and the reference at these shapes, and the logits meet check_tie_split_parity's bar (every token within
#            0.05), as the engine's tests use it on engine_q72b_model, whose token-0 tie DESIGN §2 locates.
BARS = {"llama3-70b": "port", "llama3-8b": "exact", "qwen25-72b-q5_K_M": "split", "qwen25-72b-q4_K_M": "split"}


def port_token0(arch, dims, ftype, freq_factors, seed=31):
    """Logits of the oracle port for token 0 at position 0 of the driver's TinyModel (CPU, the reference's scalar order)."""
    n_layer, n_embd, n_head, n_head_kv, n_ff, n_vocab, n_ctx = dims
    tm = TinyModel(n_layer=n_layer, n_embd=n_embd, n_head=n_head, n_head_kv=n_head_kv, n_ff=n_ff, n_vocab=n_vocab, n_ctx=n_ctx, arch=arch,
                   ftype=ftype, freq_factors=freq_factors, seed=seed, branch_scale=0.1)
    return tm.port_decode(O.Port(), [13 % n_vocab])[0][0]    # the driver's token at position 0


def check_token0(r, d, kind, arch, dims, ftype, freq_factors):
    """Token 0 (the first decode step after the clear) against the oracle port on the same bytes.  kind "port": the device agrees
    with the port to fp32 summation order.  kind "split": the port is more than 1e-3 from the CPU backend, so the CPU references
    themselves disagree on a code at token 0 (the caller pins the device's token 0 to the engine)."""
    si = next(si for si, s in enumerate(r["steps"]) if "clear" not in s)
    assert r["steps"][si]["pos"] == 0
    port = port_token0(arch, dims, ftype, freq_factors)
    dev, cpu = d[f"logits_b200_{si}"][0], d[f"logits_cpu_{si}"][0]
    e_dev, e_cpu = float(np.max(np.abs(dev - port))), float(np.max(np.abs(cpu - port)))
    print(f"  token 0: device vs CPU backend {float(np.max(np.abs(dev - cpu))):.3e}, device vs port {e_dev:.3e}, CPU backend vs port {e_cpu:.3e}")
    if kind == "port":
        bar("token-0 max-abs vs oracle port", e_dev, 1e-4)
    else:
        floor_bar("token-0 CPU backend vs oracle port (a split code)", e_cpu, 1e-3)


_runs = {}


def case_run(name, tmp_path_factory, env=None, key=None):
    """The case's DECODE_STEPS decode steps from position 0 through the plugin and the CPU backend (and the engine for ENGINE_CASES),
    run once per session and key; returns (result, dump)."""
    key = key or name
    if key not in _runs:
        c = CASES[name]
        dump = tmp_path_factory.mktemp(key) / "d.npz"
        r = run_script(c["arch"], ["clear"] + decodes(0, DECODE_STEPS), dims=c["dims"], dump=dump, ftype=c["ftype"],
                       freq_factors=c["freq_factors"], engine=name in ENGINE_CASES and env is None, env=env)
        _runs[key] = (r, np.load(dump))
    return _runs[key]


def decode_logits(r, dump, tag):
    idx = [si for si, s in enumerate(r["steps"]) if "clear" not in s]
    return np.concatenate([dump[f"logits_{tag}_{si}"] for si in idx]), idx


def check_vs_cpu(r, kind, every=None):
    """kind "exact": test_gpu_ggml_graph's multi-token bar (first token to fp32 summation order, then max-abs 0.25, NMSE 2e-3, >= 90 %
    same argmax, KV rows 0.25); "port": the same without the first-token exactness (the caller pins token 0 to the oracle port);
    "split": check_tie_split_parity's bar (every token within 0.05, NMSE, argmax) and the KV rows.  every: a measured max-abs limit
    in place of the kind's."""
    st = [s for s in r["steps"] if "clear" not in s]
    e = np.array([s["max_abs_per_row"][0] for s in st])
    nmse = sum(s["sq_err"] for s in st) / sum(s["sq_ref"] for s in st)
    agree = float(np.mean([s["argmax_agree_per_row"][0] for s in st]))
    print(f"  vs CPU backend: max-abs per token {np.array2string(e, precision=4, max_line_width=200)}, argmax agreement {agree:.3f}")
    if kind == "exact":
        bar("first-token max-abs", float(e[0]), 1e-4)
    bar("max-abs, every token", float(e.max()), every or (0.05 if kind == "split" else 0.25))
    bar("NMSE", nmse, 2e-3)
    floor_bar("argmax agreement", agree, 0.9)
    bar("KV rows max-abs", max(s["kv_max_abs"] for s in st), 0.25)


def check_vs_engine(r, d, limit=0.05):
    """The plugin against the engine, step by step.  Layer-0 K / V cells (written from the embedding alone, no upstream activation
    code) and the logits and hidden state of token 0 are bit-identical; after it every step's logits within `limit` (check_tie_split_parity's
    0.05 unless the caller measured more), NMSE 2e-3, >= 90 % same argmax.  Returns the max-abs of logits and hidden state per step."""
    idx = [si for si, s in enumerate(r["steps"]) if "clear" not in s]
    e_lg, e_hd = [], []
    for si in idx:
        n = r["steps"][si]["pos"] + 1                       # cells written so far
        for k in ("k0", "v0"):
            assert np.array_equal(d[f"{k}_b200_{si}"][:n], d[f"{k}_eng_{si}"][:n]), (si, k)
        e_lg.append(float(np.max(np.abs(d[f"logits_b200_{si}"] - d[f"logits_eng_{si}"]))))
        e_hd.append(float(np.max(np.abs(d[f"hidden_b200_{si}"] - d[f"hidden_eng_{si}"]))))
    got = np.concatenate([d[f"logits_b200_{si}"] for si in idx])
    want = np.concatenate([d[f"logits_eng_{si}"] for si in idx])
    first = next((i for i, x in enumerate(e_lg) if x > 0), len(e_lg))
    nmse = float(np.sum((got.astype(np.float64) - want) ** 2) / np.sum(want.astype(np.float64) ** 2))
    print(f"  plugin vs engine: layer-0 K / V cells bit-identical; logits bit-identical for the first {first} of {len(idx)} steps; "
          f"logits max-abs per step {np.array2string(np.array(e_lg), precision=4, max_line_width=200)}; hidden max-abs {max(e_hd):.3e}")
    assert first >= 1 and e_hd[0] == 0.0, (e_lg[0], e_hd[0])
    bar("plugin vs engine max-abs", max(e_lg), limit)
    bar("plugin vs engine NMSE", nmse, 2e-3)
    floor_bar("plugin vs engine argmax agreement", float(np.mean(got.argmax(1) == want.argmax(1))), 0.9)
    return e_lg, e_hd


@pytest.mark.parametrize("name", list(CASES))
def test_fused_decode_vs_cpu_backend(cuda, tmp_path_factory, name):
    """DECODE_STEPS decode steps of two full-size layers (n_vocab 512) through the plugin against the CPU backend, crossing n_kv
    buckets 32 -> 64 -> 96, each step on the restated launch plan."""
    r, d = case_run(name, tmp_path_factory)
    c = CASES[name]
    check_plan(r, c["arch"])
    check_vs_cpu(r, BARS[name])
    if BARS[name] != "exact":
        check_token0(r, d, BARS[name], c["arch"], c["dims"], c["ftype"], c["freq_factors"])   # token 0 vs the engine: test_plugin_vs_engine
    assert r["steps"][-1]["graph_replays"] == 1          # the plan is captured and replayed at this size too


@pytest.mark.parametrize("name", ENGINE_CASES)
def test_plugin_vs_engine(cuda, tmp_path_factory, name):
    """The plugin against the engine on the same bytes, step by step: logits, last hidden state, the layer-0 K cells, and the plugin's
    transposed V cache read back as rows against the engine's V cells.  Both run the same ring GEMVs and k_attn2's arithmetic, but
    not bit for bit over a whole run: on an H100 80GB HBM3 the layer-0 K / V cells are bit-identical at all 72 steps and the logits at
    positions 0 to 2 (to 4 for q4_K_M).  After that the logits differ in fp32 order (up to 4.8e-7), and within a few steps an
    activation code splits: up to 3.4e-2 on the logits and 2.1e-2 on the hidden state over the run.  So the bar is bit identity on the cells and on
    token 0, then check_tie_split_parity's 0.05: what bench.py's boundary leg only prints."""
    r, d = case_run(name, tmp_path_factory)
    check_vs_engine(r, d)


@pytest.mark.parametrize("golden,arch,dims,ftype,seed,tie", [
    ("engine_70b", "llama", [2, 8192, 64, 8, 28672, 512, 32], "q4_K_M", 21, False),
    ("engine_q72b", "qwen2", [2, 8192, 64, 8, 29568, 512, 64], "q5_K_M", 31, True),
], ids=["llama3-70b", "qwen25-72b-q5_K_M"])
def test_decode_vs_recorded_reference(cuda, tmp_path, golden, arch, dims, ftype, seed, tie):
    """engine_70b_model / engine_q72b_model of tests/golden/make_reference_golden.py rebuilt by the driver (same dims, seed, ftype, no freq
    factors): the plugin's 8 decode steps against the reference CPU backend's recorded logits, with the bar the engine meets on the same
    bytes (check_decode_parity; check_tie_split_parity for the Qwen2.5-72B model's documented token-0 tie)."""
    want = np.load(G / "reference_golden.npz")[f"{golden}_logits"]
    r = run_script(arch, ["clear"] + decodes(0, len(want)), dims=dims, dump=tmp_path / "d.npz", ftype=ftype, seed=seed, freq_factors=False)
    check_plan(r, arch)
    got, _ = decode_logits(r, np.load(tmp_path / "d.npz"), "b200")
    e = np.max(np.abs(got - want), axis=1)
    print(f"  vs recorded reference: max-abs per token {np.array2string(e, precision=4)}, "
          f"NMSE {float(np.sum((got - want) ** 2) / np.sum(want ** 2)):.3e}")
    (check_tie_split_parity if tie else check_decode_parity)(got, want)


# ------------------------------------------------------------------------------------------------------------- prompt graphs (1:1)
PROMPT_SCRIPT = []
for _T in (7, 9, 64, 200):
    PROMPT_SCRIPT += ["clear", prompt(_T, 0)] + decodes(_T, 4)
PROMPT_SCRIPT += ["clear", prompt(20, 0), prompt(30, 20), prompt(38, 50)] + decodes(88, 4)   # one prompt in three graphs: n_kv 32, 64, 96


@pytest.mark.parametrize("name", ["llama3-70b", "qwen25-72b-q5_K_M"])
def test_prompt_graphs_at_layer_shapes(cuda, tmp_path, name):
    """Prompts of T in {7, 9, 64, 200} at position 0, each followed by 4 fused decode steps, and one prompt cut into three graphs
    (0, 20), (20, 30), (50, 38) across n_kv buckets, then 4 decode steps.  Prompt graphs run 1:1: the per-column GEMV for T < 8, the
    tensor-core mat-mul at K 8192 (and stream-K split tiles) for T >= 8, the f16 KQ / KQV with r2 = 8, SOFT_MAX over T * 64 rows and the
    transposed V store into a 1 024-row cache (n_ctx 1024: the V cache's row stride is far from every n_kv bucket).  Layer-0 K / V rows are held to Layer0's float64 bounds, the logits to the multi-token bar."""
    c = CASES[name]
    dims = c["dims"][:6] + [1024]
    r = run_script(c["arch"], PROMPT_SCRIPT, dims=dims, reserve=200, dump=tmp_path / "d.npz", ftype=c["ftype"], freq_factors=c["freq_factors"])
    dump = np.load(tmp_path / "d.npz")
    for s in r["steps"]:
        if "clear" not in s and s["n"] > 1:
            assert s["fused_steps"] == 0 and s["unsupported_nodes"] == 0, s
    check_plan(r, c["arch"])
    l0 = Layer0(c["arch"], dims, ftype=c["ftype"], freq_factors=c["freq_factors"])
    for si, s in prompt_steps(r):
        print(f"  layer-0 K / V rows {s['pos']}..{s['pos'] + s['n'] - 1}: worst error / bound {l0.check(dump, si, s['pos'], s['n']):.3f} (limit 1)")
    for ses in sessions(r):
        # T < 8 runs per-column GEMVs like the CPU's vec_dot, but token 0 of both models holds a split activation code (BARS): their
        # token 0 is pinned to the oracle port and to the engine by the decode tests
        nmse, worst, agree, kv = check_logits(ses, first_row_exact=False)
        print(f"  session from T = {ses[0]['n']}: NMSE {nmse:.3e} (limit 2e-3), max-abs {worst:.3e} (limit 0.25), argmax {agree:.3f} "
              f"(limit 0.9), KV {kv:.3e} (limit 0.25)")


# ------------------------------------------------------------------------------------------------- full vocabulary and layer count
def test_full_vocabulary_head(cuda, tmp_path):
    """One Llama-3-70B layer with the full 128 256-token vocabulary: the head group (rms-norm prologue, Q6_K at 128 256 rows) at bench's
    size.  6 decode steps against the CPU backend, the engine and, for token 0 (1.3e-2 from the CPU backend on an H100), the oracle port."""
    dims = [1, 8192, 64, 8, 28672, 128256, 32]
    r = run_script("llama", ["clear"] + decodes(0, 6), dims=dims, dump=tmp_path / "d.npz", engine=True)
    d = np.load(tmp_path / "d.npz")
    check_plan(r, "llama")
    check_vs_cpu(r, "port")
    check_token0(r, d, "port", "llama", dims, "q4_K_M", True)
    check_vs_engine(r, d)


def test_eighty_layers(cuda, tmp_path):
    """80 layers at n_embd 1024, 8 / 2 heads: bench's layer count, so 80 layers' nodes go through the planner, its windows and the CUDA
    graph capture.  24 decode steps against the CPU backend, each on the restated plan (402 launches), and against the engine.  Token 0
    is 3.8e-2 from the CPU backend on an H100, and the oracle port is 4.3e-2 from it: a split code; token 0 is bit-identical to the
    engine."""
    dims = [80, 1024, 8, 2, 2816, 384, 96]
    r = run_script("llama", ["clear"] + decodes(0, 24), dims=dims, dump=tmp_path / "d.npz", engine=True)
    d = np.load(tmp_path / "d.npz")
    check_plan(r, "llama")
    # 80 layers carry a split code further: 0.12 at most against the CPU backend over the run on an H100, so the multi-token 0.25
    check_vs_cpu(r, "split", every=0.25)
    check_token0(r, d, "split", "llama", dims, "q4_K_M", True)
    check_vs_engine(r, d, limit=0.25)   # 80 layers carry a split further: 0.10 at most on an H100
    assert r["steps"][-1]["graph_replays"] == 1


# ------------------------------------------------------------------------------------------------ 1:1 path and direct launches
def test_unfused_path_at_70b_shape(cuda, tmp_path_factory):
    """GGML_B200_NO_FUSE=1: every node 1:1 at 64 / 8 heads (the f16 KQ / KQV with r2 = 8, the 8192-wide one-column GEMVs, the transposed
    V store), against the CPU backend with the same bars."""
    r, r_dump = case_run("llama3-70b", tmp_path_factory, env={"GGML_B200_NO_FUSE": "1"}, key="llama3-70b-nofuse")
    st = [s for s in r["steps"] if "clear" not in s]
    assert all(s["fused_steps"] == 0 and s["unsupported_nodes"] == 0 for s in st)
    assert min(s["launches"] for s in st) > 3 * plan_counts("llama", 2)[0]
    check_vs_cpu(r, BARS["llama3-70b"])
    c = CASES["llama3-70b"]
    check_token0(r, r_dump, BARS["llama3-70b"], c["arch"], c["dims"], c["ftype"], c["freq_factors"])


def test_direct_launches_equal_graph_replay_at_70b_shape(cuda, tmp_path_factory):
    """GGML_B200_NO_GRAPHS=1 issues the fused launches directly every token; the captured CUDA graph replays them with the destination
    cell read from device memory.  At the 70B shape the logits must be bit-identical, step by step."""
    a, da = case_run("llama3-70b", tmp_path_factory)
    b, db = case_run("llama3-70b", tmp_path_factory, env={"GGML_B200_NO_GRAPHS": "1"}, key="llama3-70b-nographs")
    assert sum(s.get("graph_replays", 0) for s in a["steps"]) > 0 and all(s.get("graph_replays", 0) == 0 for s in b["steps"])
    check_plan(b, "llama")
    ga, _ = decode_logits(a, da, "b200")
    gb, _ = decode_logits(b, db, "b200")
    print(f"  graph replay vs direct launches, logits max-abs {float(np.max(np.abs(ga - gb))):.3e}")
    assert np.array_equal(ga, gb)
