"""-m gpu: whole-graph parity through the drop-in boundary.  A build_llama / build_qwen2 decode graph (host/llama_graph_host.cpp,
the stand-in for libllama's builder) is computed by ggml_backend_graph_compute on the registered "B200_0" backend and on the
reference's CPU backend with identical weights and tokens; logits, last hidden state and the KV cache contents are compared, and
the launch counter proves that graph_compute ran the FUSED path (<= 6 kernels per layer instead of ~25 single ops)."""
import json
import subprocess
import sys
from pathlib import Path

import pytest

import oracle_lib as O

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent


def run(arch, n_tok, dims=None, env=None):
    import os
    if not (ROOT / "host" / "_ggml" / "libllama_graph_host.so").exists() or not (ROOT / "prima.cpp_b200" / "libggml-b200.so").exists():
        pytest.skip("host/_ggml or the plugin is not built (build() builds them only where the reference source tree is readable)")
    cmd = [sys.executable, str(ROOT / "tests" / "ggml_graph_parity.py"), arch, str(n_tok)] + ([str(d) for d in dims] if dims else [])
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=dict(os.environ, **(env or {})))
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-4000:]
    return json.loads(p.stdout.strip().splitlines()[-1])


# n_ff 29 184 (114 super-blocks): an ffn_down the fused GEMV takes, past the 28 672 of Llama-3-70B
@pytest.mark.parametrize("arch,dims", [("llama", None), ("qwen2", None), ("llama", [3, 1024, 8, 2, 29184, 384, 96])],
                         ids=["llama", "qwen2", "llama-ff29184"])
def test_whole_graph_matches_cpu_backend_and_is_fused(cuda, arch, dims):
    r = run(arch, 40, dims)
    # same bar as the engine's multi-token parity (tests/test_gpu_engine.py::check_decode_parity): first token to fp32 summation
    # order, then the quantization-flip noise that the reference's own SIMD variants show against each other
    assert r["first_token_err"] < 1e-4, r
    assert r["nmse"] < 2e-3 and r["max_abs"] < 0.25 and r["argmax_agree"] >= 0.9, r
    assert r["kv_max_abs"] < 0.25, r       # f16 cache rows of magnitude ~20: a flipped activation code upstream moves them by a few 1e-2
    per_layer = [(n - 4) / r["n_layer"] for n in r["launches_per_token"]]   # get_rows + lm_head group + slack
    assert max(per_layer) <= 6.0, (r["launches_per_token"], r["graph_nodes"])
    assert r["fused_steps"] >= 40 * (5 * r["n_layer"]), r["fused_steps"]
    assert r["graph_builds"] <= 3          # one topology per 32-cell bucket of n_kv: the plan is reused token after token
    assert r["graph_replays"] >= 40 - 2 * 3, r["graph_replays"]   # per bucket: one direct call, one capture, then CUDA-graph replays


@pytest.mark.parametrize("name,t", [("qwen2_q4_K_M", O.Q5_0), ("llama_q4_0", O.Q4_0)])
def test_golden_legacy_model_whole_graph(cuda, name, t):
    """40 decode steps of a golden legacy-type model (tiny_model.legacy_golden_models) through the plugin against the CPU backend.
    The host stand-in places every node on B200_0 and the plugin refuses a node it does not claim, so the run also shows that no node
    fell back to the CPU."""
    r = run(name, 40)
    assert r["unsupported_nodes"] == 0, r
    assert r["first_token_err"] < 1e-4, r
    assert r["nmse"] < 2e-3 and r["max_abs"] < 0.25 and r["argmax_agree"] >= 0.9, r
    assert t in r["types"], r


def test_graph_replay_equals_direct_launches(cuda):
    """GGML_B200_NO_GRAPHS=1 issues the same fused launches directly every token; replaying the captured CUDA graph (with the
    destination cell read from device memory) must give bit-identical logits, i.e. the same errors against the CPU backend."""
    a = run("qwen2", 20)
    b = run("qwen2", 20, env={"GGML_B200_NO_GRAPHS": "1"})
    assert a["graph_replays"] > 0 and b["graph_replays"] == 0
    assert a["max_abs_per_token"] == b["max_abs_per_token"] and a["kv_max_abs"] == b["kv_max_abs"]


def test_fused_equals_unfused_node_by_node(cuda):
    """GGML_B200_NO_FUSE=1 runs every node 1:1 (the path test-backend-ops validates op by op); the fused plan must agree with it
    to the same tolerance as with the CPU backend — and tightly on the first token."""
    a = run("llama", 12)
    b = run("llama", 12, env={"GGML_B200_NO_FUSE": "1"})
    assert b["fused_steps"] == 0 and a["fused_steps"] > 0
    assert max(b["launches_per_token"]) > 3 * max(a["launches_per_token"])
    assert b["first_token_err"] < 1e-4 and a["first_token_err"] < 1e-4
    assert b["nmse"] < 2e-3 and a["nmse"] < 2e-3


# ---------------------------------------------------------------------------------------------------- prompt graphs and replay
# llama_decode sends a prompt as ONE graph of T tokens.  The fusion planner declines multi-token motifs, so every node of such a
# graph runs 1:1: the tensor-core mat-mul for T >= MMQ_MIN_COLS (8), one integer-dot GEMV per column below that, the f16 KQ / KQV
# mat-muls over T query rows, SOFT_MAX with T mask rows, the strided T-row store into the transposed V cache and the CONT of the
# permuted KQV.  The fused decode plan then continues on the K / V rows that path wrote.  The host stand-in reserves its compute
# buffer once, as llama.cpp does, so a topology seen before comes back at the same addresses and the plugin replays its CUDA graph.

def run_script(arch, steps, dims=None, reserve=None, env=None, dump=None):
    import os
    if not (ROOT / "host" / "_ggml" / "libllama_graph_host.so").exists() or not (ROOT / "prima.cpp_b200" / "libggml-b200.so").exists():
        pytest.skip("host/_ggml or the plugin is not built (build() builds them only where the reference source tree is readable)")
    cmd = [sys.executable, str(ROOT / "tests" / "ggml_graph_parity.py"), arch, "--script", json.dumps(steps)]
    cmd += ["--dims", ",".join(str(d) for d in dims)] if dims else []
    cmd += ["--reserve", str(reserve)] if reserve else []
    cmd += ["--dump", str(dump)] if dump else []
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=1800, env=dict(os.environ, **(env or {})))
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-4000:]
    return json.loads(p.stdout.strip().splitlines()[-1])


def prompt(T, pos):
    return {"n": T, "pos": pos}


def decodes(pos, k):
    return [{"n": 1, "pos": pos + i} for i in range(k)]


def check_logits(rows):
    """The multi-token bar of check_decode_parity / test_whole_graph_matches_cpu_backend_and_is_fused over a session's prompt rows
    and decode steps: once an activation code flips upstream (q = round(x*127/amax) of a 1-ulp fp32 difference), the deviation is
    the noise the reference's own SIMD builds show against each other, so NMSE < 2e-3, max-abs < 0.25, >= 90 % same argmax."""
    sq_err = sum(r["sq_err"] for r in rows)
    sq_ref = sum(r["sq_ref"] for r in rows)
    agree = [a for r in rows for a in r["argmax_agree_per_row"]]
    worst = max(max(r["max_abs_per_row"]) for r in rows)
    assert sq_err / sq_ref < 2e-3 and worst < 0.25 and sum(agree) >= 0.9 * len(agree), (sq_err / sq_ref, worst, sum(agree), len(agree))
    for r in rows:
        assert r["kv_max_abs"] < 0.25, r   # f16 cache rows of magnitude ~20: a flipped activation code upstream moves them by a few 1e-2
        if r["n"] > 1 and r["n"] < 8 and r["pos"] == 0:
            # T < 8 runs one integer-dot GEMV per column, like the CPU's vec_dot: the first row depends on token 0 alone and agrees
            # to fp32 summation order
            assert r["max_abs_per_row"][0] < 1e-4, r["max_abs_per_row"]


class Layer0:
    """Bars for the layer-0 K / V cache rows a prompt writes.  Their input is rms_norm(token_embd[tok]) * attn_norm on both backends,
    so no activation code can have flipped upstream; what is left is the mat-mul's own arithmetic, RoPE and the f16 store."""

    def __init__(self, arch, dims=None):
        import numpy as np
        import oracle_lib as O
        from tiny_model import TinyModel
        n_layer, n_embd, n_head, n_head_kv, n_ff, n_vocab, n_ctx = dims or [3, 1024, 8, 2, 2816 if arch == "llama" else 3072, 384, 96]
        tm = TinyModel(n_layer=n_layer, n_embd=n_embd, n_head=n_head, n_head_kv=n_head_kv, n_ff=n_ff, n_vocab=n_vocab, n_ctx=n_ctx, arch=arch,
                       ftype="q4_K_M" if arch == "llama" else "q5_K_M", freq_factors=(arch == "llama"), seed=31, branch_scale=0.1)
        port = O.Port()
        deq = lambda name, k: port.dequantize(tm.tensors[name][0], tm.tensors[name][1], k).astype(np.float64)
        emb = deq("token_embd.weight", n_embd)
        toks = [(i * 7919 + 13) % n_vocab for i in range(n_ctx)]   # the driver's token at each position
        x = emb[toks]
        x = x / np.sqrt(np.mean(x * x, axis=1, keepdims=True) + tm.hp["rms_eps"]) * tm.tensors["blk.0.attn_norm.weight"][1].astype(np.float64)
        self.x = np.abs(x)
        self.d_x = self.x.max(axis=1, keepdims=True) / 127          # largest q8 step of each row's activation quantization
        self.neox = tm.hp["rope_mode"] == 2
        self.w = {}
        for nm, wn in (("k", "blk.0.attn_k.weight"), ("v", "blk.0.attn_v.weight")):
            W = np.abs(deq(wn, n_embd))
            sub = np.repeat(W.reshape(W.shape[0], -1, 32).max(axis=2), 32, axis=1)
            self.w[nm] = (W, W + sub)

    def pair(self, b):
        """Error bound after RoPE: a rotation mixes each pair (a, b) of a head, |R e| <= |e_a| + |e_b| per component."""
        import numpy as np
        h = b.reshape(b.shape[0], -1, 128)
        if self.neox:
            s = h[..., :64] + h[..., 64:]
            out = np.concatenate([s, s], axis=-1)
        else:
            s = h[..., 0::2] + h[..., 1::2]
            out = np.repeat(s, 2, axis=-1)
        return out.reshape(b.shape)

    def check(self, dump, si, pos, T):
        """T < 8 (integer-dot GEMVs like the CPU's): every element within one f16 ulp of the CPU's plus the fp32 summation-order
        floor 2^-22 * sum|x_j w_j|, except in at most one row, where a rare q8 code flip of the activation (~3e-4 relative, see the
        comment above test_engine_vs_port_longer_decode) is allowed up to two flips' worth, 2 * d_x * max_j |w_j|.
        T >= 8 (tensor cores): the element-wise fp16-roundings bound of tests/test_gpu_mmq.py, 2^-9 * |x| @ (|W| + sub)^T, plus the
        same floor and the f16 store's ulp."""
        import numpy as np
        rows = slice(pos, pos + T)
        x, d_x = self.x[rows], self.d_x[rows]
        for nm in ("k", "v"):
            a, b = dump[f"{nm}0_cpu_{si}"][rows].astype(np.float64), dump[f"{nm}0_b200_{si}"][rows].astype(np.float64)
            W, Wsub = self.w[nm]
            floor = 2.0 ** -22 * (x @ W.T) + 1e-7
            bound = 2.0 ** -9 * (x @ Wsub.T) + 1e-6 if T >= 8 else floor
            kick = 2 * d_x * W.max(axis=1)[None, :]
            if nm == "k":   # the f32 RoPE of the two backends differs by a few fp32 ulps of the rotated pair as well
                bound, kick = self.pair(bound) + 2.0 ** -17 * self.pair(np.abs(a)), self.pair(kick)
            ulp = np.spacing(np.maximum(np.abs(a), np.abs(b)).astype(np.float16)).astype(np.float64)
            err = np.abs(a - b)
            over = err > ulp + bound
            worst = float((err / (ulp + bound)).max())
            if T >= 8:
                assert not over.any(), f"{nm} rows {pos}..{pos + T - 1}: {int(over.sum())} elements exceed the fp16-roundings bound (worst ratio {worst:.2f})"
            else:
                rows_over = int(over.any(axis=1).sum())
                assert rows_over <= 1, f"{nm} rows {pos}..{pos + T - 1}: {rows_over} rows beyond 1 f16 ulp + fp32 order (worst ratio {worst:.2f})"
                assert (err <= ulp + bound + kick).all(), f"{nm}: deviation larger than two q8 code flips (worst {float((err / (ulp + bound + kick)).max()):.2f})"


def prompt_steps(r):
    return [(si, st) for si, st in enumerate(r["steps"]) if "clear" not in st and st["n"] > 1]


@pytest.mark.parametrize("arch", ["llama", "qwen2"])
def test_prompt_batches_match_cpu_backend(cuda, arch, tmp_path):
    """Prompts of T in {2, 7, 8, 9, 33, 64} tokens at position 0, each followed by 8 decode steps, through graph_compute vs the CPU
    backend: both sides of MMQ_MIN_COLS, a partial and a full tensor-core tile, one and two n_kv buckets."""
    import numpy as np
    steps = []
    for T in (2, 7, 8, 9, 33, 64):
        steps += ["clear", prompt(T, 0)] + decodes(T, 8)
    r = run_script(arch, steps, reserve=64, dump=tmp_path / "d.npz")
    dump, l0, L = np.load(tmp_path / "d.npz"), Layer0(arch), r["n_layer"]
    sessions = [[]]
    for st in r["steps"]:
        if "clear" in st:
            sessions.append([])
            continue
        sessions[-1].append(st)
        assert st["unsupported_nodes"] == 0, st
        if st["n"] > 1:
            assert st["fused_steps"] == 0, st                    # the planner declines multi-token motifs
        else:
            assert st["fused_steps"] >= 5 * L, st                # and the decode after it is fused again
    for si, st in prompt_steps(r):
        l0.check(dump, si, st["pos"], st["n"])
    for s in sessions[1:]:
        check_logits(s)


def test_chunked_prompt_across_buckets(cuda, tmp_path):
    """A prompt cut into three graphs, (pos 0, T 20), (20, 30) crossing n_kv 32 -> 64 and (50, 38) reaching n_kv = n_ctx = 96, then
    8 decode steps up to the last cell: later chunks attend to cache rows written by earlier prompt graphs."""
    import numpy as np
    r = run_script("llama", ["clear", prompt(20, 0), prompt(30, 20), prompt(38, 50)] + decodes(88, 8), dump=tmp_path / "d.npz")
    dump, L = np.load(tmp_path / "d.npz"), r["n_layer"]
    st = r["steps"][1:]
    assert [s["pos"] for s in st][-1] == 95
    for s in st:
        assert s["unsupported_nodes"] == 0, s
        assert (s["fused_steps"] == 0) if s["n"] > 1 else (s["fused_steps"] >= 5 * L), s
    check_logits(st)
    l0 = Layer0("llama")
    for si, s in prompt_steps(r):
        l0.check(dump, si, s["pos"], s["n"])


def test_supports_op_boundary(cuda, tmp_path):
    """qwen2 with n_ff 3104: ffn_down is Q5_1 / Q8_0 with K % 64 != 0, which the tensor-core path does not take, and 100 columns are
    more than supports_op accepts for the per-column GEMV.  So exactly one node per layer is unsupported (llama.cpp's scheduler would
    move it to the CPU).  The stand-in has no scheduler and the plugin computes it anyway: the logits must still match."""
    import numpy as np
    dims = [3, 1024, 8, 2, 3104, 384, 128]
    r = run_script("qwen2", ["clear", prompt(100, 0)] + decodes(100, 4), dims=dims, dump=tmp_path / "d.npz")
    st = r["steps"][1:]
    assert st[0]["unsupported_nodes"] == r["n_layer"], st[0]["unsupported_nodes"]
    assert all(s["unsupported_nodes"] == 0 for s in st[1:])
    # decode: ffn_down runs 1:1, so gate / up must reach it through the graph's buffers; q|k|v, attention, wo, gate and up stay fused
    assert all(s["fused_steps"] >= 5 * r["n_layer"] for s in st[1:]), [s["fused_steps"] for s in st]
    check_logits(st)
    Layer0("qwen2", dims).check(np.load(tmp_path / "d.npz"), 1, 0, 100)


def test_decode_past_attention_cell_limit(cuda, lib):
    """n_ctx beyond the largest n_kv the fused attention launch takes: the planner fuses the attention chain up to that limit and
    leaves it to the single ops past it, so q / k / v then reach them through the graph's tensors.  After a clear the stand-in
    puts the token of position p in cell p, so decode steps at positions around the limit need no long prompt."""
    max_cells = lib.c.pb200_attn_ggml_max_cells()
    assert max_cells >= 4096, max_cells
    dims = [3, 1024, 8, 2, 2816, 384, max_cells + 96]
    r = run_script("llama", ["clear"] + decodes(max_cells - 2, 6), dims=dims)
    st = r["steps"][1:]
    assert [s["pos"] for s in st] == list(range(max_cells - 2, max_cells + 4))
    for s in st:
        assert s["unsupported_nodes"] == 0, s
    # n_kv = max_cells: the fused plan (the bar of test_whole_graph_matches_cpu_backend_and_is_fused); n_kv = max_cells + 32: the
    # attention chain and q / k / v one launch per node
    per_layer = [(s["launches"] - 4) / r["n_layer"] for s in st]
    assert max(per_layer[:2]) <= 6.0 and min(per_layer[2:]) > 6.0, per_layer
    check_logits(st)


REPLAY_SCRIPT = (["clear", prompt(16, 0)] * 3 + decodes(16, 12) + ["clear", prompt(40, 0)] + ["clear", prompt(16, 0)] * 3 + decodes(16, 12))


def test_replay_across_workspace_growth(cuda, tmp_path):
    """The captured CUDA graph of a 16-token prompt holds the tensor-core workspace by value.  A 40-token prompt in between grows that
    workspace (frees it and allocates a larger one); the next 16-token prompt comes back at the same addresses and must be
    recaptured, not replayed (the plugin's workspace generation is part of what a capture is bound to)."""
    import numpy as np
    r = run_script("llama", REPLAY_SCRIPT, reserve=64, dump=tmp_path / "g.npz")
    steps = [s for s in r["steps"] if "clear" not in s]
    # precondition: the compute buffer never moved, so topologies seen before really come back at the same addresses
    assert len({s["buffer_base"] for s in steps}) == 1, [s["buffer_base"] for s in steps]
    rep = [s["graph_replays"] for s in steps]
    p16 = [s["graph_replays"] for s in steps if s["n"] == 16]
    assert p16 == [0, 0, 1, 0, 0, 1], rep                          # direct, capture, replay -- in both sessions
    assert [s["graph_replays"] for s in steps if s["n"] == 40] == [0], rep
    dec = [s["graph_replays"] for s in steps if s["n"] == 1]
    assert dec == ([0, 0] + [1] * 10) * 2, rep                       # per bucket: direct, capture, then replays
    sessions, cur = [], []
    for s in r["steps"]:
        if "clear" in s:
            if cur:
                sessions.append(cur)
            cur = []
        else:
            cur.append(s)
    sessions.append(cur)
    for s in sessions:
        check_logits(s)
    g = np.load(tmp_path / "g.npz")
    l0 = Layer0("llama")
    for si, s in prompt_steps(r):
        l0.check(g, si, s["pos"], s["n"])
    # direct launches every step: the same arithmetic up to the order of the stream-K atomics, so every step agrees with the
    # graph run to the NMSE of test_prefill_chunked_equals_whole
    d = run_script("llama", REPLAY_SCRIPT, reserve=64, env={"GGML_B200_NO_GRAPHS": "1"}, dump=tmp_path / "d.npz")
    assert all(s.get("graph_replays", 0) == 0 for s in d["steps"])
    n = np.load(tmp_path / "d.npz")
    for si, s in enumerate(r["steps"]):
        if "clear" not in s:
            a, b = g[f"logits_b200_{si}"].astype(np.float64), n[f"logits_b200_{si}"].astype(np.float64)
            assert np.sum((a - b) ** 2) / np.sum(a ** 2) <= 1e-6, (si, s)


def test_plan_cache_eviction(cuda):
    """Prompts of T = 2 .. 18 after a clear each: 17 topologies, one more than the plugin keeps plans for.  T = 2 again (its plan was
    evicted and is rebuilt) and 4 decode steps after it must still agree with the CPU backend."""
    steps = []
    for T in range(2, 19):
        steps += ["clear", prompt(T, 0)]
    steps += ["clear", prompt(2, 0)] + decodes(2, 4)
    r = run_script("qwen2", steps, reserve=18)
    sessions, cur = [], []
    for s in r["steps"]:
        if "clear" in s:
            if cur:
                sessions.append(cur)
            cur = []
        else:
            cur.append(s)
    sessions.append(cur)
    assert len(sessions) == 18
    for s in sessions:
        check_logits(s)
