"""-m gpu: whole-graph parity through the drop-in boundary.  A build_llama / build_qwen2 decode graph (host/llama_graph_host.cpp,
the stand-in for libllama's builder) is computed by ggml_backend_graph_compute on the registered "B200_0" backend and on the
reference's CPU backend with identical weights and tokens; logits, last hidden state and the KV cache contents are compared, and
the launch counter proves that graph_compute ran the FUSED path (<= 6 kernels per layer instead of ~25 single ops)."""
import json
import subprocess
import sys
from pathlib import Path

import pytest

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


@pytest.mark.parametrize("arch", ["llama", "qwen2"])
def test_whole_graph_matches_cpu_backend_and_is_fused(cuda, arch):
    r = run(arch, 40)
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
