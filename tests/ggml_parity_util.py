"""Helpers of the whole-graph plugin tests (tests/test_gpu_ggml_graph.py, tests/test_gpu_ggml_layer_shapes.py): the script runner of
tests/ggml_graph_parity.py, the multi-token logits bar and the float64 bound on the layer-0 K / V rows a prompt writes.  The model of a
run is the driver's TinyModel, named by arch, dims, seed, ftype and freq factors; Layer0 rebuilds the same one."""
import json
import os
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
DRIVER = ROOT / "tests" / "ggml_graph_parity.py"


def default_dims(arch):
    """[n_layer, n_embd, n_head, n_head_kv, n_ff, n_vocab, n_ctx] of the driver's small model."""
    return [3, 1024, 8, 2, 2816 if arch == "llama" else 3072, 384, 96]


def default_ftype(arch):
    return "q4_K_M" if arch == "llama" else "q5_K_M"


def skip_unless_built():
    if not (ROOT / "host" / "_ggml" / "libllama_graph_host.so").exists() or not (ROOT / "prima.cpp_b200" / "libggml-b200.so").exists():
        pytest.skip("host/_ggml or the plugin is not built (build() builds them only where the reference source tree is readable)")


def run_script(arch, steps, dims=None, reserve=None, env=None, dump=None, seed=None, ftype=None, freq_factors=None, engine=False,
               timeout=1800):
    """Runs the driver's script mode in a process of its own and returns its JSON line.  seed / ftype / freq_factors default to the
    driver's (31, default_ftype(arch), llama only); engine: the same model also decoded by the engine (decode steps only)."""
    skip_unless_built()
    cmd = [sys.executable, str(DRIVER), arch, "--script", json.dumps(steps)]
    cmd += ["--dims", ",".join(str(d) for d in dims)] if dims else []
    cmd += ["--reserve", str(reserve)] if reserve else []
    cmd += ["--dump", str(dump)] if dump else []
    cmd += ["--seed", str(seed)] if seed is not None else []
    cmd += ["--ftype", ftype] if ftype else []
    cmd += ["--no-freq-factors"] if freq_factors is False else []
    cmd += ["--engine"] if engine else []
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=dict(os.environ, **(env or {})))
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-4000:]
    return json.loads(p.stdout.strip().splitlines()[-1])


def prompt(T, pos):
    return {"n": T, "pos": pos}


def decodes(pos, k):
    return [{"n": 1, "pos": pos + i} for i in range(k)]


def prompt_steps(r):
    return [(si, st) for si, st in enumerate(r["steps"]) if "clear" not in st and st["n"] > 1]


def sessions(r):
    """The run's steps split at every "clear"; empty sessions dropped."""
    out, cur = [], []
    for s in r["steps"]:
        if "clear" in s:
            if cur:
                out.append(cur)
            cur = []
        else:
            cur.append(s)
    if cur:
        out.append(cur)
    return out


def check_logits(rows, first_row_exact=True):
    """The multi-token bar of check_decode_parity / test_whole_graph_matches_cpu_backend_and_is_fused over a session's prompt rows
    and decode steps: once an activation code flips upstream (q = round(x*127/amax) of a 1-ulp fp32 difference), the deviation is
    the noise the reference's own SIMD builds show against each other, so NMSE < 2e-3, max-abs < 0.25, >= 90 % same argmax.
    first_row_exact=False for models whose token 0 already holds such a flip.  Returns (nmse, max-abs, argmax agreement, kv max-abs)
    for the caller to print."""
    sq_err = sum(r["sq_err"] for r in rows)
    sq_ref = sum(r["sq_ref"] for r in rows)
    agree = [a for r in rows for a in r["argmax_agree_per_row"]]
    worst = max(max(r["max_abs_per_row"]) for r in rows)
    assert sq_err / sq_ref < 2e-3 and worst < 0.25 and sum(agree) >= 0.9 * len(agree), (sq_err / sq_ref, worst, sum(agree), len(agree))
    for r in rows:
        assert r["kv_max_abs"] < 0.25, r   # f16 cache rows of magnitude ~20: a flipped activation code upstream moves them by a few 1e-2
        if first_row_exact and r["n"] > 1 and r["n"] < 8 and r["pos"] == 0:
            # T < 8 runs one integer-dot GEMV per column, like the CPU's vec_dot: the first row depends on token 0 alone and agrees
            # to fp32 summation order
            assert r["max_abs_per_row"][0] < 1e-4, r["max_abs_per_row"]
    return sq_err / sq_ref, worst, sum(agree) / len(agree), max(r["kv_max_abs"] for r in rows)


class Layer0:
    """Bars for the layer-0 K / V cache rows a prompt writes.  Their input is rms_norm(token_embd[tok]) * attn_norm on both backends,
    so no activation code can have flipped upstream; what is left is the mat-mul's own arithmetic, RoPE and the f16 store."""

    def __init__(self, arch, dims=None, seed=31, ftype=None, freq_factors=None):
        import numpy as np
        import oracle_lib as O
        from tiny_model import TinyModel
        n_layer, n_embd, n_head, n_head_kv, n_ff, n_vocab, n_ctx = dims or default_dims(arch)
        tm = TinyModel(n_layer=n_layer, n_embd=n_embd, n_head=n_head, n_head_kv=n_head_kv, n_ff=n_ff, n_vocab=n_vocab, n_ctx=n_ctx, arch=arch,
                       ftype=ftype or default_ftype(arch), freq_factors=(arch == "llama") if freq_factors is None else freq_factors, seed=seed,
                       branch_scale=0.1)
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
        same floor and the f16 store's ulp.  Returns the worst ratio of error to bar over K and V."""
        import numpy as np
        rows = slice(pos, pos + T)
        x, d_x = self.x[rows], self.d_x[rows]
        worst_all = 0.0
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
                worst_all = max(worst_all, worst)
            else:
                rows_over = int(over.any(axis=1).sum())
                assert rows_over <= 1, f"{nm} rows {pos}..{pos + T - 1}: {rows_over} rows beyond 1 f16 ulp + fp32 order (worst ratio {worst:.2f})"
                flips = float((err / (ulp + bound + kick)).max())
                assert flips <= 1.0, f"{nm}: deviation larger than two q8 code flips (worst {flips:.2f})"
                worst_all = max(worst_all, flips)
        return worst_all
