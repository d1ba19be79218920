#!/usr/bin/env python
"""bench.py — decode tokens/s of the quantized-decode hot path (BASELINE.json metric) on N H100s of one node.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--model llama3-70b] [--impl b200|reference]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P bench.py --gpus N ...

A step = one decoded token (b=1) through every layer + lm_head of the named model with synthetic random-init weights in
the Q4_K_M / Q5_K_M type mixture, positions continuing after a 128-token prompt (llama-bench tg protocol,
examples/llama-bench/llama-bench.cpp:1433-1470).  N>1 = prima's layer-window pipeline re-targeted to NVLink: contiguous
layer ranges per rank, hidden state handed off with one NCCL send/recv per stage boundary, strictly sequential tokens
(the sampled token returns to rank 0 before the next step starts) — so per-token latency, not pipelined throughput.

Prints ONE JSON line (rank 0).  `value`: device-resident steps (token id via kernel argument, logits stay in HBM);
`e2e`: measured THROUGH THE DROP-IN BOUNDARY at N=1 — host/llama_graph_host.cpp (the stand-in for libllama's build_llama) builds
the decode graph with the host's ggml and runs it on the registered "B200_0" ggml backend: token id, position and mask row from host
memory through ggml_backend_tensor_set, ggml_backend_graph_compute (graph-level fusion inside the plugin), logits back through
ggml_backend_tensor_get, every step.  `e2e_engine` is the same step through the engine's own C call pb200_decode (what N>1 uses).
At N=1 the line also carries `prefill`: one --pp (512) token prompt batch through pb200_prefill (tensor-core mat-muls) with its
own tensor-pipe roofline — extra information next to the headline metric, measured after it, never part of `value`.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

MODELS = {
    "llama3-70b": dict(hp=dict(n_layer=80, n_embd=8192, n_head=64, n_head_kv=8, head_dim=128, n_ff=28672, n_vocab=128256, rope_mode=0,
                               n_ctx_orig=8192, rope_freq_base=500000.0, rope_freq_scale=1.0, rms_eps=1e-5), ftype=0, name="Llama-3-70B Q4_K_M"),
    "llama3-8b": dict(hp=dict(n_layer=32, n_embd=4096, n_head=32, n_head_kv=8, head_dim=128, n_ff=14336, n_vocab=128256, rope_mode=0,
                              n_ctx_orig=8192, rope_freq_base=500000.0, rope_freq_scale=1.0, rms_eps=1e-5), ftype=0, name="Llama-3-8B Q4_K_M"),
    "qwen2.5-72b": dict(hp=dict(n_layer=80, n_embd=8192, n_head=64, n_head_kv=8, head_dim=128, n_ff=29568, n_vocab=152064, rope_mode=2,
                                n_ctx_orig=32768, rope_freq_base=1000000.0, rope_freq_scale=1.0, rms_eps=1e-6), ftype=1, name="Qwen2.5-72B Q5_K_M"),
}
PROMPT = 128
METRIC = "decode tokens/sec Llama-3-70B Q4_K_M b=1 @1/2/4/8 H100; % HBM roofline"


def peaks():
    p = ROOT / "MEASURED_PEAKS.json"
    if p.exists():
        d = json.loads(p.read_text())
        return float(d["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs, STREAM-style copy)"
    return 3350.0, "H100 SXM data sheet (3.35 TB/s HBM3)"


def tensor_peak():
    p = ROOT / "MEASURED_PEAKS.json"
    if p.exists():
        d = json.loads(p.read_text())
        if "bf16_tflops" in d:
            return float(d["bf16_tflops"]), "measured (MEASURED_PEAKS.json bf16_tflops: cuBLAS bf16 8192^3 burst; the prefill batch is timed alone)"
    return 989.0, "H100 SXM data sheet (989 TFLOP/s dense fp16 at 700 W)"


def prefill_flops(hp, T):
    """Algorithmic FLOPs of one prompt batch (SURVEY 8d): 2 * sum(N*K) * T over the per-layer mat-muls, causal attention
    4 * T^2/2 * n_embd per layer, lm_head for the last token only."""
    E, F, D = hp["n_embd"], hp["n_ff"], 128
    QD, EK = hp["n_head"] * D, hp["n_head_kv"] * D
    p_mm = E * QD + 2 * E * EK + QD * E + 3 * E * F
    mm = 2.0 * p_mm * T * hp["n_layer"]
    att = 4.0 * (T * (T + 1) / 2) * QD * hp["n_layer"]
    return mm, att, 2.0 * E * hp["n_vocab"]


class ClockSampler:
    """nvidia-smi clocks / throttle reasons DURING the timed region."""
    Q = "clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown," \
        "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, index):
        self.rows, self.proc, self.index = [], None, index

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "100", "-i", str(self.index)],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except OSError:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def stop(self):
        if self.proc:
            self.proc.terminate()
        sm = sorted(int(float(r[0])) for r in self.rows if r and r[0].replace(".", "").isdigit())
        reasons = set()
        for r in self.rows:
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), r[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        mx = [int(float(r[1])) for r in self.rows if len(r) > 1 and r[1].replace(".", "").isdigit()]
        pw = [float(r[2]) for r in self.rows if len(r) > 2 and r[2].replace(".", "").isdigit()]
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None, "power_w_max": max(pw) if pw else None,
                "samples": len(sm), "reasons": sorted(reasons)}


def usable_cpus():
    """Threads the CPU arm may use: the affinity mask, capped by the cgroup CPU quota (a container often sees 128 CPUs but owns
    far fewer; ggml's spinning barriers collapse under oversubscription)."""
    try:
        n = len(os.sched_getaffinity(0))
    except AttributeError:
        n = os.cpu_count() or 1
    try:
        q, per = open("/sys/fs/cgroup/cpu.max").read().split()
        if q != "max":
            n = max(1, min(n, int(float(q) / float(per))))
    except (OSError, ValueError):
        pass
    return n


def token_at(i, n_vocab):
    return (i * 7919 + 13) % n_vocab


# ------------------------------------------------------------------------------------------------ CPU reference arm
def cpu_reference(model_key, steps, warmup, sample_layers=2):
    """Times the reference's own CPU ggml path (oracle/_ref, compiled unmodified from the reference) on a bounded sample
    of the workload: `sample_layers` full-size layers + the lm_head, extrapolated to the full layer count."""
    import numpy as np
    import oracle_lib as O
    from tiny_model import TinyModel
    cfg = MODELS[model_key]
    hp = dict(cfg["hp"])
    L = hp["n_layer"]
    kind = "reference" if O.have_ref() else "port"
    threads = usable_cpus()
    tm = TinyModel(n_layer=sample_layers, n_embd=hp["n_embd"], n_head=hp["n_head"], n_head_kv=hp["n_head_kv"], n_ff=hp["n_ff"], n_vocab=hp["n_vocab"],
                   n_ctx=PROMPT + 64, arch="llama" if hp["rope_mode"] == 0 else "qwen2", ftype="q4_K_M" if cfg["ftype"] == 0 else "q5_K_M", seed=1)
    # the sample's layers must carry the FULL model's average bytes: take one "normal" and one "more-bits" layer
    tm.hp.update({k: hp[k] for k in ("rope_freq_base", "rms_eps", "n_ctx_orig")})
    m = tm.oracle_struct()
    nv, E = hp["n_vocab"], hp["n_embd"]
    logits = np.zeros(nv, dtype=np.float32)
    if kind == "reference":
        ref = O.Ref(threads)
        # pick the thread count that is actually fastest on this host (bounded: a few lm_head mat-vecs per candidate)
        t_w, a_w = tm.tensors["output.weight"]
        xw = np.ones(E, dtype=np.float32)
        best = None
        for cand in sorted({c for c in (4, 8, 16, 32, 64, 128, threads) if c <= threads}):
            ref.mul_mat(t_w, a_w, nv, E, xw, n_threads=cand)
            t0 = time.perf_counter()
            ref.mul_mat(t_w, a_w, nv, E, xw, n_threads=cand)
            dt = time.perf_counter() - t0
            if best is None or dt < best[0]:
                best = (dt, cand)
        threads = best[1]
        h = ref.graph.gref_create(C.byref(m), threads)

        def one(i):
            tok = np.array([token_at(i, nv)], dtype=np.int32)
            rc = ref.graph.gref_decode(h, tok.ctypes.data_as(C.c_void_p), 1, PROMPT + (i % 32), logits.ctypes.data_as(C.c_void_p), None, 1 << 30)
            assert rc == 0

        def head_only():
            t, a = tm.tensors["output.weight"]
            x = np.ones(E, dtype=np.float32)
            t0 = time.perf_counter()
            ref.mul_mat(t, a, nv, E, x, n_threads=threads)
            return time.perf_counter() - t0
    else:
        port = O.Port()
        threads = 1

        def one(i):
            port.lib.port_llama_decode(C.byref(m), token_at(i, nv), PROMPT + (i % 32), logits.ctypes.data_as(C.c_void_p), None)

        def head_only():
            t, a = tm.tensors["output.weight"]
            x = np.ones(E, dtype=np.float32)
            t0 = time.perf_counter()
            port.mul_mat(t, a, nv, E, x)
            return time.perf_counter() - t0
    for i in range(warmup):
        one(i)
    t0 = time.perf_counter()
    for i in range(steps):
        one(warmup + i)
    t_sample = (time.perf_counter() - t0) / steps
    t_head = min(head_only() for _ in range(3))
    t_layer = max(t_sample - t_head, 1e-9) / sample_layers
    t_full = t_head + L * t_layer
    return {"value": 1.0 / t_full, "unit": "tokens/s", "cores": threads, "kind": kind,
            "sample": f"{steps} decode steps of {sample_layers} full-size layers + lm_head of {cfg['name']} (synthetic blocks) on the reference CPU "
                      f"ggml backend ({O.ref_variant() if kind == 'reference' else 'C port'}, OpenMP, GGML_USE_LLAMAFILE off), "
                      + (f"extrapolated to {L} layers: " if sample_layers != L else "the whole model, nothing extrapolated: ")
                      + f"t_layer={t_layer * 1e3:.2f} ms, t_head={t_head * 1e3:.2f} ms",
            "ms_per_step_sample": t_sample * 1e3, "ms_per_token_extrapolated": t_full * 1e3}


def cpu_reference_subprocess(model_key, steps, warmup):
    """The CPU leg runs in a process of its own: it loads the oracle's copy of the reference ggml, which must not share a process
    with the host ggml that bench.py's boundary leg loads (two ggml cores interpose each other's symbols)."""
    p = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--impl", "reference", "--model", model_key, "--steps", str(steps), "--warmup", str(warmup)],
                       capture_output=True, text=True, timeout=1500)
    for line in reversed(p.stdout.strip().splitlines()):
        if line.startswith("{"):
            return json.loads(line)["cpu_baseline"]
    raise RuntimeError(f"reference arm failed: {p.stderr[-500:]}")


def boundary_leg(eng, cfg, hp, args, lib):
    """e2e through the ggml-backend boundary (N=1): the model moves into the plugin's backend buffers (the engine's synthetic weights,
    staged in host memory because two resident copies of a 70B model do not fit one 80-GB GPU; the engine is released), the host's ggml
    builds the decode graph and the plugin computes it."""
    import numpy as np
    import torch
    sys.path.insert(0, str(ROOT / "host"))
    import host_graph as HG
    L = hp["n_layer"]
    names = ["token_embd.weight", "output.weight", "output_norm.weight"]
    for il in range(L):
        names += [f"blk.{il}.{w}.weight" for w in ("attn_norm", "ffn_norm") + HG.WEIGHT_ORDER]
        if hp["rope_mode"] == 2:
            names += [f"blk.{il}.attn_{x}.bias" for x in "qkv"]
    info = {n: eng.tensor_device(n) for n in names}
    types = {n: t for n, (p, b, t) in info.items() if n.endswith(".weight") and t not in (0,)}
    class U8:   # __cuda_array_interface__ view of raw device memory: torch only moves bytes here
        def __init__(self, ptr, n):
            self.__cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (ptr, False), "version": 2}

    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    nv = hp["n_vocab"]
    # the engine's logits for a token at position 0 of an empty cache, compared below with the plugin's on the same weights
    eng_logits = np.zeros(nv, dtype=np.float32)
    eng.kv_clear()
    eng.decode(token_at(1, nv), 0, eng_logits)
    need = sum(nbytes for (_, nbytes, _) in info.values())
    free = os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
    if need * 1.1 > free:
        raise RuntimeError(f"boundary leg: {need / 1e9:.1f} GB of weights to stage in host memory, {free / 1e9:.1f} GB free")
    staged = {n: torch.as_tensor(U8(ptr, nbytes), device=dev).cpu() for n, (ptr, nbytes, t) in info.items()}
    eng.close()
    hm = HG.HostModel(hp, types, "B200_0", has_bias=(hp["rope_mode"] == 2), has_freq_factors=False)
    for n, h in staged.items():
        dst, dbytes = hm.tensor_ptr(n)
        assert dbytes == h.numel(), (n, dbytes, h.numel())
        torch.as_tensor(U8(dst, dbytes), device=dev).copy_(h)
    del staged
    torch.cuda.synchronize()
    logits = np.zeros(nv, dtype=np.float32)
    first = PROMPT + args.warmup
    # same protocol as the engine arm: prompt tokens fill the cache (untimed), warm-up, then K timed steps; host wall clock, since
    # every step ends with a synchronous logits read
    for i in range(PROMPT + args.warmup):
        hm.decode([token_at(i, nv)], i, logits if i >= PROMPT else None)
    n0 = lib.c.pb200_kernel_launches()
    sampler = ClockSampler(int(os.environ.get("LOCAL_RANK", "0")))
    sampler.start()
    torch.cuda.synchronize()
    hm.phase_seconds()
    t0 = time.perf_counter()
    for i in range(args.steps):
        hm.decode([token_at(first + i, nv)], first + i, logits)
    dt = time.perf_counter() - t0
    phases = {k: v / args.steps * 1e3 for k, v in hm.phase_seconds().items()}
    clocks = sampler.stop()
    launches = lib.c.pb200_kernel_launches() - n0
    # the two paths on the same weights: a token at position 0 of an empty cache through each (later steps sit on different histories
    # of a random-init, unit-gain 80-layer net and are not comparable; the whole-graph parity test lives in tests/test_gpu_ggml_graph.py)
    hm.kv_clear()
    hm.decode([token_at(1, nv)], 0, logits)
    n_kv_pad = (first + args.steps + 32) // 32 * 32
    res = {"value": args.steps / dt, "unit": "tokens/s", "ms_per_step": dt / args.steps * 1e3,
           "h2d_bytes_per_step": 8 + n_kv_pad * 32 * 4, "d2h_bytes_per_step": nv * 4,
           "api": "ggml_backend_tensor_set(inp_tokens, inp_pos, KQ_mask) + ggml_backend_graph_compute(B200_0) + ggml_backend_tensor_get(logits) "
                  "on the graph of host/llama_graph_host.cpp (build_llama restated; the host's ggml = the reference's, unmodified)",
           "timing": "host wall clock around K synchronous steps", "gpu_launches": int(launches), "launches_per_layer": (launches / args.steps - 3) / L,
           "graph_nodes": hm.graph_nodes, "graph_builds": int(hm.graph_builds), "cuda_graph_replays": int(hm.plug.ggml_backend_b200_graph_replays()),
           "host_ms_per_step": phases, "clocks": clocks,
           "max_abs_vs_engine_first_token": float(np.max(np.abs(eng_logits - logits)))}
    hm.close()
    return res


# ------------------------------------------------------------------------------------------------ same-box GPU comparator
def ggml_cuda_arm(args, cfg, hp, config):
    """--impl ggml-cuda: the reference's OWN ggml-cuda backend (unmodified, built for sm_90a by oracle/Makefile.cudaref — BASELINE.md §3
    "the existing kernel to beat") on the same box, same synthetic weights, same host graph (host/llama_graph_host.cpp), same protocol
    as the B200 arm's e2e leg: host token / position / mask in, logits out, every step.  Measurement infrastructure: none of the
    product's kernels run inside the timed region (the engine is used before it, to synthesise the weights, and is then freed)."""
    import numpy as np
    import torch
    import pkgload
    sys.path.insert(0, str(ROOT / "host"))
    import host_graph as HG
    pkg = pkgload.load()
    lib = pkg.Lib.get()
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    L, nv, E = hp["n_layer"], hp["n_vocab"], hp["n_embd"]
    eng = pkg.Model(pkg.HParams(**hp), 0, (0, L), with_embd=True, with_head=True)
    eng.synth(cfg["ftype"], 1234)
    eng.finalize()
    names = ["token_embd.weight", "output.weight", "output_norm.weight"]
    for il in range(L):
        names += [f"blk.{il}.{w}.weight" for w in ("attn_norm", "ffn_norm") + HG.WEIGHT_ORDER]
        if hp["rope_mode"] == 2:
            names += [f"blk.{il}.attn_{x}.bias" for x in "qkv"]
    info = {n: eng.tensor_device(n) for n in names}
    types = {n: t for n, (p_, b_, t) in info.items() if n.endswith(".weight") and t not in (0,)}
    # ggml-cuda has no k-quant GET_ROWS (ggml-cuda.cu:3033-3047; llama.cpp gathers the embedding row on the CPU): the table is handed
    # over dequantized to f32 — same values, and the gather is not part of what is compared
    emb_ptr, emb_bytes, emb_type = info["token_embd.weight"]
    types["token_embd.weight"] = 0

    class U8:
        def __init__(self, ptr, n):
            self.__cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (ptr, False), "version": 2}

    eng_logits = np.zeros(nv, dtype=np.float32)
    eng.kv_clear()
    eng.decode(token_at(1, nv), 0, eng_logits)
    wbytes = eng.weight_bytes
    # two resident copies of a 70B model do not fit one 80-GB GPU: the weights are staged in host memory and the engine is freed
    # before the ggml-cuda buffers are allocated
    need = sum(nbytes for (_, nbytes, _) in info.values()) + nv * E * 4
    free = os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
    if need * 1.1 > free:
        raise RuntimeError(f"ggml-cuda arm: {need / 1e9:.1f} GB of weights to stage in host memory, {free / 1e9:.1f} GB free")
    staged = {}
    for n, (ptr, nbytes, t) in info.items():
        if n == "token_embd.weight":
            emb = torch.empty(nv * E, dtype=torch.float32)
            ids = torch.arange(nv, dtype=torch.int32, device=dev)
            step_rows = 8192
            rows = torch.empty(step_rows * E, dtype=torch.float32, device=dev)
            for r0 in range(0, nv, step_rows):
                nr = min(step_rows, nv - r0)
                lib.check(lib.c.pb200_get_rows(emb_type, C.c_void_p(emb_ptr), C.c_int64(E), C.c_void_p(ids.data_ptr() + 4 * r0), C.c_int64(nr),
                                               C.c_void_p(rows.data_ptr()), None), "get_rows")
                torch.cuda.synchronize()
                emb[r0 * E:(r0 + nr) * E].copy_(rows[:nr * E])
            staged[n] = emb.view(torch.uint8)
            del rows
            continue
        staged[n] = torch.as_tensor(U8(ptr, nbytes), device=dev).cpu()
    eng.close()
    del eng
    torch.cuda.empty_cache()
    hm = HG.HostModel(hp, types, "CUDA0", has_bias=(hp["rope_mode"] == 2), has_freq_factors=False)
    for n, h in staged.items():
        dst, dbytes = hm.tensor_ptr(n)
        assert dbytes == h.numel(), (n, dbytes, h.numel())
        torch.as_tensor(U8(dst, dbytes), device=dev).copy_(h)
    del staged
    torch.cuda.synchronize()
    logits = np.zeros(nv, dtype=np.float32)
    hm.decode([token_at(1, nv)], 0, logits)
    nmse = float(np.sum((logits - eng_logits) ** 2) / max(np.sum(eng_logits ** 2), 1e-30))
    hm.kv_clear()
    first = PROMPT + args.warmup
    for i in range(first):
        hm.decode([token_at(i, nv)], i, logits if i >= PROMPT else None)
    sampler = ClockSampler(0)
    sampler.start()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(args.steps):
        hm.decode([token_at(first + i, nv)], first + i, logits)
    dt = time.perf_counter() - t0
    clocks = sampler.stop()
    hbm, src = peaks()
    n_kv_pad = (first + args.steps + 32) // 32 * 32
    v = args.steps / dt
    line = {"impl": "ggml-cuda", "metric": METRIC, "value": v, "unit": "tokens/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": dt / args.steps * 1e3, "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
            "dtype": "q8_1 activations x k-quant weights (mul_mat_vec_q), f32 accumulate", "data": "synthetic", "config": config,
            "what": "the reference's unmodified ggml-cuda backend compiled for sm_90a (oracle/Makefile.cudaref), CUDA graphs on, same box, same weights, "
                    "same host graph and host I/O as the B200 arm's e2e leg",
            "e2e": {"value": v, "unit": "tokens/s", "h2d_bytes_per_step": 8 + n_kv_pad * 32 * 4, "d2h_bytes_per_step": nv * 4},
            "roofline": {"bound": "hbm", "achieved": wbytes * v / 1e9, "peak": hbm, "unit": "GB/s", "frac": wbytes * v / 1e9 / hbm, "peak_source": src,
                         "how": "whole step: algorithmic weight bytes per token x tokens/s"},
            "logits_nmse_vs_b200_engine_first_token": nmse, "clocks": clocks, "graph_nodes": hm.graph_nodes}
    hm.close()
    print(json.dumps(line))


def ggml_cuda_subprocess(model_key, steps, warmup, n_ctx):
    p = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--impl", "ggml-cuda", "--model", model_key, "--steps", str(steps), "--warmup", str(warmup),
                        "--n-ctx", str(n_ctx)], capture_output=True, text=True, timeout=900)
    for line in reversed(p.stdout.strip().splitlines()):
        if line.startswith("{"):
            d = json.loads(line)
            return {k: d[k] for k in ("value", "unit", "ms_per_step", "what", "roofline", "logits_nmse_vs_b200_engine_first_token", "clocks")}
    return {"unavailable": (p.stderr or p.stdout)[-300:]}


# ------------------------------------------------------------------------------------------------ main
def main():
    global PROMPT
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--model", default="llama3-70b", choices=sorted(MODELS))
    ap.add_argument("--impl", default="b200", choices=["b200", "reference", "ggml-cuda"])
    ap.add_argument("--no-gpu-comparator", action="store_true", help="skip the same-box ggml-cuda comparator leg (N=1 only)")
    ap.add_argument("--n-ctx", type=int, default=512)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-boundary", action="store_true", help="skip the e2e leg through the ggml-backend plugin (keeps pb200_decode as e2e)")
    ap.add_argument("--prompt", type=int, default=PROMPT, help="untimed prompt tokens decoded before the timed region")
    ap.add_argument("--pp", type=int, default=None, help="prompt tokens of the prompt-processing measurement that follows the decode run (0 = skip).  "
                    "N = 1: one pb200_prefill call, default 512 (llama-bench pp512).  N > 1: only when given — the prompt goes through the layer "
                    "pipeline in 512-token micro-batches (pb200_prefill_stage, NCCL hand-off of the hidden states), e.g. config C5: "
                    "--model qwen2.5-72b --gpus 8 --pp 2048 --n-ctx 4096")
    ap.add_argument("--ncu", action="store_true", help="bracket the timed region with cudaProfilerStart/Stop (ncu --profile-from-start off)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write what the timed decode path returned in its last step (logits; at N > 1 also the greedy token) as "
                         "DIR/<name>.npy, so that two builds can be compared output for output (the inputs are seeded)")
    args = ap.parse_args()
    PROMPT = args.prompt
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if args.pp is None:
        args.pp = 512 if world == 1 else 0
    local = int(os.environ.get("LOCAL_RANK", "0"))
    cfg = MODELS[args.model]
    hp = dict(cfg["hp"], n_ctx=args.n_ctx)
    config = {"workload": f"{cfg['name']} decode b=1, synthetic random-init weights, {args.prompt}-token prompt then tg steps, n_ctx {args.n_ctx}, KV f16, FA off",
              "parallelism": "single GPU" if world == 1 else f"layer pipeline pp{world} (NCCL send/recv hand-off)",
              "l2": "no explicit flush: every step streams the shard's weights (>> 50 MB L2) once"}

    if args.impl == "reference":
        if rank != 0:
            return
        steps, warm = min(args.steps, 256), min(args.warmup, 64)   # the same K / W as the B200 arm (each step = the bounded sample below)
        # Llama-3-8B (config C1) fits the bounded budget whole: every layer is timed, nothing is extrapolated
        cb = cpu_reference(args.model, steps, warm, sample_layers=(MODELS[args.model]["hp"]["n_layer"] if args.model == "llama3-8b" else 2))
        print(json.dumps({"impl": "reference", "metric": METRIC, "value": cb["value"], "unit": "tokens/s", "n_gpus": args.gpus, "steps": steps,
                          "warmup": warm, "ms_per_step": cb["ms_per_token_extrapolated"], "higher_is_better": True, "scaling": "strong",
                          "vs_baseline": None, "dtype": "int8 x k-quant dot, f32 accumulate", "data": "synthetic", "config": config,
                          "cpu_baseline": cb, "e2e": {"value": cb["value"], "unit": "tokens/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}))
        return

    if args.impl == "ggml-cuda":
        if rank == 0:
            ggml_cuda_arm(args, cfg, hp, config)
        return

    import numpy as np
    import torch
    import pkgload
    pkg = pkgload.load()
    lib = pkg.Lib.get()
    torch.cuda.set_device(local)
    dist = None
    if world > 1:
        import torch.distributed as dist
        import datetime
        # a rank that fails must take the job down in minutes, not in NCCL's default 10-minute watchdog period
        dist.init_process_group("nccl", device_id=torch.device("cuda", local), timeout=datetime.timedelta(seconds=180))
    assert args.steps + args.warmup + PROMPT <= args.n_ctx, "n_ctx too small for prompt + warmup + steps"

    L = hp["n_layer"]
    # uniform contiguous layer windows (prima: n_layer_window; 8 identical GPUs need no ILP scheduler)
    bounds = [round(r * L / world) for r in range(world + 1)]
    l0, l1 = bounds[rank], bounds[rank + 1]
    H = pkg.HParams(**hp)
    t0 = time.perf_counter()
    eng = pkg.Model(H, local, (l0, l1), with_embd=(rank == 0), with_head=(rank == world - 1))
    eng.synth(cfg["ftype"], 1234 + rank)
    if world > 1:
        eng.set_n_seq(world)          # one sequence slot per stage: the ring keeps every GPU busy (RingRunner)
    eng.finalize()
    t_load = time.perf_counter() - t0
    nv, E = hp["n_vocab"], hp["n_embd"]
    ext = torch.cuda.ExternalStream(eng.stream, device=torch.device("cuda", local))

    class DevBuf:   # __cuda_array_interface__ view of an engine buffer so torch.distributed can send/recv it in place
        def __init__(self, ptr, n):
            self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (ptr, False), "version": 2}

    hid_in = hid_out = None
    if world > 1:
        hid_in = torch.as_tensor(DevBuf(eng.hidden_in_ptr, E), device=torch.device("cuda", local))
        hid_out = torch.as_tensor(DevBuf(eng.hidden_out_ptr, E), device=torch.device("cuda", local))
    class DevI32:
        def __init__(self, ptr, n):
            self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i4", "data": (ptr, False), "version": 2}

    cuda_dev = torch.device("cuda", local)
    # latency mode (one sequence, slot 0): the last stage's device argmax lands in sample slot 0, stage 0 receives it into a scratch word
    tok_t = torch.as_tensor(DevI32(eng.sample_ptr(0), 1), device=cuda_dev) if rank == world - 1 else torch.zeros(1, dtype=torch.int32, device=cuda_dev)
    logits_t = torch.as_tensor(DevBuf(eng.logits_ptr, nv), device=torch.device("cuda", local)) if rank == world - 1 else None
    logits_host = np.zeros(nv, dtype=np.float32)

    class EngineStage:
        """adapter: the engine's device buffers as torch tensors for prima.cpp_b200.pipeline.PipelineRunner"""
        hidden_in, hidden_out, logits = hid_in, hid_out, logits_t
        host_io = False

        def decode_async(self, token, pos):
            if self.host_io and rank == world - 1:
                eng.decode(token, pos, logits_host)       # token+pos H2D from pinned memory, logits D2H, synchronised
            elif self.host_io and world == 1:
                eng.decode(token, pos, logits_host)
            else:
                eng.decode_async(token, pos)

    stage = EngineStage()
    runner = pkg.PipelineRunner(stage, rank, world, dist, tok_t, stream=ext if world > 1 else None)

    def sample_dev(_logits):
        eng.argmax_seq(0, False)      # device argmax (pb200_argmax_seq): no torch kernel, no host sync on the step path
        return tok_t

    def step(i, pos, host_io):
        """One token through the pipeline.  Synthetic token ids (llama-bench tg uses random ids, llama-bench.cpp:1452-1470);
        in pipeline mode the last stage still returns a sampled token (argmax) to rank 0 so that steps stay strictly
        sequential like real decoding."""
        stage.host_io = host_io
        with torch.cuda.stream(ext):
            runner.step(token_at(i, nv), pos, sample=sample_dev)

    def barrier():
        torch.cuda.synchronize()
        if dist is not None:
            dist.barrier()
        torch.cuda.synchronize()

    # prompt (untimed): fills the KV cache so the timed steps attend over a realistic window
    for i in range(PROMPT):
        step(i, i, False)
    for i in range(args.warmup):
        step(PROMPT + i, PROMPT + i, False)
    barrier()

    def timed(host_io, first):
        sampler = ClockSampler(local)
        sampler.start()
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n0 = lib.c.pb200_kernel_launches()
        with torch.cuda.stream(ext):
            e0.record()
        for i in range(args.steps):
            step(first + i, first + i, host_io)
        with torch.cuda.stream(ext):
            e1.record()
        barrier()
        ms = e0.elapsed_time(e1)
        launches = lib.c.pb200_kernel_launches() - n0
        clocks = sampler.stop()
        if dist is not None:
            t = torch.tensor([ms], device=torch.device("cuda", local))
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            ms = float(t.item())
            lt = torch.tensor([launches], device=torch.device("cuda", local))
            dist.all_reduce(lt)
            launches = int(lt.item())
        return ms, launches, clocks

    first = PROMPT + args.warmup
    if args.ncu:
        torch.cuda.profiler.start()
    ms_dev, launches, clocks = timed(False, first)
    if args.ncu:
        torch.cuda.profiler.stop()

    def dump_output(name, arr):
        d = Path(args.dump_outputs)
        d.mkdir(parents=True, exist_ok=True)
        np.save(d / f"{name}.npy", arr)

    if args.dump_outputs and rank == world - 1:
        # the last timed step's results as a caller of the decode path receives them: n_vocab logits, and at N > 1 the device argmax
        # that travels back to rank 0 (at N = 1 the timed path does not sample)
        dump_output("decode_logits", logits_t.cpu().numpy().astype(np.float32))
        if world > 1:
            dump_output("decode_token", tok_t.cpu().numpy().astype(np.float64))
    eng.kv_clear() if False else None
    ms_e2e, _, clocks_e2e = timed(True, first)     # same positions again: the KV rows are simply rewritten
    # pipeline only: every rank times the same number of steps of its OWN stage with no communication; the difference between
    # the pipelined step and the sum of the stage times is the exposed hand-off (NVLink + NCCL launch + token return) time
    stage_ms = None
    if world > 1:
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(ext):
            e0.record()
            for i in range(args.steps):
                eng.decode_async(token_at(first + i, nv), first + i)
            e1.record()
        barrier()
        t = torch.tensor([e0.elapsed_time(e1) / args.steps], device=torch.device("cuda", local), dtype=torch.float64)
        dist.all_reduce(t)
        stage_ms = float(t.item())
    # ring mode (N > 1): one independent sequence per stage in flight, every GPU busy in every slot; aggregate tokens/s
    ring = None
    if world > 1:
        class RingStage:
            hidden_in, hidden_out = hid_in, hid_out
            _tin = [torch.as_tensor(DevI32(eng.token_ptr(s), 1), device=cuda_dev) for s in range(world)]
            _tout = [torch.as_tensor(DevI32(eng.sample_ptr(s), 1), device=cuda_dev) for s in range(world)]

            def token_in(self, s):
                return self._tin[s]

            def token_out(self, s):
                return self._tout[s]

            def begin(self, s, token, pos):
                eng.set_tokpos_seq(s, token, pos)

            def run(self, s):
                eng.step_seq_dev(s, True)
                if rank == world - 1:
                    eng.argmax_seq(s, False)

        rr = pkg.RingRunner(RingStage(), rank, world, dist, stream=ext)
        seeds = [(token_at(1000 + s, nv), PROMPT) for s in range(world)]
        barrier()
        with torch.cuda.stream(ext):
            rr.slots(world * (1 + args.warmup), first_tokens=seeds)          # fill the pipeline + warm-up rounds
        sampler = ClockSampler(local)
        sampler.start()
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n0 = lib.c.pb200_kernel_launches()
        with torch.cuda.stream(ext):
            e0.record()
            rr.slots(world * args.steps)                                      # K rounds: every sequence advances K tokens
            e1.record()
        barrier()
        ring_ms = e0.elapsed_time(e1)
        ring_launches = lib.c.pb200_kernel_launches() - n0
        ring_clocks = sampler.stop()
        t = torch.tensor([ring_ms], device=cuda_dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        lt = torch.tensor([ring_launches], device=cuda_dev)
        dist.all_reduce(lt)
        ring = {"ms": float(t.item()), "launches": int(lt.item()), "clocks": ring_clocks, "tokens": world * args.steps}
    # live roofline of the dominant kernel (k_gemv_kquant): CUDA events around every GEMV launch of profiled steps
    prof = [eng.profile_step(token_at(first + i, nv), first + i) for i in range(4)]
    gemv_ms = sum(p["gemv_ms"] for p in prof) / len(prof)
    gemv_bytes = prof[0]["gemv_bytes"]
    gemv_launches = prof[0]["gemv_launches"]
    wb = eng.weight_bytes
    if dist is not None:
        t = torch.tensor([float(wb), gemv_ms, float(gemv_bytes), float(gemv_launches)], device=torch.device("cuda", local), dtype=torch.float64)
        dist.all_reduce(t)
        wb, gemv_ms, gemv_bytes, gemv_launches = int(t[0].item()), float(t[1].item()), int(t[2].item()), int(t[3].item())
    pp_result = None
    if world > 1 and args.pp > 0 and args.pp <= args.n_ctx:
        # Prompt processing through the layer pipeline (prima's windows during prefill): 512-token micro-batches, every stage works on a
        # different micro-batch once the pipeline is full; hidden states [512][n_embd] f32 travel stage to stage by NCCL send/recv on the
        # engine stream.  Timed on the device (events on the engine stream), max over ranks, best of 3 after a warm-up pass.
        UB = 512
        nub = (args.pp + UB - 1) // UB
        hbuf = torch.empty((UB, E), dtype=torch.float32, device=cuda_dev)
        toks_all = np.array([token_at(i, nv) for i in range(args.pp)], dtype=np.int32)

        class PrefillStage:   # adapter: pb200_prefill_stage behind the interface prima.cpp_b200.pipeline.PrefillPipeline drives
            hidden_buf = hbuf

            def prefill_stage(self, tokens, hidden_in, n, pos):
                hp_out = eng.prefill_stage(tokens, hidden_in.data_ptr() if hidden_in is not None else None, n, pos)
                return torch.as_tensor(DevBuf(hp_out, n * E), device=cuda_dev).view(n, E)

        pipe = pkg.PrefillPipeline(PrefillStage(), rank, world, dist, ubatch=UB, stream=ext)

        def pp_pass():
            pipe.run(toks_all, args.pp, 0)

        def all_ok(err):
            """Every rank learns whether any rank failed, so that no rank walks into a barrier alone."""
            if err is not None:
                print(f"[rank {rank}] pipelined prefill failed: {err}", file=sys.stderr, flush=True)
            f = torch.tensor([0 if err is None else 1], device=cuda_dev)
            dist.all_reduce(f, op=dist.ReduceOp.MAX)
            return int(f.item()) == 0

        def guarded_pass():
            try:
                pp_pass()
                torch.cuda.synchronize()
                return None
            except Exception as ex:
                return repr(ex)

        best, ok = None, True
        try:
            eng.kv_clear()
            ok = all_ok(guarded_pass())
            for _ in range(3 if ok else 0):
                barrier()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                with torch.cuda.stream(ext):
                    e0.record()
                err = guarded_pass()
                with torch.cuda.stream(ext):
                    e1.record()
                if not all_ok(err):
                    ok = False
                    break
                barrier()
                t = torch.tensor([e0.elapsed_time(e1)], device=cuda_dev)
                dist.all_reduce(t, op=dist.ReduceOp.MAX)
                best = float(t.item()) if best is None else min(best, float(t.item()))
            if not ok or best is None:
                raise RuntimeError("a rank failed (see stderr)")
            mm, att, head = prefill_flops(hp, args.pp)
            tpeak, tsrc = tensor_peak()
            pp_result = {"metric": f"prompt tokens/s, {cfg['name']}, {args.pp} tokens in {nub} micro-batches of {UB} through the {world}-stage layer pipeline",
                              "tokens": args.pp, "ms": best, "value": args.pp / (best * 1e-3), "unit": "tokens/s",
                              "timing": "CUDA events on the engine stream around the whole prompt, max over ranks, best of 3",
                              "roofline": {"bound": "tensor", "achieved": (mm + att + head) / (best * 1e-3) / 1e12 / world, "peak": tpeak, "unit": "TFLOP/s per GPU",
                                           "frac": (mm + att + head) / (best * 1e-3) / 1e12 / world / tpeak, "peak_source": tsrc,
                                           "note": f"per GPU; the pipeline is full for {nub} of {nub + world - 1} micro-batch slots (bubble {(world - 1) / (nub + world - 1):.2f})"}}
        except Exception as ex:
            pp_result = {"value": None, "unit": "tokens/s", "error": repr(ex)}
    if rank != 0:
        if dist is not None:
            dist.destroy_process_group()
        return

    peak, peak_src = peaks()
    ms_step = ms_dev / args.steps
    ms_step_e2e = ms_e2e / args.steps
    e2e_engine = {"value": 1e3 / ms_step_e2e, "unit": "tokens/s", "h2d_bytes_per_step": 8, "d2h_bytes_per_step": nv * 4,
                  "ms_per_step": ms_step_e2e, "api": "pb200_decode (token id + position from pinned host memory in, n_vocab f32 logits out)"}
    kv_bytes = 2 * L * (first + args.steps // 2) * hp["n_head_kv"] * 128 * 2
    achieved = gemv_bytes / (gemv_ms * 1e-3) / 1e9
    out = {
        "metric": METRIC, "value": 1e3 / ms_step, "unit": "tokens/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": ms_step, "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
        "dtype": "int8 activations (q8_K) x k-quant weights, int32 dot, f32 accumulate", "data": "synthetic", "config": config,
        "e2e": e2e_engine,
        "gpu_launches": launches,
        "clocks": clocks, "clocks_e2e": clocks_e2e,
        "roofline": {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                     "kernel": "k_gemv_kquant (TMA-staged k-quant GEMV)", "peak_source": peak_src,
                     "how": f"algorithmic bytes of the {gemv_launches} GEMV launches of one token ({gemv_bytes} B = sum of ggml_nbytes of the weight "
                            f"matrices read) / their summed CUDA-event durations ({gemv_ms:.3f} ms, events on the launching stream, mean of 4 profiled steps)",
                     "whole_step": {"algorithmic_bytes_per_token": wb + kv_bytes, "achieved": (wb + kv_bytes) / (ms_step * 1e-3) / 1e9,
                                    "frac": (wb + kv_bytes) / (ms_step * 1e-3) / 1e9 / peak}},
        "model_load_s": t_load,
    }
    if pp_result is not None:
        out["prefill"] = pp_result
    if ring is not None:
        # headline at N > 1: aggregate decode throughput of the ring with N sequences (each b = 1) in flight; the single-sequence
        # latency run above stays in `latency_b1` (serial across stages by nature: N GPUs cannot cut one token's latency)
        out["latency_b1"] = {"value": out["value"], "unit": "tokens/s", "ms_per_token": ms_step, "e2e": out["e2e"], "gpu_launches": launches}
        out["value"] = ring["tokens"] / (ring["ms"] * 1e-3)
        out["ms_per_step"] = ring["ms"] / args.steps
        out["scaling"] = "weak"
        out["gpu_launches"] = ring["launches"]
        out["clocks"] = ring["clocks"]
        out["config"]["parallelism"] = (f"layer pipeline pp{world}, {world} independent b=1 sequences in flight (one per stage, prima's piped ring); "
                                        f"a step = one round = {world} tokens; hand-off = grouped NCCL send/recv, tokens / positions / greedy argmax stay on the device")
        out["roofline"]["whole_step"] = {"algorithmic_bytes_per_token": wb + kv_bytes, "achieved": (wb + kv_bytes) * ring["tokens"] / (ring["ms"] * 1e-3) / 1e9 / world,
                                         "frac": (wb + kv_bytes) * ring["tokens"] / (ring["ms"] * 1e-3) / 1e9 / world / peak,
                                         "note": "per GPU: every token reads the whole model once, spread over the stages"}
        out["e2e"] = {"value": out["value"], "unit": "tokens/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0,
                      "note": "ring mode keeps tokens on the device (device argmax feeds the next step): there is no per-step host transfer to time; "
                              "the host-in / host-out call is measured in latency_b1.e2e"}
    if stage_ms is not None:
        out["pipeline"] = {"stages": world, "hand_offs_per_token": world, "sum_of_stage_ms": stage_ms, "pipelined_ms_per_token": ms_step,
                           "exposed_handoff_ms": max(0.0, ms_step - stage_ms), "exposed_frac": max(0.0, ms_step - stage_ms) / ms_step,
                           "note": "b=1 decode is serial across stages (SURVEY H7): N GPUs hold N x the model, they do not cut the token latency"}
    if world == 1 and args.pp > 0 and args.pp <= args.n_ctx:
        try:
            # prompt processing (prefill) of one ubatch through pb200_prefill: tensor-core mat-muls, batched attention
            toks = np.array([token_at(i, nv) for i in range(args.pp)], dtype=np.int32)
            eng.kv_clear()
            eng.prefill(toks, 0, logits_host)                      # warm-up (allocates the batch buffers)
            reps, best = 3, None
            for _ in range(reps):
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                eng.prefill(toks, 0, logits_host)                  # tokens from host memory in, last-token logits out: end to end
                dt = time.perf_counter() - t1
                best = dt if best is None else min(best, dt)
            mm, att, head = prefill_flops(hp, args.pp)
            tpeak, tsrc = tensor_peak()
            out["prefill"] = {"metric": f"prompt tokens/s, {cfg['name']}, one ubatch of {args.pp} tokens (llama-bench pp{args.pp})", "tokens": args.pp,
                              "ms": best * 1e3, "value": args.pp / best, "unit": "tokens/s", "timing": f"host wall clock around pb200_prefill (synchronous), best of {reps}",
                              "roofline": {"bound": "tensor", "achieved": (mm + att + head) / best / 1e12, "peak": tpeak, "unit": "TFLOP/s",
                                           "frac": (mm + att + head) / best / 1e12 / tpeak, "peak_source": tsrc,
                                           "algorithmic_flops": {"matmul": mm, "attention_causal": att, "lm_head_last_token": head},
                                           "kernel": "k_mmq_tc (wgmma k-quant mat-mul); attention on CUDA cores (k_attn_prefill_tiled: K/V tiles shared by the GQA group x 4 tokens)"}}
        except Exception as ex:   # the extra measurement must never take the headline line down
            out["prefill"] = {"value": None, "unit": "tokens/s", "error": repr(ex)}

    if world == 1 and not args.no_boundary:
        try:
            out["e2e_engine"] = e2e_engine
            out["e2e"] = boundary_leg(eng, cfg, hp, args, lib)
        except Exception as ex:   # the boundary leg needs host/_ggml (built where the reference tree exists); keep the engine number otherwise
            out["e2e_boundary_error"] = repr(ex)
    if world == 1 and not args.no_gpu_comparator:
        # same-box GPU comparator: the reference's own ggml-cuda (sm_90a build) in a process of its own, after this one released the GPU memory
        try:
            eng.close()
            torch.cuda.empty_cache()
            out["gpu_comparator"] = ggml_cuda_subprocess(args.model, min(args.steps, 64), min(args.warmup, 8), args.n_ctx)
            if out["gpu_comparator"].get("value"):
                out["gpu_comparator"]["b200_e2e_over_ggml_cuda"] = out["e2e"]["value"] / out["gpu_comparator"]["value"]
        except Exception as ex:
            out["gpu_comparator"] = {"unavailable": repr(ex)}
    if not args.no_cpu_baseline:
        try:
            out["cpu_baseline"] = cpu_reference_subprocess(args.model, args.steps, args.warmup)
        except Exception as ex:   # the checker must never take the measurement down
            out["cpu_baseline"] = {"value": None, "unit": "tokens/s", "cores": os.cpu_count(), "kind": "reference", "sample": f"failed: {ex!r}"}
    print(json.dumps(out))
    if dist is not None:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
