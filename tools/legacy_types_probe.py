"""GPU: what the legacy 32-element weight types cost.  python tools/legacy_types_probe.py --out DIR  (writes DIR/legacy_types_probe.json)

* GEMV weight bytes per second of Q4_0 / Q4_1 / Q5_0 beside Q5_1 / Q8_0 at Qwen2.5-72B's ffn_down shape (8 192 x 29 568) and at
  8 192 x 8 192: CUDA events over 200 launches of the bulk-copy ring, rotating through 4 weight copies (more than L2 holds).
* Decode (device-resident steps, 4 warm-up + 32 timed, two alternating runs): synthetic Qwen2.5-72B Q4_K_M (ffn_down Q5_0 / Q8_0)
  against Q5_K_M, loaded, measured and freed in turn (one at a time fits 80 GB), and Llama-3-8B Q4_0 against Q4_K_M.
* pp512: one 512-token prompt through pb200_prefill on Qwen2.5-72B Q4_K_M.
The card's name and power limit are read in the same run."""
import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
import torch  # noqa: E402

import pkgload  # noqa: E402

TYPES = {"q4_0": 2, "q4_1": 3, "q5_0": 6, "q5_1": 7, "q8_0": 8}
QWEN72 = dict(n_layer=80, n_embd=8192, n_head=64, n_head_kv=8, head_dim=128, n_ff=29568, n_vocab=152064, rope_mode=2, n_ctx_orig=32768,
              rope_freq_base=1e6, rope_freq_scale=1.0, rms_eps=1e-6)
LLAMA8 = dict(n_layer=32, n_embd=4096, n_head=32, n_head_kv=8, head_dim=128, n_ff=14336, n_vocab=128256, rope_mode=0, n_ctx_orig=8192,
              rope_freq_base=500000.0, rope_freq_scale=1.0, rms_eps=1e-5)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None}


def gemv_rates(lib):
    p = lambda a: C.c_void_p(a.data_ptr())
    out = {}
    for N, K in ((8192, 29568), (8192, 8192)):
        x = torch.randn(K, device="cuda")
        y = torch.zeros(N, device="cuda")
        for name, t in TYPES.items():
            rb = lib.c.pb200_row_bytes(t, K)
            W = [torch.randint(0, 255, (N * rb + 64,), dtype=torch.uint8, device="cuda") for _ in range(4)]
            ws = torch.zeros(lib.c.pb200_act_workspace_bytes(K) + 64, dtype=torch.uint8, device="cuda")
            lib.check(lib.c.pb200_quantize_act(t, p(x), K, p(ws), None), "q")
            for i in range(8):
                lib.check(lib.c.pb200_mul_mat_vec_q(t, p(W[i % 4]), N, K, p(ws), p(y), None, None, None), "gemv")
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            reps = 200
            e0.record()
            for i in range(reps):
                lib.c.pb200_mul_mat_vec_q(t, p(W[i % 4]), N, K, p(ws), p(y), None, None, None)
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) / reps * 1e3
            out[f"{name}_{N}x{K}"] = {"us": round(us, 2), "TB_s": round(N * rb / us / 1e6, 3), "bytes": N * rb}
            print(name, N, K, out[f"{name}_{N}x{K}"], flush=True)
            del W
            torch.cuda.empty_cache()
    return out


def decode_run(pkg, hp, ftype, steps=32, warm=4, pp=0):
    m = pkg.Model(pkg.HParams(**hp, n_ctx=1024), 0, None, True, True)
    m.synth(ftype, 1234)
    m.finalize()
    nv = hp["n_vocab"]
    for i in range(warm):
        m.decode_async((i * 7919 + 13) % nv, i)
    m.synchronize()
    t0 = time.perf_counter()
    for i in range(warm, warm + steps):
        m.decode_async((i * 7919 + 13) % nv, i)
    m.synchronize()
    dt = time.perf_counter() - t0
    r = {"tok_s": round(steps / dt, 2), "ms_per_token": round(dt / steps * 1e3, 3), "weight_bytes": m.weight_bytes,
         "GB_s": round(m.weight_bytes / (dt / steps) / 1e9, 1)}
    if pp:
        toks = [(i * 7919 + 13) % nv for i in range(pp)]
        m.kv_clear()
        m.prefill(toks, 0)
        m.kv_clear()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.prefill(toks, 0)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        r["pp_ms"] = round(dt * 1e3, 1)
        r["pp_tok_s"] = round(pp / dt, 1)
    m.close()
    del m
    torch.cuda.empty_cache()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    out_dir = Path(args.out)
    out_dir.mkdir(parents=True, exist_ok=True)
    assert torch.cuda.is_available(), "the probe measures on a CUDA device"
    torch.cuda.set_device(0)
    pkg = pkgload.load()
    lib = pkg.Lib.get()
    res = {"card": card(), "gemv": gemv_rates(lib), "decode": {}}
    for run in range(2):
        for key, hp, ftype in (("qwen2.5-72b q4_K_M", QWEN72, 0), ("qwen2.5-72b q5_K_M", QWEN72, 1), ("llama3-8b q4_0", LLAMA8, 2),
                               ("llama3-8b q4_K_M", LLAMA8, 0)):
            r = decode_run(pkg, hp, ftype, pp=512 if (run == 1 and ftype == 0 and hp is QWEN72) else 0)
            res["decode"].setdefault(key, []).append(r)
            print(key, run, r, flush=True)
    res["card_after"] = card()
    (out_dir / "legacy_types_probe.json").write_text(json.dumps(res, indent=1))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
