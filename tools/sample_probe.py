"""Device sampling (pb200_sample) against the copy-to-host path, and a Llama-3-8B-shape decode step with sampling vs with argmax.

    python tools/sample_probe.py --out DIR

Writes DIR/sample_probe.json and prints a table.  Times are CUDA events over back-to-back launches (device sampler, decode steps) or a
host clock around work that ends in a synchronise (host path: D2H of the logits into pinned memory, the reference's chain from
oracle/_ref/libsampling_ref.so, H2D of the token).  The card's name and power limit are recorded in the same run.
"""
import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tests" / "golden"))

import pkgload  # noqa: E402
import sampling_ref as S  # noqa: E402

CHAINS = {"defaults": (40, 0.95, 0.05, 0.8, 0), "top_k 0 / top_p 0.9": (0, 0.9, 0.0, 0.8, 0), "pure temperature": (0, 1.0, 0.0, 0.8, 0)}
LLAMA3_8B = dict(n_layer=32, n_embd=4096, n_head=32, n_head_kv=8, head_dim=128, n_ff=14336, n_vocab=128256, n_ctx=512, rope_mode=0,
                 n_ctx_orig=8192, rope_freq_base=500000.0, rope_freq_scale=1.0, rms_eps=1e-5)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def ev_time(fn, iters, warm=20):
    for _ in range(warm):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / iters   # us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--iters", type=int, default=500)
    args = ap.parse_args()
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    assert torch.cuda.is_available(), "sample_probe measures on a CUDA device"
    pkg = pkgload.load()
    lib = pkg.Lib.get()
    res = {"card": card(), "device_us": {}, "host_us": {}, "step_ms": {}}
    state = torch.zeros(lib.sampler_state_bytes(), dtype=torch.uint8, device="cuda")
    tok = torch.zeros(1, dtype=torch.int32, device="cuda")
    ref = None
    ref_lib = ROOT / "oracle" / "_ref" / "libsampling_ref.so"
    if ref_lib.exists():
        from make_sampling_golden import RefChain
        ref = C.CDLL(str(ref_lib))
    for n in (128256, 152064):
        logits_np = S.make_logits(n, n)
        logits = torch.from_numpy(logits_np).cuda()
        host = torch.empty(n, dtype=torch.float32).pin_memory()
        for name, ch in CHAINS.items():
            p = pkg.Sampling(*ch, 1)
            lib.sampler_seed(state.data_ptr(), 1)
            key = f"{name} @ {n}"
            res["device_us"][key] = ev_time(lambda: lib.sample(logits.data_ptr(), n, p, state.data_ptr(), tok.data_ptr()), args.iters)
            if ref is not None:
                chain = RefChain(ref, *ch, 1)
                it = 20 if ch[0] <= 0 else 100
                ts = []
                for i in range(it + 3):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    host.copy_(logits, non_blocking=True)
                    torch.cuda.synchronize()
                    t_ref, _, _, _ = chain(host.numpy())
                    tok.fill_(t_ref)
                    torch.cuda.synchronize()
                    if i >= 3:
                        ts.append(time.perf_counter() - t0)
                chain.close()
                res["host_us"][key] = float(np.median(ts)) * 1e6
    # Llama-3-8B-shape synthetic decode step + sample vs + argmax (graph-replayed step, device-resident token)
    eng = pkg.Model(pkg.HParams(**LLAMA3_8B), 0, None, True, True)
    eng.synth(0, 7)
    eng.finalize()
    eng.set_sampling(0, seed=5)
    stream = torch.cuda.ExternalStream(eng.stream)
    for mode in ("argmax", "sample", "argmax", "sample"):
        eng.set_tokpos_seq(0, 1, 0)

        def step():
            eng.step_seq_dev(0, False)
            (eng.argmax_seq if mode == "argmax" else eng.sample_seq)(0, True)
        with torch.cuda.stream(stream):
            res["step_ms"][mode] = ev_time(step, 100) / 1e3
    eng.close()
    (out / "sample_probe.json").write_text(json.dumps(res, indent=1))
    print(f"card: {res['card']}")
    print(f"{'chain @ n_vocab':34s} {'device us':>10s} {'host path us':>13s}")
    for k, v in res["device_us"].items():
        h = res["host_us"].get(k)
        print(f"{k:34s} {v:10.1f} {h if h is None else round(h, 1)!s:>13s}")
    print(f"Llama-3-8B-shape step + argmax {res['step_ms']['argmax']:.3f} ms, step + sample {res['step_ms']['sample']:.3f} ms")


if __name__ == "__main__":
    main()
