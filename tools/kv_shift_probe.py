"""Context shift on the device (pb200_kv_seq_shift) against what a host without it has to do instead (pb200_kv_clear + pb200_prefill of
the kept half), on synthetic Llama-3-8B and Llama-3-70B models (Q4_K_M mixture, n_ctx 8192, llama-cli's rule at a full context with
n_keep 0: n_discard 4096, cells [4096, 8192) move to [0, 4096)).

    python tools/kv_shift_probe.py --out DIR

Writes DIR/kv_shift_probe.json and prints a table.  Shift times are CUDA events around back-to-back shifts on the model stream; the
alternative is timed with CUDA events around kv_clear + prefill (both end in a synchronise).  Bytes moved by a shift:
2 tensors x 2 (read + write) x n_layer x (p1 - p0) x n_head_kv x 128 x 2 B, set against the H100 SXM data-sheet 3.35 TB/s.  The card's
name and power limit are recorded in the same run.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import pkgload  # noqa: E402

N_CTX, N_KEEP, N_DISCARD = 8192, 0, 4096
MODELS = {
    "llama3-8b": dict(n_layer=32, n_embd=4096, n_head=32, n_head_kv=8, head_dim=128, n_ff=14336, n_vocab=128256),
    "llama3-70b": dict(n_layer=80, n_embd=8192, n_head=64, n_head_kv=8, head_dim=128, n_ff=28672, n_vocab=128256),
}
HBM_TBS = 3.35


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def probe(pkg, name, shape, iters, reps):
    hp = pkg.HParams(**shape, n_ctx=N_CTX, rope_mode=0, n_ctx_orig=8192, rope_freq_base=500000.0, rope_freq_scale=1.0, rms_eps=1e-5)
    eng = pkg.Model(hp, 0)
    eng.synth(0, 7)
    eng.finalize()
    st = torch.cuda.ExternalStream(eng.stream)
    p0, p1, delta = N_KEEP + N_DISCARD, N_CTX, -N_DISCARD
    kept = p1 - p0
    toks = (np.arange(kept) * 7919 + 13) % shape["n_vocab"]
    eng.prefill(toks, 0)             # warm-up of the prefill path (and a filled cache)
    for _ in range(5):
        eng.kv_shift(0, p0, p1, delta)
    eng.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(st):
        a.record()
        for _ in range(iters):
            eng.kv_shift(0, p0, p1, delta)
        b.record()
    b.synchronize()
    shift_ms = a.elapsed_time(b) / iters
    alt = []
    for _ in range(reps):
        with torch.cuda.stream(st):
            a.record()
        eng.kv_clear()
        eng.prefill(toks, 0)
        with torch.cuda.stream(st):
            b.record()
        b.synchronize()
        alt.append(a.elapsed_time(b))
    eng.close()
    nbytes = 2 * 2 * shape["n_layer"] * kept * shape["n_head_kv"] * 128 * 2
    return dict(model=name, n_ctx=N_CTX, p0=p0, p1=p1, delta=delta, shift_ms=shift_ms, shift_bytes=nbytes, shift_tbs=nbytes / shift_ms / 1e9,
                shift_share_of_3_35=nbytes / shift_ms / 1e9 / HBM_TBS, clear_prefill_ms_median=float(np.median(alt)),
                clear_prefill_ms_all=alt, prefill_tokens=kept)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    assert torch.cuda.is_available(), "kv_shift_probe measures on a CUDA device"
    pkg = pkgload.load()
    res = {"card": card(), "rows": [probe(pkg, n, s, args.iters, args.reps) for n, s in MODELS.items()]}
    (out / "kv_shift_probe.json").write_text(json.dumps(res, indent=1))
    print(f"card, power limit: {res['card']}")
    print(f"{'model':<12} {'shift ms':>9} {'GB moved':>9} {'TB/s':>6} {'of 3.35':>8} {'clear+prefill ms':>17}")
    for r in res["rows"]:
        print(f"{r['model']:<12} {r['shift_ms']:9.3f} {r['shift_bytes'] / 1e9:9.3f} {r['shift_tbs']:6.2f} {r['shift_share_of_3_35']:8.1%} "
              f"{r['clear_prefill_ms_median']:17.1f}")


if __name__ == "__main__":
    main()
