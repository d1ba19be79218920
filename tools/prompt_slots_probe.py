"""Prompts into a sequence slot other than 0 (pb200_prefill_seq) and the KV copy between slots (pb200_kv_seq_cp), on a synthetic
Llama-3-70B (Q4_K_M mixture) with 4 slots and n_ctx 4096.

    python tools/prompt_slots_probe.py --out DIR

Writes DIR/prompt_slots_probe.json and prints a table:
- pp512 and pp2048 into slot 0 and slot 3, alternated and repeated (CUDA events on the model stream around each prefill call, which
  ends in a synchronise), and whether the two slots' last-token logits are bit-identical;
- kv_seq_cp of 512 and 4096 cells from slot 0 to slot 3: time per copy over back-to-back copies, and the rate of the bytes copied
  (2 caches x n_layer x cells x n_head_kv x 128 x 2 B; the copy engine reads and writes each byte once), against prefilling the same
  prefix;
- device-resident decode (pb200_step_seq_dev + pb200_argmax_seq with feed-back) of slot 3 after its 2048-token prompt against slot 0
  after the same prompt, alternated.
The card's name and power limit are recorded in the same run.
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

SHAPE = dict(n_layer=80, n_embd=8192, n_head=64, n_head_kv=8, head_dim=128, n_ff=28672, n_vocab=128256)
N_CTX, N_SEQ, SLOTS = 4096, 4, (0, 3)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--steps", type=int, default=64)
    args = ap.parse_args()
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    assert torch.cuda.is_available(), "prompt_slots_probe measures on a CUDA device"
    pkg = pkgload.load()
    res = {"card": card(), "model": "llama3-70b synthetic Q4_K_M", "n_ctx": N_CTX, "n_seq": N_SEQ}
    hp = pkg.HParams(**SHAPE, n_ctx=N_CTX, rope_mode=0, n_ctx_orig=8192, rope_freq_base=500000.0, rope_freq_scale=1.0, rms_eps=1e-5)
    eng = pkg.Model(hp, 0)
    eng.set_n_seq(N_SEQ)
    eng.synth(0, 7)
    eng.finalize()
    st = torch.cuda.ExternalStream(eng.stream)
    nv = SHAPE["n_vocab"]
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(f):
        with torch.cuda.stream(st):
            a.record()
        f()
        with torch.cuda.stream(st):
            b.record()
        b.synchronize()
        return a.elapsed_time(b)

    toks = {n: (np.arange(n) * 7919 + 13) % nv for n in (512, 2048, 4096)}
    # prompt processing into slot 0 and slot 3, alternated
    for n in (512, 2048):
        for s in SLOTS:
            eng.prefill(toks[n], 0, seq=s)                                 # warm-up of every shape and slot
    pp = {(n, s): [] for n in (512, 2048) for s in SLOTS}
    lg = {(n, s): [] for n in (512, 2048) for s in SLOTS}

    def prefill(n, s):
        lg[(n, s)].append(eng.prefill(toks[n], 0, seq=s))
    for _ in range(args.reps):
        for n in (512, 2048):
            for s in SLOTS:
                pp[(n, s)].append(timed(lambda: prefill(n, s)))
    # The tensor-core mat-mul adds the partial sums of a tile that two or more CTAs share with fp32 atomics (mmq.cu), so at these shapes
    # the logits of one prompt vary from run to run in any slot.  Each run is set against slot 0's first run: slot 0's own later runs
    # show the mat-mul's spread, slot 3's runs whether the slot adds anything to it.
    ref = {n: lg[(n, 0)][0] for n in (512, 2048)}
    res["pp"] = [dict(n_tokens=n, seq=s, ms_all=v, ms_median=float(np.median(v)), tok_s=n / float(np.median(v)) * 1e3,
                      bit_identical_to_slot_0_run_0=[bool(np.array_equal(x.view(np.uint32), ref[n].view(np.uint32))) for x in lg[(n, s)]],
                      max_abs_diff_to_slot_0_run_0=[float(np.max(np.abs(x - ref[n]))) for x in lg[(n, s)]],
                      argmax_equal_to_slot_0_run_0=[int(np.argmax(x)) == int(np.argmax(ref[n])) for x in lg[(n, s)]])
                 for (n, s), v in pp.items()]
    # KV copy against prefilling the same prefix
    row = SHAPE["n_head_kv"] * 128 * 2
    cp = []
    pf4096 = [timed(lambda: eng.prefill(toks[4096], 0, seq=0)) for _ in range(2)]
    for cells in (512, 4096):
        eng.kv_copy(0, 3, 0, cells)
        eng.synchronize()

        def copies():
            for _ in range(args.iters):
                eng.kv_copy(0, 3, 0, cells)
        ms = timed(copies) / args.iters
        nbytes = 2 * SHAPE["n_layer"] * cells * row
        pf_ms = float(np.median(pp[(512, 0)])) if cells == 512 else float(np.median(pf4096))
        cp.append(dict(cells=cells, ms=ms, bytes=nbytes, gb_s=nbytes / ms / 1e6, prefill_same_prefix_ms=pf_ms, prefill_over_copy=pf_ms / ms))
    res["kv_copy"] = cp
    res["prefill_4096_ms_all"] = pf4096
    # device-resident decode after a 2048-token prompt, slot 3 against slot 0
    dec = {s: [] for s in SLOTS}
    for s in SLOTS:
        eng.prefill(toks[2048], 0, seq=s)
        eng.set_tokpos_seq(s, 0, 2048)
        eng.argmax_seq(s, True)                       # the first token from the prompt's logits
    for rep in range(args.reps):                      # both slots advance alike: 4 + steps positions per repetition
        for s in SLOTS:
            for _ in range(4):
                eng.step_seq_dev(s, True)
                eng.argmax_seq(s, True)
            eng.synchronize()

            def steps():
                for _ in range(args.steps):
                    eng.step_seq_dev(s, True)
                    eng.argmax_seq(s, True)
            dec[s].append(args.steps / timed(steps) * 1e3)
    res["decode"] = [dict(seq=s, tok_s_all=v, tok_s_median=float(np.median(v))) for s, v in dec.items()]
    eng.close()
    (out / "prompt_slots_probe.json").write_text(json.dumps(res, indent=1))
    print(f"card, power limit: {res['card']}")
    for r in res["pp"]:
        print(f"pp{r['n_tokens']:<5} slot {r['seq']}: median {r['ms_median']:8.2f} ms  {r['tok_s']:8.1f} tok/s  all {['%.2f' % x for x in r['ms_all']]}"
              f"  vs slot 0 run 0: bit-identical {r['bit_identical_to_slot_0_run_0']}, max |diff| "
              f"{['%.2e' % x for x in r['max_abs_diff_to_slot_0_run_0']]}, same argmax {r['argmax_equal_to_slot_0_run_0']}")
    for r in cp:
        print(f"kv_seq_cp {r['cells']:5d} cells: {r['ms']:.3f} ms, {r['bytes'] / 1e9:.3f} GB, {r['gb_s']:.0f} GB/s;  prefill of the same prefix "
              f"{r['prefill_same_prefix_ms']:.1f} ms ({r['prefill_over_copy']:.0f}x)")
    for r in res["decode"]:
        print(f"decode slot {r['seq']} after pp2048: median {r['tok_s_median']:.2f} tok/s  all {['%.2f' % x for x in r['tok_s_all']]}")


if __name__ == "__main__":
    main()
