"""Logit bias + penalties on the device: apply + sample + accept against pb200_sample alone, and a Llama-3-8B-shape decode step with
pb200_sample_seq with and without penalties.

    python tools/penalty_probe.py --out DIR

Writes DIR/penalty_probe.json and prints a table.  Times are CUDA events over back-to-back launches (default chain: top-k 40,
top-p 0.95, min-p 0.05, temp 0.8); the history is filled to last_n before timing.  The card's name and power limit are recorded in the
same run.
"""
import argparse
import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tools"))

import pkgload  # noqa: E402
import sampling_ref as S  # noqa: E402
from sample_probe import LLAMA3_8B, card, ev_time  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--iters", type=int, default=500)
    args = ap.parse_args()
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    assert torch.cuda.is_available(), "penalty_probe measures on a CUDA device"
    pkg = pkgload.load()
    lib = pkg.Lib.get()
    res = {"card": card(), "sample_us": {}, "apply_us": {}, "apply_sample_accept_us": {}, "step_ms": {}}
    state = torch.zeros(lib.sampler_state_bytes(), dtype=torch.uint8, device="cuda")
    tok = torch.zeros(1, dtype=torch.int32, device="cuda")
    sp = pkg.Sampling(40, 0.95, 0.05, 0.8, 0, 1)
    g = np.random.default_rng(1)
    for n in (128256, 152064):
        x = torch.from_numpy(S.make_logits(n, n)).cuda()
        row = torch.empty_like(x)
        lib.sampler_seed(state.data_ptr(), 1)
        res["sample_us"][str(n)] = ev_time(lambda: lib.sample(x.data_ptr(), n, sp, state.data_ptr(), tok.data_ptr()), args.iters)
        for last_n in (64, 4096):
            for nb in (0, 1000):
                bias = [(int(t), float(v)) for t, v in zip(g.integers(0, n, nb), g.standard_normal(nb))]
                p = pkg.penalties(last_n=last_n, repeat=1.1, freq=0.05, present=0.05, nl_token=13, eos_token=2, logit_bias=bias)
                pst = torch.zeros(lib.penalty_state_bytes(n, p), dtype=torch.uint8, device="cuda")
                lib.penalty_init(pst.data_ptr(), n, p)
                hist = torch.from_numpy(g.integers(0, n, last_n).astype(np.int32)).cuda()
                lib.penalty_accept(pst.data_ptr(), hist.data_ptr(), last_n)
                key = f"{n} last_n {last_n} bias {nb}"
                res["apply_us"][key] = ev_time(lambda: lib.penalty_apply(x.data_ptr(), n, pst.data_ptr(), row.data_ptr()), args.iters)

                def chain():
                    lib.penalty_apply(x.data_ptr(), n, pst.data_ptr(), row.data_ptr())
                    lib.sample(row.data_ptr(), n, sp, state.data_ptr(), tok.data_ptr())
                    lib.penalty_accept(pst.data_ptr(), tok.data_ptr(), 1)
                res["apply_sample_accept_us"][key] = ev_time(chain, args.iters)
    # Llama-3-8B-shape synthetic decode step + pb200_sample_seq, without and with penalties (llama-cli's --repeat-penalty 1.1 over 64)
    eng = pkg.Model(pkg.HParams(**LLAMA3_8B), 0, None, True, True)
    eng.synth(0, 7)
    eng.finalize()
    eng.set_sampling(0, seed=5)
    stream = torch.cuda.ExternalStream(eng.stream)
    for mode in ("sample", "sample + penalties", "sample", "sample + penalties"):
        eng.set_penalties(0, last_n=64, repeat=1.1) if mode != "sample" else eng.set_penalties(0, None)
        eng.set_tokpos_seq(0, 1, 0)

        def step():
            eng.step_seq_dev(0, False)
            eng.sample_seq(0, True)
        with torch.cuda.stream(stream):
            res["step_ms"].setdefault(mode, []).append(ev_time(step, 100) / 1e3)
    eng.close()
    (out / "penalty_probe.json").write_text(json.dumps(res, indent=1))
    print(f"card: {res['card']}")
    for n, v in res["sample_us"].items():
        print(f"pb200_sample alone @ {n}: {v:.1f} us")
    print(f"{'n_vocab / last_n / bias entries':34s} {'apply us':>9s} {'apply+sample+accept us':>23s}")
    for k, v in res["apply_us"].items():
        print(f"{k:34s} {v:9.1f} {res['apply_sample_accept_us'][k]:23.1f}")
    for k, v in res["step_ms"].items():
        print(f"Llama-3-8B-shape step + {k}: {', '.join(f'{t:.3f}' for t in v)} ms")


if __name__ == "__main__":
    main()
