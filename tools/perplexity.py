"""llama-perplexity on the engine: the reference's chunk loop (prima.cpp_b200/perplexity.py) over a GGUF model or synthetic weights.

    python tools/perplexity.py --gguf MODEL.gguf --tokens ids.npy --ctx 512 [--chunks N] [--bos ID]
    python tools/perplexity.py --synth llama3-70b --ctx 512 --chunks 4 [--out DIR]

Token ids come from a .npy int32 file (tokenization is not provided) or, without --tokens, from a seeded generator.  Each chunk is
prefilled in ubatches of at most 512 tokens, and pb200_prompt_head scores the rows at positions >= ctx / 2 of each ubatch on the device.
Prints the reference's "[i]ppl," lines and "Final estimate", then seconds per chunk, the share of pb200_prompt_head in it (CUDA events on the
model stream around each call, which ends in a synchronise), scored tokens per second, and the card's name and power limit (read in the
same run).  --out DIR also writes DIR/perplexity.json."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import pkgload  # noqa: E402
from bench import MODELS  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--gguf", help="GGUF model file (llama / qwen2)")
    src.add_argument("--synth", choices=sorted(MODELS), help="synthetic weights of this shape and type mixture")
    ap.add_argument("--tokens", help=".npy int32 token ids (default: seeded random ids)")
    ap.add_argument("--ctx", type=int, default=512)
    ap.add_argument("--chunks", type=int, default=-1, help="at most this many chunks (default: all)")
    ap.add_argument("--bos", type=int, default=None, help="replace each chunk's first token with this id")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", help="directory for perplexity.json")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "tools/perplexity.py runs the engine on a CUDA device"
    pkg = pkgload.load()
    if args.gguf:
        eng = pkg.Model.from_gguf(args.gguf, 0, n_ctx=args.ctx)
        name = Path(args.gguf).name
    else:
        cfg = MODELS[args.synth]
        eng = pkg.Model(pkg.HParams(**cfg["hp"], n_ctx=args.ctx), 0)
        eng.synth(cfg["ftype"], 7)
        eng.finalize()
        name = f"{cfg['name']} (synthetic)"
    nv = eng.hp.n_vocab
    if args.tokens:
        toks = np.load(args.tokens).astype(np.int32).reshape(-1)
    else:
        toks = np.random.default_rng(args.seed).integers(0, nv, max(args.chunks, 2) * args.ctx).astype(np.int32)

    st = torch.cuda.ExternalStream(eng.stream)
    head_ms = []
    prompt_head = eng.prompt_head

    def timed_head(*a, **kw):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(st):
            e0.record()
        r = prompt_head(*a, **kw)
        with torch.cuda.stream(st):
            e1.record()
        e1.synchronize()
        head_ms.append(e0.elapsed_time(e1))
        return r
    eng.prompt_head = timed_head
    run = pkg.perplexity.model_run_chunk(eng)
    chunk_s, chunk_head = [], []

    def run_chunk(tokens, first):
        n0 = len(head_ms)
        t0 = time.perf_counter()
        s = run(tokens, first)                          # ends in prompt_head's synchronise
        chunk_s.append(time.perf_counter() - t0)
        chunk_head.append(sum(head_ms[n0:]) / 1e3)
        return s

    print(f"{name}: n_vocab {nv}, ctx {args.ctx}, {len(toks)} tokens, bos {args.bos}")
    res = pkg.perplexity.perplexity(toks, args.ctx, run_chunk, args.chunks, args.bos)
    c = card()
    per_chunk = res.count // len(chunk_s)
    # the first chunk includes the first launches of every shape (module loading, the head buffer's allocation)
    steady = chunk_s[1:] or chunk_s
    steady_head = chunk_head[1:] or chunk_head
    sec, hsec = float(np.mean(steady)), float(np.mean(steady_head))
    print(f"seconds per chunk: {sec:.4f} (first chunk {chunk_s[0]:.4f}); pb200_prompt_head {hsec * 1e3:.2f} ms of it ({100 * hsec / sec:.1f} %)")
    print(f"scored tokens per second: {per_chunk / sec:.1f} ({per_chunk} scored of {args.ctx} per chunk)")
    print(f"card, power limit: {c}")
    if args.out:
        out = Path(args.out)
        out.mkdir(parents=True, exist_ok=True)
        (out / "perplexity.json").write_text(json.dumps(dict(
            model=name, ctx=args.ctx, chunks=len(chunk_s), bos=args.bos, ppl=res.ppl, uncertainty=res.uncertainty, chunk_ppl=res.chunk_ppl,
            chunk_seconds=chunk_s, chunk_head_seconds=chunk_head, seconds_per_chunk=sec, head_seconds_per_chunk=hsec,
            scored_tokens_per_second=per_chunk / sec, card=c), indent=1))
    eng.close()


if __name__ == "__main__":
    main()
