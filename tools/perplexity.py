"""llama-perplexity on the engine: the reference's chunk loop (prima.cpp_b200/perplexity.py) over a GGUF model or synthetic weights.

    python tools/perplexity.py --gguf MODEL.gguf --tokens ids.npy --ctx 512 [--chunks N] [--bos ID]
    python tools/perplexity.py --synth llama3-70b --ctx 512 --chunks 4 [--out DIR]
    python tools/perplexity.py --synth llama3-70b --ctx 512 --chunks 4 --kl-divergence-base BASE     (write the base file)
    python tools/perplexity.py --synth llama3-70b --kl-divergence-base BASE --kl-divergence           (compare against it)

Token ids come from a .npy int32 file (tokenization is not provided) or, without --tokens, from a seeded generator.  Each chunk is
prefilled in ubatches of at most 512 tokens, and pb200_prompt_head scores the rows at positions >= ctx / 2 of each ubatch on the device.
Prints the reference's "[i]ppl," lines and "Final estimate", then seconds per chunk, the share of pb200_prompt_head in it (CUDA events on the
model stream around each call, which ends in a synchronise), scored tokens per second, and the card's name and power limit (read in the
same run).  --out DIR also writes DIR/perplexity.json.

--kl-divergence-base FILE alone writes llama-perplexity's base file of u16 log-probability records (pb200_prompt_head_kld in writer
mode); with --kl-divergence it compares the model against FILE instead (tokens, n_ctx and chunk count come from the file) and prints the
reference's KL-divergence table and statistics.  Both report the share of pb200_prompt_head_kld in each chunk and the bytes it copied
between host and device per chunk."""
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
    ap.add_argument("--kl-divergence-base", dest="kld_base", help="the base file of log-probabilities: written, or read with --kl-divergence")
    ap.add_argument("--kl-divergence", dest="kld", action="store_true", help="compare against --kl-divergence-base FILE")
    args = ap.parse_args()
    if args.kld and not args.kld_base:
        ap.error("--kl-divergence needs --kl-divergence-base FILE")
    if args.kld:
        args.ctx = pkgload.load().perplexity.read_base_header(args.kld_base).n_ctx
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
    copied = []                                         # host <-> device bytes of each pb200_prompt_head_kld call
    rec_u16s = pkg.record_u16s(nv)

    def timed(f):                                       # CUDA events on the model stream around each call, which ends in a synchronise
        def call(*a, **kw):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(st):
                e0.record()
            r = f(*a, **kw)
            with torch.cuda.stream(st):
                e1.record()
            e1.synchronize()
            head_ms.append(e0.elapsed_time(e1))
            return r
        return call
    head_kld = timed(eng.prompt_head_kld)

    def timed_head_kld(row0, n, targets, records=False, base=None):
        copied.append(4 * n + (2 * n * rec_u16s + 4 * n if records else 0) + (2 * n * rec_u16s + 24 * n if base is not None else 0))
        return head_kld(row0, n, targets, records=records, base=base)
    eng.prompt_head = timed(eng.prompt_head)
    eng.prompt_head_kld = timed_head_kld
    run = pkg.perplexity.model_run_chunk(eng)
    chunk_s, chunk_head, chunk_bytes = [], [], []

    def run_chunk(tokens, first, **kw):
        n0, c0 = len(head_ms), len(copied)
        t0 = time.perf_counter()
        s = run(tokens, first, **kw)                    # ends in the head call's synchronise
        chunk_s.append(time.perf_counter() - t0)
        chunk_head.append(sum(head_ms[n0:]) / 1e3)
        chunk_bytes.append(sum(copied[c0:]))
        return s
    run_chunk.n_vocab, run_chunk.n_ctx = run.n_vocab, run.n_ctx

    mode = "compare" if args.kld else "writer" if args.kld_base else "score"
    head_name = "pb200_prompt_head" if mode == "score" else "pb200_prompt_head_kld"
    print(f"{name}: n_vocab {eng.hp.n_vocab}, ctx {args.ctx}, {len(toks)} tokens, bos {args.bos}, mode {mode}")
    kld = None
    if mode == "compare":
        kld = pkg.perplexity.kl_divergence(args.kld_base, run_chunk, args.bos)
        count = kld.sums.count
    else:
        res = pkg.perplexity.perplexity(toks, args.ctx, run_chunk, args.chunks, args.bos, logits_file=args.kld_base)
        count = res.count
    c = card()
    per_chunk = count // len(chunk_s)
    # the first chunk includes the first launches of every shape (module loading, the head buffer's allocation)
    steady = chunk_s[1:] or chunk_s
    steady_head = chunk_head[1:] or chunk_head
    sec, hsec = float(np.mean(steady)), float(np.mean(steady_head))
    print(f"seconds per chunk: {sec:.4f} (first chunk {chunk_s[0]:.4f}); {head_name} {hsec * 1e3:.2f} ms of it ({100 * hsec / sec:.1f} %)")
    print(f"scored tokens per second: {per_chunk / sec:.1f} ({per_chunk} scored of {args.ctx} per chunk)")
    if mode != "score":
        print(f"bytes copied between host and device per chunk by {head_name}: {chunk_bytes[-1]} ({chunk_bytes[-1] / 2**20:.1f} MiB)")
    print(f"card, power limit: {c}")
    if args.out:
        out = Path(args.out)
        out.mkdir(parents=True, exist_ok=True)
        d = dict(model=name, mode=mode, ctx=args.ctx, chunks=len(chunk_s), bos=args.bos, chunk_seconds=chunk_s, chunk_head_seconds=chunk_head,
                 seconds_per_chunk=sec, head_seconds_per_chunk=hsec, scored_tokens_per_second=per_chunk / sec, card=c)
        if mode == "compare":
            d.update(mean_kld=kld.sums.sum_kld / kld.sums.count, same_top=kld.sums.n_same_top / kld.sums.count, chunk_rows=kld.chunk_rows,
                     bytes_per_chunk=chunk_bytes[-1])
        else:
            d.update(ppl=res.ppl, uncertainty=res.uncertainty, chunk_ppl=res.chunk_ppl)
            if mode == "writer":
                d.update(bytes_per_chunk=chunk_bytes[-1])
        (out / f"perplexity_{mode}.json" if mode != "score" else out / "perplexity.json").write_text(json.dumps(d, indent=1))
    eng.close()


if __name__ == "__main__":
    main()
