"""llama-perplexity's chunk loop (examples/perplexity/perplexity.cpp:475-687) as host logic over a run_chunk callable, and run_chunk for a
whole model and for the last rank of a layer pipeline.

The token ids are split into chunks of n_ctx tokens.  Each chunk is evaluated from position 0 (with its first token replaced by BOS when
one is given) and positions [first, n_ctx - 1), first = n_ctx // 2, are scored against the ORIGINAL next token, so every scored position
has at least n_ctx // 2 tokens of context.  run_chunk(tokens, first) gets the chunk's input ids (n_ctx of them) and returns one
TokenScore record per scored position p, scored against tokens[p + 1] (positions >= first >= 1 never read the BOS-replaced token 0), or
None on a pipeline rank that does not hold the head.

Not provided: ppl_stride (perplexity_v2), KL-divergence, HellaSwag / Winogrande / multiple choice, several chunks as sequences of one
batch, and tokenization (token ids come from the caller)."""
from __future__ import annotations

import math
import sys
from dataclasses import dataclass, field

import numpy as np


@dataclass
class Result:
    ppl: float                  # exp(mean nll)
    nll: float                  # mean nll over the scored positions
    uncertainty: float | None   # the reference's +/- on ppl (None where its variance estimate is not positive)
    count: int                  # scored positions
    chunk_ppl: list = field(default_factory=list)   # running ppl after each chunk, the numbers of the [i]ppl, lines


def perplexity(tokens, n_ctx: int, run_chunk, n_chunks: int = -1, bos: int | None = None, out=None) -> Result | None:
    """The reference's perplexity() over token ids: at least 2 * n_ctx tokens, len // n_ctx chunks (at most n_chunks when n_chunks >= 0).
    nll and nll^2 accumulate in double.  out (default stdout) gets the reference's output: "[i]ppl," after each chunk on one line, then
    "Final estimate: PPL = ... +/- ...".  Returns None when run_chunk returns None (a pipeline rank without the head)."""
    out = out or sys.stdout
    tokens = np.asarray(tokens, dtype=np.int32)
    if n_ctx < 3:
        raise ValueError(f"n_ctx {n_ctx}: a chunk needs at least 3 tokens to score one")
    if len(tokens) < 2 * n_ctx:
        raise ValueError(f"you need at least {2 * n_ctx} tokens to evaluate perplexity with a context of {n_ctx} (got {len(tokens)})")
    n_chunk_max = len(tokens) // n_ctx
    n_chunk = n_chunk_max if n_chunks < 0 else min(n_chunks, n_chunk_max)
    first = n_ctx // 2
    nll = nll2 = 0.0
    count = 0
    res = Result(0.0, 0.0, None, 0)
    for i in range(n_chunk):
        chunk = tokens[i * n_ctx:(i + 1) * n_ctx].copy()
        if bos is not None:
            chunk[0] = bos
        s = run_chunk(chunk, first)
        if s is None:
            return None
        v = np.asarray(s["nll"], dtype=np.float64)
        if v.shape != (n_ctx - 1 - first,):
            raise ValueError(f"run_chunk returned {v.shape} scores, expected {n_ctx - 1 - first}")
        nll += float(v.sum())
        nll2 += float((v * v).sum())
        count += v.size
        res.chunk_ppl.append(math.exp(nll / count))
        out.write(f"[{i + 1}]{res.chunk_ppl[-1]:.4f},")
        out.flush()
    out.write("\n")
    nll /= count
    nll2 /= count
    res.ppl, res.nll, res.count = math.exp(nll), nll, count
    nll2 -= nll * nll
    if nll2 > 0:
        res.uncertainty = math.sqrt(nll2 / (count - 1)) * res.ppl
        out.write(f"Final estimate: PPL = {res.ppl:.4f} +/- {res.uncertainty:.5f}\n")
    else:
        out.write("Unexpected negative standard deviation of log(prob)\n")
    return res


def _scored_rows(j0: int, n: int, first: int, n_ctx: int):
    """Rows [a - j0, b - j0) of the micro-batch [j0, j0 + n) hold the scored positions [a, b), or None."""
    a, b = max(first, j0), min(j0 + n, n_ctx - 1)
    return (a, b) if a < b else None


def model_run_chunk(model, ubatch: int = 512):
    """run_chunk for a whole model (Model): the chunk is prefilled in ubatches of at most 512 tokens at positions 0.., each followed by
    prompt_head on its scored rows.  No kv_clear is needed between chunks: the engine keeps cell == position, and every cell a chunk
    reads has been rewritten by that chunk first."""
    def run_chunk(tokens, first):
        n_ctx, out = len(tokens), []
        for j0 in range(0, n_ctx, ubatch):
            n = min(ubatch, n_ctx - j0)
            model.prefill(tokens[j0:j0 + n], j0)
            ab = _scored_rows(j0, n, first, n_ctx)
            if ab:
                out.append(model.prompt_head(ab[0] - j0, ab[1] - ab[0], targets=tokens[ab[0] + 1:ab[1] + 1], logits=False)[1])
        return np.concatenate(out)
    return run_chunk


def pipeline_run_chunk(pipe, model=None):
    """run_chunk for one rank of a PrefillPipeline (call it on every rank with the same chunks).  model: this rank's Model on the last
    rank, whose prompt_head scores each micro-batch from the pipeline's outputs hook; the other ranks pass None and get None back."""
    last = pipe.rank == pipe.world - 1

    def run_chunk(tokens, first):
        n_ctx, out = len(tokens), []

        def outputs(j0, n):
            ab = _scored_rows(j0, n, first, n_ctx)
            if ab:
                out.append(model.prompt_head(ab[0] - j0, ab[1] - ab[0], targets=tokens[ab[0] + 1:ab[1] + 1], logits=False)[1])

        pipe.run(tokens, n_ctx, 0, outputs=outputs if last else None)
        return np.concatenate(out) if last else None
    return run_chunk
