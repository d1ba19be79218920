"""CPU: llama-perplexity's chunk loop (prima.cpp_b200/perplexity.py) with a fake run_chunk, the pb200_token_score layout of the ctypes
binding, and PrefillPipeline's outputs hook over gloo at world 2 and 3."""
import ctypes as C
import io
import math
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import pkgload

pkg = pkgload.load()
PPL = pkg.perplexity


def fake_scores(tokens, first):
    """A deterministic nll per scored position p, from the target tokens[p + 1] and the position."""
    n_ctx = len(tokens)
    s = np.zeros(n_ctx - 1 - first, dtype=np.dtype(pkg.TokenScore))
    p = np.arange(first, n_ctx - 1)
    s["nll"] = 0.5 + (tokens[first + 1:].astype(np.float64) % 7) * 0.25 + p * 1e-3
    return s


def restated(tokens, n_ctx, n_chunk, bos):
    """The reference's arithmetic (perplexity.cpp:640-683) on fake_scores, summed serially."""
    nll = nll2 = 0.0
    count = 0
    running = []
    for i in range(n_chunk):
        ch = tokens[i * n_ctx:(i + 1) * n_ctx].copy()
        if bos is not None:
            ch[0] = bos
        for v in fake_scores(ch, n_ctx // 2)["nll"]:
            nll += v
            nll2 += v * v
            count += 1
        running.append(math.exp(nll / count))
    nll, nll2 = nll / count, nll2 / count
    ppl = math.exp(nll)
    return ppl, math.sqrt((nll2 - nll * nll) / (count - 1)) * ppl, count, running


@pytest.mark.parametrize("n_ctx,n_tok,n_chunks,bos", [(64, 200, -1, 1), (64, 200, 2, None), (9, 40, -1, 0), (512, 1100, 1, 128000)])
def test_chunk_loop(n_ctx, n_tok, n_chunks, bos):
    toks = (np.arange(n_tok) * 7919 + 13).astype(np.int32) % 1000 + 5
    calls = []

    def run_chunk(tokens, first):
        calls.append((tokens.copy(), first))
        return fake_scores(tokens, first)
    out = io.StringIO()
    res = PPL.perplexity(toks, n_ctx, run_chunk, n_chunks, bos, out=out)
    n_chunk = n_tok // n_ctx if n_chunks < 0 else min(n_chunks, n_tok // n_ctx)
    assert len(calls) == n_chunk
    for i, (t, first) in enumerate(calls):
        orig = toks[i * n_ctx:(i + 1) * n_ctx]
        assert first == n_ctx // 2 and len(t) == n_ctx
        assert t[0] == (orig[0] if bos is None else bos)       # BOS in the input ...
        assert np.array_equal(t[1:], orig[1:])                  # ... and every target is the original token
    ppl, unc, count, running = restated(toks, n_ctx, n_chunk, bos)
    assert count == res.count == n_chunk * (n_ctx - 1 - n_ctx // 2)
    assert res.ppl == pytest.approx(ppl, rel=1e-13) and res.uncertainty == pytest.approx(unc, rel=1e-9)
    assert res.chunk_ppl == pytest.approx(running, rel=1e-13)
    lines = out.getvalue().split("\n")
    assert lines[0] == "".join(f"[{i + 1}]{p:.4f}," for i, p in enumerate(res.chunk_ppl))
    assert lines[1] == f"Final estimate: PPL = {res.ppl:.4f} +/- {res.uncertainty:.5f}"


def test_chunk_loop_errors():
    toks = np.arange(127, dtype=np.int32)
    with pytest.raises(ValueError, match="at least 128 tokens"):
        PPL.perplexity(toks, 64, fake_scores, out=io.StringIO())
    with pytest.raises(ValueError, match="expected 31"):
        PPL.perplexity(np.arange(128), 64, lambda t, f: fake_scores(t, f)[1:], out=io.StringIO())
    assert PPL.perplexity(np.arange(128), 64, lambda t, f: None, out=io.StringIO()) is None   # a pipeline rank without the head


def test_token_score_layout():
    T = pkg.TokenScore
    assert C.sizeof(T) == 24
    assert [(n, getattr(T, n).offset) for n, _ in T._fields_] == [("nll", 0), ("logit", 8), ("prob", 12), ("top", 16), ("_pad", 20)]
    d = np.dtype(T)
    assert d.itemsize == 24 and d["nll"] == np.float64 and d["top"] == np.int32


# ---- PrefillPipeline's outputs hook ----
UB = 4


class ToyStage:
    """prefill_stage logs its call into a log shared with the outputs hook; hidden states are a toy function of the input."""

    def __init__(self, first, log):
        self.first, self.log = first, log
        self.hidden_buf = torch.zeros(UB, 3, dtype=torch.float64)

    def prefill_stage(self, tokens, hidden_in, n, pos0):
        self.log.append(("stage", pos0, n))
        x = torch.tensor([[float(t)] * 3 for t in tokens], dtype=torch.float64) if self.first else hidden_in.clone()
        return x * 1.5 + pos0


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _outputs_worker(rank, world, port, q, n_tokens):
    import sys
    from pathlib import Path
    sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
    import pkgload
    import torch.distributed as dist
    pkg = pkgload.load()
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    log = []
    st = ToyStage(rank == 0, log)
    pipe = pkg.PrefillPipeline(st, rank, world, dist, ubatch=UB)
    pipe.run(list(range(n_tokens)), n_tokens, pos0=3, outputs=lambda j0, n: log.append(("outputs", j0, n)))
    q.put((rank, log))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world,n_tokens", [(2, 10), (3, 8)])
def test_prefill_pipeline_outputs_hook(world, n_tokens):
    """outputs(j0, n) runs on the last rank only, once per micro-batch, in order, right after that micro-batch's prefill_stage."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_outputs_worker, args=(r, world, port, q, n_tokens)) for r in range(world)]
    [p.start() for p in procs]
    logs = dict(q.get(timeout=120) for _ in range(world))
    [p.join(60) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    mb = [(j0, min(UB, n_tokens - j0)) for j0 in range(0, n_tokens, UB)]
    for r in range(world - 1):
        assert logs[r] == [("stage", 3 + j0, n) for j0, n in mb]
    assert logs[world - 1] == [e for j0, n in mb for e in (("stage", 3 + j0, n), ("outputs", j0, n))]
