"""CPU: ring sequences that start from prompts (RingRunner.prefill), the KV copy between sequences (RingRunner.copy) and the slot argument
of PrefillPipeline, over gloo at world 2 and 3, against one process that runs every layer.

The toy stage keeps a per-slot cache of each layer's inputs and lets every token read the cells [0, pos] of its slot, so a prompt that
went to the wrong slot, a wrong position, a copy at the wrong point or of the wrong cells all change the tokens.  Every token is computed
with the same operations whether it comes in a prompt micro-batch or as a single step, so the results are bit-identical."""
import os
import socket

import pytest
import torch
import torch.multiprocessing as mp

E, V, L, N_CTX, UB = 16, 11, 6, 64, 4


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


class ToyPromptStage:
    """Layers [l0, l1) of a toy model with a cache per sequence slot: layer l stores its input x at cell pos of the slot and returns
    tanh(W_l x + 0.1 * sum of the slot's cells [0, pos]) + 0.01 * pos.  The RingRunner / PrefillPipeline stage interface."""

    def __init__(self, l0, l1, first, last, n_seq):
        g = torch.Generator().manual_seed(0)
        self.W = [torch.randn(E, E, generator=g) / 4 for _ in range(L)]
        self.emb = torch.randn(V, E, generator=g)
        self.head = torch.randn(V, E, generator=g)
        self.l0, self.l1, self.first, self.last = l0, l1, first, last
        self.cache = [torch.zeros(L, N_CTX, E) for _ in range(n_seq)]
        self.hidden_in, self.hidden_out, self.logits = torch.zeros(E), torch.zeros(E), torch.zeros(V)
        self.hidden_buf = torch.zeros(UB, E)
        self.tok = [torch.zeros(1, dtype=torch.int32) for _ in range(n_seq)]
        self.smp = [torch.zeros(1, dtype=torch.int32) for _ in range(n_seq)]
        self.pos = [0] * n_seq
        self.history = [[] for _ in range(n_seq)]
        self.copy_log = []

    def _layers(self, x, s, p):
        for l in range(self.l0, self.l1):
            self.cache[s][l, p] = x
            x = torch.tanh(self.W[l] @ x + 0.1 * self.cache[s][l, :p + 1].sum(0)) + 0.01 * p
        return x

    def prefill_stage(self, tokens, hidden_in, n, pos0, seq=0):
        out = torch.zeros(n, E)
        for i in range(n):
            x = self.emb[int(tokens[i])].clone() if self.first else hidden_in[i].clone()
            out[i] = self._layers(x, seq, pos0 + i)
        if self.last:
            self.logits.copy_(self.head @ out[n - 1])
        return out

    def token_in(self, s):
        return self.tok[s]

    def token_out(self, s):
        return self.smp[s]

    def begin(self, s, token, pos):
        self.tok[s][0] = token
        self.pos[s] = pos

    def sample(self, s):
        self.smp[s][0] = int(torch.argmax(self.logits))
        self.history[s].append(int(self.smp[s][0]))

    def run(self, s):
        x = self.emb[int(self.tok[s][0])].clone() if self.first else self.hidden_in.clone()
        y = self._layers(x, s, self.pos[s])
        self.hidden_out.copy_(y)
        self.pos[s] += 1
        if self.last:
            self.logits.copy_(self.head @ y)
            self.sample(s)

    def kv_copy(self, src, dst, p0, p1):
        self.copy_log.append((src, dst, self.pos[src], self.pos[dst]))
        p0 = max(p0, 0)
        p1 = N_CTX if p1 < 0 or p1 > N_CTX else p1
        if src != dst and p0 < p1:
            self.cache[dst][:, p0:p1] = self.cache[src][:, p0:p1]


def prompts_for(world):
    return [[(5 * s + 3 * i + 1) % V for i in range(6 + 3 * s)] for s in range(world)]   # lengths 6, 9, 12: one to three micro-batches


def reference(prompts, rounds, copies=()):
    """One stage with every layer: each prompt into its slot and its first token, then rounds of one step per sequence in ring order
    (sequence 0, 1, ...), each copy (src, dst, at_step, p0, p1) applied right before step at_step of dst."""
    n = len(prompts)
    st = ToyPromptStage(0, L, True, True, n)
    for s, p in enumerate(prompts):
        st.prefill_stage(p, None, len(p), 0, seq=s)
        st.begin(s, 0, len(p))
        st.sample(s)
        st.tok[s][0] = st.smp[s][0]
    for k in range(rounds):
        for s in range(n):
            for src, dst, at, p0, p1 in copies:
                if dst == s and at == k:
                    st.kv_copy(src, dst, p0, p1)
            st.run(s)
            st.tok[s][0] = st.smp[s][0]
    return st.history, st.copy_log


def _worker(rank, world, port, q, rounds, copies):
    import sys
    from pathlib import Path
    sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
    import pkgload
    import torch.distributed as dist
    pkg = pkgload.load()
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    b = pkg.layer_windows(L, world)
    st = ToyPromptStage(b[rank], b[rank + 1], rank == 0, rank == world - 1, world)
    rr = pkg.RingRunner(st, rank, world, dist)
    rr.prefill(prompts_for(world), ubatch=UB)
    for c in copies:
        rr.copy(*c)
    rr.slots(world * rounds + world - 1)          # + world - 1: let the last stage finish the last round
    q.put((rank, st.history, st.copy_log, st.pos))
    dist.barrier()
    dist.destroy_process_group()


def _run(world, target, *args):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=target, args=(r, world, port, q) + args) for r in range(world)]
    [p.start() for p in procs]
    got = sorted([q.get(timeout=120) for _ in range(world)], key=lambda x: x[0])
    [p.join(60) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    return got


@pytest.mark.parametrize("world", [2, 3])
def test_ring_prefill_then_slots_matches_single_stage(world):
    rounds = 5
    want, _ = reference(prompts_for(world), rounds)
    got = _run(world, _worker, rounds, [])
    hist = got[-1][1]
    assert [h[:rounds + 1] for h in hist] == want               # the first token of every sequence comes from its prompt
    for _, _, _, pos in got:                                     # the last stage ran `rounds` steps of every sequence from len(prompt) on
        assert all(pos[s] >= len(p) + rounds for s, p in enumerate(prompts_for(world)))
    assert got[-1][3] == [len(p) + rounds for p in prompts_for(world)]


@pytest.mark.parametrize("world", [2, 3])
def test_ring_copy_lands_between_the_same_two_tokens_on_every_rank(world):
    rounds = 5
    # sequence 0's first 6 cells (its whole prompt) into sequence 1 before its step 2; all of sequence 1 into the last one before step 3
    copies = [(0, 1, 2, 0, 6), (1, world - 1, 3, -1, -1)]
    want, want_log = reference(prompts_for(world), rounds, copies)
    plain, _ = reference(prompts_for(world), rounds)
    assert want != plain                                         # the copies change the tokens that follow them
    got = _run(world, _worker, rounds, copies)
    assert [h[:rounds + 1] for h in got[-1][1]] == want
    for _, _, log, _ in got:                                     # the same positions of src and dst at the copy on every rank
        assert log == want_log


def _four_arg_worker(rank, world, port, q, n_tokens):
    import sys
    from pathlib import Path
    sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
    import pkgload
    import torch.distributed as dist
    pkg = pkgload.load()
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    b = pkg.layer_windows(L, world)
    toy = ToyPromptStage(b[rank], b[rank + 1], rank == 0, rank == world - 1, 1)

    class FourArgStage:   # the shape of bench.py's adapter: prefill_stage(tokens, hidden_in, n, pos), slot 0 only
        hidden_buf = toy.hidden_buf

        def prefill_stage(self, tokens, hidden_in, n, pos):
            return toy.prefill_stage(tokens, hidden_in, n, pos)

    pipe = pkg.PrefillPipeline(FourArgStage(), rank, world, dist, ubatch=UB)
    toks = [(7 * i + 3) % V for i in range(n_tokens)]
    out = pipe.run(toks, n_tokens, 2)
    q.put((rank, out.clone(), toy.logits.clone()))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_prefill_pipeline_keeps_four_argument_stages(world):
    n = 10
    single = ToyPromptStage(0, L, True, True, 1)
    toks = [(7 * i + 3) % V for i in range(n)]
    want = single.prefill_stage(toks, None, n, 2)
    got = _run(world, _four_arg_worker, n)
    _, out, logits = got[-1]
    assert torch.equal(out, want[8:]) and torch.equal(logits, single.logits)


def test_ring_prefill_argument_rules(pkg):
    st = ToyPromptStage(0, L, True, True, 2)
    rr = pkg.RingRunner(st, 0, 2, dist=object())
    with pytest.raises(ValueError):
        rr.prefill([[1, 2]])                                     # one prompt per sequence
    with pytest.raises(ValueError):
        rr.prefill([[1, 2], []])
    rr.t = 1
    with pytest.raises(ValueError):
        rr.prefill([[1, 2], [3]])                                # after the first slots()
    rr.runs[1] = 3
    with pytest.raises(ValueError):
        rr.copy(0, 1, 2)                                         # sequence 1 is already past step 2
