"""CPU: the host side of the context shift.  RingRunner.shift lands between the same two tokens of a sequence on every rank of the ring
(gloo, world 2 and 3, fake stages), also while the ring fills; pb200_kv_seq_shift / pb200_rope_f16 reject bad arguments without a GPU."""
import ctypes as C
import os
import socket

import pytest
import torch
import torch.multiprocessing as mp

ROUNDS = 7
N_KEEP = 1


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def shifts_for(world):
    """(seq, at_step, p0, p1, delta): sequence s is shifted before its run number at_step; at_step 0 and 1 fall into the ring's fill
    on the later ranks."""
    out = []
    for s in range(world):
        at = [0, 1, 3][s % 3]
        out.append((s, at, 1, 2 * s + at + 1, -1))     # sequence 0 at step 0 sits at position 0 < p0: its position stays
        out.append((s, 5, 2 * s + 3, 2 * s + 5, -2))
    return out


class ShiftStage:
    """Stands in for the engine: layer l mixes the hidden state with a fixed matrix and adds the position, so a shift (which moves the
    sequence's position like pb200_kv_seq_shift does) applied at a different token on one rank changes the result."""
    E, V, L = 12, 13, 6

    def __init__(self, l0, l1, first, last, n_seq):
        g = torch.Generator().manual_seed(0)
        self.W = [torch.randn(self.E, self.E, generator=g) / 4 for _ in range(self.L)]
        self.emb = torch.randn(self.V, self.E, generator=g)
        self.head = torch.randn(self.V, self.E, generator=g)
        self.l0, self.l1, self.first, self.last = l0, l1, first, last
        self.hidden_in, self.hidden_out, self.logits = torch.zeros(self.E), torch.zeros(self.E), torch.zeros(self.V)
        self.tok = [torch.zeros(1, dtype=torch.int32) for _ in range(n_seq)]
        self.smp = [torch.zeros(1, dtype=torch.int32) for _ in range(n_seq)]
        self.pos = [0] * n_seq
        self.runs = [0] * n_seq
        self.events = []                 # ("shift", seq, runs of seq so far)
        self.history = [[] for _ in range(n_seq)]

    def layers(self, x, pos):
        for l in range(self.l0, self.l1):
            x = torch.tanh(self.W[l] @ x) + 0.01 * pos
        return x

    def token_in(self, s): return self.tok[s]
    def token_out(self, s): return self.smp[s]

    def begin(self, s, token, pos):
        self.tok[s][0] = token
        self.pos[s] = pos

    def kv_shift(self, s, p0, p1, delta):
        self.events.append(("shift", s, self.runs[s]))
        if self.pos[s] >= p0:
            self.pos[s] += delta

    def run(self, s):
        x = self.emb[int(self.tok[s][0])].clone() if self.first else self.hidden_in.clone()
        x = self.layers(x, self.pos[s])
        self.hidden_out.copy_(x)
        self.pos[s] += 1
        self.runs[s] += 1
        if self.last:
            self.smp[s][0] = int(torch.argmax(self.head @ x))
            self.history[s].append(int(self.smp[s][0]))


def _worker(rank, world, port, q):
    import sys
    from pathlib import Path
    sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
    import pkgload
    import torch.distributed as dist
    pkg = pkgload.load()
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    b = pkg.layer_windows(ShiftStage.L, world)
    st = ShiftStage(b[rank], b[rank + 1], rank == 0, rank == world - 1, world)
    rr = pkg.RingRunner(st, rank, world, dist)
    for sh in shifts_for(world):
        rr.shift(*sh)
    seeds = [(3 + s, 2 * s) for s in range(world)]
    rr.slots(world * ROUNDS + world - 1, first_tokens=seeds)
    q.put((rank, st.events, st.history if rank == world - 1 else None, rr.shifts))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_ring_shift_lands_between_the_same_tokens_on_every_rank(world):
    # single process: sequence s decoded token by token, shifted before its token number at_step
    want = []
    for s in range(world):
        st = ShiftStage(0, ShiftStage.L, True, True, 1)
        tok, pos, hist = 3 + s, 2 * s, []
        for k in range(ROUNDS):
            for (sq, at, p0, p1, delta) in shifts_for(world):
                if sq == s and at == k and pos >= p0:
                    pos += delta
            x = st.layers(st.emb[tok].clone(), pos)
            tok = int(torch.argmax(st.head @ x)); pos += 1
            hist.append(tok)
        want.append(hist)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    [p.start() for p in procs]
    res = [q.get(timeout=120) for _ in range(world)]
    [p.join(60) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    expect = sorted(("shift", s, at) for (s, at, *_rest) in shifts_for(world))
    for rank, events, hist, pending in res:
        assert sorted(events) == expect, (rank, events)          # every rank applied every shift right before run number at_step
        assert all(not v for v in pending.values()), pending
        if hist is not None:
            assert [h[:ROUNDS] for h in hist] == want


def test_ring_shift_in_the_past_is_refused(pkg):
    class Dist:
        pass
    rr = pkg.RingRunner(object(), 0, 2, Dist())
    rr.runs[1] = 4
    with pytest.raises(ValueError):
        rr.shift(1, 3, 10, 20, -5)
    rr.shift(1, 4, 10, 20, -5)
    assert rr.shifts[1] == [(4, 10, 20, -5)]


def test_kv_seq_shift_argument_errors(lib):
    c = lib.c
    EINVAL, ESTATE = -1, -4
    assert c.pb200_kv_seq_shift(None, 0, 10, 20, 0) == EINVAL       # delta must be negative (positive shifts are not supported)
    assert c.pb200_kv_seq_shift(None, 0, 10, 20, 3) == EINVAL
    assert c.pb200_kv_seq_shift(None, 0, 10, 20, -11) == EINVAL     # p0 + delta < 0
    assert c.pb200_kv_seq_shift(None, 0, 20, 20, -5) == EINVAL      # empty range
    assert c.pb200_kv_seq_shift(None, 0, 21, 20, -5) == EINVAL
    assert c.pb200_kv_seq_shift(None, 0, 10, 20, -10) == ESTATE     # valid arguments, no model
    assert c.pb200_kv_device(None, 0) is None
    assert c.pb200_rope_f16(None, None, 1, 1, 128, 128, 0, None, 1e4, 1.0, 0.0, 1.0, 32.0, 1.0, 4096, None, None) == EINVAL
    x = C.c_void_p(256)
    assert c.pb200_rope_f16(x, x, 1, 1, 64, 128, 0, x, 1e4, 1.0, 0.0, 1.0, 32.0, 1.0, 4096, None, None) == EINVAL   # n_dims > head_dim
    assert c.pb200_rope_f16(x, x, 1, 1, 128, 63, 0, x, 1e4, 1.0, 0.0, 1.0, 32.0, 1.0, 4096, None, None) == EINVAL   # odd n_dims
    assert c.pb200_rope_f16(x, x, 0, 1, 128, 128, 0, x, 1e4, 1.0, 0.0, 1.0, 32.0, 1.0, 4096, None, None) == EINVAL  # no rows
