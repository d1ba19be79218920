"""-m gpu: sequence slots of the engine, device-resident token / position / greedy argmax, and (with >= 2 GPUs) the ring of
sequences across NCCL ranks against single-process decoding — bit for bit (same kernels, same order; SURVEY §8e)."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch

from tiny_model import TinyModel

pytestmark = pytest.mark.gpu


def _model(n_layer=4):
    return TinyModel(n_layer=n_layer, n_embd=512, n_head=4, n_head_kv=2, n_ff=1024, n_vocab=320, n_ctx=48, seed=9, branch_scale=0.3)


def _i32(ptr):
    class V:
        __cuda_array_interface__ = {"shape": (1,), "typestr": "<i4", "data": (ptr, False), "version": 2}
    return torch.as_tensor(V(), device="cuda")


def _load(tm, pkg, n_seq, **kw):
    hp = pkg.HParams(**tm.hp)
    eng = pkg.Model(hp, 0, kw.get("layers"), kw.get("with_embd", True), kw.get("with_head", True))
    for name, (t, a) in tm.tensors.items():
        eng.set_tensor(name, t, a)
    eng.set_n_seq(n_seq)
    eng.finalize()
    return eng


def greedy_reference(tm, pkg, seeds, rounds):
    """Single process, one sequence slot per seed, host-driven greedy decoding through pb200_decode."""
    out = []
    for tok, pos in seeds:
        eng = tm.load_engine(pkg)
        logits = np.zeros(tm.hp["n_vocab"], np.float32)
        hist = []
        for _ in range(rounds):
            eng.decode(tok, pos, logits)
            tok = int(logits.argmax()); pos += 1
            hist.append(tok)
        eng.close()
        out.append(hist)
    return out


def test_sequence_slots_are_independent_and_device_argmax_matches(cuda, pkg):
    tm = _model()
    seeds = [(5, 0), (77, 3), (200, 1)]
    want = greedy_reference(tm, pkg, seeds, 6)
    eng = _load(tm, pkg, len(seeds))
    toks = [_i32(eng.token_ptr(s)) for s in range(len(seeds))]
    smps = [_i32(eng.sample_ptr(s)) for s in range(len(seeds))]
    for s, (tok, pos) in enumerate(seeds):
        eng.set_tokpos_seq(s, tok, pos)
    got = [[] for _ in seeds]
    for _ in range(6):                       # interleaved slots, nothing but the final read-back crosses the host
        for s in range(len(seeds)):
            eng.step_seq_dev(s, True)
            eng.argmax_seq(s, True)          # feeds the sample back into the slot's token on the device
        eng.synchronize()
        for s in range(len(seeds)):
            got[s].append(int(smps[s].item()))
            assert int(toks[s].item()) == got[s][-1]
    eng.close()
    assert got == want


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _ring_rank(rank, world, port, rounds, q):
    import sys
    from pathlib import Path
    root = Path(__file__).resolve().parent.parent
    sys.path.insert(0, str(root)); sys.path.insert(0, str(root / "tests"))
    import pkgload
    import torch.distributed as dist
    pkg = pkgload.load()
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    tm = _model()
    b = pkg.layer_windows(tm.hp["n_layer"], world)
    hp = pkg.HParams(**tm.hp)
    eng = pkg.Model(hp, rank, (b[rank], b[rank + 1]), rank == 0, rank == world - 1)
    for name, (t, a) in tm.tensors.items():
        eng.set_tensor(name, t, a)
    eng.set_n_seq(world)
    eng.finalize()
    dev = torch.device("cuda", rank)
    E = tm.hp["n_embd"]

    class F32:
        def __init__(self, ptr, n):
            self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (ptr, False), "version": 2}

    class I32:
        def __init__(self, ptr):
            self.__cuda_array_interface__ = {"shape": (1,), "typestr": "<i4", "data": (ptr, False), "version": 2}

    hist = [[] for _ in range(world)]

    class Stage:
        hidden_in = torch.as_tensor(F32(eng.hidden_in_ptr, E), device=dev)
        hidden_out = torch.as_tensor(F32(eng.hidden_out_ptr, E), device=dev)
        tin = [torch.as_tensor(I32(eng.token_ptr(s)), device=dev) for s in range(world)]
        tout = [torch.as_tensor(I32(eng.sample_ptr(s)), device=dev) for s in range(world)]

        def token_in(self, s): return self.tin[s]
        def token_out(self, s): return self.tout[s]
        def begin(self, s, token, pos): eng.set_tokpos_seq(s, token, pos)

        def run(self, s):
            eng.step_seq_dev(s, True)
            if rank == world - 1:
                eng.argmax_seq(s, False)
                eng.synchronize()
                hist[s].append(int(self.tout[s].item()))

    ext = torch.cuda.ExternalStream(eng.stream, device=dev)
    rr = pkg.RingRunner(Stage(), rank, world, dist)
    with torch.cuda.stream(ext):
        rr.slots(world * rounds + world - 1, first_tokens=[(5 + 9 * s, s) for s in range(world)])
    torch.cuda.synchronize()
    if rank == world - 1:
        q.put(hist)
    dist.barrier()
    eng.close()
    dist.destroy_process_group()


def test_ring_across_nccl_ranks_bit_identical_to_single_process(cuda, pkg):
    world = 2
    if torch.cuda.device_count() < world:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    rounds = 5
    want = greedy_reference(_model(), pkg, [(5 + 9 * s, s) for s in range(world)], rounds)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_ring_rank, args=(r, world, port, rounds, q)) for r in range(world)]
    [p.start() for p in procs]
    got = q.get(timeout=300)
    [p.join(120) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    assert [h[:rounds] for h in got] == want
