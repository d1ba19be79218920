"""Driver (run in a process of its own by tests/test_gpu_kv_shift.py): llama-cli's context shift through the drop-in boundary.  The host
stand-in (host/llama_graph_host.cpp) keeps the reference's cell bookkeeping; both the registered "B200_0" backend and the reference CPU
backend run a prompt, then decode steps, and whenever the context is full they get llama_kv_cache_seq_rm + seq_add
(examples/main/main.cpp:578-608).  The next decode runs the K-shift graph (one in-place f16 ROPE per layer) and places new tokens in
the freed cells, below the live shifted ones.  Prints one JSON line.

    python tests/ggml_kshift_parity.py <llama|qwen2> <n_head_kv> <n_keep> <n_shifts>
"""
import ctypes as C
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests")); sys.path.insert(0, str(ROOT / "host"))
from tiny_model import TinyModel   # noqa: E402  (weights as raw GGUF blocks; loads no ggml)
import host_graph as HG            # noqa: E402

arch, n_head_kv, n_keep, n_shifts = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4])
n_layer, n_embd, n_head, n_vocab, n_ctx, PROMPT = 3, 1024, 8, 384, 64, 8
n_ff = 2816 if arch == "llama" else 3072
tm = TinyModel(n_layer=n_layer, n_embd=n_embd, n_head=n_head, n_head_kv=n_head_kv, n_ff=n_ff, n_vocab=n_vocab, n_ctx=n_ctx, arch=arch,
               ftype="q4_K_M" if arch == "llama" else "q5_K_M", freq_factors=(arch == "llama"), seed=31, branch_scale=0.1)
types = {name: t for name, (t, a) in tm.tensors.items() if name.endswith(".weight") and a.dtype == np.uint8}
g, plug = HG.load(with_plugin=True)
plug.ggml_backend_b200_nodes_computed.restype = C.c_ulonglong
models = {}
for be in ("CPU", "B200_0"):
    m = HG.HostModel(tm.hp, types, be, n_threads=8, has_bias=(arch == "qwen2"), has_freq_factors=("rope_freqs.weight" in tm.tensors), n_tokens_max=PROMPT)
    for name, (t, a) in tm.tensors.items():
        m.set_tensor(name, a)
    m.kv_clear()
    models[be] = m
EK = n_head_kv * 128


def cache(be, il):
    return models[be].get_tensor(f"blk.{il}.cache_k", EK * n_ctx * 2).view(np.float16).astype(np.float32)


def token(i):
    return (i * 7919 + 13) % n_vocab


steps = []
n_past, i, shifts_done, after_last = 0, 0, 0, 0
shift_pending = False
while after_last < 20:
    if n_past == 0:
        T, toks = PROMPT, [token(j) for j in range(PROMPT)]
    else:
        T, toks = 1, [token(i)]
        if n_past + T >= n_ctx:   # llama-cli's context shift
            n_discard = (n_past - n_keep) // 2
            for m in models.values():
                m.kv_seq_rm(n_keep, n_keep + n_discard)
                m.kv_seq_add(n_keep + n_discard, n_past, -n_discard)
            n_past -= n_discard
            shifts_done += 1
            shift_pending = True
    lg = {be: np.zeros((T, n_vocab), np.float32) for be in models}
    r0, f0, n0 = plug.ggml_backend_b200_graph_replays(), plug.ggml_backend_b200_fused_steps(), plug.ggml_backend_b200_nodes_computed()
    for be, m in models.items():
        m.decode(toks, n_past, lg[be], all_logits=True)
    r1, f1, n1 = plug.ggml_backend_b200_graph_replays(), plug.ggml_backend_b200_fused_steps(), plug.ggml_backend_b200_nodes_computed()
    cells = {be: m.kv_cells() for be, m in models.items()}
    a, b = lg["CPU"], lg["B200_0"]
    cell = int(np.where(cells["B200_0"] == n_past + T - 1)[0][0])
    live = np.where(cells["B200_0"] >= 0)[0]
    st = {"n": T, "pos": n_past, "shift": shift_pending, "cell": cell, "live_above": int((live > cell).sum()),
          "cells_equal": bool(np.array_equal(cells["CPU"], cells["B200_0"])),
          "max_abs_per_row": [float(x) for x in np.max(np.abs(a - b), axis=1)],
          "sq_err": float(np.sum((a.astype(np.float64) - b) ** 2)), "sq_ref": float(np.sum(a.astype(np.float64) ** 2)),
          "argmax_agree_per_row": [bool(x) for x in a.argmax(1) == b.argmax(1)],
          "graph_replays": int(r1 - r0), "fused_steps": int(f1 - f0), "nodes": int(n1 - n0),
          "unsupported_nodes": int(models["B200_0"].unsupported_nodes)}
    if shift_pending:
        st["kv_max_abs"] = max(float(np.max(np.abs(cache("CPU", il) - cache("B200_0", il)))) for il in range(n_layer))
    steps.append(st)
    shift_pending = False
    n_past += T
    i += T
    if shifts_done >= n_shifts:
        after_last += 1
print(json.dumps({"arch": arch, "n_layer": n_layer, "n_head_kv": n_head_kv, "shifts": shifts_done,
                  "k_shifts": {be: int(m.k_shifts) for be, m in models.items()},
                  "kshift_nodes": int(models["B200_0"].kshift_nodes), "kshift_unsupported": int(models["B200_0"].kshift_unsupported_nodes),
                  "steps": steps}))
