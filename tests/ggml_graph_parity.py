"""Driver (run in a process of its own by tests/test_gpu_ggml_graph.py): a whole build_llama / build_qwen2 decode graph through
ggml_backend_graph_compute on the registered "B200_0" backend vs the reference CPU backend, same weights, same tokens, HOST tensors
in and out (ggml_backend_tensor_set / _get) — what llama_decode does.  Prints one JSON line.

    python tests/ggml_graph_parity.py <llama|qwen2> <n_tokens> [n_layer n_embd n_head n_head_kv n_ff n_vocab n_ctx]
    python tests/ggml_graph_parity.py <qwen2_q4_K_M|llama_q4_0> <n_tokens>     (a model of tiny_model.legacy_golden_models())

Script mode drives both backends through a list of steps the way llama_decode would: a prompt of n tokens at position pos is one
graph of n tokens (a decode step is n = 1), "clear" empties both KV caches.  Every step computes all its rows' logits.

    python tests/ggml_graph_parity.py <llama|qwen2> --script STEPS_JSON [--dims n_layer,n_embd,n_head,n_head_kv,n_ff,n_vocab,n_ctx]
                                      [--reserve N_TOKENS_MAX] [--dump FILE.npz]

STEPS_JSON is a JSON list of {"n": T, "pos": p} and "clear".  The compute buffers are reserved for the largest T of the script
unless --reserve says otherwise.  One JSON line per run with one entry per step; --dump also writes every step's logits of both
backends and the layer-0 K / V cache contents after it.
"""
import ctypes as C
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests")); sys.path.insert(0, str(ROOT / "host"))
from tiny_model import TinyModel, legacy_golden_models   # noqa: E402  (weights as raw GGUF blocks; loads no ggml)
import host_graph as HG            # noqa: E402

arch = sys.argv[1]
script_mode = sys.argv[2] == "--script"
opts = dict(zip(sys.argv[2::2], sys.argv[3::2])) if script_mode else {}
if script_mode:
    steps = json.loads(opts["--script"])
    n_tok = max([st["n"] for st in steps if st != "clear"])
    dims = [int(x) for x in opts["--dims"].split(",")] if "--dims" in opts else None
else:
    n_tok = int(sys.argv[2])
    dims = [int(x) for x in sys.argv[3:10]] if len(sys.argv) >= 10 else None
reserve = int(opts.get("--reserve", n_tok)) if script_mode else 1   # the token-by-token run keeps the one-token reservation
if arch in ("llama", "qwen2"):
    dims = dims or [3, 1024, 8, 2, 2816 if arch == "llama" else 3072, 384, 96]
    n_layer, n_embd, n_head, n_head_kv, n_ff, n_vocab, n_ctx = dims
    tm = TinyModel(n_layer=n_layer, n_embd=n_embd, n_head=n_head, n_head_kv=n_head_kv, n_ff=n_ff, n_vocab=n_vocab, n_ctx=n_ctx, arch=arch,
                   ftype="q4_K_M" if arch == "llama" else "q5_K_M", freq_factors=(arch == "llama"), seed=31, branch_scale=0.1)
else:
    tm = legacy_golden_models()[arch][0]
    n_layer, n_embd, n_head, n_head_kv, n_ff, n_vocab, n_ctx = (tm.hp[k] for k in ("n_layer", "n_embd", "n_head", "n_head_kv", "n_ff",
                                                                                   "n_vocab", "n_ctx"))
types = {name: t for name, (t, a) in tm.tensors.items() if name.endswith(".weight") and a.dtype == np.uint8}
has_bias = tm.arch == "qwen2"
has_ff = "rope_freqs.weight" in tm.tensors
g, plug = HG.load(with_plugin=True)
libpb = C.CDLL(str(ROOT / "prima.cpp_b200" / "libprima_b200.so"))
libpb.pb200_kernel_launches.restype = C.c_uint64
models = {}
for be in ("CPU", "B200_0"):
    m = HG.HostModel(tm.hp, types, be, n_threads=8, has_bias=has_bias, has_freq_factors=has_ff, n_tokens_max=reserve)
    for name, (t, a) in tm.tensors.items():
        m.set_tensor(name, a)
    models[be] = m
EK = n_head_kv * 128


def cache(be, il, nm):
    return models[be].get_tensor(f"blk.{il}.{nm}", EK * n_ctx * 2).view(np.float16).astype(np.float32)


if script_mode:
    toks = [(i * 7919 + 13) % n_vocab for i in range(n_ctx)]   # the token at a position does not depend on how the prompt is cut
    out_steps, dump = [], {}
    for si, st in enumerate(steps):
        if st == "clear":
            for m in models.values():
                m.kv_clear()
            out_steps.append({"clear": True})
            continue
        T, pos = st["n"], st["pos"]
        lg = {be: np.zeros((T, n_vocab), np.float32) for be in models}
        hd = {}
        r0, f0, n0 = plug.ggml_backend_b200_graph_replays(), plug.ggml_backend_b200_fused_steps(), libpb.pb200_kernel_launches()
        for be, m in models.items():
            m.decode(toks[pos:pos + T], pos, lg[be], all_logits=True)
            hd[be] = m.hidden(T)
        r1, f1, n1 = plug.ggml_backend_b200_graph_replays(), plug.ggml_backend_b200_fused_steps(), libpb.pb200_kernel_launches()
        a, b = lg["CPU"], lg["B200_0"]
        kv = {(be, il, nm): cache(be, il, nm) for be in models for il in range(n_layer) for nm in ("cache_k", "cache_v")}
        kv_err = [max(float(np.max(np.abs(kv[("CPU", il, nm)] - kv[("B200_0", il, nm)]))) for nm in ("cache_k", "cache_v")) for il in range(n_layer)]
        out_steps.append({"n": T, "pos": pos,
                          "max_abs_per_row": [float(x) for x in np.max(np.abs(a - b), axis=1)],
                          "nmse_per_row": [float(x) for x in np.sum((a - b) ** 2, axis=1) / np.sum(a ** 2, axis=1)],
                          "sq_err": float(np.sum((a.astype(np.float64) - b) ** 2)), "sq_ref": float(np.sum(a.astype(np.float64) ** 2)),
                          "argmax_agree_per_row": [bool(x) for x in a.argmax(1) == b.argmax(1)],
                          "hidden_max_abs": float(np.max(np.abs(hd["CPU"] - hd["B200_0"]))),
                          "graph_replays": int(r1 - r0), "fused_steps": int(f1 - f0), "launches": int(n1 - n0),
                          "unsupported_nodes": int(models["B200_0"].unsupported_nodes),
                          "buffer_base": int(models["B200_0"].compute_buffer_base),
                          "kv_max_abs": max(kv_err), "kv0_max_abs": kv_err[0]})
        if "--dump" in opts:
            for be in models:
                tag = "cpu" if be == "CPU" else "b200"
                dump[f"logits_{tag}_{si}"] = lg[be]
                dump[f"k0_{tag}_{si}"] = kv[(be, 0, "cache_k")].reshape(n_ctx, EK)    # row = cell
                dump[f"v0_{tag}_{si}"] = kv[(be, 0, "cache_v")].reshape(EK, n_ctx).T  # transposed cache: row = cell
    if "--dump" in opts:
        np.savez(opts["--dump"], **dump)
    print(json.dumps({"arch": arch, "n_layer": n_layer, "n_tokens_max": reserve, "steps": out_steps}))
    sys.exit(0)

toks = [(i * 7919 + 13) % n_vocab for i in range(n_tok)]
out = {be: np.zeros((n_tok, n_vocab), np.float32) for be in models}
hid = {be: np.zeros((n_tok, n_embd), np.float32) for be in models}
launches = []
fused0 = plug.ggml_backend_b200_fused_steps()
for i, t in enumerate(toks):
    for be, m in models.items():
        n0 = libpb.pb200_kernel_launches()
        m.decode([t], i, out[be][i])
        if be == "B200_0":
            launches.append(int(libpb.pb200_kernel_launches() - n0))
        hid[be][i] = m.hidden()[0]
kv_err = 0.0
for il in range(n_layer):
    for nm in ("cache_k", "cache_v"):
        kv_err = max(kv_err, float(np.max(np.abs(cache("CPU", il, nm) - cache("B200_0", il, nm)))))
e = np.max(np.abs(out["CPU"] - out["B200_0"]), axis=1)
res = {"arch": arch, "n_tokens": n_tok, "max_abs_per_token": [float(x) for x in e], "max_abs": float(e.max()), "first_token_err": float(e[0]),
       "nmse": float(np.sum((out["CPU"] - out["B200_0"]) ** 2) / np.sum(out["CPU"] ** 2)),
       "hidden_max_abs": float(np.max(np.abs(hid["CPU"] - hid["B200_0"]))), "kv_max_abs": kv_err,
       "argmax_agree": float(np.mean(out["CPU"].argmax(1) == out["B200_0"].argmax(1))),
       "launches_per_token": launches, "n_layer": n_layer, "graph_nodes": models["B200_0"].graph_nodes,
       "unsupported_nodes": int(models["B200_0"].unsupported_nodes),
       "fused_steps": int(plug.ggml_backend_b200_fused_steps() - fused0), "graph_builds": int(models["B200_0"].graph_builds),
       "graph_replays": int(plug.ggml_backend_b200_graph_replays()), "types": sorted({int(t) for t in types.values()})}
print(json.dumps(res))
