"""Driver (run in a process of its own by tests/test_gpu_legacy_types.py): one of the two golden legacy-type models
(tests/legacy_types.py: a Qwen2 Q4_K_M with a Q5_0 ffn_down, a llama Q4_0) decoded token by token through
ggml_backend_graph_compute on the registered "B200_0" backend and on the reference CPU backend, same weights, same tokens.  Prints one
JSON line.

    python tests/legacy_graph_parity.py <qwen2_q4_K_M|llama_q4_0> <n_tokens>
"""
import ctypes as C
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests")); sys.path.insert(0, str(ROOT / "host"))
import legacy_types as L                              # noqa: E402
import host_graph as HG                              # noqa: E402

name, n_tok = sys.argv[1], int(sys.argv[2])
tm, toks = L.models()[name]
toks = toks[:n_tok]
types = {k: t for k, (t, a) in tm.tensors.items() if k.endswith(".weight") and a.dtype == np.uint8}
g, plug = HG.load(with_plugin=True)
libpb = C.CDLL(str(ROOT / "prima.cpp_b200" / "libprima_b200.so"))
libpb.pb200_kernel_launches.restype = C.c_uint64
models = {}
for be in ("CPU", "B200_0"):
    m = HG.HostModel(tm.hp, types, be, n_threads=8, has_bias=tm.arch == "qwen2", has_freq_factors=False, n_tokens_max=1)
    for k, (t, a) in tm.tensors.items():
        m.set_tensor(k, a)
    models[be] = m
nv = tm.hp["n_vocab"]
out = {be: np.zeros((len(toks), nv), np.float32) for be in models}
launches = []
for i, t in enumerate(toks):
    for be, m in models.items():
        n0 = libpb.pb200_kernel_launches()
        m.decode([t], i, out[be][i])
        if be == "B200_0":
            launches.append(int(libpb.pb200_kernel_launches() - n0))
a, b = out["CPU"], out["B200_0"]
e = np.max(np.abs(a - b), axis=1)
print(json.dumps({"model": name, "n_tokens": len(toks), "max_abs": float(e.max()), "first_token_err": float(e[0]),
                  "nmse": float(np.sum((a - b) ** 2) / np.sum(a ** 2)), "argmax_agree": float(np.mean(a.argmax(1) == b.argmax(1))),
                  "unsupported_nodes": int(models["B200_0"].unsupported_nodes), "launches_per_token": launches,
                  "types": sorted({int(t) for t in types.values()})}))
