"""GPU: bandwidth of the Q8_0 / Q5_1 GEMV at Qwen2.5-72B's ffn_down shape (K = 29568 -> N = 8192).  python tools/b32_probe.py"""
import ctypes as C, sys
from pathlib import Path
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
import torch
import pkgload
pkg = pkgload.load(); lib = pkg.Lib.get()
p = lambda a: C.c_void_p(a.data_ptr())
N, K = 8192, 29568
# 16-byte aligned weights take the bulk-copy ring kernel, 8-byte aligned ones the per-warp cp.async kernel k_gemv_blk32
for t, name in ((8, "q8_0"), (7, "q5_1")):
    rb = lib.c.pb200_row_bytes(t, K)
    copies = 8                                       # rotate through > L2 worth of weights
    W = [torch.randint(0, 255, (N * rb + 64,), dtype=torch.uint8, device="cuda") for _ in range(copies)]
    x = torch.randn(K, device="cuda"); y = torch.zeros(N, device="cuda")
    ws = torch.zeros(lib.c.pb200_act_workspace_bytes(K) + 64, dtype=torch.uint8, device="cuda")
    lib.check(lib.c.pb200_quantize_act(t, p(x), K, p(ws), None), "q")
    for off, kernel in ((0, "ring"), (8, "blk32")):
        w = lambda i: C.c_void_p(W[i % copies].data_ptr() + off)
        for i in range(4): lib.c.pb200_mul_mat_vec_q(t, w(i), N, K, p(ws), p(y), None, None, None)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = 32
        e0.record()
        for i in range(reps): lib.c.pb200_mul_mat_vec_q(t, w(i), N, K, p(ws), p(y), None, None, None)
        e1.record(); torch.cuda.synchronize()
        us = e0.elapsed_time(e1) / reps * 1e3
        print(f"{name} {kernel} N {N} K {K}: {us:.1f} us/launch  {N * rb / us / 1e6:.2f} TB/s", flush=True)
