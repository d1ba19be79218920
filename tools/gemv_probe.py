"""GPU: the k-quant GEMV at the Llama-3-70B launch shapes, back to back through the C ABI (events), and the target of the ncu captures:

    ncu --set full --clock-control none --import-source on -k regex:k_gemv_kquant -s 10 -c 5 -o gemv python tools/gemv_probe.py 1
"""
import sys, ctypes as C
from pathlib import Path
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
import torch
import pkgload
pkg = pkgload.load(); lib = pkg.Lib.get()
reps = int(sys.argv[1]) if len(sys.argv) > 1 else 30
Q4, Q5, Q6 = 12, 13, 14
pool = torch.randint(0, 255, (3 << 30,), dtype=torch.uint8, device="cuda")
shapes = [("qkv", 8192, [(Q4, 8192), (Q4, 1024), (Q5, 1024)]), ("wo", 8192, [(Q4, 8192)]), ("gate|up", 8192, [(Q4, 28672), (Q4, 28672)]),
          ("down q4", 28672, [(Q4, 8192)]), ("down q6", 28672, [(Q6, 8192)]), ("head", 8192, [(Q6, 128256)])]
y = torch.zeros(1 << 20, device="cuda")
for name, K, mats in shapes:
    x = torch.randn(K, device="cuda")
    ws = torch.zeros(lib.c.pb200_act_workspace_bytes(K) + 64, dtype=torch.uint8, device="cuda")
    lib.check(lib.c.pb200_quantize_act(Q4, C.c_void_p(x.data_ptr()), K, C.c_void_p(ws.data_ptr()), None), "q")
    n = len(mats)
    types = (C.c_int * n)(*[t for t, _ in mats])
    Ns = (C.c_int64 * n)(*[N for _, N in mats])
    sizes = [lib.c.pb200_row_bytes(t, K) * N for t, N in mats]
    total = sum(sizes)
    ncopies = max(1, min(8, pool.numel() // (total + 4096)))
    def go(i):
        base = pool.data_ptr() + (i % ncopies) * ((total + 4095) // 4096 * 4096)
        W = (C.c_void_p * n)(); Y = (C.c_void_p * n)()
        off = 0; yo = 0
        for j in range(n):
            W[j] = base + off; off += (sizes[j] + 255) // 256 * 256
            Y[j] = y.data_ptr() + yo * 4; yo += mats[j][1]
        lib.check(lib.c.pb200_mul_mat_vec_fused(n, types, W, Ns, K, C.c_void_p(ws.data_ptr()), Y, None), name)
    for i in range(3):
        go(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(reps):
        go(i)
    e1.record(); torch.cuda.synchronize()
    us = e0.elapsed_time(e1) / reps * 1e3
    print(f"{name:8s} K={K:6d} {total / 1e6:8.1f} MB  {us:8.2f} us  {total / us / 1e6:6.2f} TB/s")
