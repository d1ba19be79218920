"""-m gpu: every op the ggml-backend plugin claims, computed by the kernel the plugin dispatches it to (through the C ABI) and compared
with the reference's own CPU backend on the same seeded inputs.  The reference's results are recorded in golden/reference_golden.npz
(golden/make_reference_golden.py builds each op with the reference's ggml and computes it on its CPU backend), so the comparison needs
no reference tree.  Bars: the reference's own NMSE thresholds (tests/test-backend-ops.cpp: MUL_MAT 5e-4 :1660, SOFT_MAX 1e-6 :2077,
others 1e-7 :320), and bit-exact results where the op only moves or converts values."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest
import torch

import oracle_lib as O
from golden import make_reference_golden as RG
from gpu_util import act_ws, dev_f32, dev_u8, ptr, sync

pytestmark = pytest.mark.gpu
G = Path(__file__).resolve().parent / "golden"


@pytest.fixture(scope="module")
def refgold():
    return np.load(G / "reference_golden.npz")


def nmse(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return float(np.sum((got - want) ** 2) / max(np.sum(want ** 2), 1e-30))


def copy_strided(lib, x, ne, src_strides, dst_strides, shape, f16=False):
    # device buffers stay referenced until the kernel has run: a freed temporary could be handed to the next allocation
    xd = dev_f32(x)
    y = torch.zeros(x.size, dtype=torch.float16 if f16 else torch.float32, device="cuda")
    arr = lambda v: (C.c_int64 * 4)(*v)  # noqa: E731
    lib.check(lib.c.pb200_copy_strided(ptr(xd), ptr(y), C.c_int(int(f16)), arr(ne), arr(src_strides), arr(dst_strides), None), "copy_strided")
    sync()
    return y.cpu().numpy().reshape(shape)


@pytest.mark.parametrize("op", RG.OPS)
def test_op_matches_reference_cpu_backend(cuda, lib, refgold, op):
    inp = RG.op_inputs(op)
    if op in ("MUL_MAT", "MUL_MAT_BATCHED"):
        N, K, x = inp["N"], inp["K"], inp["x"]
        T = x.shape[0]
        for t in RG.MM_TYPES:
            want = refgold[f"op_{op}_{O.TYPE_NAME[t]}"]
            Wd, xd = dev_u8(inp[f"w_{O.TYPE_NAME[t]}"]), dev_f32(x)
            y = torch.full((T * N,), float("nan"), device="cuda")
            if op == "MUL_MAT":      # decode GEMV: the CPU's activation quantization, integer dots, fp32 order only
                ws = act_ws(lib, K)
                lib.check(lib.c.pb200_mul_mat_vec(t, ptr(Wd), N, K, ptr(xd), ptr(y), ptr(ws), None), "mul_mat_vec")
                sync()
                got = y.cpu().numpy().reshape(T, N)
                assert np.max(np.abs(got - want)) <= 4e-6 * max(1.0, float(np.max(np.abs(want)))), O.TYPE_NAME[t]
            else:                    # prefill tensor-core product: fp16 operands, fp32 accumulation
                ws = torch.zeros(lib.c.pb200_mul_mat_q_workspace_bytes(K, T) + 256, dtype=torch.uint8, device="cuda")
                lib.check(lib.c.pb200_mul_mat_q(t, ptr(Wd), N, K, ptr(xd), K, T, ptr(y), None, None, ptr(ws), None), "mul_mat_q")
                sync()
                got = y.cpu().numpy().reshape(T, N)
            assert nmse(got, want) < 5e-4, (O.TYPE_NAME[t], nmse(got, want))
        return
    want = refgold[f"op_{op}"]
    if op == "RMS_NORM":
        x = inp["x"]
        xd, y = dev_f32(x), torch.zeros(x.size, device="cuda")
        lib.check(lib.c.pb200_rms_norm(ptr(xd), ptr(y), x.shape[1], x.shape[0], C.c_float(inp["eps"]), None), "rms_norm")
        sync()
        got = y.cpu().numpy().reshape(x.shape)
        assert np.max(np.abs(got - want) / np.maximum(np.abs(want), 1e-6)) < 3e-7
    elif op == "ROPE":
        x, pos = inp["x"], inp["pos"]
        Tn, H, D = x.shape
        got = []
        xd = dev_f32(x)
        for mode, ff in ((0, None), (2, None), (0, inp["ff"])):
            y = torch.zeros(x.size, device="cuda")
            pd, fd = torch.from_numpy(pos).cuda(), (dev_f32(ff) if ff is not None else None)
            lib.check(lib.c.pb200_rope(ptr(xd), ptr(y), Tn, H, D, D, mode, ptr(pd), C.c_float(500000.0), C.c_float(1.0), C.c_float(0.0),
                                       C.c_float(1.0), C.c_float(32.0), C.c_float(1.0), 8192, ptr(fd) if fd is not None else None, None), "rope")
            sync()
            got.append(y.cpu().numpy().reshape(x.shape))
        got = np.stack(got)
        # cosf / sinf of CUDA and glibc differ by <= 2 ulp
        assert np.max(np.abs(got - want)) < 4e-6 * np.max(np.abs(x))
    elif op == "SOFT_MAX":
        x, mask = inp["x"], inp["mask"]
        xd, md, y = dev_f32(x), dev_f32(mask), torch.zeros(x.size, device="cuda")
        lib.check(lib.c.pb200_soft_max(ptr(xd), ptr(md), ptr(y), x.shape[1], x.shape[0], mask.shape[0],
                                       C.c_float(inp["scale"]), None), "soft_max")
        sync()
        got = y.cpu().numpy().reshape(x.shape)
        assert np.max(np.abs(got - want)) < 3e-7
        assert nmse(got, want) < 1e-6
        return
    elif op in ("ADD", "MUL"):
        a, b = inp["a"], inp["b"]
        ad, bd, y = dev_f32(a), dev_f32(b), torch.zeros(a.size, device="cuda")
        lib.check(lib.c.pb200_binary(C.c_int(0 if op == "ADD" else 1), ptr(ad), ptr(bd), ptr(y), C.c_int64(a.size), C.c_int64(b.size), None),
                  "binary")
        sync()
        got = y.cpu().numpy().reshape(a.shape)
        assert np.array_equal(got, want)
    elif op == "SILU":
        x = inp["x"]
        xd, y = dev_f32(x), torch.zeros(x.size, device="cuda")
        lib.check(lib.c.pb200_silu(ptr(xd), ptr(y), C.c_int64(x.size), None), "silu")
        sync()
        got = y.cpu().numpy().reshape(x.shape)
    elif op == "CPY":        # f32 -> f16 (the KV-cache store)
        x = inp["x"]
        R, K = x.shape
        got = copy_strided(lib, x, [K, R, 1, 1], [4, 4 * K, 4 * K * R, 4 * K * R], [2, 2 * K, 2 * K * R, 2 * K * R], x.shape, f16=True)
        assert np.array_equal(got.view(np.uint16), want.view(np.uint16))
    elif op == "CONT":       # a transposed view made contiguous (the transposed V-cache layout)
        x = inp["x"]
        R, K = x.shape
        got = copy_strided(lib, x, [R, K, 1, 1], [4 * K, 4, 4 * K * R, 4 * K * R], [4, 4 * R, 4 * K * R, 4 * K * R], (K, R))
        assert np.array_equal(got, want)
    elif op == "DUP":        # a permuted 3-D view (permute 0, 2, 1, 3) duplicated into contiguous memory
        x = inp["x"]
        D2, D1, D0 = x.shape
        got = copy_strided(lib, x, [D0, D2, D1, 1], [4, 4 * D0 * D1, 4 * D0, 4 * x.size], [4, 4 * D0, 4 * D0 * D2, 4 * x.size], (D1, D2, D0))
        assert np.array_equal(got, want)
    elif op == "GET_ROWS":   # k-quant rows dequantized on the gather
        ids = inp["ids"]
        y = torch.zeros(len(ids) * 1024, device="cuda")
        idd, tabd = torch.from_numpy(ids).cuda(), dev_u8(inp["table"])
        lib.check(lib.c.pb200_get_rows(O.Q4_K, ptr(tabd), 1024, ptr(idd), len(ids), ptr(y), None), "get_rows")
        sync()
        got = y.cpu().numpy().reshape(len(ids), 1024)
        assert np.array_equal(got, want)
    assert nmse(got, want) < 1e-7, nmse(got, want)
