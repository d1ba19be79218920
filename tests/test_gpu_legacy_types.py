"""-m gpu: the legacy 32-element weight types Q4_0, Q4_1 and Q5_0 on every path, against the CPU oracles: the activation quantizer,
the decode GEMV on each of its kernels (bulk-copy ring, split rows, k_gemv_blk32, k_gemv_generic), the tensor-core prefill product,
get_rows, the engine (decode, prefill, GGUF load, synthetic Qwen2.5-72B Q4_K_M types) and whole decode graphs through the ggml-backend
plugin."""
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import legacy_types as L
import oracle_lib as O
from gpu_util import act_ws, act_ws_fields, dev_f32, dev_u8, ptr, sync
from test_gpu_engine import check_decode_parity
from test_gpu_mmq import check, mmq_plan, run_mmq

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
G = ROOT / "tests" / "golden"
LT = L.LEGACY_TYPES
ACT = {L.Q4_0: "q8_0", L.Q4_1: "q8_1", L.Q5_0: "q8_0"}


def rel_tol(ref, r=4e-6):
    return r * max(1.0, float(np.max(np.abs(ref))))


@pytest.mark.parametrize("t", LT, ids=lambda t: L.NAME[t])
def test_quantize_act_bit_exact(cuda, lib, port, t):
    """q8_0 for Q4_0 / Q5_0, q8_1 (with s = d * sum q) for Q4_1, as the CPU quantizes the activation for each type."""
    for K in (512, 7392, 29568):
        x = np.random.default_rng(K + t).standard_normal(K).astype(np.float32)
        ws = act_ws(lib, K)
        lib.check(lib.c.pb200_quantize_act(t, ptr(dev_f32(x)), K, ptr(ws), None), "quantize_act")
        sync()
        assert np.array_equal(act_ws_fields(ws, K, ACT[t]), L.quantize_act(port, t, x)), K


def gemv(lib, t, W, N, K, x, shift=0, bias=None, resid=None, trace_slots=0):
    """pb200_quantize_act + pb200_mul_mat_vec_q with W placed `shift` bytes past a 256-byte boundary; returns (y, launches, ring launches)."""
    buf = torch.zeros(W.size + 320, dtype=torch.uint8, device="cuda")
    buf[shift: shift + W.size] = torch.from_numpy(np.ascontiguousarray(W).view(np.uint8).reshape(-1))
    ws = act_ws(lib, K)
    lib.check(lib.c.pb200_quantize_act(t, ptr(dev_f32(x)), K, ptr(ws), None), "q")
    y = torch.full((N,), float("nan"), device="cuda")
    bd = dev_f32(bias) if bias is not None else None
    rd = dev_f32(resid) if resid is not None else None
    trace = torch.zeros(4 * 4096, dtype=torch.int64, device="cuda")
    lib.c.pb200_debug_set_trace.argtypes = [C.c_void_p, C.c_int]
    lib.check(lib.c.pb200_debug_set_trace(trace.data_ptr(), 4), "trace")
    try:
        sync()
        n0 = lib.c.pb200_kernel_launches()
        lib.check(lib.c.pb200_mul_mat_vec_q(t, C.c_void_p(buf.data_ptr() + shift), N, K, ptr(ws), ptr(y), ptr(bd) if bd is not None else None,
                                            ptr(rd) if rd is not None else None, None), "mul_mat_vec_q")
        sync()
        n = lib.c.pb200_kernel_launches() - n0
    finally:
        lib.c.pb200_debug_set_trace(None, 0)
    ring = int((trace.view(4, 4096) != 0).any(dim=1).sum().item())
    assert lib.c.pb200_aborted() == 0
    return y.cpu().numpy(), n, ring


# (N, K, W shift, ring expected): the ring (whole rows, K = 8 192 and Llama-3-8B's 4 096 / 14 336), split rows at Qwen2.5-72B's ffn_down
# (8 192 x 29 568: rows 8- but not 16-byte aligned) and a ragged N; a W 8 bytes off a 16-byte boundary (k_gemv_blk32); W 2 bytes off
# and K = 1 056, whose rows are not 8-byte multiples (k_gemv_generic)
GEMV_CASES = [(1000, 8192, 0, True), (333, 4096, 0, True), (200, 14336, 0, True), (8192, 29568, 0, True), (77, 29568, 0, True),
              (300, 8192, 8, False), (129, 29568, 8, False), (300, 4096, 2, False), (100, 1056, 0, False)]


@pytest.mark.parametrize("t", LT, ids=lambda t: L.NAME[t])
@pytest.mark.parametrize("N,K,shift,ring", GEMV_CASES)
def test_gemv_every_route(cuda, lib, port, t, N, K, shift, ring):
    rng = np.random.default_rng(N + K + t)
    W = L.synth_blocks(t, N, K, seed=7 * t + N)
    x = rng.standard_normal(K).astype(np.float32)
    bias, resid = rng.standard_normal(N).astype(np.float32), rng.standard_normal(N).astype(np.float32)
    y, n, rl = gemv(lib, t, W, N, K, x, shift, bias, resid)
    assert n == 1
    assert (rl == 1) == ring, (rl, ring)
    want = (L.mul_mat(port, t, W, N, K, x)[0] + bias) + resid
    assert np.max(np.abs(y - want)) <= rel_tol(want), np.max(np.abs(y - want))


@pytest.mark.parametrize("t", LT, ids=lambda t: L.NAME[t])
def test_gemv_weight_bit_patterns(cuda, lib, port, t):
    """All-zero / all-one quant bytes, d = 0 blocks: the same on the ring and on the generic kernel."""
    N, K = 96, 4096
    W = L.synth_blocks(t, N, K, seed=3).reshape(N, K // 32, -1)
    W[1::4, :, -16:] = 0x00
    W[2::4, :, -16:] = 0xFF
    W[3::4, ::2, 0:2] = 0x00
    W = W.reshape(-1)
    x = np.random.default_rng(1).standard_normal(K).astype(np.float32)
    want = L.mul_mat(port, t, W, N, K, x)[0]
    for shift in (0, 2):
        y, _, _ = gemv(lib, t, W, N, K, x, shift)
        assert np.max(np.abs(y - want)) <= rel_tol(want), shift


@pytest.mark.parametrize("t", LT, ids=lambda t: L.NAME[t])
@pytest.mark.parametrize("N,K,T", [(136, 448, 1), (136, 448, 24), (136, 448, 100), (136, 448, 512), (128, 29568, 24), (200, 4096, 33)])
def test_mmq_vs_oracle(cuda, lib, port, t, N, K, T):
    """Every token-tile rung (BN 16 / 32 / 128, four token tiles), Qwen2.5-72B's ffn_down K, under the bar of tests/test_gpu_mmq.py."""
    rng = np.random.default_rng(N + K + T + t)
    X = rng.standard_normal((T, K)).astype(np.float32)
    if T > 1:
        X[0] = 0.0
    W = L.synth_blocks(t, N, K, seed=5 * t + N)
    got = run_mmq(lib, t, W, N, K, X)
    Wf = L.dequantize(t, W, K)
    check(got, L.mul_mat(port, t, W, N, K, X), Wf, X)
    if T > 1:
        assert np.all(got[0] == 0.0)


@pytest.mark.parametrize("t", LT, ids=lambda t: L.NAME[t])
def test_mmq_split_tiles_bias_residual(cuda, lib, port, t):
    """Stream-K tiles shared by several CTAs, the short last 256-K group in a partial segment (K = 4 160), bias and residual once."""
    N, T, K = 200, 150, 4160
    p = mmq_plan(lib, N, K, T)
    assert p.split and p.ctas_per_tile >= 3 and p.short_group_split, p
    rng = np.random.default_rng(50 + t)
    W = L.synth_blocks(t, N, K, seed=29 + t)
    X = rng.standard_normal((T, K)).astype(np.float32)
    bias, resid = rng.standard_normal(N).astype(np.float32), rng.standard_normal((T, N)).astype(np.float32)
    got = run_mmq(lib, t, W, N, K, X, bias=bias, resid=resid)
    Wf = L.dequantize(t, W, K)
    check(got, (L.mul_mat(port, t, W, N, K, X) + bias[None, :]) + resid, Wf, X)


@pytest.mark.parametrize("t", LT, ids=lambda t: L.NAME[t])
def test_get_rows_bit_exact(cuda, lib, port, t):
    n_rows, K = 64, 4096
    W = L.synth_blocks(t, n_rows, K, seed=11 + t)
    ids = np.array([0, 63, 5, 5, 17, 32], np.int32)
    y = torch.full((ids.size, K), float("nan"), device="cuda")
    idd = torch.from_numpy(ids).cuda()
    lib.check(lib.c.pb200_get_rows(t, ptr(dev_u8(W)), K, ptr(idd), ids.size, ptr(y), None), "get_rows")
    sync()
    assert np.array_equal(y.cpu().numpy(), L.dequantize(t, W, K)[ids])


@pytest.fixture(scope="module")
def gold():
    return np.load(G / "legacy_types_golden.npz")


@pytest.mark.parametrize("name", ["qwen2_q4_K_M", "llama_q4_0"])
def test_engine_decode_vs_reference(cuda, pkg, gold, name):
    """40 tokens against the compiled reference's graph on the same weights (recorded), under the multi-token parity bar."""
    tm, toks = L.models()[name]
    eng = tm.load_engine(pkg)
    got = np.zeros((len(toks), tm.hp["n_vocab"]), np.float32)
    for i, tk in enumerate(toks):
        eng.decode(int(tk), i, got[i])
    eng.close()
    check_decode_parity(got, gold[f"{name}_logits"])


@pytest.mark.parametrize("name", ["qwen2_q4_K_M", "llama_q4_0"])
def test_engine_prefill_then_decode(cuda, pkg, name):
    """A 24-token prompt through pb200_prefill (tensor-core mat-muls, the Q5_0 / Q4_0 weights expanded to fp16), then 8 decode steps:
    the prompt's last logits and every step after it agree with token-by-token decode (NMSE 1e-3, the prefill bar of the smoke run)."""
    tm, toks = L.models()[name]
    nv = tm.hp["n_vocab"]
    eng = tm.load_engine(pkg)
    seq = np.zeros((32, nv), np.float32)
    for i in range(32):
        eng.decode(int(toks[i]), i, seq[i])
    eng.close()
    eng = tm.load_engine(pkg)
    got = [eng.prefill(toks[:24], 0)]
    for i in range(24, 32):
        got.append(eng.decode(int(toks[i]), i, np.zeros(nv, np.float32)))
    eng.close()
    for j, g in enumerate(got):
        w = seq[23 + j]
        assert np.sum((g - w) ** 2) / np.sum(w ** 2) < 1e-3, j


def test_gguf_loaded_model_decodes_like_set_tensor_model(cuda, pkg, tmp_path):
    """A Q4_0 file with a Q4_1 ffn_down and a Q5_0 attn_output, loaded from disk: bit-identical to the same weights set tensor by tensor."""
    from test_legacy_types_cpu import gguf_model
    tm = gguf_model()
    path = tmp_path / "q4_0.gguf"
    L.write_gguf(tm, path)
    toks = [(i * 7919 + 13) % 320 for i in range(8)]
    ref = tm.load_engine(pkg)
    want = np.zeros((len(toks), 320), np.float32)
    for i, tk in enumerate(toks):
        ref.decode(int(tk), i, want[i])
    ref.close()
    eng = pkg.Model.from_gguf(path, n_ctx=64)
    got = np.zeros_like(want)
    for i, tk in enumerate(toks):
        eng.decode(int(tk), i, got[i])
    eng.close()
    assert np.array_equal(got, want)


def test_synth_qwen72b_q4_K_M_types(cuda, pkg):
    """pb200_model_synth(ftype 0) on two Qwen2.5-72B layers: the reference's Q4_K_M types tensor by tensor (80 layers = MODEL_70B: attn_v
    Q5_K; n_ff 29 568: ffn_down Q4_K -> Q5_0, or Q6_K -> Q8_0 in the use_more_bits layers), and ftype 2 gives Q4_0 everywhere."""
    hp = pkg.HParams(n_layer=80, n_embd=8192, n_head=64, n_head_kv=8, head_dim=128, n_ff=29568, n_vocab=152064, n_ctx=64, rope_mode=2,
                     n_ctx_orig=32768, rope_freq_base=1e6, rope_freq_scale=1.0, rms_eps=1e-6)
    want = {0: {11: {"attn_v": O.Q5_K, "ffn_down": L.Q5_0}, 12: {"attn_v": O.Q6_K, "ffn_down": O.Q8_0}},
            2: {11: {"attn_v": L.Q4_0, "ffn_down": L.Q4_0}, 12: {"attn_v": L.Q4_0, "ffn_down": L.Q4_0}}}
    for ftype, layers in want.items():
        m = pkg.Model(hp, 0, (11, 13), False, False)
        m.synth(ftype, 5)
        default = O.Q4_K if ftype == 0 else L.Q4_0
        for il, special in layers.items():
            for w, K in (("attn_q", 8192), ("attn_k", 8192), ("attn_v", 8192), ("attn_output", 8192), ("ffn_gate", 8192), ("ffn_up", 8192),
                         ("ffn_down", 29568)):
                _, nbytes, t = m.tensor_device(f"blk.{il}.{w}.weight")
                assert t == special.get(w, default), (ftype, il, w, t)
                N = {"attn_k": 1024, "attn_v": 1024, "ffn_gate": 29568, "ffn_up": 29568}.get(w, 8192)
                assert nbytes == L.row_size(t, K) * N
        m.close()


@pytest.mark.parametrize("name", ["qwen2_q4_K_M", "llama_q4_0"])
def test_plugin_whole_graph_decode(cuda, name):
    """40 decode steps of the whole graph through ggml_backend_graph_compute on B200_0 against the CPU backend.  The host stand-in places
    every node on B200_0 and the plugin refuses a node it does not claim, so the run also shows that no node fell back to the CPU."""
    if not (ROOT / "host" / "_ggml" / "libllama_graph_host.so").exists() or not (ROOT / "prima.cpp_b200" / "libggml-b200.so").exists():
        pytest.skip("host/_ggml or the plugin is not built (build() builds them only where the reference source tree is readable)")
    p = subprocess.run([sys.executable, str(ROOT / "tests" / "legacy_graph_parity.py"), name, "40"], capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-4000:]
    r = json.loads(p.stdout.strip().splitlines()[-1])
    assert r["unsupported_nodes"] == 0, r
    assert r["first_token_err"] < 1e-4, r
    assert r["nmse"] < 2e-3 and r["max_abs"] < 0.25 and r["argmax_agree"] >= 0.9, r
    assert (L.Q5_0 in r["types"]) if name.startswith("qwen2") else (L.Q4_0 in r["types"]), r
