"""CPU: the C-ABI library loads and exports every symbol include/prima_b200.h declares; argument validation works
without a GPU (no compute calls)."""
import ctypes as C
import re
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent


def declared_symbols(header):
    txt = (ROOT / "include" / header).read_text()
    return sorted(set(re.findall(r"PB200_API[^;]*?\b(pb200_\w+)\s*\(", txt)))


def test_header_symbols_exported(pkg):
    so = C.CDLL(str(pkg.lib_path()))
    syms = declared_symbols("prima_b200.h")
    assert len(syms) >= 30
    for s in syms:
        assert hasattr(so, s), f"{s} declared in include/prima_b200.h but not exported"


def test_row_bytes_and_workspace(lib):
    c = lib.c
    assert c.pb200_row_bytes(12, 8192) == 4608      # Q4_K 144 B / 256
    assert c.pb200_row_bytes(13, 8192) == 5632
    assert c.pb200_row_bytes(14, 8192) == 6720
    assert c.pb200_row_bytes(8, 29568) == 29568 // 32 * 34
    assert c.pb200_row_bytes(7, 29568) == 29568 // 32 * 24
    assert c.pb200_act_workspace_bytes(8192) == 8192 + 8192 // 32 * 8 + 8192 // 16 * 2
    assert c.pb200_error_string(-3).decode().startswith("unsupported")
    assert "watchdog" in c.pb200_error_string(-5).decode()


def test_argument_validation_no_gpu(lib, pkg):
    c = lib.c
    assert c.pb200_quantize_act(12, None, 256, None, None) == -1
    assert c.pb200_mul_mat_vec_q(3, None, 1, 256, None, None, None, None, None) == -1
    # matrices that need different activation formats (q8_K for Q4_K, q8_0 for Q8_0) cannot share one activation
    fake = (C.c_void_p * 2)(256, 512)
    assert c.pb200_mul_mat_vec_fused(2, (C.c_int * 2)(12, 8), fake, (C.c_int64 * 2)(16, 16), 256, C.c_void_p(1024), fake, None) == -1
    hp = pkg.HParams(n_layer=2, n_embd=250, n_head=2, n_head_kv=1, head_dim=128, n_ff=512, n_vocab=100, n_ctx=16, rope_mode=0,
                     n_ctx_orig=8192, rope_freq_base=5e5, rope_freq_scale=1.0, rms_eps=1e-5)
    assert not c.pb200_model_create(C.byref(hp), 0, 0, 2, 1, 1)   # n_embd % 256 != 0 -> NULL, no abort
    assert c.pb200_decode(None, 0, 0, None) == -4
    assert c.pb200_prefill(None, None, 1, 0, None) == -4
    # batched tensor-core product: workspace = padded rows x (K fp16 + one f32 row scale); argument errors before any CUDA call
    assert c.pb200_mul_mat_q_workspace_bytes(8192, 512) == 512 * (8192 * 2 + 4)
    assert c.pb200_mul_mat_q_workspace_bytes(8192, 20) == 32 * (8192 * 2 + 4)      # 20 rows -> one 32-column tile
    assert c.pb200_mul_mat_q(12, None, 128, 256, None, 256, 8, None, None, None, None, None) == -1
    assert c.pb200_attn_prefill(None, None, None, None, 8, 2, 128, None, 4, 4, 0.1, None) == -1


def test_fused_path_limits(lib):
    """What the ggml-backend plugin plans with: the fused GEMV takes k-quant rows up to K = 29 696 (116 super-blocks), the
    tensor-core product Q8_0 rows in 64-element steps."""
    c = lib.c
    assert c.pb200_gemv_fused_supported(12, C.c_int64(29696)) == 1
    assert c.pb200_gemv_fused_supported(12, C.c_int64(29952)) == 0
    assert c.pb200_gemv_fused_supported(8, C.c_int64(4096)) == 0     # Q8_0 is not a k-quant
    assert c.pb200_mul_mat_q_supported(8, C.c_int64(4096)) == 1
    assert c.pb200_mul_mat_q_supported(8, C.c_int64(4064)) == 0


def test_hparams_layout_matches_header(pkg):
    assert C.sizeof(pkg.HParams) == 10 * 4 + 3 * 4


def test_missing_library_fails_loudly(pkg, monkeypatch, tmp_path):
    import pytest
    host = __import__("sys").modules["prima_cpp_b200.host"]
    monkeypatch.setattr(host, "lib_path", lambda: tmp_path / "nope.so")
    with pytest.raises(host.Pb200Error):
        host.Lib()
