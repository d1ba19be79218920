"""ctypes access to the two CPU oracles (TEST INFRASTRUCTURE — never imported by the product package).

* ``port``  : oracle/liboracle_port.so — our plain-C restatement (oracle/kquants_port.c).
* ``ref``   : oracle/_ref/{v3,v4}/libggml_ref.so + libgraph_ref.so — the UNMODIFIED reference CPU ggml
              compiled from the reference source tree (oracle/Makefile).
Also: synthetic GGUF-block generators shared by the tests and bench.py's cpu legs.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
ORACLE = ROOT / "oracle"

# enum ggml_type (ggml/include/ggml.h:356-395)
F32, F16, Q5_1, Q8_0, Q4_K, Q5_K, Q6_K = 0, 1, 7, 8, 12, 13, 14
TYPE_NAME = {F32: "f32", F16: "f16", Q5_1: "q5_1", Q8_0: "q8_0", Q4_K: "q4_K", Q5_K: "q5_K", Q6_K: "q6_K"}
BLOCK = {Q4_K: (256, 144), Q5_K: (256, 176), Q6_K: (256, 210), Q8_0: (32, 34), Q5_1: (32, 24), F32: (1, 4), F16: (1, 2)}
QUANT_TYPES = [Q4_K, Q5_K, Q6_K, Q8_0, Q5_1]


def row_size(t: int, k: int) -> int:
    be, bb = BLOCK[t]
    assert k % be == 0
    return k // be * bb


def _cpu_flags() -> set:
    try:
        for line in open("/proc/cpuinfo"):
            if line.startswith("flags"):
                return set(line.split(":", 1)[1].split())
    except OSError:
        pass
    return set()


def ref_variant() -> str:
    forced = os.environ.get("PB200_REF_VARIANT")          # tests/test_reference_self_divergence.py runs both builds
    if forced in ("v3", "v4") and (ORACLE / "_ref" / forced / "libggml_ref.so").exists():
        return forced
    need_v4 = {"avx512f", "avx512bw", "avx512cd", "avx512dq", "avx512vl"}
    return "v4" if need_v4 <= _cpu_flags() and (ORACLE / "_ref" / "v4" / "libggml_ref.so").exists() else "v3"


def ref_dir() -> Path:
    return ORACLE / "_ref" / ref_variant()


def have_ref() -> bool:
    return (ref_dir() / "libggml_ref.so").exists() and (ref_dir() / "libgraph_ref.so").exists()


def build_port() -> Path:
    so = ORACLE / "liboracle_port.so"
    src = ORACLE / "kquants_port.c"
    if not so.exists() or so.stat().st_mtime < src.stat().st_mtime:
        subprocess.check_call(["make", "-C", str(ORACLE), "port"], stdout=subprocess.DEVNULL)
    return so


def have_reference_tree() -> bool:
    """Whether the reference source tree oracle/Makefile points at (REF) is present and readable by this user."""
    return subprocess.call(["make", "-s", "-C", str(ORACLE), "have-ref"], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL) == 0


def build_ref() -> bool:
    """(Re)build oracle/_ref from the reference source tree when that tree is readable."""
    if not have_reference_tree():
        return have_ref()
    subprocess.check_call(["make", "-C", str(ORACLE), "-j8", "ref"], stdout=subprocess.DEVNULL)
    return have_ref()


# ----------------------------------------------------------------------------------------------
# model description structs shared by port_llama_decode and gref_decode (identical layout)
class HParams(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("n_layer", "n_embd", "n_head", "n_head_kv", "head_dim", "n_ff", "n_vocab", "n_ctx",
                                          "rope_mode", "n_ctx_orig")] + \
               [(n, C.c_float) for n in ("rope_freq_base", "rope_freq_scale", "rms_eps")]


class Weight(C.Structure):
    _fields_ = [("type", C.c_int32), ("_pad", C.c_int32), ("data", C.c_void_p)]


class Layer(C.Structure):
    _fields_ = [("attn_norm", C.c_void_p), ("ffn_norm", C.c_void_p)] + \
               [(n, Weight) for n in ("wq", "wk", "wv", "wo", "gate", "up", "down")] + \
               [(n, C.c_void_p) for n in ("bq", "bk", "bv")]


class Model(C.Structure):
    _fields_ = [("hp", HParams), ("tok_embd", Weight), ("output_norm", C.c_void_p), ("output", Weight),
                ("layers", C.POINTER(Layer)), ("rope_freq_factors", C.c_void_p),
                ("k_cache", C.c_void_p), ("v_cache", C.c_void_p)]


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


class Port:
    """Plain-C restatement (oracle/kquants_port.c)."""

    def __init__(self):
        self.lib = C.CDLL(str(build_port()))
        L = self.lib
        L.port_fp16_to_fp32.restype = C.c_float
        L.port_fp16_to_fp32.argtypes = [C.c_uint16]
        L.port_fp32_to_fp16.restype = C.c_uint16
        L.port_fp32_to_fp16.argtypes = [C.c_float]
        L.port_row_size.restype = C.c_int64
        L.port_row_size.argtypes = [C.c_int, C.c_int64]
        L.port_act_row_size.restype = C.c_int64
        L.port_act_row_size.argtypes = [C.c_int, C.c_int64]
        L.port_dequantize_row.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int64]
        L.port_quantize_act.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int64]
        L.port_mul_mat.argtypes = [C.c_int, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]
        L.port_rms_norm.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_float]
        L.port_rope.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int32] + [C.c_float] * 6 + [C.c_int, C.c_void_p]
        L.port_soft_max.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_float]
        L.port_silu_mul.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]
        L.port_attention_decode.argtypes = [C.c_void_p] * 4 + [C.c_int] * 4 + [C.c_float]
        L.port_llama_decode.argtypes = [C.POINTER(Model), C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]

    def dequantize(self, t: int, blocks: np.ndarray, k: int) -> np.ndarray:
        rs = row_size(t, k)
        b = np.ascontiguousarray(blocks, dtype=np.uint8).reshape(-1, rs)
        out = np.empty((b.shape[0], k), dtype=np.float32)
        for i in range(b.shape[0]):
            self.lib.port_dequantize_row(t, _ptr(b[i]), _ptr(out[i]), k)
        return out

    def quantize_act(self, wtype: int, x: np.ndarray) -> np.ndarray:
        x = np.ascontiguousarray(x, dtype=np.float32)
        n = self.lib.port_act_row_size(wtype, x.size)
        q = np.zeros(n, dtype=np.uint8)
        self.lib.port_quantize_act(wtype, _ptr(x), _ptr(q), x.size)
        return q

    def mul_mat(self, t: int, W: np.ndarray, N: int, K: int, x: np.ndarray) -> np.ndarray:
        x = np.ascontiguousarray(x, dtype=np.float32).reshape(-1, K)
        W = np.ascontiguousarray(W, dtype=np.uint8)
        out = np.empty((x.shape[0], N), dtype=np.float32)
        self.lib.port_mul_mat(t, _ptr(W), N, K, _ptr(x), x.shape[0], _ptr(out))
        return out

    def rms_norm(self, x, eps):
        x = np.ascontiguousarray(x, dtype=np.float32)
        y = np.empty_like(x)
        self.lib.port_rms_norm(_ptr(x), _ptr(y), x.size, eps)
        return y

    def rope(self, x, n_head, head_dim, mode, pos, freq_base=500000.0, freq_scale=1.0, n_ctx_orig=8192, freq_factors=None,
             ext_factor=0.0, attn_factor=1.0, beta_fast=32.0, beta_slow=1.0, n_dims=None):
        x = np.ascontiguousarray(x, dtype=np.float32)
        y = np.empty_like(x)
        ff = None if freq_factors is None else np.ascontiguousarray(freq_factors, dtype=np.float32)
        self.lib.port_rope(_ptr(x), _ptr(y), n_head, head_dim, n_dims or head_dim, mode, pos, freq_base, freq_scale, ext_factor,
                           attn_factor, beta_fast, beta_slow, n_ctx_orig, None if ff is None else _ptr(ff))
        return y

    def soft_max(self, x, mask, scale):
        x = np.ascontiguousarray(x, dtype=np.float32)
        y = np.empty_like(x)
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.float32)
        self.lib.port_soft_max(_ptr(x), None if m is None else _ptr(m), _ptr(y), x.size, scale)
        return y

    def silu_mul(self, g, u):
        g = np.ascontiguousarray(g, dtype=np.float32)
        u = np.ascontiguousarray(u, dtype=np.float32)
        y = np.empty_like(g)
        self.lib.port_silu_mul(_ptr(g), _ptr(u), _ptr(y), g.size)
        return y

    def attention_decode(self, q, Kc, Vc, n_head, n_head_kv, head_dim, n_kv, scale):
        q = np.ascontiguousarray(q, dtype=np.float32)
        Kc = np.ascontiguousarray(Kc, dtype=np.uint16)
        Vc = np.ascontiguousarray(Vc, dtype=np.uint16)
        out = np.empty(n_head * head_dim, dtype=np.float32)
        self.lib.port_attention_decode(_ptr(q), _ptr(Kc), _ptr(Vc), _ptr(out), n_head, n_head_kv, head_dim, n_kv, scale)
        return out


class Ref:
    """The compiled, unmodified reference (oracle/_ref)."""

    def __init__(self, n_threads: int | None = None):
        d = ref_dir()
        self.ggml = C.CDLL(str(d / "libggml_ref.so"), mode=C.RTLD_GLOBAL)
        self.graph = C.CDLL(str(d / "libgraph_ref.so"))
        self.n_threads = n_threads or min(os.cpu_count() or 1, 64)
        g = self.ggml
        # ggml_init() fills the fp16->fp32 lookup table used by GGML_FP16_TO_FP32 (ggml.c ggml_init); do it once.
        class _IP(C.Structure):
            _fields_ = [("mem_size", C.c_size_t), ("mem_buffer", C.c_void_p), ("no_alloc", C.c_bool)]
        g.ggml_init.restype = C.c_void_p
        g.ggml_init.argtypes = [_IP]
        g.ggml_free.argtypes = [C.c_void_p]
        g.ggml_free(g.ggml_init(_IP(1 << 16, None, False)))
        g.ggml_quantize_chunk.restype = C.c_size_t
        g.ggml_quantize_chunk.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p]
        g.quantize_row_q8_K.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        g.quantize_row_q8_0.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        g.quantize_row_q8_1.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        for n in ("q4_K", "q5_K", "q6_K", "q8_0", "q5_1"):
            getattr(g, f"dequantize_row_{n}").argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        self.graph.gref_mul_mat.argtypes = [C.c_int, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int]
        self.graph.gref_create.restype = C.c_void_p
        self.graph.gref_create.argtypes = [C.POINTER(Model), C.c_int]
        self.graph.gref_free.argtypes = [C.c_void_p]
        self.graph.gref_decode.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t]

    def quantize(self, t: int, w: np.ndarray) -> np.ndarray:
        """f32 [N,K] -> raw GGUF blocks via ggml_quantize_chunk (ggml.c)."""
        w = np.ascontiguousarray(w, dtype=np.float32)
        N, K = w.shape
        out = np.zeros(N * row_size(t, K), dtype=np.uint8)
        n = self.ggml.ggml_quantize_chunk(t, _ptr(w), _ptr(out), 0, N, K, None)
        assert n == out.size
        return out

    def dequantize(self, t: int, blocks: np.ndarray, k: int) -> np.ndarray:
        rs = row_size(t, k)
        b = np.ascontiguousarray(blocks, dtype=np.uint8).reshape(-1, rs)
        out = np.empty((b.shape[0], k), dtype=np.float32)
        fn = getattr(self.ggml, f"dequantize_row_{TYPE_NAME[t]}")
        for i in range(b.shape[0]):
            fn(_ptr(b[i]), _ptr(out[i]), k)
        return out

    def quantize_act(self, wtype: int, x: np.ndarray) -> np.ndarray:
        x = np.ascontiguousarray(x, dtype=np.float32)
        if wtype in (Q4_K, Q5_K, Q6_K):
            q = np.zeros(x.size // 256 * 292, dtype=np.uint8)
            self.ggml.quantize_row_q8_K(_ptr(x), _ptr(q), x.size)
        elif wtype == Q8_0:
            q = np.zeros(x.size // 32 * 34, dtype=np.uint8)
            self.ggml.quantize_row_q8_0(_ptr(x), _ptr(q), x.size)
        else:
            q = np.zeros(x.size // 32 * 36, dtype=np.uint8)
            self.ggml.quantize_row_q8_1(_ptr(x), _ptr(q), x.size)
        return q

    def mul_mat(self, t: int, W: np.ndarray, N: int, K: int, x: np.ndarray, n_threads: int | None = None) -> np.ndarray:
        x = np.ascontiguousarray(x, dtype=np.float32).reshape(-1, K)
        W = np.ascontiguousarray(W, dtype=np.uint8)
        out = np.empty((x.shape[0], N), dtype=np.float32)
        rc = self.graph.gref_mul_mat(t, _ptr(W), N, K, _ptr(x), x.shape[0], _ptr(out), n_threads or self.n_threads)
        assert rc == 0
        return out


# ----------------------------------------------------------------------------------------------
# synthetic raw blocks (valid bit patterns, sane fp16 scales) — no quantizer needed
def _f16_bits(a: np.ndarray) -> np.ndarray:
    return a.astype(np.float16).view(np.uint16)


def synth_blocks(t: int, N: int, K: int, seed: int, scale: float = 1.0) -> np.ndarray:
    """Random weight blocks of type t for an [N,K] matrix, as uint8[N*row_size]. Weight std ~ scale/sqrt(K)."""
    rng = np.random.default_rng(seed)
    be, bb = BLOCK[t]
    nb = N * K // be
    out = np.zeros((nb, bb), dtype=np.uint8)
    s = scale / np.sqrt(K)
    if t == Q4_K or t == Q5_K:
        qmax = 15 if t == Q4_K else 31
        d = (rng.uniform(0.5, 1.5, nb) * s / (qmax / 2 * 32)).astype(np.float32)
        dmin = d * (qmax / 2) * rng.uniform(0.9, 1.1, nb).astype(np.float32)
        out[:, 0:2] = _f16_bits(d).view(np.uint8).reshape(nb, 2)
        out[:, 2:4] = _f16_bits(dmin).view(np.uint8).reshape(nb, 2)
        out[:, 4:] = rng.integers(0, 256, (nb, bb - 4), dtype=np.uint8)
    elif t == Q6_K:
        out[:, :192] = rng.integers(0, 256, (nb, 192), dtype=np.uint8)
        out[:, 192:208] = rng.integers(-128, 128, (nb, 16), dtype=np.int8).view(np.uint8)
        d = (rng.uniform(0.5, 1.5, nb) * s / (18.0 * 64)).astype(np.float32)
        out[:, 208:210] = _f16_bits(d).view(np.uint8).reshape(nb, 2)
    elif t == Q8_0:
        d = (rng.uniform(0.5, 1.5, nb) * s / 73.0).astype(np.float32)
        out[:, 0:2] = _f16_bits(d).view(np.uint8).reshape(nb, 2)
        out[:, 2:] = rng.integers(-127, 128, (nb, 32), dtype=np.int8).view(np.uint8)
    elif t == Q5_1:
        d = (rng.uniform(0.5, 1.5, nb) * s / 9.0).astype(np.float32)
        m = -d * 15.5 * rng.uniform(0.9, 1.1, nb).astype(np.float32)
        out[:, 0:2] = _f16_bits(d).view(np.uint8).reshape(nb, 2)
        out[:, 2:4] = _f16_bits(m).view(np.uint8).reshape(nb, 2)
        out[:, 4:] = rng.integers(0, 256, (nb, 20), dtype=np.uint8)
    else:
        raise ValueError(t)
    return out.reshape(-1)


# byte ranges of the quants and of the block scale d inside one block
_QBYTES = {Q4_K: slice(16, 144), Q5_K: slice(16, 176), Q6_K: slice(0, 192), Q8_0: slice(2, 34), Q5_1: slice(4, 24)}
_DBYTES = {Q4_K: slice(0, 2), Q5_K: slice(0, 2), Q6_K: slice(208, 210), Q8_0: slice(0, 2), Q5_1: slice(0, 2)}


def edge_blocks(t: int, N: int, K: int, seed: int) -> np.ndarray:
    """synth_blocks with the bit patterns random blocks (almost) never hold, by row r % 6: 0 random; 1 every quant byte 0x00; 2 every
    quant byte 0xFF; 3 the type's extreme: Q8_0 q = -128, Q6_K sub-block scales -128 with q = -32, Q4_K / Q5_K 6-bit scales and mins all
    63, Q5_1 offset m = 0 with q = 31; 4 d = 0 in every block; 5 d = 0 in every other block."""
    be, bb = BLOCK[t]
    b = synth_blocks(t, N, K, seed).reshape(N, K // be, bb)
    q, dd = _QBYTES[t], _DBYTES[t]
    b[1::6, :, q] = 0x00
    b[2::6, :, q] = 0xFF
    if t == Q8_0:
        b[3::6, :, q] = 0x80
    elif t == Q6_K:
        b[3::6, :, q] = 0x00
        b[3::6, :, 192:208] = 0x80
    elif t in (Q4_K, Q5_K):
        b[3::6, :, 4:16] = 0xFF
    else:
        b[3::6, :, 2:4] = 0x00
        b[3::6, :, q] = 0xFF
    b[4::6, :, dd] = 0x00
    b[5::6, ::2, dd] = 0x00
    return b.reshape(-1)


def f32_to_f16_bits(a: np.ndarray) -> np.ndarray:
    return np.asarray(a, dtype=np.float32).astype(np.float16).view(np.uint16)
