"""The legacy 32-element weight types Q4_0, Q4_1 and Q5_0 for the tests (TEST INFRASTRUCTURE — never imported by the product package).

* A restatement of the reference's CPU arithmetic for them, in numpy, written from the block formats (ggml/src/ggml-common.h:143-170):
  dequantize_row_q4_0 / _q4_1 / _q5_0 (ggml-quants.c:1522-1580) and the scalar loops of ggml_vec_dot_q4_0_q8_0 / _q4_1_q8_1 /
  _q5_0_q8_0 (:3921, :4502, :4789): an exact integer dot per block, then the block's fp32 scale product added in the CPU's order.
  The activation is the q8_0 (Q4_0, Q5_0) or q8_1 (Q4_1) block the C port (oracle/kquants_port.c) already quantizes for Q8_0 / Q5_1.
* Synthetic blocks, GGUF writing and the two tiny models of tests/golden/legacy_types_golden.npz (a Qwen2 Q4_K_M whose n_ff % 256 != 0
  turns ffn_down into Q5_0, a llama Q4_0), built on tests/tiny_model.py's TinyModel.
* Access to the compiled reference's quantizer and dequantizers for the three types (oracle/_ref, through oracle_lib.Ref).

Element j < 16 of a block is the low nibble of qs[j], element j + 16 its high nibble; Q5_0's fifth bit of element j is bit j of qh."""
from __future__ import annotations

import ctypes as C

import numpy as np

import oracle_lib as O
from tiny_model import TinyModel

Q4_0, Q4_1, Q5_0 = 2, 3, 6                        # enum ggml_type (ggml/include/ggml.h)
LEGACY_TYPES = [Q4_0, Q4_1, Q5_0]
NAME = {Q4_0: "q4_0", Q4_1: "q4_1", Q5_0: "q5_0"}
BLOCK_BYTES = {Q4_0: 18, Q4_1: 20, Q5_0: 22}      # [d f16][qs 16] | [d f16][m f16][qs 16] | [d f16][qh u32][qs 16]
QOFF = {Q4_0: 2, Q4_1: 4, Q5_0: 6}
ACT_TYPE = {Q4_0: O.Q8_0, Q4_1: O.Q5_1, Q5_0: O.Q8_0}   # the weight type whose activation format (q8_0 / q8_1) the CPU uses


def row_size(t: int, k: int) -> int:
    if t in BLOCK_BYTES:
        assert k % 32 == 0
        return k // 32 * BLOCK_BYTES[t]
    return O.row_size(t, k)


def _f16(b: np.ndarray) -> np.ndarray:
    """little-endian f16 in the last axis (2 bytes) -> f32"""
    return np.ascontiguousarray(b).view(np.float16)[..., 0].astype(np.float32)


def _fields(t: int, W: np.ndarray, K: int):
    """(q [rows, nb, 32] int32 with the type's offset applied, d [rows, nb] f32, m [rows, nb] f32 or None)"""
    nb = K // 32
    b = np.ascontiguousarray(W, dtype=np.uint8).reshape(-1, nb, BLOCK_BYTES[t])
    qs = b[..., QOFF[t]:QOFF[t] + 16].astype(np.int32)
    q = np.concatenate([qs & 0xF, qs >> 4], axis=-1)
    if t == Q5_0:
        qh = np.ascontiguousarray(b[..., 2:6]).view(np.uint32)[..., 0]
        q |= ((qh[..., None] >> np.arange(32, dtype=np.uint32)) & 1).astype(np.int32) << 4
        q -= 16
    elif t == Q4_0:
        q -= 8
    m = _f16(b[..., 2:4]) if t == Q4_1 else None
    return q, _f16(b[..., 0:2]), m


def dequantize(t: int, W: np.ndarray, K: int) -> np.ndarray:
    """rows [rows, K] f32: (q - 8) d, q d + m, (q - 16) d"""
    q, d, m = _fields(t, W, K)
    y = q.astype(np.float32) * d[..., None]
    if m is not None:
        y = y + m[..., None]
    return y.reshape(q.shape[0], K)


def quantize_act(port, t: int, x: np.ndarray) -> np.ndarray:
    """the activation blocks the CPU quantizes for weight type t: q8_0 (34 B) or q8_1 (36 B, with s = d * sum q)"""
    return port.quantize_act(ACT_TYPE[t], x)


def mul_mat(port, t: int, W: np.ndarray, N: int, K: int, X: np.ndarray, chunk: int = 1024) -> np.ndarray:
    """dst[T, N] = W . quant(X), block by block in the CPU's order"""
    X = np.ascontiguousarray(X, dtype=np.float32).reshape(-1, K)
    T, nb = X.shape[0], K // 32
    acts = [quantize_act(port, t, X[i]) for i in range(T)]
    ab = np.stack([a.reshape(nb, -1) for a in acts])                   # [T, nb, 34 | 36]
    da = _f16(ab[..., 0:2])
    sa = _f16(ab[..., 2:4]) if t == Q4_1 else None
    aq = ab[..., -32:].view(np.int8).astype(np.int32)                  # [T, nb, 32]
    out = np.empty((T, N), np.float32)
    Wr = np.ascontiguousarray(W, dtype=np.uint8).reshape(N, -1)
    for r0 in range(0, N, chunk):
        q, dw, m = _fields(t, Wr[r0:r0 + chunk], K)
        sumi = np.einsum("nbk,tbk->tnb", q, aq).astype(np.float32)     # exact: |sumi| < 2^24
        acc = np.zeros((T, q.shape[0]), np.float32)
        for ib in range(nb):
            if t == Q4_0:
                acc += (sumi[:, :, ib] * dw[None, :, ib]) * da[:, ib, None]
            elif t == Q4_1:
                acc += (dw[None, :, ib] * da[:, ib, None]) * sumi[:, :, ib] + m[None, :, ib] * sa[:, ib, None]
            else:
                acc += (dw[None, :, ib] * da[:, ib, None]) * sumi[:, :, ib]
        out[:, r0:r0 + q.shape[0]] = acc
    return out


def synth_blocks(t: int, N: int, K: int, seed: int, scale: float = 1.0) -> np.ndarray:
    """Random blocks of type t for an [N, K] matrix (valid bit patterns, sane fp16 scales), weight std ~ scale / sqrt(K)."""
    if t not in BLOCK_BYTES:
        return O.synth_blocks(t, N, K, seed, scale)
    rng = np.random.default_rng(seed)
    nb, bb = N * K // 32, BLOCK_BYTES[t]
    out = np.zeros((nb, bb), np.uint8)
    s = scale / np.sqrt(K)
    d = (rng.uniform(0.5, 1.5, nb) * s / (9.0 if t == Q5_0 else 4.5)).astype(np.float32)   # q uniform: (q - 8), q, (q - 16)
    out[:, 0:2] = d.astype(np.float16).view(np.uint8).reshape(nb, 2)
    if t == Q4_1:
        m = -d * 7.5 * rng.uniform(0.9, 1.1, nb).astype(np.float32)
        out[:, 2:4] = m.astype(np.float16).view(np.uint8).reshape(nb, 2)
        out[:, 4:] = rng.integers(0, 256, (nb, 16), dtype=np.uint8)
    else:
        out[:, 2:] = rng.integers(0, 256, (nb, bb - 2), dtype=np.uint8)
    return out.reshape(-1)


def retype(tm: TinyModel, name: str, t: int, seed: int) -> None:
    """Replaces a weight matrix of the model by synthetic blocks of type t (same shape)."""
    t0, a = tm.tensors[name]
    K = tm._row_len(name)
    N = a.size // row_size(t0, K)
    # the scales TinyModel gives its matrices: sqrt(n_embd) for the embedding, branch_scale 0.1 for the residual branches' outputs
    scale = np.sqrt(K) if name == "token_embd.weight" else 0.1 if name.endswith(("attn_output.weight", "ffn_down.weight")) else 1.0
    tm.tensors[name] = (t, synth_blocks(t, N, K, seed, scale))


def q4_0_model(seed: int, **kw) -> TinyModel:
    """The reference's Q4_0 mixture without an imatrix (src/llama.cpp:19271-19556): every matrix and the embedding Q4_0, the head Q6_K."""
    tm = TinyModel(arch="llama", ftype="q4_K_M", seed=seed, branch_scale=0.1, **kw)
    for i, (name, (t, a)) in enumerate(list(tm.tensors.items())):
        if a.dtype == np.uint8 and name != "output.weight":
            retype(tm, name, Q4_0, 1000 * seed + i)
    return tm


def models():
    """name -> (TinyModel, tokens) of the golden file: a Qwen2 Q4_K_M with n_ff 1 152 (not a multiple of 256: ffn_down Q4_K -> Q5_0 in
    layer 0, Q6_K -> Q8_0 in the use_more_bits layer 1) and a llama Q4_0."""
    qwen = TinyModel(n_layer=2, n_embd=512, n_head=4, n_head_kv=2, n_ff=1152, n_vocab=320, n_ctx=64, arch="qwen2", ftype="q4_K_M", seed=41,
                     branch_scale=0.1, types={"ffn_down": O.Q5_K})   # TinyModel's own fallback table ends at Q5_1 / Q8_0: retyped below
    retype(qwen, "blk.0.ffn_down.weight", Q5_0, 4101)
    retype(qwen, "blk.1.ffn_down.weight", O.Q8_0, 4102)
    llama = q4_0_model(43, n_layer=2, n_embd=512, n_head=4, n_head_kv=2, n_ff=1024, n_vocab=320, n_ctx=64)
    toks = [(i * 7919 + 13) % 320 for i in range(40)]
    return {"qwen2_q4_K_M": (qwen, toks), "llama_q4_0": (llama, toks)}


def write_gguf(tm: TinyModel, path) -> None:
    """TinyModel.write_gguf for models that hold the legacy types (GGUF v3 by the upstream gguf-py writer)."""
    import gguf
    w = gguf.GGUFWriter(str(path), tm.arch)
    hp = tm.hp
    w.add_block_count(hp["n_layer"]); w.add_embedding_length(hp["n_embd"]); w.add_head_count(hp["n_head"])
    w.add_head_count_kv(hp["n_head_kv"]); w.add_feed_forward_length(hp["n_ff"]); w.add_context_length(hp["n_ctx_orig"])
    w.add_rope_dimension_count(128); w.add_rope_freq_base(hp["rope_freq_base"]); w.add_layer_norm_rms_eps(hp["rms_eps"])
    for name, (t, a) in tm.tensors.items():
        if t == O.F32:
            w.add_tensor(name, np.ascontiguousarray(a, dtype=np.float32))
        else:
            rb = row_size(t, tm._row_len(name))
            w.add_tensor(name, np.ascontiguousarray(a).view(np.uint8).reshape(-1, rb), raw_dtype=gguf.GGMLQuantizationType(t))
    w.write_header_to_file(); w.write_kv_data_to_file(); w.write_tensors_to_file(); w.close()


# ---- the compiled reference (oracle/_ref) on the three types ----
def ref_quantize(ref: "O.Ref", t: int, w: np.ndarray) -> np.ndarray:
    """f32 [N, K] -> blocks by ggml_quantize_chunk"""
    w = np.ascontiguousarray(w, dtype=np.float32)
    N, K = w.shape
    out = np.zeros(N * row_size(t, K), np.uint8)
    assert ref.ggml.ggml_quantize_chunk(t, w.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), 0, N, K, None) == out.size
    return out


def ref_dequantize(ref: "O.Ref", t: int, blocks: np.ndarray, K: int) -> np.ndarray:
    fn = getattr(ref.ggml, f"dequantize_row_{NAME[t]}")
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
    b = np.ascontiguousarray(blocks, dtype=np.uint8).reshape(-1, row_size(t, K))
    out = np.empty((b.shape[0], K), np.float32)
    for i in range(b.shape[0]):
        fn(b[i].ctypes.data_as(C.c_void_p), out[i].ctypes.data_as(C.c_void_p), K)
    return out


def ref_quantize_act(ref: "O.Ref", t: int, x: np.ndarray) -> np.ndarray:
    return ref.quantize_act(ACT_TYPE[t], x)
