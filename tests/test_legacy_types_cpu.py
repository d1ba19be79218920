"""CPU: the legacy 32-element weight types Q4_0, Q4_1 and Q5_0 (Q4_0 files; Qwen2.5-72B Q4_K_M's ffn_down, where n_ff % 256 != 0 turns
Q4_K into Q5_0).  Their restatement (tests/legacy_types.py) against the reference's recorded outputs (golden/legacy_types_golden.npz) and,
where oracle/_ref is built, against the compiled reference itself; the library's row sizes; the GGUF parser on files holding the three
types."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest

import legacy_types as L
import oracle_lib as O
from golden import make_legacy_types_golden as LG

G = Path(__file__).resolve().parent / "golden"


@pytest.fixture(scope="module")
def gold():
    return np.load(G / "legacy_types_golden.npz")


@pytest.mark.parametrize("t", L.LEGACY_TYPES, ids=lambda t: L.NAME[t])
def test_restatement_matches_golden(port, gold, t):
    """Dequantization and the activation quantization bit-exact; mul_mat within fp32 summation order (the bar of
    test_qwen72b_ffn_down_fallback_types: 3e-6 of the largest output)."""
    n = L.NAME[t]
    for i, (N, K, T) in enumerate(LG.MULMAT_CASES):
        _, x = LG.mulmat_inputs(t, i, N, K, T)
        blocks = gold[f"{n}_{i}_blocks"]
        assert np.array_equal(L.dequantize(t, blocks, K), gold[f"{n}_{i}_dequant"]), (n, K)
        for j in range(T):
            assert np.array_equal(L.quantize_act(port, t, x[j]), gold[f"{n}_{i}_act"][j]), (n, K, j)
        y, ref = L.mul_mat(port, t, blocks, N, K, x), gold[f"{n}_{i}_mulmat"]
        assert np.max(np.abs(y - ref)) <= 3e-6 * max(1.0, float(np.max(np.abs(ref)))), (n, K)


@pytest.mark.parametrize("t", L.LEGACY_TYPES, ids=lambda t: L.NAME[t])
def test_restatement_matches_compiled_reference(port, ref, t):
    """Fresh seeds straight through the compiled reference: the reference quantizer's blocks and synthetic blocks."""
    rng = np.random.default_rng(70 + t)
    for N, K in ((8, 1024), (5, 29568 // 4)):
        w = (rng.standard_normal((N, K)) * 0.03).astype(np.float32)
        for blocks in (L.ref_quantize(ref, t, w), L.synth_blocks(t, N, K, seed=t + K)):
            assert np.array_equal(L.dequantize(t, blocks, K), L.ref_dequantize(ref, t, blocks, K))
            x = rng.standard_normal((2, K)).astype(np.float32)
            for j in range(2):
                assert np.array_equal(L.quantize_act(port, t, x[j]), L.ref_quantize_act(ref, t, x[j]))
            y, r = L.mul_mat(port, t, blocks, N, K, x), ref.mul_mat(t, blocks, N, K, x)
            assert np.max(np.abs(y - r)) <= 3e-6 * max(1.0, float(np.max(np.abs(r))))


def test_tiny_model_types_follow_the_reference_rules(gold):
    """The type of every tensor of the two golden models, as llama_tensor_get_type picks it (src/llama.cpp:19271-19556)."""
    for name, (tm, _) in L.models().items():
        want = {k: int(v) for k, v in (s.rsplit("|", 1) for s in gold[f"{name}_types"])}
        assert {k: v[0] for k, v in tm.tensors.items()} == want
    qwen, _ = L.models()["qwen2_q4_K_M"]
    assert qwen.tensors["blk.0.ffn_down.weight"][0] == L.Q5_0 and qwen.tensors["blk.1.ffn_down.weight"][0] == O.Q8_0
    llama, _ = L.models()["llama_q4_0"]
    assert llama.tensors["output.weight"][0] == O.Q6_K
    assert all(t in (L.Q4_0, O.F32) for k, (t, _) in llama.tensors.items() if k != "output.weight")


def test_golden_models_rebuild_bit_for_bit(ref, gold):
    """The compiled reference decodes the rebuilt models to the recorded logits (the seeds regenerate the same weights)."""
    for name, (tm, toks) in L.models().items():
        logits, _ = tm.ref_decode(ref, toks[:3])
        assert np.max(np.abs(logits - gold[f"{name}_logits"][:3])) < 1e-5, name


@pytest.mark.parametrize("t,bpb", [(L.Q4_0, 18), (L.Q4_1, 20), (L.Q5_0, 22)])
def test_row_bytes(lib, t, bpb):
    for k in (32, 4096, 7392, 29568):
        assert lib.c.pb200_row_bytes(t, k) == k // 32 * bpb == L.row_size(t, k)


def gguf_model():
    """A Q4_0 model whose ffn_down are Q4_1 (the reference's imatrix rule for the first layers) and attn_output Q5_0."""
    tm = L.q4_0_model(4, n_layer=2, n_embd=512, n_head=4, n_head_kv=2, n_ff=1024, n_vocab=320, n_ctx=64)
    for il in range(2):
        L.retype(tm, f"blk.{il}.ffn_down.weight", L.Q4_1, 70 + il)
        L.retype(tm, f"blk.{il}.attn_output.weight", L.Q5_0, 80 + il)
    return tm


def test_gguf_probe_accepts_the_legacy_types(pkg, tmp_path):
    """A Q4_0 file with a Q4_1 ffn_down and a Q5_0 attn_output: the parser sizes every tensor of the three types."""
    tm = gguf_model()
    assert {t for t, _ in tm.tensors.values()} == {O.F32, L.Q4_0, L.Q4_1, L.Q5_0, O.Q6_K}
    path = tmp_path / "q4_0.gguf"
    L.write_gguf(tm, path)
    lib = pkg.Lib.get()
    hp = pkg.HParams()
    n, nbytes, a = C.c_int32(), C.c_int64(), C.create_string_buffer(16)
    assert lib.c.pb200_gguf_probe(str(path).encode(), C.byref(hp), C.byref(n), C.byref(nbytes), a) == 0
    assert a.value.decode() == "llama" and n.value == len(tm.tensors) and hp.n_ff == 1024
    assert nbytes.value >= sum(np.asarray(a_).nbytes for _, a_ in tm.tensors.values())
