"""GGUF -> device loader (SURVEY N2).  CPU: the container parser (pb200_gguf_probe) against files written by the upstream gguf-py writer
and against malformed files.  -m gpu: a model loaded by pb200_model_load_gguf decodes bit-identically to the same bytes handed over
tensor by tensor with pb200_model_set_tensor, whole and as a layer-window shard."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O
from tiny_model import TinyModel


def _tiny(arch="llama", **kw):
    return TinyModel(n_layer=2, n_embd=512, n_head=4, n_head_kv=2, n_ff=1024, n_vocab=320, n_ctx=64, arch=arch,
                     ftype="q4_K_M" if arch == "llama" else "q5_K_M", seed=4, branch_scale=0.1, freq_factors=(arch == "llama"), **kw)


def _q4_0_mix():
    """A Q4_0 model whose ffn_down are Q4_1 (the reference's imatrix rule for the first layers) and attn_output Q5_0."""
    tm = TinyModel.q4_0(4, n_layer=2, n_embd=512, n_head=4, n_head_kv=2, n_ff=1024, n_vocab=320, n_ctx=64)
    for il in range(2):
        tm.retype(f"blk.{il}.ffn_down.weight", O.Q4_1, 70 + il)
        tm.retype(f"blk.{il}.attn_output.weight", O.Q5_0, 80 + il)
    return tm


@pytest.mark.parametrize("t,bpb", [(O.Q4_0, 18), (O.Q4_1, 20), (O.Q5_0, 22)])
def test_row_bytes(lib, t, bpb):
    for k in (32, 4096, 7392, 29568):
        assert lib.c.pb200_row_bytes(t, k) == k // 32 * bpb == O.row_size(t, k)


def test_probe_accepts_the_legacy_types(pkg, tmp_path):
    """A Q4_0 file with a Q4_1 ffn_down and a Q5_0 attn_output: the parser sizes every tensor of the three types."""
    tm = _q4_0_mix()
    assert {t for t, _ in tm.tensors.values()} == {O.F32, O.Q4_0, O.Q4_1, O.Q5_0, O.Q6_K}
    path = tmp_path / "q4_0.gguf"
    tm.write_gguf(path)
    lib = pkg.Lib.get()
    hp = pkg.HParams()
    n, nbytes, a = C.c_int32(), C.c_int64(), C.create_string_buffer(16)
    assert lib.c.pb200_gguf_probe(str(path).encode(), C.byref(hp), C.byref(n), C.byref(nbytes), a) == 0
    assert a.value.decode() == "llama" and n.value == len(tm.tensors) and hp.n_ff == 1024
    assert nbytes.value >= sum(np.asarray(a_).nbytes for _, a_ in tm.tensors.values())


@pytest.mark.parametrize("arch", ["llama", "qwen2"])
def test_probe_reads_what_gguf_py_wrote(pkg, tmp_path, arch):
    tm = _tiny(arch)
    path = tmp_path / "m.gguf"
    tm.write_gguf(path)
    lib = pkg.Lib.get()
    hp = pkg.HParams()
    n, nbytes, a = C.c_int32(), C.c_int64(), C.create_string_buffer(16)
    assert lib.c.pb200_gguf_probe(str(path).encode(), C.byref(hp), C.byref(n), C.byref(nbytes), a) == 0
    assert a.value.decode() == arch
    assert n.value == len(tm.tensors)
    for k in ("n_layer", "n_embd", "n_head", "n_head_kv", "n_ff", "n_vocab", "rope_mode"):
        assert getattr(hp, k) == tm.hp[k], k
    assert hp.head_dim == 128 and hp.n_ctx_orig == tm.hp["n_ctx_orig"]
    assert abs(hp.rope_freq_base - tm.hp["rope_freq_base"]) < 1e-3 and abs(hp.rms_eps - tm.hp["rms_eps"]) < 1e-12
    # the data section holds at least every tensor's bytes (plus alignment padding)
    assert nbytes.value >= sum(np.asarray(a_).nbytes for _, a_ in tm.tensors.values())


def test_probe_rejects_bad_files(pkg, tmp_path):
    lib = pkg.Lib.get()
    hp = pkg.HParams()
    bad = tmp_path / "bad.gguf"
    bad.write_bytes(b"GGML" + b"\0" * 64)
    assert lib.c.pb200_gguf_probe(str(bad).encode(), C.byref(hp), None, None, None) != 0        # wrong magic
    assert lib.c.pb200_gguf_probe(str(tmp_path / "missing.gguf").encode(), C.byref(hp), None, None, None) != 0
    good = tmp_path / "m.gguf"
    _tiny().write_gguf(good)
    raw = good.read_bytes()
    (tmp_path / "trunc.gguf").write_bytes(raw[: len(raw) // 2])                                  # tensor data cut off
    assert lib.c.pb200_gguf_probe(str(tmp_path / "trunc.gguf").encode(), C.byref(hp), None, None, None) != 0
    (tmp_path / "v1.gguf").write_bytes(raw[:4] + (1).to_bytes(4, "little") + raw[8:])           # version 1: not supported
    assert lib.c.pb200_gguf_probe(str(tmp_path / "v1.gguf").encode(), C.byref(hp), None, None, None) != 0


def test_probe_accepts_version_2_and_custom_alignment(pkg, tmp_path):
    """GGUF v2 has the v3 layout (64-bit counts and lengths); general.alignment moves the data section (gguf_init_from_file honours both)."""
    import gguf
    lib = pkg.Lib.get()
    tm = _tiny()
    v3 = tmp_path / "v3.gguf"
    tm.write_gguf(v3)
    raw = v3.read_bytes()
    v2 = tmp_path / "v2.gguf"
    v2.write_bytes(raw[:4] + (2).to_bytes(4, "little") + raw[8:])
    hp = pkg.HParams()
    n = C.c_int32()
    assert lib.c.pb200_gguf_probe(str(v2).encode(), C.byref(hp), C.byref(n), None, None) == 0
    assert hp.n_layer == tm.hp["n_layer"] and n.value == len(tm.tensors)
    # a writer with 64-byte alignment: every tensor offset and the data section start move
    al = tmp_path / "al.gguf"
    w = gguf.GGUFWriter(str(al), "llama")
    w.add_custom_alignment(64)
    h = tm.hp
    w.add_block_count(h["n_layer"]); w.add_embedding_length(h["n_embd"]); w.add_head_count(h["n_head"]); w.add_head_count_kv(h["n_head_kv"])
    w.add_feed_forward_length(h["n_ff"]); w.add_context_length(h["n_ctx_orig"]); w.add_rope_dimension_count(128)
    for name, (t, a) in tm.tensors.items():
        if t == 0:
            w.add_tensor(name, np.ascontiguousarray(a, dtype=np.float32))
        else:
            w.add_tensor(name, np.ascontiguousarray(a).view(np.uint8).reshape(-1, O.row_size(t, tm._row_len(name))), raw_dtype=gguf.GGMLQuantizationType(t))
    w.write_header_to_file(); w.write_kv_data_to_file(); w.write_tensors_to_file(); w.close()
    nb = C.c_int64()
    assert lib.c.pb200_gguf_probe(str(al).encode(), C.byref(hp), C.byref(n), C.byref(nb), None) == 0
    assert hp.n_embd == h["n_embd"] and hp.rope_freq_base == 10000.0      # rope base absent: the loader's default, like llm_load_hparams
    assert (al.stat().st_size - nb.value) % 64 == 0                          # the data section starts on the custom alignment


def check_gguf_load(pkg, tmp_path, tm):
    path = tmp_path / "m.gguf"
    tm.write_gguf(path)
    toks = [(i * 7919 + 13) % 320 for i in range(8)]
    ref = tm.load_engine(pkg)
    want = np.zeros((len(toks), 320), np.float32)
    for i, t in enumerate(toks):
        ref.decode(int(t), i, want[i])
    ref.close()
    eng = pkg.Model.from_gguf(path, n_ctx=64)
    assert eng.load_bytes == sum(np.asarray(a).nbytes for _, a in tm.tensors.values())
    got = np.zeros_like(want)
    for i, t in enumerate(toks):
        eng.decode(int(t), i, got[i])
    eng.close()
    assert np.array_equal(got, want)
    # a two-stage pipeline straight from the file: every shard reads only its window
    s0 = pkg.Model.from_gguf(path, layers=(0, 1), n_ctx=64)
    s1 = pkg.Model.from_gguf(path, layers=(1, 2), n_ctx=64)
    assert s0.load_bytes < eng.load_bytes and s1.load_bytes < eng.load_bytes
    got2 = np.zeros_like(want)
    for i, t in enumerate(toks):
        s0.decode(int(t), i, None)
        s1.set_hidden(s0.hidden())
        s1.decode(int(t), i, got2[i])
    s0.close(); s1.close()
    assert np.array_equal(got2, want)


@pytest.mark.gpu
@pytest.mark.parametrize("arch", ["llama", "qwen2"])
def test_gguf_loaded_model_decodes_like_set_tensor_model(cuda, pkg, tmp_path, arch):
    check_gguf_load(pkg, tmp_path, _tiny(arch))


@pytest.mark.gpu
def test_gguf_loaded_legacy_types_model_decodes_like_set_tensor_model(cuda, pkg, tmp_path):
    """A Q4_0 file with a Q4_1 ffn_down and a Q5_0 attn_output."""
    check_gguf_load(pkg, tmp_path, _q4_0_mix())
