"""Tiny Llama/Qwen2-shaped models for parity tests: same quantized bytes go to the port oracle, the compiled reference
graph (oracle/_ref) and the CUDA engine.  TEST INFRASTRUCTURE."""
from __future__ import annotations

import ctypes as C

import numpy as np

import oracle_lib as O


def use_more_bits(i, n):  # src/llama.cpp:19278-19280
    return i < n // 8 or i >= 7 * n // 8 or (i - n // 8) % 3 == 2


class TinyModel:
    """Weights as raw GGUF blocks (uint8 arrays) + f32 vectors, keyed by GGUF tensor names."""

    def __init__(self, n_layer=2, n_embd=512, n_head=4, n_head_kv=2, n_ff=1024, n_vocab=320, n_ctx=64, arch="llama", ftype="q4_K_M",
                 seed=0, quantizer=None, freq_factors=False, types=None, branch_scale=1.0):
        self.hp = dict(n_layer=n_layer, n_embd=n_embd, n_head=n_head, n_head_kv=n_head_kv, head_dim=128, n_ff=n_ff, n_vocab=n_vocab,
                       n_ctx=n_ctx, rope_mode=0 if arch == "llama" else 2, n_ctx_orig=8192,
                       rope_freq_base=500000.0 if arch == "llama" else 1000000.0, rope_freq_scale=1.0,
                       rms_eps=1e-5 if arch == "llama" else 1e-6)
        self.arch = arch
        self.tensors: dict[str, tuple[int, np.ndarray]] = {}
        rng = np.random.default_rng(seed)
        E, QD, EK, F = n_embd, n_head * 128, n_head_kv * 128, n_ff
        default = O.Q4_K if ftype == "q4_K_M" else O.Q5_K
        self._seed = seed * 1000

        def fallback(t, K):   # rows that are not whole 256-element super-blocks (src/llama.cpp:19516-19551)
            if K % 256 == 0:
                return t
            return {O.Q4_K: O.Q5_0, O.Q5_K: O.Q5_1, O.Q6_K: O.Q8_0}[t]

        def qmat(name, t, N, K, scale=1.0):
            if types and name.split(".")[-2] in types:
                t = types[name.split(".")[-2]]
            t = fallback(t, K)
            self._seed += 1
            if quantizer is not None:
                w = (rng.standard_normal((N, K)) * (scale / np.sqrt(K))).astype(np.float32)
                self.tensors[name] = (t, quantizer(t, w))
            else:
                self.tensors[name] = (t, O.synth_blocks(t, N, K, self._seed, scale))

        def fvec(name, n, base, jit):
            self.tensors[name] = (O.F32, (base + jit * rng.standard_normal(n)).astype(np.float32))

        qmat("token_embd.weight", default, n_vocab, E, scale=np.sqrt(E))
        qmat("output.weight", O.Q6_K, n_vocab, E)
        fvec("output_norm.weight", E, 1.0, 0.05)
        if freq_factors:
            self.tensors["rope_freqs.weight"] = (O.F32, (1.0 + rng.uniform(0, 7, 64)).astype(np.float32))
        for il in range(n_layer):
            more = use_more_bits(il, n_layer)
            p = f"blk.{il}."
            fvec(p + "attn_norm.weight", E, 1.0, 0.05)
            fvec(p + "ffn_norm.weight", E, 1.0, 0.05)
            qmat(p + "attn_q.weight", default, QD, E)
            qmat(p + "attn_k.weight", default, EK, E)
            qmat(p + "attn_v.weight", O.Q6_K if more else (O.Q5_K if default == O.Q4_K else default), EK, E)
            qmat(p + "attn_output.weight", default, E, QD, scale=branch_scale)
            qmat(p + "ffn_gate.weight", default, F, E)
            qmat(p + "ffn_up.weight", default, F, E)
            qmat(p + "ffn_down.weight", O.Q6_K if more else default, E, F, scale=branch_scale)
            if arch == "qwen2":
                fvec(p + "attn_q.bias", QD, 0.0, 0.05)
                fvec(p + "attn_k.bias", EK, 0.0, 0.05)
                fvec(p + "attn_v.bias", EK, 0.0, 0.05)

    @classmethod
    def q4_0(cls, seed, **kw):
        """The reference's Q4_0 mixture without an imatrix (src/llama.cpp:19271-19556): every matrix and the embedding Q4_0, the head
        Q6_K."""
        tm = cls(arch="llama", ftype="q4_K_M", seed=seed, branch_scale=0.1, **kw)
        for i, (name, (t, a)) in enumerate(list(tm.tensors.items())):
            if a.dtype == np.uint8 and name != "output.weight":
                tm.retype(name, O.Q4_0, 1000 * seed + i)
        return tm

    def retype(self, name, t, seed):
        """Replaces a weight matrix by synthetic blocks of type t (same shape)."""
        t0, a = self.tensors[name]
        K = self._row_len(name)
        N = a.size // O.row_size(t0, K)
        # the scales __init__ gives its matrices: sqrt(n_embd) for the embedding, branch_scale 0.1 for the residual branches' outputs
        scale = np.sqrt(K) if name == "token_embd.weight" else 0.1 if name.endswith(("attn_output.weight", "ffn_down.weight")) else 1.0
        self.tensors[name] = (t, O.synth_blocks(t, N, K, seed, scale))

    # ---- oracle-side model struct (shared by port_llama_decode and gref_decode) ----
    def oracle_struct(self):
        hp = O.HParams(**self.hp)
        L = (O.Layer * self.hp["n_layer"])()
        keep = []

        def W(name):
            t, a = self.tensors[name]
            keep.append(a)
            return O.Weight(t, 0, a.ctypes.data_as(C.c_void_p).value)

        def V(name):
            if name not in self.tensors:
                return None
            a = self.tensors[name][1]
            keep.append(a)
            return a.ctypes.data_as(C.c_void_p).value

        for il in range(self.hp["n_layer"]):
            p = f"blk.{il}."
            L[il].attn_norm = V(p + "attn_norm.weight")
            L[il].ffn_norm = V(p + "ffn_norm.weight")
            L[il].wq, L[il].wk, L[il].wv = W(p + "attn_q.weight"), W(p + "attn_k.weight"), W(p + "attn_v.weight")
            L[il].wo = W(p + "attn_output.weight")
            L[il].gate, L[il].up, L[il].down = W(p + "ffn_gate.weight"), W(p + "ffn_up.weight"), W(p + "ffn_down.weight")
            L[il].bq, L[il].bk, L[il].bv = V(p + "attn_q.bias"), V(p + "attn_k.bias"), V(p + "attn_v.bias")
        EK = self.hp["n_head_kv"] * 128
        kc = np.zeros(self.hp["n_layer"] * self.hp["n_ctx"] * EK, dtype=np.uint16)
        vc = np.zeros_like(kc)
        m = O.Model()
        m.hp = hp
        m.tok_embd = W("token_embd.weight")
        m.output_norm = V("output_norm.weight")
        m.output = W("output.weight")
        m.layers = L
        m.rope_freq_factors = V("rope_freqs.weight")
        m.k_cache = kc.ctypes.data_as(C.c_void_p).value
        m.v_cache = vc.ctypes.data_as(C.c_void_p).value
        keep += [L, kc, vc]
        m._keep = keep
        return m

    def port_decode(self, port: "O.Port", tokens):
        m = self.oracle_struct()
        nv, E = self.hp["n_vocab"], self.hp["n_embd"]
        logits = np.zeros((len(tokens), nv), dtype=np.float32)
        hidden = np.zeros((len(tokens), E), dtype=np.float32)
        for i, t in enumerate(tokens):
            port.lib.port_llama_decode(C.byref(m), int(t), i, logits[i].ctypes.data_as(C.c_void_p), hidden[i].ctypes.data_as(C.c_void_p))
        return logits, hidden

    def ref_decode(self, ref: "O.Ref", tokens, batch_prefill=0):
        """Runs the restated graph on the reference CPU backend, token by token (decode), optionally a batched prompt first."""
        m = self.oracle_struct()
        nv, E = self.hp["n_vocab"], self.hp["n_embd"]
        h = ref.graph.gref_create(C.byref(m), ref.n_threads)
        logits = np.zeros((len(tokens), nv), dtype=np.float32)
        hidden = np.zeros((len(tokens), E), dtype=np.float32)
        toks = np.asarray(tokens, dtype=np.int32)
        mem = 256 << 20
        i = 0
        if batch_prefill > 1:
            rc = ref.graph.gref_decode(h, toks.ctypes.data_as(C.c_void_p), batch_prefill, 0, logits.ctypes.data_as(C.c_void_p),
                                       hidden.ctypes.data_as(C.c_void_p), mem)
            assert rc == 0
            i = batch_prefill
        while i < len(tokens):
            rc = ref.graph.gref_decode(h, toks[i:].ctypes.data_as(C.c_void_p), 1, i, logits[i].ctypes.data_as(C.c_void_p),
                                       hidden[i].ctypes.data_as(C.c_void_p), mem)
            assert rc == 0
            i += 1
        ref.graph.gref_free(h)
        return logits, hidden

    def load_engine(self, pkg, device=0, layers=None, with_embd=True, with_head=True):
        hp = pkg.HParams(**self.hp)
        eng = pkg.Model(hp, device, layers, with_embd, with_head)
        for name, (t, a) in self.tensors.items():
            eng.set_tensor(name, t, a)
        eng.finalize()
        return eng


    def write_gguf(self, path, with_tokenizer_array=True):
        """The model as a GGUF v3 file written by the upstream gguf-py writer (raw quantized blocks, the KV pairs llm_load_hparams reads,
        a string-array KV like a tokenizer table so that the parser's array skipping is exercised)."""
        import gguf
        w = gguf.GGUFWriter(str(path), self.arch)
        hp = self.hp
        w.add_block_count(hp["n_layer"]); w.add_embedding_length(hp["n_embd"]); w.add_head_count(hp["n_head"])
        w.add_head_count_kv(hp["n_head_kv"]); w.add_feed_forward_length(hp["n_ff"]); w.add_context_length(hp["n_ctx_orig"])
        w.add_rope_dimension_count(128); w.add_rope_freq_base(hp["rope_freq_base"]); w.add_layer_norm_rms_eps(hp["rms_eps"])
        if with_tokenizer_array:
            w.add_array("tokenizer.ggml.tokens", [f"t{i}" for i in range(hp["n_vocab"])])
            w.add_array("tokenizer.ggml.scores", [float(i) for i in range(hp["n_vocab"])])
        for name, (t, a) in self.tensors.items():
            if t == O.F32:
                w.add_tensor(name, np.ascontiguousarray(a, dtype=np.float32))
            else:
                K = self._row_len(name)
                rb = O.row_size(t, K)
                w.add_tensor(name, np.ascontiguousarray(a).view(np.uint8).reshape(-1, rb), raw_dtype=gguf.GGMLQuantizationType(t))
        w.write_header_to_file(); w.write_kv_data_to_file(); w.write_tensors_to_file(); w.close()

    def _row_len(self, name):
        E, F, QD = self.hp["n_embd"], self.hp["n_ff"], self.hp["n_head"] * 128
        if name.endswith("ffn_down.weight"):
            return F
        if name.endswith("attn_output.weight"):
            return QD
        return E


def from_golden(path):
    """Rebuilds a TinyModel (weights + hparams) and its reference outputs from a committed golden fixture."""
    z = np.load(path)
    tm = TinyModel.__new__(TinyModel)
    keys = [str(k) for k in z["hp_keys"]]
    vals = z["hp_vals"]
    ints = {"n_layer", "n_embd", "n_head", "n_head_kv", "head_dim", "n_ff", "n_vocab", "n_ctx", "rope_mode", "n_ctx_orig"}
    tm.hp = {k: (int(v) if k in ints else float(v)) for k, v in zip(keys, vals)}
    tm.arch = "llama" if tm.hp["rope_mode"] == 0 else "qwen2"
    tm.tensors = {}
    for k in z.files:
        if k.startswith("T|"):
            _, name, t = k.split("|")
            tm.tensors[name] = (int(t), np.ascontiguousarray(z[k]))
    return tm, z["tokens"], z["logits"], z["hidden"]


def legacy_golden_models():
    """name -> (TinyModel, tokens) of tests/golden/legacy_types_golden.npz: a Qwen2 Q4_K_M with n_ff 1 152 (not a multiple of 256: ffn_down
    Q4_K -> Q5_0 in layer 0, Q6_K -> Q8_0 in the use_more_bits layer 1) and a llama Q4_0.  The Qwen2's two ffn_down are the retyped
    blocks the reference's logits were recorded on."""
    qwen = TinyModel(n_layer=2, n_embd=512, n_head=4, n_head_kv=2, n_ff=1152, n_vocab=320, n_ctx=64, arch="qwen2", ftype="q4_K_M", seed=41,
                     branch_scale=0.1, types={"ffn_down": O.Q5_K})
    qwen.retype("blk.0.ffn_down.weight", O.Q5_0, 4101)
    qwen.retype("blk.1.ffn_down.weight", O.Q8_0, 4102)
    llama = TinyModel.q4_0(43, n_layer=2, n_embd=512, n_head=4, n_head_kv=2, n_ff=1024, n_vocab=320, n_ctx=64)
    toks = [(i * 7919 + 13) % 320 for i in range(40)]
    return {"qwen2_q4_K_M": (qwen, toks), "llama_q4_0": (llama, toks)}
