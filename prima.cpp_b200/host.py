"""ctypes binding of include/prima_b200.h (plain pointers and sizes; torch only provides device memory in callers)."""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

PKG = Path(__file__).resolve().parent
ROOT = PKG.parent

TYPES = {"f32": 0, "f16": 1, "q4_0": 2, "q4_1": 3, "q5_0": 6, "q5_1": 7, "q8_0": 8, "q4_K": 12, "q5_K": 13, "q6_K": 14}


def lib_path() -> Path:
    import os
    alt = os.environ.get("PB200_LIB")   # development only: A/B of two builds of the library on one box (tools/runs/*.sh)
    return Path(alt) if alt else PKG / "libprima_b200.so"


def build(force: bool = False) -> Path:
    """Compile libprima_b200.so for sm_90a with nvcc (cross-compiles without a GPU)."""
    if force:
        subprocess.check_call(["make", "-C", str(PKG / "csrc"), "clean"], stdout=subprocess.DEVNULL)
    subprocess.check_call(["make", "-C", str(PKG / "csrc"), "-j4"], stdout=subprocess.DEVNULL)
    return lib_path()


class HParams(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("n_layer", "n_embd", "n_head", "n_head_kv", "head_dim", "n_ff", "n_vocab", "n_ctx",
                                          "rope_mode", "n_ctx_orig")] + \
               [(n, C.c_float) for n in ("rope_freq_base", "rope_freq_scale", "rms_eps")]


class Sampling(C.Structure):
    """pb200_sampling: the reference's sampler chain (top-k -> top-p -> min-p -> temperature -> dist); temp <= 0 is greedy."""
    _fields_ = [("top_k", C.c_int32), ("top_p", C.c_float), ("min_p", C.c_float), ("temp", C.c_float), ("min_keep", C.c_int32),
                ("seed", C.c_uint32)]


def sampling(top_k: int = 40, top_p: float = 0.95, min_p: float = 0.05, temp: float = 0.8, min_keep: int = 0, seed: int | None = None) -> Sampling:
    """Defaults of llama-cli (common/common.h:103-137); seed None draws a random one, like LLAMA_DEFAULT_SEED."""
    if seed is None:
        import secrets
        seed = secrets.randbits(32)
    return Sampling(int(top_k), float(top_p), float(min_p), float(temp), int(min_keep), int(seed) & 0xFFFFFFFF)


class LogitBias(C.Structure):
    """pb200_logit_bias (llama_logit_bias)."""
    _fields_ = [("token", C.c_int32), ("bias", C.c_float)]


class Penalties(C.Structure):
    """pb200_penalties: logit bias, ignore_eos and the repeat / frequency / presence penalties over the last last_n accepted tokens."""
    _fields_ = [("last_n", C.c_int32), ("repeat", C.c_float), ("freq", C.c_float), ("present", C.c_float), ("penalize_nl", C.c_int32),
                ("ignore_eos", C.c_int32), ("nl_token", C.c_int32), ("eos_token", C.c_int32), ("n_logit_bias", C.c_int32),
                ("logit_bias", C.POINTER(LogitBias))]


def penalties(last_n: int = 64, repeat: float = 1.0, freq: float = 0.0, present: float = 0.0, penalize_nl: bool = False,
              ignore_eos: bool = False, nl_token: int = -1, eos_token: int = -1, logit_bias=()) -> Penalties:
    """Defaults of llama-cli (common/common.h:118-126): last_n 64, every penalty off, the newline not penalised.  logit_bias: pairs
    (token, bias).  The vocabulary's newline / EOS ids are the caller's to pass (-1: none).  The returned structure keeps its list alive."""
    arr = (LogitBias * max(len(logit_bias), 1))(*[LogitBias(int(t), float(b)) for t, b in logit_bias])
    p = Penalties(int(last_n), float(repeat), float(freq), float(present), int(bool(penalize_nl)), int(bool(ignore_eos)), int(nl_token),
                  int(eos_token), len(logit_bias), C.cast(arr, C.POINTER(LogitBias)))
    p._keep = arr
    return p


class Pb200Error(RuntimeError):
    pass


class Lib:
    """Loads the CUDA library; raises loudly if it is missing (there is no CPU fallback)."""

    _inst = None

    def __init__(self):
        p = lib_path()
        if not p.exists():
            raise Pb200Error(f"{p} is missing: run __graft_entry__.build() (nvcc, sm_90a); no CPU fallback exists")
        self.c = C.CDLL(str(p))
        c = self.c
        vp, i32, i64, f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float
        c.pb200_version.restype = C.c_char_p
        c.pb200_error_string.restype = C.c_char_p
        c.pb200_error_string.argtypes = [C.c_int]
        c.pb200_row_bytes.restype = i64
        c.pb200_row_bytes.argtypes = [C.c_int, i64]
        c.pb200_kernel_launches.restype = C.c_uint64
        c.pb200_act_workspace_bytes.restype = C.c_size_t
        c.pb200_act_workspace_bytes.argtypes = [i64]
        c.pb200_quantize_act.argtypes = [C.c_int, vp, i64, vp, vp]
        c.pb200_mul_mat_vec_q.argtypes = [C.c_int, vp, i64, i64, vp, vp, vp, vp, vp]
        c.pb200_mul_mat_vec.argtypes = [C.c_int, vp, i64, i64, vp, vp, vp, vp]
        c.pb200_mul_mat_vec_fused.argtypes = [C.c_int, C.POINTER(C.c_int), C.POINTER(vp), C.POINTER(i64), i64, vp, C.POINTER(vp), vp]
        c.pb200_mul_mat_vec_host.argtypes = [C.c_int, vp, i64, i64, vp, vp]
        c.pb200_rms_norm.argtypes = [vp, vp, i64, i64, f32, vp]
        c.pb200_rope.argtypes = [vp, vp, i64, C.c_int, C.c_int, C.c_int, C.c_int, vp, f32, f32, f32, f32, f32, f32, C.c_int, vp, vp]
        c.pb200_soft_max.argtypes = [vp, vp, vp, i64, i64, i64, f32, vp]
        c.pb200_silu_mul.argtypes = [vp, vp, vp, i64, vp]
        c.pb200_get_rows.argtypes = [C.c_int, vp, i64, vp, i64, vp, vp]
        c.pb200_mul_mat_q_workspace_bytes.restype = C.c_size_t
        c.pb200_mul_mat_q_workspace_bytes.argtypes = [i64, i64]
        c.pb200_mul_mat_q.argtypes = [C.c_int, vp, i64, i64, vp, i64, i64, vp, vp, vp, vp, vp]
        c.pb200_attn_decode.argtypes = [vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, vp, C.c_int, f32, vp]
        c.pb200_attn_prefill.argtypes = [vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, vp, C.c_int, C.c_int, f32, vp]
        c.pb200_model_create.restype = vp
        c.pb200_model_create.argtypes = [C.POINTER(HParams), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
        c.pb200_model_free.argtypes = [vp]
        c.pb200_model_set_tensor.argtypes = [vp, C.c_char_p, C.c_int, vp, C.c_size_t]
        c.pb200_model_synth.argtypes = [vp, C.c_int, C.c_uint64]
        c.pb200_model_finalize.argtypes = [vp]
        c.pb200_model_weight_bytes.restype = i64
        c.pb200_model_weight_bytes.argtypes = [vp]
        c.pb200_kv_clear.argtypes = [vp]
        c.pb200_kv_seq_shift.argtypes = [vp, C.c_int, i32, i32, i32]
        c.pb200_kv_device.restype = vp
        c.pb200_kv_device.argtypes = [vp, C.c_int]
        c.pb200_rope_f16.argtypes = [vp, vp, i64, C.c_int, C.c_int, C.c_int, C.c_int, vp, f32, f32, f32, f32, f32, f32, C.c_int, vp, vp]
        c.pb200_decode.argtypes = [vp, i32, i32, vp]
        c.pb200_prefill.argtypes = [vp, vp, i32, i32, vp]
        c.pb200_prefill_stage.argtypes = [vp, vp, vp, i32, i32, vp, i32]
        c.pb200_gguf_probe.argtypes = [C.c_char_p, C.POINTER(HParams), C.POINTER(i32), C.POINTER(i64), C.c_char_p]
        c.pb200_model_load_gguf.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(vp), C.POINTER(C.c_double), C.POINTER(i64)]
        c.pb200_model_tensor_alloc.argtypes = [vp, C.c_char_p, C.c_int, C.c_size_t, C.POINTER(vp)]
        c.pb200_prefill_hidden_device.restype = vp
        c.pb200_prefill_hidden_device.argtypes = [vp]
        c.pb200_decode_async.argtypes = [vp, i32, i32]
        c.pb200_synchronize.argtypes = [vp]
        for n in ("pb200_logits_device", "pb200_hidden_in_device", "pb200_hidden_out_device", "pb200_stream"):
            getattr(c, n).restype = vp
            getattr(c, n).argtypes = [vp]
        c.pb200_get_hidden.argtypes = [vp, vp]
        c.pb200_set_hidden.argtypes = [vp, vp]
        c.pb200_debug_read.argtypes = [vp, C.c_char_p, vp, i64]
        c.pb200_profile_step.argtypes = [vp, i32, i32, C.POINTER(C.c_double), C.POINTER(i64), C.POINTER(i32), C.POINTER(C.c_double)]
        c.pb200_set_use_graph.argtypes = [vp, C.c_int]
        c.pb200_model_tensor_device.argtypes = [vp, C.c_char_p, C.POINTER(vp), C.POINTER(C.c_size_t), C.POINTER(C.c_int)]
        c.pb200_aborted.restype = C.c_int
        c.pb200_model_set_n_seq.argtypes = [vp, C.c_int]
        c.pb200_decode_seq_async.argtypes = [vp, C.c_int, i32, i32]
        c.pb200_step_seq_dev.argtypes = [vp, C.c_int, C.c_int]
        c.pb200_set_tokpos_seq.argtypes = [vp, C.c_int, i32, i32]
        c.pb200_argmax_seq.argtypes = [vp, C.c_int, C.c_int]
        for n in ("pb200_token_device", "pb200_sample_device"):
            getattr(c, n).restype = vp
            getattr(c, n).argtypes = [vp, C.c_int]
        c.pb200_sampler_state_bytes.restype = C.c_size_t
        c.pb200_sampler_seed.argtypes = [vp, C.c_uint32, vp]
        c.pb200_sample.argtypes = [vp, C.c_int, C.POINTER(Sampling), vp, vp, vp]
        c.pb200_sampling_set_seq.argtypes = [vp, C.c_int, C.POINTER(Sampling)]
        c.pb200_sample_seq.argtypes = [vp, C.c_int, C.c_int]
        c.pb200_penalty_state_bytes.restype = C.c_size_t
        c.pb200_penalty_state_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
        c.pb200_penalty_init.argtypes = [vp, C.c_int, C.POINTER(Penalties), vp]
        c.pb200_penalty_accept.argtypes = [vp, vp, C.c_int, vp]
        c.pb200_penalty_apply.argtypes = [vp, C.c_int, vp, vp, vp]
        c.pb200_penalties_set_seq.argtypes = [vp, C.c_int, C.POINTER(Penalties)]
        c.pb200_sampler_accept_seq.argtypes = [vp, C.c_int, vp, C.c_int]

    @classmethod
    def get(cls) -> "Lib":
        if cls._inst is None:
            cls._inst = Lib()
        return cls._inst

    def check(self, rc: int, what: str = "") -> None:
        if rc != 0:
            raise Pb200Error(f"{what}: {self.c.pb200_error_string(rc).decode()} ({rc})")

    def sampler_state_bytes(self) -> int:
        return self.c.pb200_sampler_state_bytes()

    def sampler_seed(self, state_ptr: int, seed: int, stream: int = 0) -> None:
        """state = std::mt19937(seed) in device memory of sampler_state_bytes()."""
        self.check(self.c.pb200_sampler_seed(C.c_void_p(state_ptr), seed & 0xFFFFFFFF, C.c_void_p(stream)), "sampler_seed")

    def sample(self, logits_ptr: int, n_vocab: int, p: Sampling, state_ptr: int, token_ptr: int, stream: int = 0) -> None:
        """pb200_sample: one token from n_vocab device logits into the int32 at token_ptr (enqueued on stream)."""
        self.check(self.c.pb200_sample(C.c_void_p(logits_ptr), n_vocab, C.byref(p), C.c_void_p(state_ptr), C.c_void_p(token_ptr), C.c_void_p(stream)),
                   "sample")

    def penalty_state_bytes(self, n_vocab: int, p: Penalties) -> int:
        return self.c.pb200_penalty_state_bytes(n_vocab, p.last_n, p.n_logit_bias)

    def penalty_init(self, state_ptr: int, n_vocab: int, p: Penalties, stream: int = 0) -> None:
        """A fresh penalties sampler in device memory of penalty_state_bytes(): configuration uploaded, history cleared."""
        self.check(self.c.pb200_penalty_init(C.c_void_p(state_ptr), n_vocab, C.byref(p), C.c_void_p(stream)), "penalty_init")

    def penalty_accept(self, state_ptr: int, tokens_ptr: int, n: int, stream: int = 0) -> None:
        """llama_sampler_accept for n int32 device tokens at tokens_ptr."""
        self.check(self.c.pb200_penalty_accept(C.c_void_p(state_ptr), C.c_void_p(tokens_ptr), n, C.c_void_p(stream)), "penalty_accept")

    def penalty_apply(self, logits_ptr: int, n_vocab: int, state_ptr: int, out_ptr: int, stream: int = 0) -> None:
        """out = the row with logit bias and penalties applied (a copy; out must not alias logits)."""
        self.check(self.c.pb200_penalty_apply(C.c_void_p(logits_ptr), n_vocab, C.c_void_p(state_ptr), C.c_void_p(out_ptr), C.c_void_p(stream)),
                   "penalty_apply")


class Model:
    """One model shard (layers [l0, l1)) resident on one GPU."""

    def __init__(self, hp: HParams, device: int = 0, layers: tuple[int, int] | None = None, with_embd: bool = True, with_head: bool = True):
        self.lib = Lib.get()
        self.hp = hp
        l0, l1 = layers if layers is not None else (0, hp.n_layer)
        self.h = self.lib.c.pb200_model_create(C.byref(hp), device, l0, l1, int(with_embd), int(with_head))
        if not self.h:
            raise Pb200Error("pb200_model_create failed (bad hparams or no CUDA device)")

    @classmethod
    def from_gguf(cls, path, device: int = 0, layers: tuple[int, int] | None = None, n_ctx: int = 0, with_embd: int = -1, with_head: int = -1) -> "Model":
        """pb200_model_load_gguf: a finalized shard straight from a GGUF file (pinned double-buffered stream to the device)."""
        lib = Lib.get()
        h = C.c_void_p()
        secs, nbytes = C.c_double(), C.c_int64()
        hp = HParams()
        lib.check(lib.c.pb200_gguf_probe(str(path).encode(), C.byref(hp), None, None, None), "gguf_probe")
        l0, l1 = layers if layers is not None else (0, -1)
        lib.check(lib.c.pb200_model_load_gguf(str(path).encode(), device, l0, l1, n_ctx, with_embd, with_head, C.byref(h), C.byref(secs), C.byref(nbytes)),
                  "model_load_gguf")
        m = cls.__new__(cls)
        m.lib = lib
        if n_ctx > 0:
            hp.n_ctx = n_ctx
        m.hp = hp
        m.h = h.value
        m.load_seconds, m.load_bytes = secs.value, nbytes.value
        return m

    def set_tensor(self, name: str, ttype: int, data) -> None:
        import numpy as np
        a = np.ascontiguousarray(data)
        self.lib.check(self.lib.c.pb200_model_set_tensor(self.h, name.encode(), ttype, a.ctypes.data_as(C.c_void_p), a.nbytes), f"set_tensor {name}")

    def synth(self, ftype: int, seed: int) -> None:
        self.lib.check(self.lib.c.pb200_model_synth(self.h, ftype, seed), "model_synth")

    def finalize(self) -> None:
        self.lib.check(self.lib.c.pb200_model_finalize(self.h), "model_finalize")

    @property
    def weight_bytes(self) -> int:
        return self.lib.c.pb200_model_weight_bytes(self.h)

    def kv_clear(self) -> None:
        self.lib.check(self.lib.c.pb200_kv_clear(self.h), "kv_clear")

    def kv_shift(self, seq: int, p0: int, p1: int, delta: int) -> None:
        """prima's context shift of slot seq (pb200_kv_seq_shift): cells [p0, p1) move to c + delta (delta < 0), K re-rotated by delta,
        and the slot's device position moves with them.  Enqueued on the model stream.  llama-cli's rule when the context fills:
        n_discard = (n_past - n_keep) // 2, kv_shift(seq, n_keep + n_discard, n_past, -n_discard)."""
        self.lib.check(self.lib.c.pb200_kv_seq_shift(self.h, seq, int(p0), int(p1), int(delta)), "kv_seq_shift")

    def kv_ptr(self, v: bool = False) -> int:
        """Device address of the f16 K (or V) cache: [n_seq][layers of this shard][n_ctx][n_head_kv * 128]."""
        return self.lib.c.pb200_kv_device(self.h, int(v)) or 0

    def decode(self, token: int, pos: int, logits_out=None):
        ptr = None if logits_out is None else logits_out.ctypes.data_as(C.c_void_p)
        self.lib.check(self.lib.c.pb200_decode(self.h, token, pos, ptr), "decode")
        return logits_out

    def prefill(self, tokens, pos0: int = 0, logits_out=None):
        """Prompt processing: all tokens as one batch (tensor-core mat-muls); returns the last token's logits."""
        import numpy as np
        toks = np.ascontiguousarray(tokens, dtype=np.int32)
        out = logits_out if logits_out is not None else np.empty(self.hp.n_vocab, dtype=np.float32)
        self.lib.check(self.lib.c.pb200_prefill(self.h, toks.ctypes.data_as(C.c_void_p), int(toks.size), int(pos0), out.ctypes.data_as(C.c_void_p)),
                       "prefill")
        return out

    def prefill_stage(self, tokens, hidden_in_ptr: int | None, n_tokens: int, pos0: int, logits_out=None, synchronize: bool = False) -> int:
        """One ubatch through this shard (pb200_prefill_stage); returns the device pointer of the stage's output hidden states."""
        import numpy as np
        tp = None
        if tokens is not None:
            self._pf_toks = np.ascontiguousarray(tokens, dtype=np.int32)   # kept alive until the (possibly asynchronous) copy has run
            tp = self._pf_toks.ctypes.data_as(C.c_void_p)
        lp = None if logits_out is None else logits_out.ctypes.data_as(C.c_void_p)
        self.lib.check(self.lib.c.pb200_prefill_stage(self.h, tp, C.c_void_p(hidden_in_ptr) if hidden_in_ptr else None, int(n_tokens), int(pos0), lp,
                                                      1 if synchronize else 0), "prefill_stage")
        return self.lib.c.pb200_prefill_hidden_device(self.h)

    def decode_async(self, token: int, pos: int) -> None:
        self.lib.check(self.lib.c.pb200_decode_async(self.h, token, pos), "decode_async")

    def synchronize(self) -> None:
        self.lib.check(self.lib.c.pb200_synchronize(self.h), "synchronize")

    def hidden(self):
        import numpy as np
        out = np.empty(self.hp.n_embd, dtype=np.float32)
        self.lib.check(self.lib.c.pb200_get_hidden(self.h, out.ctypes.data_as(C.c_void_p)), "get_hidden")
        return out

    def profile_step(self, token: int, pos: int) -> dict:
        g, b, n, st = C.c_double(), C.c_int64(), C.c_int32(), C.c_double()
        self.lib.check(self.lib.c.pb200_profile_step(self.h, token, pos, C.byref(g), C.byref(b), C.byref(n), C.byref(st)), "profile_step")
        return {"gemv_ms": g.value, "gemv_bytes": b.value, "gemv_launches": n.value, "step_ms": st.value}

    def debug_read(self, name: str, n: int):
        import numpy as np
        out = np.empty(n, dtype=np.float32)
        self.lib.check(self.lib.c.pb200_debug_read(self.h, name.encode(), out.ctypes.data_as(C.c_void_p), n), "debug_read")
        return out

    def set_hidden(self, h) -> None:
        import numpy as np
        a = np.ascontiguousarray(h, dtype=np.float32)
        self.lib.check(self.lib.c.pb200_set_hidden(self.h, a.ctypes.data_as(C.c_void_p)), "set_hidden")

    def tensor_device(self, name: str) -> tuple[int, int, int]:
        """(device address, bytes, ggml type) of a tensor held by this shard."""
        p, n, t = C.c_void_p(), C.c_size_t(), C.c_int()
        self.lib.check(self.lib.c.pb200_model_tensor_device(self.h, name.encode(), C.byref(p), C.byref(n), C.byref(t)), f"tensor_device {name}")
        return p.value, n.value, t.value

    def set_n_seq(self, n: int) -> None:
        self.lib.check(self.lib.c.pb200_model_set_n_seq(self.h, n), "set_n_seq")

    def decode_seq_async(self, seq: int, token: int, pos: int) -> None:
        self.lib.check(self.lib.c.pb200_decode_seq_async(self.h, seq, token, pos), "decode_seq_async")

    def step_seq_dev(self, seq: int, advance_pos: bool = True) -> None:
        self.lib.check(self.lib.c.pb200_step_seq_dev(self.h, seq, int(advance_pos)), "step_seq_dev")

    def set_tokpos_seq(self, seq: int, token: int, pos: int) -> None:
        self.lib.check(self.lib.c.pb200_set_tokpos_seq(self.h, seq, token, pos), "set_tokpos_seq")

    def argmax_seq(self, seq: int, feed_back: bool = False) -> None:
        self.lib.check(self.lib.c.pb200_argmax_seq(self.h, seq, int(feed_back)), "argmax_seq")

    def set_sampling(self, seq: int, top_k: int = 40, top_p: float = 0.95, min_p: float = 0.05, temp: float = 0.8, min_keep: int = 0,
                     seed: int | None = None) -> None:
        """Sampling parameters of slot seq (llama-cli's defaults); seeds the slot's generator (None: a random seed)."""
        p = sampling(top_k, top_p, min_p, temp, min_keep, seed)
        self.lib.check(self.lib.c.pb200_sampling_set_seq(self.h, seq, C.byref(p)), "sampling_set_seq")

    def sample_seq(self, seq: int, feed_back: bool = False) -> None:
        """argmax_seq with the slot's sampling parameters: the token goes to sample_ptr(seq) (and with feed_back to the slot)."""
        self.lib.check(self.lib.c.pb200_sample_seq(self.h, seq, int(feed_back)), "sample_seq")

    def set_penalties(self, seq: int, p: Penalties | None = None, **kw) -> None:
        """Logit bias and penalties of slot seq (a Penalties, or penalties()'s keywords); clears its history.  None without keywords
        removes them.  Sampling parameters and generator are left alone."""
        if p is None and kw:
            p = penalties(**kw)
        self.lib.check(self.lib.c.pb200_penalties_set_seq(self.h, seq, C.byref(p) if p is not None else None), "penalties_set_seq")

    def accept(self, seq: int, tokens) -> None:
        """Host tokens into slot seq's penalty history (the prompt, as llama-cli accepts it)."""
        import numpy as np
        t = np.ascontiguousarray(tokens, dtype=np.int32)
        self.lib.check(self.lib.c.pb200_sampler_accept_seq(self.h, seq, t.ctypes.data_as(C.c_void_p), int(t.size)), "sampler_accept_seq")

    def token_ptr(self, seq: int) -> int:
        return self.lib.c.pb200_token_device(self.h, seq)

    def sample_ptr(self, seq: int) -> int:
        return self.lib.c.pb200_sample_device(self.h, seq)

    def set_use_graph(self, on: bool) -> None:
        self.lib.c.pb200_set_use_graph(self.h, int(on))

    @property
    def stream(self) -> int:
        return self.lib.c.pb200_stream(self.h) or 0

    @property
    def hidden_in_ptr(self) -> int:
        return self.lib.c.pb200_hidden_in_device(self.h)

    @property
    def hidden_out_ptr(self) -> int:
        return self.lib.c.pb200_hidden_out_device(self.h)

    @property
    def logits_ptr(self) -> int:
        return self.lib.c.pb200_logits_device(self.h)

    def close(self) -> None:
        if self.h:
            self.lib.c.pb200_model_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
