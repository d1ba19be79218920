"""ctypes binding of host/llama_graph_host.cpp — the stand-in for libllama used by the whole-graph parity test and by bench.py's
end-to-end leg.  Loads, in this order and process-wide (RTLD_GLOBAL): the host's ggml core (host/_ggml/libggml_host.so, the
reference's own, unmodified), the plugin prima.cpp_b200/libggml-b200.so (its constructor registers the "B200" backend with that ggml:
ggml_backend_register), then the graph driver.  Must not share a process with oracle/_ref's copy of ggml (two ggml cores would
interpose each other's symbols): callers run it in a process of its own, or before / without the oracle."""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
HOST = ROOT / "host"
PLUGIN = ROOT / "prima.cpp_b200" / "libggml-b200.so"
# same-box GPU comparator (measurement infrastructure, oracle/Makefile.cudaref): the reference's own ggml-cuda backend built for sm_90a
CUDAREF = ROOT / "oracle" / "_ref" / "cuda" / "libggml-cuda-ref.so"


class HParams(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("n_layer", "n_embd", "n_head", "n_head_kv", "head_dim", "n_ff", "n_vocab", "n_ctx", "rope_mode", "n_ctx_orig")] + \
               [(n, C.c_float) for n in ("rope_freq_base", "rope_freq_scale", "rms_eps")] + \
               [(n, C.c_int32) for n in ("has_bias", "has_freq_factors", "type_default", "type_v_even", "type_v_odd", "type_down_even", "type_down_odd", "type_output")]


def build() -> None:
    # the reference tree oracle/Makefile points at (REF) must be readable by this user
    if subprocess.call(["make", "-s", "-C", str(ROOT / "oracle"), "have-ref"], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL) == 0:
        subprocess.check_call(["make", "-C", str(HOST), "-j8"], stdout=subprocess.DEVNULL)


_libs = None


def load(with_plugin: bool = True, with_cudaref: bool = False):
    """Returns (graph_lib, plugin_lib or None)."""
    global _libs
    if _libs is not None:
        return _libs
    if with_cudaref and not CUDAREF.exists():
        raise RuntimeError(f"{CUDAREF} is missing: make -C oracle -f Makefile.cudaref (needs the reference source tree)")
    core = HOST / "_ggml" / "libggml_host.so"
    drv = HOST / "_ggml" / "libllama_graph_host.so"
    if not core.exists() or not drv.exists():
        build()
    if not core.exists() or not drv.exists():
        raise RuntimeError("host/_ggml is not built (needs the reference tree: run __graft_entry__.build() where it is readable)")
    C.CDLL(str(core), mode=C.RTLD_GLOBAL)
    plug = None
    if with_plugin:
        if not PLUGIN.exists():
            raise RuntimeError(f"{PLUGIN} is missing: run __graft_entry__.build(); there is no CPU fallback for the B200 backend")
        plug = C.CDLL(str(PLUGIN), mode=C.RTLD_GLOBAL)
        plug.ggml_backend_b200_nodes_computed.restype = C.c_ulonglong
        plug.ggml_backend_b200_fused_steps.restype = C.c_ulonglong
        plug.ggml_backend_b200_graph_replays.restype = C.c_ulonglong
    if with_cudaref:
        C.CDLL(str(CUDAREF), mode=C.RTLD_GLOBAL)   # its constructor registers the "CUDA" backend (oracle/cudaref_register.cpp)
    g = C.CDLL(str(drv), mode=C.RTLD_GLOBAL)
    vp = C.c_void_p
    g.lgh_create.restype = vp
    g.lgh_create.argtypes = [C.POINTER(HParams), C.POINTER(C.c_int32), C.c_char_p, C.c_int]
    g.lgh_free.argtypes = [vp]
    g.lgh_set_tensor.argtypes = [vp, C.c_char_p, vp, C.c_size_t]
    g.lgh_tensor_data.restype = vp
    g.lgh_tensor_data.argtypes = [vp, C.c_char_p, C.POINTER(C.c_size_t)]
    g.lgh_get_tensor.argtypes = [vp, C.c_char_p, vp, C.c_size_t]
    g.lgh_kv_clear.argtypes = [vp]
    g.lgh_graph_builds.restype = C.c_uint64
    g.lgh_graph_builds.argtypes = [vp]
    g.lgh_graph_nodes.argtypes = [vp]
    g.lgh_reserve.argtypes = [vp, C.c_int]
    g.lgh_compute_buffer_base.restype = vp
    g.lgh_compute_buffer_base.argtypes = [vp]
    g.lgh_unsupported_nodes.argtypes = [vp]
    g.lgh_decode.argtypes = [vp, vp, C.c_int, C.c_int, vp, C.c_int]
    g.lgh_get_hidden.argtypes = [vp, vp]
    g.lgh_phase_seconds.argtypes = [vp, C.POINTER(C.c_double)]
    g.lgh_kv_seq_rm.argtypes = [vp, C.c_int32, C.c_int32]
    g.lgh_kv_seq_add.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32]
    g.lgh_kv_cells.argtypes = [vp, vp]
    g.lgh_kshift_unsupported_nodes.argtypes = [vp]
    g.lgh_kshift_nodes.argtypes = [vp]
    g.lgh_k_shifts.restype = C.c_uint64
    g.lgh_k_shifts.argtypes = [vp]
    _libs = (g, plug)
    return _libs


WEIGHT_ORDER = ("attn_q", "attn_k", "attn_v", "attn_output", "ffn_gate", "ffn_up", "ffn_down")


class HostModel:
    """A model living in the buffers of one ggml backend ("CPU", "B200_0", ...), driven like llama_decode drives it."""

    def __init__(self, hp: dict, types: dict, backend: str, n_threads: int = 8, has_bias: bool = False, has_freq_factors: bool = False,
                 n_tokens_max: int = 1):
        """types: tensor name -> ggml_type for "token_embd.weight", "output.weight" and "blk.N.<WEIGHT_ORDER>.weight".
        n_tokens_max: the largest batch the compute buffer is reserved for (llama.cpp's n_ubatch); a larger batch still runs, but
        grows (moves) the buffer."""
        self.g, self.plug = load(with_plugin=backend.startswith("B200"), with_cudaref=backend.startswith("CUDA"))
        self.hp = hp
        H = HParams(**{k: hp[k] for k in ("n_layer", "n_embd", "n_head", "n_head_kv", "head_dim", "n_ff", "n_vocab", "n_ctx", "rope_mode", "n_ctx_orig",
                                          "rope_freq_base", "rope_freq_scale", "rms_eps")}, has_bias=int(has_bias), has_freq_factors=int(has_freq_factors))
        tl = [types["token_embd.weight"], types["output.weight"]]
        for il in range(hp["n_layer"]):
            tl += [types[f"blk.{il}.{w}.weight"] for w in WEIGHT_ORDER]
        arr = (C.c_int32 * len(tl))(*tl)
        self.h = self.g.lgh_create(C.byref(H), arr, backend.encode(), n_threads)
        if not self.h:
            raise RuntimeError(f"lgh_create failed for backend {backend}")
        rc = self.g.lgh_reserve(self.h, int(n_tokens_max))
        if rc != 0:
            self.close()
            raise RuntimeError(f"lgh_reserve({n_tokens_max}) failed for backend {backend}: {rc}")

    def set_tensor(self, name: str, data) -> None:
        import numpy as np
        a = np.ascontiguousarray(data)
        rc = self.g.lgh_set_tensor(self.h, name.encode(), a.ctypes.data_as(C.c_void_p), a.nbytes)
        if rc != 0:
            raise RuntimeError(f"lgh_set_tensor {name}: {rc}")

    def tensor_ptr(self, name: str) -> tuple[int, int]:
        n = C.c_size_t()
        p = self.g.lgh_tensor_data(self.h, name.encode(), C.byref(n))
        if not p:
            raise KeyError(name)
        return p, n.value

    def decode(self, tokens, pos0: int, logits_out=None, all_logits: bool = False):
        import numpy as np
        toks = np.ascontiguousarray(tokens, dtype=np.int32)
        ptr = None if logits_out is None else logits_out.ctypes.data_as(C.c_void_p)
        rc = self.g.lgh_decode(self.h, toks.ctypes.data_as(C.c_void_p), int(toks.size), int(pos0), ptr, int(all_logits))
        if rc != 0:
            raise RuntimeError(f"lgh_decode: {rc}")
        return logits_out

    def hidden(self, n_tokens: int = 1):
        import numpy as np
        out = np.empty((n_tokens, self.hp["n_embd"]), dtype=np.float32)
        self.g.lgh_get_hidden(self.h, out.ctypes.data_as(C.c_void_p))
        return out

    def get_tensor(self, name: str, nbytes: int):
        import numpy as np
        out = np.empty(nbytes, dtype=np.uint8)
        rc = self.g.lgh_get_tensor(self.h, name.encode(), out.ctypes.data_as(C.c_void_p), nbytes)
        if rc != 0:
            raise RuntimeError(f"lgh_get_tensor {name}: {rc}")
        return out

    def kv_clear(self) -> None:
        self.g.lgh_kv_clear(self.h)

    def kv_seq_rm(self, p0: int, p1: int) -> None:
        """llama_kv_cache_seq_rm of the one sequence: cells holding positions [p0, p1) become empty (holes)."""
        self.g.lgh_kv_seq_rm(self.h, int(p0), int(p1))

    def kv_seq_add(self, p0: int, p1: int, delta: int) -> None:
        """llama_kv_cache_seq_add: cells holding positions [p0, p1) now hold position + delta; the next decode first runs the
        K-shift graph (one in-place f16 ROPE per layer) on the backend."""
        self.g.lgh_kv_seq_add(self.h, int(p0), int(p1), int(delta))

    def kv_cells(self):
        """Position held by each cell (-1 = empty)."""
        import numpy as np
        out = np.empty(self.hp["n_ctx"], dtype=np.int32)
        self.g.lgh_kv_cells(self.h, out.ctypes.data_as(C.c_void_p))
        return out

    @property
    def kshift_unsupported_nodes(self) -> int:
        """Non-view nodes of the K-shift graph the backend does not support (the scheduler aborts on such a node of a cache it owns)."""
        return self.g.lgh_kshift_unsupported_nodes(self.h)

    @property
    def kshift_nodes(self) -> int:
        return self.g.lgh_kshift_nodes(self.h)

    @property
    def k_shifts(self) -> int:
        """K-shift graphs computed so far."""
        return self.g.lgh_k_shifts(self.h)

    def phase_seconds(self) -> dict:
        """Host seconds since the last call in: graph (re)build + allocation, input upload, graph_compute (enqueue), wait + logits read."""
        a = (C.c_double * 4)()
        self.g.lgh_phase_seconds(self.h, a)
        return {"graph_build": a[0], "set_inputs": a[1], "graph_compute_call": a[2], "wait_and_get": a[3]}

    @property
    def graph_builds(self) -> int:
        return self.g.lgh_graph_builds(self.h)

    @property
    def graph_nodes(self) -> int:
        return self.g.lgh_graph_nodes(self.h)

    @property
    def compute_buffer_base(self) -> int:
        """Device / host address of the compute buffer (0 before the first decode); constant while every graph fits the reservation."""
        return self.g.lgh_compute_buffer_base(self.h) or 0

    @property
    def unsupported_nodes(self) -> int:
        """Non-view nodes of the current graph for which ggml_backend_supports_op is false (llama.cpp would run them on the CPU)."""
        return self.g.lgh_unsupported_nodes(self.h)

    def close(self) -> None:
        if self.h:
            self.g.lgh_free(self.h)
            self.h = None
