"""prima.cpp_b200 — H100-native (sm_90a) quantized-decode hot path of prima.cpp behind a C ABI.

The product is ``libprima_b200.so`` (CUDA kernels + C++ decode engine, ``include/prima_b200.h``) and
``libggml-b200.so`` (the same kernels behind the reference's ggml-backend vtables, ``include/ggml_b200.h``).
This Python package is only the thin ctypes binding used by tests and bench.py; it never falls back to a CPU
path: importing :mod:`host` raises if the CUDA library is missing.
"""
from .host import Lib, Model, HParams, Sampling, sampling, Penalties, LogitBias, penalties, Pb200Error, lib_path, build, TYPES  # noqa: F401
from .pipeline import PipelineRunner, RingRunner, PrefillPipeline, layer_windows  # noqa: F401
