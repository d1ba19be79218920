"""Writes tests/golden/sampling_golden.npz: the reference's own sampler chain (oracle/_ref/libsampling_ref.so, built by
`make -C oracle -f Makefile.sampling` from the reference's unmodified src/llama-sampling.cpp) on seeded logits.

Chain per case, as gpt_sampler_init builds it (common/sampling.cpp:140-224): top_k -> top_p(p, min_keep) -> min_p(p, min_keep) ->
temp_ext(t, 0, 1) -> softmax -> dist(seed).  Logits are regenerated from (seed, n, scale, spike) by sampling_ref.make_logits.
Recorded per single-draw case: the selected token, the survivor count, the first survivors' p (up to P_HEAD) and the double running
sums around the pick.  Sequences carry one chain (one generator) across SEQ_STEPS draws; every spike_every-th step has a spiked
maximum that min-p leaves alone, a single survivor that must not advance the generator.

    python tests/golden/make_sampling_golden.py
"""
import ctypes as C
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
import sampling_ref as S  # noqa: E402

LIB = HERE.parent.parent / "oracle" / "_ref" / "libsampling_ref.so"
P_HEAD = 64
SEQ_STEPS = 1000
VOCABS = (128256, 152064, 1000)
# name: (top_k, top_p, min_p, temp, min_keep, spike)
PARAMS = {
    "defaults": (40, 0.95, 0.05, 0.8, 0, 0.0),
    "top_k_1": (1, 0.95, 0.05, 0.8, 0, 0.0),
    "top_p_0.9": (0, 0.9, 0.0, 0.8, 0, 0.0),
    "min_p_0.05": (0, 1.0, 0.05, 0.8, 0, 0.0),
    "temp_1.0": (0, 1.0, 0.0, 1.0, 0, 0.0),
    "temp_1.5": (0, 1.0, 0.0, 1.5, 0, 0.0),
    "temp_0.01": (40, 0.95, 0.05, 0.01, 0, 0.0),
    "min_keep_30": (40, 0.5, 0.3, 0.8, 30, 0.0),
    "single": (40, 0.95, 0.05, 0.8, 0, 12.0),
}
SEEDS_PER = 8
# sequences: (n_vocab, params name, dist seed, logit seed base, spike_every)
SEQS = ((1000, "defaults", 1234, 7000000, 5), (152064, "defaults", 4321, 9000000, 7))

TokenData = np.dtype([("id", "<i4"), ("logit", "<f4"), ("p", "<f4")], align=True)


class TokenDataArray(C.Structure):
    _fields_ = [("data", C.c_void_p), ("size", C.c_size_t), ("selected", C.c_int64), ("sorted", C.c_bool)]


class ChainParams(C.Structure):
    _fields_ = [("no_perf", C.c_bool)]


class RefChain:
    """One llama_sampler chain of the live reference library."""

    def __init__(self, lib, top_k, top_p, min_p, temp, min_keep, seed):
        self.lib = lib
        vp = C.c_void_p
        lib.llama_sampler_chain_init.restype = vp
        lib.llama_sampler_chain_init.argtypes = [ChainParams]
        lib.llama_sampler_chain_add.argtypes = [vp, vp]
        for f, at in (("top_k", [C.c_int32]), ("top_p", [C.c_float, C.c_size_t]), ("min_p", [C.c_float, C.c_size_t]),
                      ("temp_ext", [C.c_float, C.c_float, C.c_float]), ("softmax", []), ("dist", [C.c_uint32])):
            fn = getattr(lib, "llama_sampler_init_" + f)
            fn.restype, fn.argtypes = vp, at
        lib.llama_sampler_apply.argtypes = [vp, C.POINTER(TokenDataArray)]
        lib.llama_sampler_free.argtypes = [vp]
        self.h = lib.llama_sampler_chain_init(ChainParams(True))
        for s in (lib.llama_sampler_init_top_k(top_k), lib.llama_sampler_init_top_p(top_p, min_keep), lib.llama_sampler_init_min_p(min_p, min_keep),
                  lib.llama_sampler_init_temp_ext(temp, 0.0, 1.0), lib.llama_sampler_init_softmax(), lib.llama_sampler_init_dist(seed)):
            lib.llama_sampler_chain_add(self.h, s)

    def __call__(self, logits):
        n = logits.size
        d = np.zeros(n, TokenData)
        d["id"] = np.arange(n)
        d["logit"] = logits
        arr = TokenDataArray(d.ctypes.data, n, -1, False)
        self.lib.llama_sampler_apply(self.h, C.byref(arr))
        sel = int(arr.selected)
        size = int(arr.size)
        return int(d["id"][sel]), size, d["p"][:size].copy(), sel

    def close(self):
        self.lib.llama_sampler_free(self.h)


def cum_around(p, sel):
    pd = p.astype(np.float64)
    cp = np.cumsum(pd / np.cumsum(pd)[-1])
    cp[-1] = 1.0
    return np.array([cp[sel - 1] if sel > 0 else 0.0, cp[sel]])


def main():
    lib = C.CDLL(str(LIB))
    rows = []
    for n in VOCABS:
        for pi, (name, (tk, tp, mp, t, mk, spike)) in enumerate(PARAMS.items()):
            for s in range(SEEDS_PER):
                lseed = 1000003 * n + 101 * pi + s
                dseed = (lseed * 2654435761) & 0xFFFFFFFF
                logits = S.make_logits(lseed, n, 3.0, spike)
                ch = RefChain(lib, tk, tp, mp, t, mk, dseed)
                tok, size, p, sel = ch(logits)
                ch.close()
                head = np.zeros(P_HEAD, np.float32)
                head[: min(size, P_HEAD)] = p[:P_HEAD]
                rows.append((n, tk, tp, mp, t, mk, spike, lseed, dseed, tok, size, head, cum_around(p, sel) if size > 1 else np.ones(2)))
                print(f"n={n:6d} {name:12s} seed {s}: token {tok:6d}, {size} survivors", flush=True)
    out = {
        "n_vocab": np.array([r[0] for r in rows], np.int32), "top_k": np.array([r[1] for r in rows], np.int32),
        "top_p": np.array([r[2] for r in rows], np.float32), "min_p": np.array([r[3] for r in rows], np.float32),
        "temp": np.array([r[4] for r in rows], np.float32), "min_keep": np.array([r[5] for r in rows], np.int32),
        "spike": np.array([r[6] for r in rows], np.float32), "logit_seed": np.array([r[7] for r in rows], np.int64),
        "dist_seed": np.array([r[8] for r in rows], np.uint32), "token": np.array([r[9] for r in rows], np.int32),
        "n_surv": np.array([r[10] for r in rows], np.int32), "p_head": np.stack([r[11] for r in rows]),
        "cum_sel": np.stack([r[12] for r in rows]),
    }
    seq_tok, seq_surv = [], []
    for n, name, dseed, base, every in SEQS:
        tk, tp, mp, t, mk, _ = PARAMS[name]
        ch = RefChain(lib, tk, tp, mp, t, mk, dseed)
        toks, survs = [], []
        for i in range(SEQ_STEPS):
            tok, size, _, _ = ch(S.make_logits(base + i, n, 3.0, 12.0 if i % every == 0 else 0.0))
            toks.append(tok); survs.append(size)
        ch.close()
        print(f"sequence n={n}: {sum(1 for x in survs if x == 1)} single-survivor steps of {SEQ_STEPS}", flush=True)
        seq_tok.append(toks); seq_surv.append(survs)
    out.update({
        "seq_n_vocab": np.array([s[0] for s in SEQS], np.int32),
        "seq_params": np.array([PARAMS[s[1]][:5] for s in SEQS], np.float64),
        "seq_dist_seed": np.array([s[2] for s in SEQS], np.uint32), "seq_logit_base": np.array([s[3] for s in SEQS], np.int64),
        "seq_spike_every": np.array([s[4] for s in SEQS], np.int32),
        "seq_token": np.array(seq_tok, np.int32), "seq_n_surv": np.array(seq_surv, np.int32),
    })
    np.savez_compressed(HERE / "sampling_golden.npz", **out)


if __name__ == "__main__":
    main()
