"""Writes tests/golden/penalties_golden.npz: the reference's logit-bias and penalties samplers (oracle/_ref/libsampling_ref.so, built by
`make -C oracle -f Makefile.sampling` from the reference's unmodified src/llama-sampling.cpp) in front of its chains.

Chains, as gpt_sampler_init builds them (common/sampling.cpp:156-224):
  logit_bias -> penalties -> top_k -> top_p -> min_p -> temp_ext -> softmax -> dist     ("dist", llama-cli's defaults)
  logit_bias -> penalties -> greedy                                                      ("greedy", temp <= 0)
History: llama_sampler_accept of a prompt (and, in the sequences, of every sampled token), as llama-cli does
(examples/main/main.cpp:702, 720).  The penalised row is read from a second chain of logit_bias -> penalties alone with the same
configuration and history, and recorded as a sparse diff against the input row.

Single rows: every case of CASES at 1 000, 128 256 and 152 064 logits.  Sequences: SEQ_STEPS steps whose logits are raised on the last
sampled tokens (penalties_ref.seq_logits), so the penalty decides the token.

    python tests/golden/make_penalties_golden.py
"""
import ctypes as C
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE))
import penalties_ref as P  # noqa: E402
import sampling_ref as S  # noqa: E402
from make_sampling_golden import ChainParams, TokenData, TokenDataArray  # noqa: E402

LIB = HERE.parent.parent / "oracle" / "_ref" / "libsampling_ref.so"
VOCABS = (1000, 128256, 152064)
N_HIST = 300
SEQ_STEPS = 1000
NL, EOS = 13, 2        # newline / EOS ids of the synthetic vocabulary (always in the history)
# name: (last_n, repeat, freq, present, penalize_nl, ignore_eos, bias kind)
CASES = {
    "neutral": (64, 1.0, 0.0, 0.0, False, False, None),
    "repeat_1.05": (64, 1.05, 0.0, 0.0, False, False, None),
    "repeat_1.1": (64, 1.1, 0.0, 0.0, False, False, None),
    "repeat_1.3": (64, 1.3, 0.0, 0.0, False, False, None),
    "repeat_0.9": (64, 0.9, 0.0, 0.0, False, False, None),
    "last_n_-1": (-1, 1.3, 0.5, 0.5, False, False, None),
    "last_n_0_bias": (0, 1.3, 0.5, 0.5, False, False, "mixed"),
    "last_n_1": (1, 1.3, 0.5, 0.5, False, False, None),
    "last_n_4096": (4096, 1.1, 0.0, 0.0, False, False, None),
    "freq_present": (300, 1.0, 0.1, 0.7, False, False, None),
    "freq_present_repeat": (256, 1.1, 0.05, 0.3, False, False, None),
    "penalize_nl_on": (64, 1.3, 0.1, 0.2, True, False, None),
    "penalize_nl_off": (64, 1.3, 0.1, 0.2, False, False, None),
    "ignore_eos": (64, 1.0, 0.0, 0.0, False, True, None),
    "ignore_eos_penalties": (64, 1.1, 0.1, 0.1, False, True, None),
    "bias_only": (64, 1.0, 0.0, 0.0, False, False, "mixed"),
    "bias_penalties": (64, 1.3, 0.1, 0.2, False, True, "mixed"),
    "bias_1000": (64, 1.1, 0.0, 0.0, False, False, "many"),
}
# sequences: (name, n_vocab, chain, penalties, dist seed, logit seed base)
SEQS = (
    ("greedy", 1000, "greedy", dict(last_n=64, repeat=1.3, freq=0.1, present=0.2, ignore_eos=True, nl_token=NL, eos_token=EOS,
                                   logit_bias=[(5, -np.inf), (7, 1.5)]), 0, 11000000),
    ("dist", 32000, "dist", dict(last_n=64, repeat=1.1, freq=0.05, present=0.1, nl_token=NL, eos_token=EOS), 777, 12000000),
)


def bias_list(kind, n, rng):
    if kind is None:
        return []
    if kind == "mixed":     # duplicates (applied twice, in order), out-of-range ids, -inf, a bias on EOS and on the newline
        return [(17, 1.25), (42, -3.5), (17, 0.1), (-5, 9.0), (n, 9.0), (n + 100, -9.0), (99, -np.inf), (EOS, 2.0), (NL, -0.75),
                (42, 0.3), (17, -0.4), (n - 1, 5.0)]
    ids = rng.integers(-3, n + 3, 1000)
    ids[::50] = 17                                        # repeated entries spread over the list
    b = (rng.standard_normal(1000) * 2).astype(np.float32)
    b[7] = -np.inf
    return [(int(t), float(v)) for t, v in zip(ids, b)]


def history(n, rng):
    """N_HIST accepted tokens: a small pool so counts run up to a dozen, the newline and EOS among them, two ids outside [0, n)."""
    pool = rng.choice(n, size=min(40, n), replace=False)
    h = rng.choice(pool, size=N_HIST).astype(np.int64)
    h[-5:] = [NL, -7, n + 3, NL, EOS]
    h[-20:-15] = pool[:5]
    return h


class RefSampler:
    """logit_bias -> penalties [-> tail] as one llama_sampler chain of the live reference library."""

    def __init__(self, lib, n, p: P.Penalties, tail=None):
        vp = C.c_void_p
        self.lib = lib
        lib.llama_sampler_chain_init.restype = vp
        lib.llama_sampler_chain_init.argtypes = [ChainParams]
        lib.llama_sampler_chain_add.argtypes = [vp, vp]
        lib.llama_sampler_init_logit_bias.restype = vp
        lib.llama_sampler_init_logit_bias.argtypes = [C.c_int32, C.c_int32, vp]
        lib.llama_sampler_init_penalties.restype = vp
        lib.llama_sampler_init_penalties.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_float, C.c_float, C.c_bool, C.c_bool]
        for f, at in (("top_k", [C.c_int32]), ("top_p", [C.c_float, C.c_size_t]), ("min_p", [C.c_float, C.c_size_t]),
                      ("temp_ext", [C.c_float, C.c_float, C.c_float]), ("softmax", []), ("dist", [C.c_uint32]), ("greedy", [])):
            fn = getattr(lib, "llama_sampler_init_" + f)
            fn.restype, fn.argtypes = vp, at
        lib.llama_sampler_apply.argtypes = [vp, C.POINTER(TokenDataArray)]
        lib.llama_sampler_accept.argtypes = [vp, C.c_int32]
        lib.llama_sampler_free.argtypes = [vp]
        lb = np.array([(t, b) for t, b in p.logit_bias], dtype=[("token", "<i4"), ("bias", "<f4")])
        self.h = lib.llama_sampler_chain_init(ChainParams(True))
        lib.llama_sampler_chain_add(self.h, lib.llama_sampler_init_logit_bias(n, len(lb), lb.ctypes.data if len(lb) else None))
        lib.llama_sampler_chain_add(self.h, lib.llama_sampler_init_penalties(n, p.eos_token, p.nl_token, p.last_n, p.repeat, p.freq, p.present,
                                                                             p.penalize_nl, p.ignore_eos))
        if tail == "greedy":
            lib.llama_sampler_chain_add(self.h, lib.llama_sampler_init_greedy())
        elif tail is not None:           # llama-cli's default chain, dist seeded with `tail`
            for s in (lib.llama_sampler_init_top_k(40), lib.llama_sampler_init_top_p(0.95, 0), lib.llama_sampler_init_min_p(0.05, 0),
                      lib.llama_sampler_init_temp_ext(0.8, 0.0, 1.0), lib.llama_sampler_init_softmax(), lib.llama_sampler_init_dist(tail)):
                lib.llama_sampler_chain_add(self.h, s)

    def accept(self, tokens):
        for t in np.atleast_1d(tokens):
            self.lib.llama_sampler_accept(self.h, int(t))

    def __call__(self, logits):
        """(selected token or -1, the row in id order; for a chain with a tail the row is the one it left, not in id order)"""
        n = logits.size
        d = np.zeros(n, TokenData)
        d["id"] = np.arange(n)
        d["logit"] = logits
        arr = TokenDataArray(d.ctypes.data, n, -1, False)
        self.lib.llama_sampler_apply(self.h, C.byref(arr))
        sel = int(arr.selected)
        assert (d["id"] == np.arange(n)).all() or sel >= 0
        return (int(d["id"][sel]) if sel >= 0 else -1), d["logit"].copy()

    def close(self):
        self.lib.llama_sampler_free(self.h)


def penalties_of(args, n, rng):
    last_n, rep, freq, pres, pnl, ieos, kind = args
    return P.Penalties(last_n, rep, freq, pres, pnl, ieos, NL, EOS, bias_list(kind, n, rng))


def main():
    lib = C.CDLL(str(LIB))
    rows = []
    for n in VOCABS:
        for ci, (name, args) in enumerate(CASES.items()):
            seed = 7919 * n + ci
            rng = np.random.default_rng(seed)
            p = penalties_of(args, n, rng)
            hist = history(n, rng)
            x = S.make_logits(seed, n, 3.0)
            hid = hist[(hist >= 0) & (hist < n)]
            x[hid[:6]] = 0.0                          # history tokens whose logit is exactly 0, the rest negative and positive
            x[hid[6]] = -0.0
            dseed = (seed * 2654435761) & 0xFFFFFFFF
            pre, grd, dst = RefSampler(lib, n, p), RefSampler(lib, n, p, "greedy"), RefSampler(lib, n, p, dseed)
            for s in (pre, grd, dst):
                s.accept(hist)
            _, row = pre(x)
            tok_g, _ = grd(x)
            tok_d, _ = dst(x)
            for s in (pre, grd, dst):
                s.close()
            idx, val = P.diff(row, x)
            rows.append((n, ci, seed, dseed, hist, p, tok_g, tok_d, idx, val))
            print(f"n={n:6d} {name:22s}: {idx.size:4d} logits changed, greedy {tok_g:6d}, dist {tok_d:6d}", flush=True)
    names = list(CASES)
    cat = lambda k, dt: np.concatenate([np.asarray(r[k], dt) for r in rows]) if rows else np.zeros(0, dt)  # noqa: E731
    off = lambda k: np.cumsum([0] + [len(r[k]) for r in rows]).astype(np.int64)  # noqa: E731
    bias = [r[5].logit_bias for r in rows]
    out = {
        "case_names": np.array(names), "n_vocab": np.array([r[0] for r in rows], np.int32), "case": np.array([r[1] for r in rows], np.int32),
        "logit_seed": np.array([r[2] for r in rows], np.int64), "dist_seed": np.array([r[3] for r in rows], np.uint32),
        "cfg": np.array([(r[5].last_n, r[5].penalize_nl, r[5].ignore_eos, r[5].nl_token, r[5].eos_token) for r in rows], np.int32),
        "cfg_f": np.array([(r[5].repeat, r[5].freq, r[5].present) for r in rows], np.float32),
        "hist": cat(4, np.int32), "hist_off": off(4),
        "bias_tok": np.concatenate([np.array([t for t, _ in b], np.int32) for b in bias]),
        "bias_val": np.concatenate([np.array([v for _, v in b], np.float32) for b in bias]),
        "bias_off": np.cumsum([0] + [len(b) for b in bias]).astype(np.int64),
        "token_greedy": np.array([r[6] for r in rows], np.int32), "token_dist": np.array([r[7] for r in rows], np.int32),
        "diff_idx": cat(8, np.int32), "diff_val": cat(9, np.float32), "diff_off": off(8),
    }
    for name, n, chain, kw, dseed, base in SEQS:
        p = P.Penalties(**kw)
        rng = np.random.default_rng(base)
        prompt = rng.integers(0, n, 32)
        ref = RefSampler(lib, n, p, "greedy" if chain == "greedy" else dseed)
        ref.accept(prompt)
        toks = []
        for i in range(SEQ_STEPS):
            tok, _ = ref(P.seq_logits(base + i, n, list(prompt) + toks))
            ref.accept(tok)
            toks.append(tok)
        ref.close()
        print(f"sequence {name}: {len(set(toks))} distinct tokens in {SEQ_STEPS} steps", flush=True)
        out.update({
            f"seq_{name}_n_vocab": np.int32(n), f"seq_{name}_dist_seed": np.uint32(dseed), f"seq_{name}_logit_base": np.int64(base),
            f"seq_{name}_prompt": prompt.astype(np.int32), f"seq_{name}_token": np.array(toks, np.int32),
            f"seq_{name}_cfg": np.array([p.last_n, p.penalize_nl, p.ignore_eos, p.nl_token, p.eos_token], np.int32),
            f"seq_{name}_cfg_f": np.array([p.repeat, p.freq, p.present], np.float32),
            f"seq_{name}_bias_tok": np.array([t for t, _ in p.logit_bias], np.int32),
            f"seq_{name}_bias_val": np.array([v for _, v in p.logit_bias], np.float32),
        })
    np.savez_compressed(HERE / "penalties_golden.npz", **out)


if __name__ == "__main__":
    main()
