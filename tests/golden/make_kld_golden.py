"""Writes tests/golden/kld_golden.npz: llama-perplexity's log-probability writer and KL-divergence functions (oracle/_ref/libppl_ref.so,
built by `make -C oracle -f Makefile.perplexity` from the reference's unmodified examples/perplexity/perplexity.cpp) on seeded rows.

Per vocabulary V, case r has the kind KINDS[kinds[r]] and seed seeds[r]; tests/kld_ref.make_rows(V, seed, kind) regenerates its logits
row x, its base row y and its target.  Stored per V:
  - the writer on the rows [x_0..x_n-1, y_0..y_n-1]: the header floats (scale, min_log_prob) and the float nll; the whole records where
    V <= 32 000, else the SHA-256 of each record's entries (pad included);
  - the KLD function on x_r against y_r's record: kld (double), nll, nll_base, p_diff (float), same_top;
  - process_logits over all n rows: the accumulated kl_divergence_result sums and the per-row kld / p_diff values it stores.

    python tests/golden/make_kld_golden.py"""
import hashlib
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
import kld_ref as K  # noqa: E402

VOCABS = (160, 1001, 32000, 128256, 152064, 262144)
WHOLE_RECORDS_UP_TO = 32000


def entries_sha(rec) -> bytes:
    return hashlib.sha256(np.ascontiguousarray(rec[4:], dtype="<u2").tobytes()).digest()


def main():
    ref = K.RefPpl()
    out = {"vocabs": np.array(VOCABS, np.int32)}
    for V in VOCABS:
        kinds = np.array([k for k in range(len(K.KINDS))] * (2 if V <= 1001 else 1), np.int32)
        seeds = (1000 * V + np.arange(kinds.size)).astype(np.int64) % (2 ** 31)
        xs, ys, toks = [], [], []
        for k, s in zip(kinds, seeds):
            x, y, t = K.make_rows(V, int(s), K.KINDS[k])
            xs.append(x); ys.append(y); toks.append(t)
        rows, row_toks = xs + ys, toks + toks
        recs, nll = [], []
        for x, t in zip(rows, row_toks):
            r, v = ref.logprobs_u16(x, t)
            recs.append(r); nll.append(v)
        recs = np.stack(recs)
        p = f"V{V}_"
        out[p + "kinds"], out[p + "seeds"], out[p + "targets"] = kinds, seeds, np.array(toks, np.int32)
        sc, mlp = K.header(recs)
        out[p + "scale"], out[p + "min_log_prob"], out[p + "nll"] = sc.copy(), mlp.copy(), np.array(nll, np.float32)
        if V <= WHOLE_RECORDS_UP_TO:
            out[p + "records"] = recs
        else:
            out[p + "sha"] = np.stack([np.frombuffer(entries_sha(r), np.uint8) for r in recs])
        n = len(xs)
        base = recs[n:]
        kl = [ref.kld_row(x, b, t) for x, b, t in zip(xs, base, toks)]
        out[p + "kld"] = np.array([v[0] for v in kl], np.float64)
        for j, name in ((1, "kld_nll"), (2, "kld_nll_base"), (3, "p_diff")):
            out[p + name] = np.array([v[j] for v in kl], np.float32)
        out[p + "same_top"] = np.array([v[4] for v in kl], np.int32)
        acc, kv, pv = ref.process_kld(np.stack(xs), base, toks)
        out[p + "sums"] = np.array([getattr(acc, f) for f, _ in K.KldResultC._fields_[:10]], np.float64)
        out[p + "max_p_diff"] = np.float32(acc.max_p_diff)
        out[p + "n_same_top"], out[p + "count"] = np.int64(acc.n_same_top), np.int64(acc.count)
        out[p + "kld_values"], out[p + "p_diff_values"] = kv, pv
        print(f"V {V}: {n} cases, same_top {acc.n_same_top}/{acc.count}, mean KLD {acc.sum_kld / acc.count:.6g}")
    np.savez_compressed(K.GOLDEN, **out)
    print(f"wrote {K.GOLDEN} ({K.GOLDEN.stat().st_size} bytes)")


if __name__ == "__main__":
    main()
