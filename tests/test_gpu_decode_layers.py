"""Decode layer by layer: every launch of every decode step (engine.cu enqueue_step) against the CPU oracle on the device's own input.

Each layer runs as its own one-layer shard (pb200_model_create with a one-layer window, as the pipeline stages do), fed with
set_hidden the previous shard's output.  After every step the shard's buffers are read back (pb200_debug_read) and each launch is
checked on the values the device itself handed it, so errors never compound and a failure names its layer, launch and position:

  launch                  reference                                                                     bar
  get_rows (layer 0)      the dequantized embedding row                                                 bit-exact
  q | k | v (+ biases)    oracle mat-vec of rms_norm(x_in) * attn_norm                                  GEMV bar
  K / V cache cell pos    f16(pb200_rope(k)), f16(v) of the device's own k / v                          bit-exact
  every other cell/slot   unchanged (cells past pos start as f16 NaN)                                   bit-exact
  att                     port.attention_decode on rope(q) and the device's own cache                  3e-4 / 2e-5 + flips
  wo + residual           oracle mat-vec of the device's att, + x_in                                    GEMV bar
  gate | up               oracle mat-vec of rms_norm(ffn_inp) * ffn_norm                                GEMV bar
  ffn_down + residual     oracle mat-vec of pb200_silu_mul(g, u), + ffn_inp                             GEMV bar
  head                    oracle mat-vec (Q6_K) of rms_norm(x_out) * output_norm                        GEMV bar

The attention bar is test_attn_decode's (max 3e-4, mean 2e-5) plus f16_flip_slack: for the few cells whose probability lies within
the derived f32 error of an f16 rounding boundary, one f16 step times |V|.  Both sides round p to f16, and where the device's expf
ulps tip one to the other side of a boundary near p = 1 that is worth up to |V| 2^-11.  The GEMV bar is that of test_gpu_gemv_shapes.Scattered.check: 4e-6 max(1, max |ref|), the
fp32 summation order.  The oracle is the C port; it quantizes the activation exactly as the device's
producers do (same f32 input, same block scale arithmetic), so a quantization code that differs shows up as a GEMV error.

decode_launches() restates the branch choices of launch_gemv (gemv.cu) and launch_attn_step (ops.cu): the distributed prologue inside
the ring kernel; a producer kernel and the ring per matrix group; the several-modes route of a Q8_0 matrix beside k-quants; the ring
or k_gemv_generic per matrix; k_attn2, or k_attn_rows plus a quantize kernel in front of wo.  The launch count of every
step must equal it, and a CPU-only test checks that each case reaches the branches it is there for.  The same tokens then go through
the unsplit model (logits bit-identical to the shard composition), and direct launches must equal the CUDA-graph replay bit for bit.

Long positions cost no long decodes: cells [0, pos) are filled with seeded f16 rows through the cache view and the step runs at pos."""
import functools

import numpy as np
import pytest
import torch

import oracle_lib as O
from gpu_util import dev_f32, ptr, sync
from test_gpu_gemv_shapes import gemv_plan
from test_gpu_kv_shift import _dev, kv_tensors, load
from tiny_model import TinyModel, use_more_bits

D = 128
F16_NAN = 0x7E00
ACT_Q8_K, ACT_Q8_0, ACT_Q8_1 = 0, 1, 2
ACT_MAX_NBLK = 116


def act_mode(t):
    """common.cuh act_mode_for: the CPU's vec_dot_type of the weight type."""
    return {"q8_K": ACT_Q8_K, "q8_0": ACT_Q8_0, "q8_1": ACT_Q8_1}[O.ACT_TYPE[t]]


# ---- the branch choices of one decode step, restated ----
def gemv_kernels(types, Ns, K):
    """gemv.cu gemv_kernels: the ring for the whole group, else per matrix the ring (32-element types on their own) or
    k_gemv_generic.  Weights are 256-byte aligned in the engine."""
    if gemv_plan(types, Ns, K):
        return 1, "ring"
    kinds = ["ring" if t in O.BLK32 and gemv_plan((t,), (N,), K) else "generic" for t, N in zip(types, Ns)]
    return len(kinds), ",".join(kinds)


def gemv_launches(types, Ns, K, pro):
    """gemv.cu launch_gemv: (kernel launches, branch).  pro: "rms_norm" / "silu_mul" / "quantize" / "none" (activation ready).
    1. rms_norm / silu_mul on a k-quant group that fits the ring: one launch, the prologue distributed over its CTAs ("dist");
    2. one activation mode: a producer kernel unless the activation is ready, then the kernels ("producer" / "ready");
    3. several modes: rms_norm * w to an f32 scratch, then per mode a quantize kernel and that mode's kernels ("modes")."""
    if pro in ("rms_norm", "silu_mul") and all(t in O.KQ for t in types) and gemv_plan(types, Ns, K):
        return 1, "dist"
    modes = list(dict.fromkeys(act_mode(t) for t in types))
    if len(modes) == 1:
        n, kinds = gemv_kernels(types, Ns, K)
        return n + (pro != "none"), ("producer+" if pro != "none" else "ready+") + kinds
    assert pro in ("rms_norm", "quantize"), pro
    n, parts = int(pro == "rms_norm"), []
    for m in modes:
        sub = [(t, N) for t, N in zip(types, Ns) if act_mode(t) == m]
        c, kinds = gemv_kernels([t for t, _ in sub], [N for _, N in sub], K)
        n += 1 + c
        parts.append(kinds)
    return n, "modes+" + "|".join(parts)


def uses_attn2(types, hp, attn2_max):
    """ops.cu launch_attn_step: k_attn2 when wo takes q8_K, its K fits the ring's activation staging and the scores fit shared
    memory (n_ctx <= pb200_attn_ggml_max_cells()), else k_attn_rows<true> and wo's own quantize kernel."""
    QD = hp["n_head"] * D
    return act_mode(types["o"]) == ACT_Q8_K and QD % 256 == 0 and QD // 256 <= ACT_MAX_NBLK and hp["n_head"] % 2 == 0 and hp["n_ctx"] <= attn2_max


def decode_launches(types, hp, with_embd, head_type, attn2_max):
    """enqueue_step's kernel launches for a one-layer shard, and the branch of each launch group (head_type None: no head)."""
    E, QD, EK, F, V = hp["n_embd"], hp["n_head"] * D, hp["n_head_kv"] * D, hp["n_ff"], hp["n_vocab"]
    n, br = int(with_embd), {}
    c, br["qkv"] = gemv_launches([types["q"], types["k"], types["v"]], [QD, EK, EK], E, "rms_norm")
    n += c
    a2 = uses_attn2(types, hp, attn2_max)
    br["attn"] = "attn2" if a2 else "rows"
    c, br["wo"] = gemv_launches([types["o"]], [E], QD, "none" if a2 else "quantize")
    n += 1 + c
    c, br["gu"] = gemv_launches([types["gate"], types["up"]], [F, F], E, "rms_norm")
    n += c
    c, br["down"] = gemv_launches([types["down"]], [E], F, "silu_mul")
    n += c
    if head_type is not None:
        c, br["head"] = gemv_launches([head_type], [V], E, "rms_norm")
        n += c
    return n, br


def hidden_names(with_embd):
    """enqueue_step's buffer rotation for a one-layer shard: (layer input, ffn_inp).  The input is x_in, or x_a holding get_rows'
    row; ffn_inp goes to the first of x_a, x_b, xn that is not the input; the last layer writes x_out."""
    x = "x_a" if with_embd else "x_in"
    return x, next(b for b in ("x_a", "x_b", "xn") if b != x)


# ---- cases: tiny models, E 1024, 8 / 2 heads, 3 layers ----
def layer_types(tensors, il):
    return {k: tensors[f"blk.{il}.{n}.weight"][0] for k, n in (("q", "attn_q"), ("k", "attn_k"), ("v", "attn_v"), ("o", "attn_output"),
                                                                 ("gate", "ffn_gate"), ("up", "ffn_up"), ("down", "ffn_down"))}


def _qwen2_q4_K_M(seed, n_ctx):
    """The Qwen2.5-72B Q4_K_M mixture in small: n_ff % 256 != 0 turns ffn_down Q4_K into Q5_0 and Q6_K (layer 2) into Q8_0."""
    tm = TinyModel(n_layer=3, n_embd=1024, n_head=8, n_head_kv=2, n_ff=1152, n_vocab=512, n_ctx=n_ctx, arch="qwen2", ftype="q4_K_M",
                   seed=seed, branch_scale=0.1, types={"ffn_down": O.Q5_K})
    for il in range(3):
        tm.retype(f"blk.{il}.ffn_down.weight", O.Q8_0 if use_more_bits(il, 3) else O.Q5_0, 500 + il)
    return tm


def _llama_q4_0(seed, n_ctx):
    """The Q4_0 mixture (a Q6_K head) with the imatrix rule's Q4_1 ffn_down in layers 0 and 1 and a Q5_0 attn_output in layer 0."""
    tm = TinyModel.q4_0(seed, n_layer=3, n_embd=1024, n_head=8, n_head_kv=2, n_ff=2048, n_vocab=512, n_ctx=n_ctx)
    for il in range(2):
        tm.retype(f"blk.{il}.ffn_down.weight", O.Q4_1, 600 + il)
    tm.retype("blk.0.attn_output.weight", O.Q5_0, 610)
    return tm


def _tiny(**kw):
    return lambda seed, n_ctx: TinyModel(n_layer=3, n_embd=1024, n_head=8, n_head_kv=2, n_vocab=512, n_ctx=n_ctx, seed=seed, branch_scale=0.1, **kw)


# name -> (model builder, decode steps, branches the case is there for: "launch:branch" over its three layers)
CASES = {
    "llama_q4_K_M": (_tiny(arch="llama", ftype="q4_K_M", n_ff=2048, freq_factors=True), 40,
                     {"qkv:dist", "attn:attn2", "wo:ready+ring", "gu:dist", "down:dist", "head:dist"}),
    "qwen2_q5_K_M_ring": (_tiny(arch="qwen2", ftype="q5_K_M", n_ff=1152), 40,          # Q5_1 and Q8_0 ffn_down on the ring
                          {"qkv:dist", "attn:attn2", "down:producer+ring", "head:dist"}),
    "qwen2_q5_K_M_generic": (_tiny(arch="qwen2", ftype="q5_K_M", n_ff=1056), 40,       # Q8_0 rows of 1 122 bytes: k_gemv_generic
                             {"down:producer+ring", "down:producer+generic"}),
    "qwen2_q5_K_M_longK": (_tiny(arch="qwen2", ftype="q5_K_M", n_ff=29824), 8,         # Q5_1 / Q8_0 K past the ring's 116 super-blocks
                           {"down:producer+generic"}),
    "qwen2_q4_K_M": (_qwen2_q4_K_M, 40, {"qkv:dist", "attn:attn2", "down:producer+ring"}),
    "llama_q4_0": (_llama_q4_0, 40, {"qkv:producer+ring,ring,ring", "attn:rows", "wo:producer+ring", "gu:producer+ring,ring",
                                     "down:producer+ring", "head:dist"}),
    "qkv_mixed": (_tiny(arch="llama", ftype="q4_K_M", n_ff=2048, types={"attn_k": O.Q8_0}), 40, {"qkv:modes+ring|ring", "attn:attn2"}),
    "gu_mixed": (_tiny(arch="llama", ftype="q4_K_M", n_ff=2048, types={"ffn_up": O.Q8_0}), 40, {"gu:modes+ring|ring"}),
}


@functools.lru_cache(maxsize=None)
def case_model(name, n_ctx=64):
    return CASES[name][0](len(name), n_ctx)


def case_branches(tm, attn2_max):
    hp, got = tm.hp, set()
    for il in range(hp["n_layer"]):
        _, br = decode_launches(layer_types(tm.tensors, il), hp, il == 0, tm.tensors["output.weight"][0] if il == hp["n_layer"] - 1 else None,
                                attn2_max)
        got |= {f"{k}:{v}" for k, v in br.items()}
    return got


def test_decode_cases_reach_their_branches():
    """No GPU: every case takes the branches it is named for (H100 plans, k_attn2 for n_ctx 64), and the launch arithmetic matches
    counts worked out by hand."""
    big = 1 << 20
    for name, (_, _, want) in CASES.items():
        got = case_branches(case_model(name), big)
        assert want <= got, (name, want - got, got)
    tm = case_model("llama_q4_0")
    n, br = decode_launches(layer_types(tm.tensors, 0), tm.hp, True, O.Q6_K, big)
    #       get_rows, norm+q+k+v, k_attn_rows, quantize+wo, norm+gate+up, silu+down, head
    assert n == 1 + 4 + 1 + 2 + 3 + 2 + 1, (n, br)
    tm = case_model("qkv_mixed")
    n, br = decode_launches(layer_types(tm.tensors, 1), tm.hp, False, None, big)
    #       norm to f32, q8_K + q|v ring, q8_0 + k ring, k_attn2, wo, gate|up, down
    assert n == 1 + 2 + 2 + 1 + 1 + 1 + 1 and br["qkv"] == "modes+ring|ring", (n, br)
    # the attention fallback past k_attn2's shared-memory limit
    tm = case_model("llama_q4_K_M")
    hp = dict(tm.hp, n_ctx=2048)
    assert decode_launches(layer_types(tm.tensors, 1), hp, False, None, 1024)[1]["attn"] == "rows"
    assert decode_launches(layer_types(tm.tensors, 1), hp, False, None, 2048)[1]["attn"] == "attn2"


# ---- device helpers ----
def f16_bits(a):
    return np.asarray(a, np.float32).astype(np.float16).view(np.uint16)


def rope_dev(lib, hp, x, n_head, pos, ff):
    """pb200_rope of one token's [n_head][128] vector with the engine's RoPE parameters (rope_params_init in finalize)."""
    xd, y = dev_f32(x), torch.full((n_head * D,), float("nan"), device="cuda")
    pd = torch.tensor([pos], dtype=torch.int32, device="cuda")
    fd = dev_f32(ff) if ff is not None else None
    lib.check(lib.c.pb200_rope(ptr(xd), ptr(y), 1, n_head, D, D, hp["rope_mode"], ptr(pd), hp["rope_freq_base"], hp["rope_freq_scale"], 0.0, 1.0,
                               32.0, 1.0, hp["n_ctx_orig"], ptr(fd) if fd is not None else None, None), "rope")
    sync()
    return y.cpu().numpy()


def silu_mul_dev(lib, g, u):
    gd, ud = dev_f32(g), dev_f32(u)
    y = torch.full_like(gd, float("nan"))
    lib.check(lib.c.pb200_silu_mul(ptr(gd), ptr(ud), ptr(y), gd.numel(), None), "silu_mul")
    sync()
    return y.cpu().numpy()


U32 = 2.0 ** -24             # unit roundoff of f32; one ulp is at most 2 U32 relative
EXPF_ULPS = 2                # CUDA's expf: at most 2 ulp (CUDA C++ Programming Guide, single-precision functions); glibc's: under 1
DEV_SCORE_ROUNDINGS = 8      # roundings in a device score: 3 fmaf per lane, then 5 levels of warp_sum (k_attn2, k_attn_rows)


def f16_flip_slack(q_rot, Kc, Vc, H, HK, scale):
    """[H * D] what rounding the probabilities to f16 can legitimately make the device and the CPU disagree by.  Both round p to f16
    before P.V.  Each side's f32 p is within tau_c p_c of the exact p_c (f64, from the same f16 q and K):
      score s_c:        products of f16 values are exact in f32.  The CPU's sequential f32 sum is restated here, so its error is
                        known; the device's is at most DEV_SCORE_ROUNDINGS U32 sum |q k|.  The larger of the two counts
      t = fl(s scale):  + U32 |t|;  d = fl(t - t_max): the errors of t_c and t_max, + U32 |d|
      e = expf(d):      expm1(|error of d|) + 2 EXPF_ULPS U32 relative
      p = fl(e fl(1 / sum e)), the sum in double: the sum is off by the p-weighted mean of the e's relative errors, + 3 U32
    A cell rounds to different f16 values on the two sides only if an f16 rounding boundary lies in p_c (1 -+ tau_c), and then they
    differ by the f16 step there.  The slack is that step times |V| over such cells; every other cell gets none."""
    gqa = H // HK
    qf = q_rot.astype(np.float16).astype(np.float64).reshape(H, D)
    K = Kc.view(np.float16).astype(np.float64).reshape(-1, HK, D)
    V = np.abs(Vc.view(np.float16).astype(np.float64).reshape(-1, HK, D))
    out = np.zeros((H, D))
    for h in range(H):
        Kh = K[:, h // gqa]
        s64 = Kh @ qf[h]
        s32 = np.zeros(len(Kh), np.float32)
        for i in range(D):                                   # port_attention_decode's order, every product exact in f32
            s32 += (Kh[:, i] * qf[h, i]).astype(np.float32)
        ds = np.maximum(np.abs(s32 - s64), DEV_SCORE_ROUNDINGS * U32 * (np.abs(Kh) @ np.abs(qf[h])))
        t = s64 * scale
        dt = ds * scale + U32 * np.abs(t)
        m = int(np.argmax(t))
        p = np.exp(t - t[m])
        p /= p.sum()
        rel_e = np.expm1(dt + dt[m] + U32 * np.abs(t - t[m])) + 2 * EXPF_ULPS * U32
        tau = rel_e + p @ rel_e + 3 * U32
        step = np.abs((p * (1 + tau)).astype(np.float16).astype(np.float64) - (p * (1 - tau)).astype(np.float16).astype(np.float64))
        out[h] = step @ V[:, h // gqa]
    return out.reshape(-1)


def check_gemv(where, got, want):
    bad = ~np.isfinite(got)
    assert not bad.any(), f"{where}: {int(bad.sum())} of {got.size} rows not finite, first {np.flatnonzero(bad)[:8]}"
    err = np.abs(got.astype(np.float64) - want.astype(np.float64))
    tol = 4e-6 * max(1.0, float(np.max(np.abs(want))))
    r = int(np.argmax(err))
    assert err[r] <= tol, f"{where}: row {r} off by {err[r]:.3e} > {tol:.3e}; {int((err > tol).sum())} rows over"


def check_bits(where, got, want):
    bad = np.flatnonzero(np.asarray(got).view(np.uint32) != np.asarray(want).view(np.uint32))
    assert bad.size == 0, f"{where}: {bad.size} values differ, first at {bad[0]}: {got[bad[0]]!r} vs {want[bad[0]]!r}"


def dequant_row(port, t, W, K, row):
    rb = O.row_size(t, K)
    blk = np.ascontiguousarray(W.reshape(-1)[row * rb:(row + 1) * rb])
    return port.dequantize(t, blk, K)[0]


class Shard:
    """One finalized one-layer shard (or a wider one for the unsplit run) with host copies of the weights it holds."""

    def __init__(self, eng, hp, weights, il, with_embd, with_head, n_seq):
        self.eng, self.hp, self.w, self.il = eng, hp, weights, il
        self.with_embd, self.with_head, self.n_seq = with_embd, with_head, n_seq
        EK = hp["n_head_kv"] * D
        self.exp_k = np.full((n_seq, hp["n_ctx"], EK), F16_NAN, np.uint16)   # the cache this shard must hold
        self.exp_v = self.exp_k.copy()

    def kv(self):
        """Host copies of the engine's K / V caches of this shard's layer, [n_seq][n_ctx][EK] uint16 (views stay in here)."""
        k, v = kv_tensors(self.eng, None, self.n_seq, 1, self.hp)
        return k[:, 0].cpu().numpy().view(np.uint16), v[:, 0].cpu().numpy().view(np.uint16)

    def fill(self, slot, pos0, rng):
        """Cells [0, pos0) of the slot: seeded f16 rows (|K| ~ 0.5, |V| ~ 1); cells from pos0 on: f16 NaN."""
        n_ctx, EK = self.exp_k.shape[1:]
        self.exp_k[slot, :pos0] = f16_bits(rng.standard_normal((pos0, EK)) * 0.5)
        self.exp_v[slot, :pos0] = f16_bits(rng.standard_normal((pos0, EK)))
        self.exp_k[slot, pos0:] = F16_NAN
        self.exp_v[slot, pos0:] = F16_NAN
        k, v = kv_tensors(self.eng, None, self.n_seq, 1, self.hp)
        k[slot, 0] = torch.from_numpy(self.exp_k[slot].view(np.int16)).cuda()
        v[slot, 0] = torch.from_numpy(self.exp_v[slot].view(np.int16)).cuda()
        sync()

    def read(self, name, n):
        return self.eng.debug_read(name, n)


def check_step(lib, port, s, tag, pos, slot=0, check_att=True, f32_scratch_att=False):
    """Every launch of the shard's last step at pos (one layer), on the device's own inputs; updates and compares the caches."""
    hp, w, il = s.hp, s.w, s.il
    E, H, HK, F, V = hp["n_embd"], hp["n_head"], hp["n_head_kv"], hp["n_ff"], hp["n_vocab"]
    QD, EK, eps, p = H * D, HK * D, hp["rms_eps"], f"blk.{il}."
    where = f"{tag} layer {il} pos {pos}"
    xname, x1name = hidden_names(s.with_embd)
    x = s.read(xname, E)
    if s.with_embd:
        t, Wt = w["token_embd.weight"]
        check_bits(f"{where} get_rows", x, dequant_row(port, t, Wt, E, s.last_token))

    def mm(name, xin, N, K):
        t, W = w[name]
        return port.mul_mat(t, W, N, K, xin)[0]

    def bias(name, n):
        return w[name][1] if name in w else np.zeros(n, np.float32)

    # q | k | v
    xn = port.rms_norm(x, eps) * w[p + "attn_norm.weight"][1]
    q, k, v = s.read("q", QD), s.read("k", EK), s.read("v", EK)
    for nm, got, N in (("attn_q", q, QD), ("attn_k", k, EK), ("attn_v", v, EK)):
        check_gemv(f"{where} {nm}", got, mm(p + nm + ".weight", xn, N, E) + bias(p + nm + ".bias", N))
    # the cache: cell pos of this slot = f16(rope(k)), f16(v); nothing else changed
    ff = w["rope_freqs.weight"][1] if "rope_freqs.weight" in w else None
    q_rot, k_rot = rope_dev(lib, hp, q, H, pos, ff), rope_dev(lib, hp, k, HK, pos, ff)
    s.exp_k[slot, pos], s.exp_v[slot, pos] = f16_bits(k_rot), f16_bits(v)
    gk, gv = s.kv()
    for nm, g, e in (("K", gk, s.exp_k), ("V", gv, s.exp_v)):
        bad = np.argwhere((g != e).any(axis=2))
        assert bad.size == 0, f"{where}: {nm} cache cells (slot, cell) {bad[:8].tolist()} differ ({len(bad)} cells; the step wrote slot {slot} cell {pos})"
    # attention over the device's own cache
    x1 = s.read(x1name, E)
    if check_att:
        att = s.read("att", QD)
        scale = float(np.float32(1.0) / np.sqrt(np.float32(D)))
        want = port.attention_decode(q_rot, gk[slot, :pos + 1], gv[slot, :pos + 1], H, HK, D, pos + 1, scale)
        err = np.abs(att.astype(np.float64) - want)
        slack = f16_flip_slack(q_rot, gk[slot, :pos + 1], gv[slot, :pos + 1], H, HK, scale)
        assert np.isfinite(att).all() and np.all(err < 3e-4 + slack) and np.mean(err) < 2e-5 + np.mean(slack), \
            (f"{where} att: max {np.max(err):.3e} mean {np.mean(err):.3e} (f16 rounding slack: max {np.max(slack):.3e}, "
             f"mean {np.mean(slack):.3e}), worst head {int(np.argmax(err - slack)) // D}")
        check_gemv(f"{where} attn_output + residual", x1, mm(p + "attn_output.weight", att, E, QD) + x)
    # gate | up
    xn2 = port.rms_norm(x1, eps) * w[p + "ffn_norm.weight"][1]
    if f32_scratch_att:   # the several-modes route of gate | up leaves rms_norm(ffn_inp) * ffn_norm in att (its f32 scratch)
        check_bits(f"{where} gate|up f32 scratch (att)", s.read("att", E), xn2)
    g, u = s.read("g", F), s.read("u", F)
    check_gemv(f"{where} ffn_gate", g, mm(p + "ffn_gate.weight", xn2, F, E))
    check_gemv(f"{where} ffn_up", u, mm(p + "ffn_up.weight", xn2, F, E))
    # ffn_down + residual
    out = s.read("x_out", E)
    check_gemv(f"{where} ffn_down + residual", out, mm(p + "ffn_down.weight", silu_mul_dev(lib, g, u), E, F) + x1)
    if s.with_head:
        xo = port.rms_norm(out, eps) * w["output_norm.weight"][1]
        check_gemv(f"{where} head", s.read("logits", V), mm("output.weight", xo, V, E))
    return out


def step(lib, s, tok, pos, x_in=None, slot=None):
    """One decode step of the shard (x_in: its input hidden state); returns the kernel launches it made."""
    if x_in is not None:
        s.eng.set_hidden(x_in)
    s.last_token = tok
    n0 = lib.c.pb200_kernel_launches()
    if slot is None:
        s.eng.decode(tok, pos)
    else:
        s.eng.decode_seq_async(slot, tok, pos)
        s.eng.synchronize()
    n = lib.c.pb200_kernel_launches() - n0
    assert lib.c.pb200_aborted() == 0, "an in-kernel wait gave up (watchdog)"
    return n


def load_shard(pkg, tm, il, with_embd, with_head, n_seq=1, hp=None):
    eng = load(tm, pkg, n_seq, (il, il + 1), with_embd, with_head, hp)
    return Shard(eng, hp or tm.hp, tm.tensors, il, with_embd, with_head, n_seq)


def check_launches(lib, s, n, tag, pos, head_type):
    want, br = decode_launches(layer_types(s.w, s.il), s.hp, s.with_embd, head_type, lib.c.pb200_attn_ggml_max_cells())
    assert n == want, f"{tag} layer {s.il} pos {pos}: {n} launches, the branches {br} make {want}"


def tokens(n, V):
    return [(i * 7919 + 13) % V for i in range(n)]


# ---- 1. every step of a 40-token decode, layer by layer; the unsplit model and the graph replay against it ----
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_decode_layers_vs_oracle(cuda, lib, pkg, port, name):
    tm = case_model(name)
    hp, nl, E, V = tm.hp, tm.hp["n_layer"], tm.hp["n_embd"], tm.hp["n_vocab"]
    toks = tokens(CASES[name][1], V)
    head_t = tm.tensors["output.weight"][0]
    shards = [load_shard(pkg, tm, il, il == 0, il == nl - 1) for il in range(nl)]
    logits = []
    try:
        for s in shards:
            s.fill(0, 0, np.random.default_rng(0))       # every cell f16 NaN
        for pos, tok in enumerate(toks):
            x = None
            for s in shards:
                n = step(lib, s, tok, pos, x)
                check_launches(lib, s, n, name, pos, head_t if s.with_head else None)
                x = check_step(lib, port, s, name, pos, check_att=name != "gu_mixed", f32_scratch_att=name == "gu_mixed")
            logits.append(shards[-1].read("logits", V))
    finally:
        for s in shards:
            s.eng.close()
    # the unsplit model: logits bit-identical to the shard composition; then direct launches bit-identical to the graph replay
    eng = tm.load_engine(pkg)
    try:
        got = np.zeros((len(toks), V), np.float32)
        for pos, tok in enumerate(toks):
            eng.decode(tok, pos, got[pos])
        for pos in range(len(toks)):
            check_bits(f"{name} unsplit model vs shards, pos {pos} logits", got[pos], logits[pos])
        kg, vg = (c.cpu().numpy() for c in kv_tensors(eng, tm, 1, nl))
        eng.kv_clear()
        eng.set_use_graph(False)
        for pos, tok in enumerate(toks[:6]):
            out = np.zeros(V, np.float32)
            eng.decode(tok, pos, out)
            check_bits(f"{name} direct launches vs graph replay, pos {pos} logits", out, got[pos])
        kd, vd = (c.cpu().numpy() for c in kv_tensors(eng, tm, 1, nl))
        assert np.array_equal(kd[:, :, :6], kg[:, :, :6]) and np.array_equal(vd[:, :, :6], vg[:, :, :6]), f"{name}: direct launches' cache"
    finally:
        eng.close()


# ---- 2. cache positions: every chunk refill and mbarrier parity flip of k_attn2, the k_attn_rows fallback, a Q4_0 model ----
POSITIONS = [("attn2", p) for p in (0, 1, 127, 128, 255, 256, 511, 512, 1000)] + [("attn2", "max-1"), ("rows", 200), ("rows", "max-1"),
                                                                                   ("q4_0", 1500)]


@pytest.mark.gpu
@pytest.mark.parametrize("rung,pos", POSITIONS, ids=[f"{r}-p{p}" for r, p in POSITIONS])
def test_decode_at_position(cuda, lib, pkg, port, rung, pos):
    limit = lib.c.pb200_attn_ggml_max_cells()
    tm = case_model("llama_q4_0" if rung == "q4_0" else "llama_q4_K_M")
    n_ctx = {"attn2": limit if pos == "max-1" else 1024, "rows": limit + 32, "q4_0": 2048}[rung]
    pos = n_ctx - 1 if pos == "max-1" else pos
    hp = dict(tm.hp, n_ctx=n_ctx)
    s = load_shard(pkg, tm, 1, False, False, hp=hp)
    try:
        assert uses_attn2(layer_types(tm.tensors, 1), hp, limit) == (rung == "attn2"), (rung, n_ctx, limit)
        rng = np.random.default_rng(pos)
        s.fill(0, pos, rng)
        for p in (pos, pos + 1)[:2 if pos + 1 < n_ctx else 1]:
            x = rng.standard_normal(tm.hp["n_embd"]).astype(np.float32)
            n = step(lib, s, 5, p, x)
            check_launches(lib, s, n, rung, p, None)
            check_step(lib, port, s, f"{rung} n_ctx {n_ctx}", p)
    finally:
        s.eng.close()


# ---- 3. sequence slots: a step of slot 2 leaves slots 0 and 1 alone ----
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["llama_q4_K_M", "llama_q4_0"])
def test_decode_slot_leaves_other_slots(cuda, lib, pkg, port, name):
    tm = case_model(name)
    s = load_shard(pkg, tm, 1, False, False, n_seq=3)
    try:
        rng = np.random.default_rng(3)
        for slot, p0 in ((0, 64), (1, 64), (2, 20)):
            s.fill(slot, p0, rng)
        for p in (20, 21):
            n = step(lib, s, 7, p, rng.standard_normal(tm.hp["n_embd"]).astype(np.float32), slot=2)
            check_launches(lib, s, n, f"{name} slot 2", p, None)
            check_step(lib, port, s, f"{name} slot 2", p, slot=2)
    finally:
        s.eng.close()


# ---- 4. full-size layers from pb200_model_synth ----
QWEN72B = dict(n_layer=80, n_embd=8192, n_head=64, n_head_kv=8, head_dim=128, n_ff=29568, n_vocab=152064, n_ctx=64, rope_mode=2,
               n_ctx_orig=32768, rope_freq_base=1e6, rope_freq_scale=1.0, rms_eps=1e-6)
LLAMA8B = dict(n_layer=32, n_embd=4096, n_head=32, n_head_kv=8, head_dim=128, n_ff=14336, n_vocab=128256, n_ctx=64, rope_mode=0,
               n_ctx_orig=8192, rope_freq_base=500000.0, rope_freq_scale=1.0, rms_eps=1e-5)
FULL = [("qwen2.5-72b", 0, 11), ("qwen2.5-72b", 0, 12), ("llama3-8b", 2, 5), ("qwen2.5-72b", 2, 11)]


def synth_weights(eng, hp, il):
    """Host copies of a synthesized shard's layer tensors: name -> (type, uint8 blocks or f32 vector).  pb200_model_synth gives Qwen2
    (rope_mode 2) its q / k / v biases."""
    names = ["attn_q.weight", "attn_k.weight", "attn_v.weight", "attn_output.weight", "ffn_gate.weight", "ffn_up.weight", "ffn_down.weight",
             "attn_norm.weight", "ffn_norm.weight"] + (["attn_q.bias", "attn_k.bias", "attn_v.bias"] if hp["rope_mode"] == 2 else [])
    out = {}
    for n in names:
        p, nbytes, t = eng.tensor_device(f"blk.{il}.{n}")
        a = _dev(p, (nbytes,), "|u1").cpu().numpy()
        out[f"blk.{il}.{n}"] = (t, a.view(np.float32).copy() if t == O.F32 else a)
    return out


@pytest.mark.gpu
def test_synth_qwen72b_types(cuda, pkg):
    """pb200_model_synth(ftype 0) on two Qwen2.5-72B layers: the reference's Q4_K_M types tensor by tensor (80 layers = MODEL_70B: attn_v
    Q5_K; n_ff 29 568: ffn_down Q4_K -> Q5_0, or Q6_K -> Q8_0 in the use_more_bits layers), and ftype 2 gives Q4_0 everywhere."""
    hp = pkg.HParams(**QWEN72B)
    want = {0: {11: {"attn_v": O.Q5_K, "ffn_down": O.Q5_0}, 12: {"attn_v": O.Q6_K, "ffn_down": O.Q8_0}},
            2: {11: {"attn_v": O.Q4_0, "ffn_down": O.Q4_0}, 12: {"attn_v": O.Q4_0, "ffn_down": O.Q4_0}}}
    for ftype, layers in want.items():
        m = pkg.Model(hp, 0, (11, 13), False, False)
        m.synth(ftype, 5)
        default = O.Q4_K if ftype == 0 else O.Q4_0
        for il, special in layers.items():
            for w, K in (("attn_q", 8192), ("attn_k", 8192), ("attn_v", 8192), ("attn_output", 8192), ("ffn_gate", 8192), ("ffn_up", 8192),
                         ("ffn_down", 29568)):
                _, nbytes, t = m.tensor_device(f"blk.{il}.{w}.weight")
                assert t == special.get(w, default), (ftype, il, w, t)
                N = {"attn_k": 1024, "attn_v": 1024, "ffn_gate": 29568, "ffn_up": 29568}.get(w, 8192)
                assert nbytes == O.row_size(t, K) * N
        m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("model,ftype,il", FULL, ids=[f"{m}-ftype{f}-layer{il}" for m, f, il in FULL])
def test_full_size_layer_vs_oracle(cuda, lib, pkg, port, model, ftype, il):
    hp = dict(QWEN72B if model == "qwen2.5-72b" else LLAMA8B)
    eng = pkg.Model(pkg.HParams(**hp), 0, (il, il + 1), False, False)
    eng.synth(ftype, 17 + il)
    eng.finalize()
    s = Shard(eng, hp, synth_weights(eng, hp, il), il, False, False, 1)
    try:
        types = layer_types(s.w, il)
        if model == "qwen2.5-72b" and ftype == 0:
            assert (types["down"], types["v"]) == ((O.Q5_0, O.Q5_K) if il == 11 else (O.Q8_0, O.Q6_K)), types
        rng = np.random.default_rng(il)
        s.fill(0, 37, rng)
        for p in (37, 38):
            n = step(lib, s, 1, p, rng.standard_normal(hp["n_embd"]).astype(np.float32))
            check_launches(lib, s, n, f"{model} ftype {ftype}", p, None)
            check_step(lib, port, s, f"{model} ftype {ftype}", p)
    finally:
        eng.close()
