"""Prompt processing layer by layer: the tensor-core activation image bit for bit against the CPU quantizer, and every layer of a
prefill ubatch bit-identical to the same layer built from single-op entry points.

A. k_mmq_prep (mmq.cu) quantizes each activation row like the CPU backend (q8_K for k-quants, q8_0 / q8_1 per 32 values for Q8_0 /
   Q5_1), scales it by a power of two and rounds it to fp16 in the tiled, swizzled image the wgmma consumers read.  After
   pb200_mul_mat_q returns, the workspace holds that image and the row scales; image_rows() undoes the layout and the rows are
   compared as uint16 / uint32 with the restatement built from port.quantize_act, for all five weight types, every T rung of
   test_gpu_mmq.py, short last 256-K groups, ldx > K and activation rows from 2^-60 to 2^60.

B. prefill_ubatch (engine.cu) against compose_layer(), a restatement from the C ABI's single ops on the engine's own weights.  Each
   layer runs in its own pipeline shard (pb200_prefill_stage) fed the composition's input hidden state, so a difference names its layer;
   the unsplit model then runs the same calls through pb200_prefill.  K / V cache rows and output hidden states must be bit-identical,
   and cache rows past the ubatch (f16 NaN before the call) untouched.  That pins the engine's own code: the rms_norm and silu * mul
   producers fused into the activation pass (the same roundings as the separate kernels), the reuse of q's image by k and v and of
   gate's by up, and the branch each layer takes.  prefill_launches() restates that branch choice; the launch count of every shard
   without the head must equal it, and a CPU-only test checks that each case reaches the branch it is named after.
   The last-token logits are held to the GEMV bar (4e-6 of the largest |logit|) against rms_norm * w -> pb200_mul_mat_vec: the head's
   fused producer sums the squares in another order than block_rms_scale.

Bit-identity holds only where every output tile of a mat-mul is computed by one CTA: stream-K splits (mmq.cu) add partial tiles with
fp32 atomics in an order that varies from run to run.  Every product here has K <= 2048 and is asserted unsplit (mmq_plan on this
device's SM count); split shapes are covered by the bounds of test_gpu_mmq.py, test_gpu_engine.py and test_gpu_prefill_attention.py."""
import ctypes as C
import functools
from collections import namedtuple

import numpy as np
import pytest
import torch

import oracle_lib as O
from gpu_util import act_ws, dev_f32, dev_u8, ptr, sync
from test_gpu_kv_shift import _dev, kv_tensors
from test_gpu_mmq import BLK32, KQ, T_RUNGS, mmq_plan, range_rows
from tiny_model import TinyModel

D = 128
F16_NAN = 0x7E00
HALF_ORDER = np.array([0, 2, 1, 3, 4, 6, 5, 7])   # k offsets held by the 8 halves of a 16-byte piece (an involution)


def is_kquant(t):
    return t in KQ


def mmq_supported(t, K):
    """mmq.cu mmq_supported."""
    if is_kquant(t):
        return K % 256 == 0 and K >= 256
    return t in BLK32 and K % 64 == 0 and K >= 256


def pf_tc(t, K, T):
    """engine.cu pf_tc: the tensor-core path, else per-token GEMV."""
    return mmq_supported(t, K) and T >= 8


# ---- A. the activation image ----
def image_rows(ws, tpad, K, BN):
    """The fp16 image at the head of the workspace back in row order, [tpad][K] uint16.  Layout (k_mmq_prep): token tile tt = t / BN,
    64-wide K chunk kc, then row tl = t % BN of 128 bytes; the 16-byte piece j = (k & 63) >> 3 sits at slot j ^ (tl & 7), and inside
    a piece the halves hold k + 0, 2, 1, 3, 4, 6, 5, 7."""
    img = ws[:tpad * K * 2].view(np.uint16).reshape(tpad // BN, K // 64, BN, 8, 8)
    slot = np.arange(8)[None, :] ^ (np.arange(BN)[:, None] & 7)                 # [tl][j] -> slot, an involution per row
    img = np.take_along_axis(img, slot[None, None, :, :, None], axis=3)[..., HALF_ORDER]
    return img.transpose(0, 2, 1, 3, 4).reshape(tpad, K)


def expected_image(port, t, X, tpad):
    """(image [tpad][K] uint16, rscale [tpad] uint32) from the CPU quantizer: q8_K (d f32) for k-quants, q8_0 / q8_1 (d f16) for
    Q8_0 / Q5_1; rmax = max |fl(d q)|, e = min(14 - floor(log2 rmax), 126) (0 for a zero row), image = fp16(fl(d q) 2^e),
    rscale = 2^-e; padding rows zero with rscale 1."""
    T, K = X.shape
    q = port.quantize_act(t, X.reshape(-1))
    if is_kquant(t):
        b = q.reshape(-1, 292)
        d, qs = b[:, 0:4].copy().view(np.float32), b[:, 4:260].view(np.int8)
    else:
        b = q.reshape(-1, 34 if t == O.Q8_0 else 36)
        d = b[:, 0:2].copy().view(np.float16).astype(np.float32)
        qs = b[:, 2:34].view(np.int8) if t == O.Q8_0 else b[:, 4:36].view(np.int8)
    dq = (d * qs.astype(np.float32)).reshape(T, K)                              # float32 products, rounded like __fmul_rn
    rmax = np.abs(dq).max(axis=1)
    e = np.where(rmax > 0, np.minimum(14 - (np.frexp(rmax)[1] - 1), 126), 0)
    up = np.ldexp(np.float32(1.0), e).astype(np.float32)
    img = np.zeros((tpad, K), np.float16)
    img[:T] = (dq * up[:, None]).astype(np.float16)
    rs = np.ones(tpad, np.float32)
    rs[:T] = np.ldexp(np.float32(1.0), -e).astype(np.float32)
    return img.view(np.uint16), rs.view(np.uint32)


K_IMAGE = {t: (256, 1024, 8192) for t in KQ} | {t: (448, 4160, 29568) for t in BLK32}
IMAGE_CASES = [(t, K, T) for t in KQ + BLK32 for K in K_IMAGE[t] for T in T_RUNGS]


def image_inputs(t, K, T, seed):
    """T rows cycled from test_gpu_mmq.range_rows: 2^-60 .. 2^60 (k-quants) / 2^20 and 8e6 (Q8_0, Q5_1), amax 65 000 / 66 000, one hot
    block among 1e-3 blocks, a single nonzero, a zero row.  Below K = 1024 the columns around the hot block's edge (256) and the single
    nonzero (777) are kept, both windows starting at an even column so that Q5_1's (v, -v) pairs stay whole."""
    rows = range_rows(t, max(K, 1024), np.random.default_rng(seed))
    if K < rows.shape[1]:
        h = K // 4
        rows = rows[:, np.r_[256 - h:256 + h, 776 - h:776 + h]]
    return rows[(np.arange(T) * 5 + T) % len(rows)]


@pytest.mark.gpu
@pytest.mark.parametrize("t,K,T", IMAGE_CASES, ids=[f"{O.TYPE_NAME[t]}-K{K}-T{T}" for t, K, T in IMAGE_CASES])
def test_mmq_prep_image_bit_exact(cuda, lib, port, t, K, T):
    """The workspace after pb200_mul_mat_q, at ldx = K and K + 64 (NaN in the 64 extra columns): image and row scales bit for bit,
    padding rows zero with scale 1, and the bytes behind the workspace untouched."""
    X = image_inputs(t, K, T, seed=7 * t + K + T)
    p = mmq_plan(lib, 16, K, T)
    assert (p.bn, p.ttiles) == T_RUNGS[T], p
    want_img, want_rs = expected_image(port, t, X, p.tpad)
    nbytes = lib.c.pb200_mul_mat_q_workspace_bytes(K, T)
    assert nbytes == p.tpad * (2 * K + 4)
    Wd = dev_u8(O.synth_blocks(t, 16, K, seed=t + K))
    for ldx in (K, K + 64):
        Xp = np.full((T, ldx), np.nan, np.float32)
        Xp[:, :K] = X
        xd = dev_f32(Xp)
        y = torch.empty((T, 16), dtype=torch.float32, device="cuda")
        ws = torch.full((nbytes + 64,), 0xA5, dtype=torch.uint8, device="cuda")
        lib.check(lib.c.pb200_mul_mat_q(t, ptr(Wd), 16, K, ptr(xd), ldx, T, ptr(y), None, None, ptr(ws), None), "mul_mat_q")
        sync()
        assert lib.c.pb200_aborted() == 0, "tensor-core pipeline gave up (watchdog)"
        raw = ws.cpu().numpy()
        got = image_rows(raw, p.tpad, K, p.bn)
        bad = np.argwhere(got != want_img)
        assert bad.size == 0, (f"ldx {ldx}: {len(bad)} image halves differ, first at (t, k) = {tuple(bad[0])}: "
                               f"got {got[tuple(bad[0])]:#06x}, want {want_img[tuple(bad[0])]:#06x}; rows {np.unique(bad[:, 0])[:16]}")
        rs = raw[p.tpad * K * 2:nbytes].view(np.uint32)
        assert np.array_equal(rs, want_rs), (ldx, np.nonzero(rs != want_rs)[0][:16])
        assert np.all(raw[nbytes:] == 0xA5), f"ldx {ldx}: write past the workspace"


# ---- B. prefill ubatches against single ops ----
LayerPlan = namedtuple("LayerPlan", "launches qkv gu down reuse")


def layer_types(tm, il):
    return {k: tm.tensors[f"blk.{il}.{n}.weight"][0] for k, n in (("q", "attn_q"), ("k", "attn_k"), ("v", "attn_v"), ("o", "attn_output"),
                                                                    ("gate", "ffn_gate"), ("up", "ffn_up"), ("down", "ffn_down"))}


def prefill_launches(types, hp, T, with_embd):
    """prefill_ubatch's kernel launches for a shard of one layer without the head (engine.cu), and the branches it takes.
    A tensor-core product costs 2 launches (k_mmq_prep + k_mmq_tc), 1 when it reuses the previous product's image (pf_matmul: both on
    the tensor-core path, the same K, both k-quants or both not); per-token GEMV costs 2 per token (quantize + GEMV).  q|k|v and
    gate|up fuse rms_norm * w into the first product's activation pass when all of them are k-quants on the tensor-core path, else
    k_rms_norm_rows runs first; ffn_down fuses silu(g) * u when it is a k-quant on the tensor-core path, else k_silu_mul runs first."""
    E, QD, EK, F = hp["n_embd"], hp["n_head"] * D, hp["n_head_kv"] * D, hp["n_ff"]
    n = 1 + int(with_embd)                                   # k_iota_pos, get_rows
    reuse = {}

    def mm(name, K, same_as=None):
        t = types[name]
        if not pf_tc(t, K, T):
            return 2 * T
        s = types.get(same_as)
        reuse[name] = same_as is not None and pf_tc(s, K, T) and is_kquant(s) == is_kquant(t)   # same K: q|k|v and gate|up share x
        return 1 if reuse[name] else 2

    def group(names, K):
        tc = all(pf_tc(types[m], K, T) for m in names)
        kind = "fused" if tc and all(is_kquant(types[m]) for m in names) else ("split" if tc else "gemv")
        return kind, (kind != "fused") + sum(mm(m, K, names[i - 1] if i else None) for i, m in enumerate(names))

    qkv, c = group(("q", "k", "v"), E)
    n += c + 2 + 2 + 1 + mm("o", QD)                         # rope q, k; f16 K / V store; attention; wo (+ residual)
    gu, c = group(("gate", "up"), E)
    n += c
    if pf_tc(types["down"], F, T) and is_kquant(types["down"]):
        down = "fused"
    else:
        down = "silu_tc" if pf_tc(types["down"], F, T) else "silu_gemv"
        n += 1
    n += mm("down", F)
    return LayerPlan(n, qkv, gu, down, reuse)


def plan_tag(p):
    if p.qkv == p.gu == "gemv":
        return "gemv"
    return f"qkv_{p.qkv}-gu_{p.gu}-down_{p.down}"


# name -> TinyModel arguments, [(pos0, T)], the branch tag every layer of every call must reach.  8 / 2 heads, E 1024, three layers.
LAYER_CASES = {
    "llama_fused": (dict(arch="llama", ftype="q4_K_M", n_ff=2048, n_ctx=192, freq_factors=True),
                    [(0, 129), (129, 31), (160, 8), (168, 5)],
                    ["qkv_fused-gu_fused-down_fused"] * 3 + ["gemv"]),
    "llama_fused_t512": (dict(arch="llama", ftype="q4_K_M", n_ff=2048, n_ctx=512, freq_factors=True), [(0, 512)],
                         ["qkv_fused-gu_fused-down_fused"]),
    "qwen2_bias_blk32_down": (dict(arch="qwen2", ftype="q5_K_M", n_ff=1088, n_ctx=128), [(0, 64), (64, 33)],
                              ["qkv_fused-gu_fused-down_silu_tc"] * 2),
    "qwen2_gemv_down": (dict(arch="qwen2", ftype="q5_K_M", n_ff=1056, n_ctx=128), [(0, 12)], ["qkv_fused-gu_fused-down_silu_gemv"]),
    "llama_mixed_q8_0": (dict(arch="llama", ftype="q4_K_M", n_ff=2048, n_ctx=128, types={"attn_k": O.Q8_0, "ffn_up": O.Q8_0}),
                         [(0, 40)], ["qkv_split-gu_split-down_fused"]),
}


@functools.lru_cache(maxsize=None)
def layer_model(name, seed):
    kw = dict(LAYER_CASES[name][0])
    return TinyModel(n_layer=3, n_embd=1024, n_head=8, n_head_kv=2, n_vocab=512, seed=seed, branch_scale=0.1, **kw)


def case_id(name):
    _, calls, tags = LAYER_CASES[name]
    return name + "-" + "-".join(f"p{p}t{T}_{tag}" for (p, T), tag in zip(calls, tags))


def test_layer_cases_reach_their_branches():
    """No GPU: every layer of every call takes the branch its case is named after, the reuse rule gives what the case is there for, and
    the launch arithmetic matches two counts worked out by hand."""
    for name, (_, calls, tags) in LAYER_CASES.items():
        tm = layer_model(name, seed=1)
        hp = tm.hp
        assert max(hp["n_embd"], hp["n_ff"], hp["n_head"] * D) <= 2048, name
        assert calls[-1][0] + calls[-1][1] <= hp["n_ctx"] and all(T <= 512 for _, T in calls), name
        for (pos0, T), tag in zip(calls, tags):
            for il in range(hp["n_layer"]):
                p = prefill_launches(layer_types(tm, il), hp, T, il == 0)
                assert plan_tag(p) == tag, (name, pos0, T, il, p)
                if name == "llama_mixed_q8_0":
                    assert not any(p.reuse.values()), p             # q8_K / q8_0 images must not be shared
                elif p.qkv == "fused":
                    assert p.reuse["k"] and p.reuse["v"] and p.reuse["up"] and not p.reuse["q"] and not p.reuse["gate"], p
    tm = layer_model("llama_mixed_q8_0", seed=1)
    assert prefill_launches(layer_types(tm, 1), tm.hp, 40, False).launches == 1 + 1 + 2 + 2 + 2 + 2 + 2 + 1 + 2 + 1 + 2 + 2 + 2
    tm = layer_model("llama_fused", seed=1)
    assert prefill_launches(layer_types(tm, 0), tm.hp, 5, True).launches == 2 + 1 + 30 + 5 + 10 + 1 + 20 + 1 + 10
    kinds = {layer_types(layer_model(n, 1), il)["down"] for n in ("qwen2_bias_blk32_down", "qwen2_gemv_down") for il in range(3)}
    assert kinds == {O.Q5_1, O.Q8_0}                               # both 32-element block types as ffn_down


class Compose:
    """prefill_ubatch restated from the C ABI's single ops, on the device, with its own f16 K / V caches [layer][n_ctx][EK]."""

    def __init__(self, lib, tm, engines):
        self.lib, self.tm, self.hp = lib, tm, tm.hp
        self.w = {}
        for name in tm.tensors:
            for eng in engines:
                try:
                    p, _, t = eng.tensor_device(name)
                except Exception:
                    continue
                self.w[name] = (p, t)
                break
        assert set(self.w) == set(tm.tensors), set(tm.tensors) - set(self.w)
        hp = self.hp
        self.kc = [torch.zeros((hp["n_ctx"], hp["n_head_kv"] * D), dtype=torch.int16, device="cuda") for _ in range(hp["n_layer"])]
        self.vc = [torch.zeros_like(k) for k in self.kc]

    def wp(self, name):
        return C.c_void_p(self.w[name][0]) if name in self.w else None

    def norm(self, x, rows, wname):
        E, c = self.hp["n_embd"], self.lib.c
        y = torch.full_like(x, float("nan"))
        self.lib.check(c.pb200_rms_norm(ptr(x), ptr(y), E, rows, self.hp["rms_eps"], None), "rms_norm")
        out = torch.full_like(x, float("nan"))
        self.lib.check(c.pb200_binary(C.c_int(1), ptr(y), self.wp(wname), ptr(out), C.c_int64(rows * E), C.c_int64(E), None), "binary mul")
        return out

    def mm(self, name, x, T, N, K, bias=None, resid=None):
        """The engine's pf_matmul: pb200_mul_mat_q on the tensor-core path, else pb200_quantize_act + pb200_mul_mat_vec_q per token."""
        c = self.lib.c
        W, t = self.w[name]
        y = torch.full((T, N), float("nan"), dtype=torch.float32, device="cuda")
        b = self.wp(bias) if bias else None
        assert bool(c.pb200_mul_mat_q_supported(t, C.c_int64(K))) == mmq_supported(t, K), (name, t, K)
        if pf_tc(t, K, T):
            assert not mmq_plan(self.lib, N, K, T).split, (name, N, K, T, mmq_plan(self.lib, N, K, T))
            ws = torch.empty(c.pb200_mul_mat_q_workspace_bytes(K, T), dtype=torch.uint8, device="cuda")
            self.lib.check(c.pb200_mul_mat_q(t, C.c_void_p(W), N, K, ptr(x), K, T, ptr(y), b, ptr(resid) if resid is not None else None,
                                         ptr(ws), None), f"mul_mat_q {name}")
            return y
        aws = act_ws(self.lib, K)
        for i in range(T):
            r = C.c_void_p(resid.data_ptr() + i * N * 4) if resid is not None else None
            self.lib.check(c.pb200_quantize_act(t, C.c_void_p(x.data_ptr() + i * K * 4), K, ptr(aws), None), "quantize_act")
            self.lib.check(c.pb200_mul_mat_vec_q(t, C.c_void_p(W), N, K, ptr(aws), C.c_void_p(y.data_ptr() + i * N * 4), b, r, None),
                       f"mul_mat_vec_q {name}")
        return y

    def rope(self, x, T, n_head, pos):
        hp = self.hp
        y = torch.full_like(x, float("nan"))
        self.lib.check(self.lib.c.pb200_rope(ptr(x), ptr(y), T, n_head, D, D, hp["rope_mode"], ptr(pos), hp["rope_freq_base"],
                                         hp["rope_freq_scale"], 0.0, 1.0, 32.0, 1.0, hp["n_ctx_orig"], self.wp("rope_freqs.weight"), None),
                   "rope")
        return y

    def store(self, src, cache, pos0, T):
        EK = self.hp["n_head_kv"] * D
        ne = (C.c_int64 * 4)(EK, T, 1, 1)
        sb = (C.c_int64 * 4)(4, EK * 4, T * EK * 4, T * EK * 4)
        db = (C.c_int64 * 4)(2, EK * 2, T * EK * 2, T * EK * 2)
        self.lib.check(self.lib.c.pb200_copy_strided(ptr(src), C.c_void_p(cache.data_ptr() + pos0 * EK * 2), C.c_int(1), ne, sb, db, None),
                   "copy_strided")

    def embed(self, toks):
        E = self.hp["n_embd"]
        W, t = self.w["token_embd.weight"]
        ids = torch.from_numpy(np.ascontiguousarray(toks, np.int32)).cuda()
        x = torch.full((len(toks), E), float("nan"), dtype=torch.float32, device="cuda")
        self.lib.check(self.lib.c.pb200_get_rows(t, C.c_void_p(W), E, ptr(ids), len(toks), ptr(x), None), "get_rows")
        return x

    def layer(self, il, x, pos0, T):
        hp, c = self.hp, self.lib.c
        E, H, HK, F = hp["n_embd"], hp["n_head"], hp["n_head_kv"], hp["n_ff"]
        QD, EK, p = H * D, HK * D, f"blk.{il}."
        pos = torch.arange(pos0, pos0 + T, dtype=torch.int32, device="cuda")
        xn = self.norm(x, T, p + "attn_norm.weight")
        q = self.mm(p + "attn_q.weight", xn, T, QD, E, bias=p + "attn_q.bias")
        k = self.mm(p + "attn_k.weight", xn, T, EK, E, bias=p + "attn_k.bias")
        v = self.mm(p + "attn_v.weight", xn, T, EK, E, bias=p + "attn_v.bias")
        q, k = self.rope(q, T, H, pos), self.rope(k, T, HK, pos)
        self.store(k, self.kc[il], pos0, T)
        self.store(v, self.vc[il], pos0, T)
        att = torch.full((T, QD), float("nan"), dtype=torch.float32, device="cuda")
        scale = float(np.float32(1.0) / np.sqrt(np.float32(D)))    # the engine's 1.0f / sqrtf(128.f)
        self.lib.check(c.pb200_attn_prefill(ptr(q), ptr(self.kc[il]), ptr(self.vc[il]), ptr(att), H, HK, D, ptr(pos), T, pos0 + T, scale, None),
                   "attn_prefill")
        x1 = self.mm(p + "attn_output.weight", att, T, E, QD, resid=x)
        xn = self.norm(x1, T, p + "ffn_norm.weight")
        g = self.mm(p + "ffn_gate.weight", xn, T, F, E)
        u = self.mm(p + "ffn_up.weight", xn, T, F, E)
        a = torch.full_like(g, float("nan"))
        self.lib.check(c.pb200_silu_mul(ptr(g), ptr(u), ptr(a), T * F, None), "silu_mul")
        return self.mm(p + "ffn_down.weight", a, T, E, F, resid=x1)

    def head(self, x_last):
        hp, c = self.hp, self.lib.c
        xn = self.norm(x_last.reshape(1, -1).contiguous(), 1, "output_norm.weight")
        W, t = self.w["output.weight"]
        y = torch.full((hp["n_vocab"],), float("nan"), dtype=torch.float32, device="cuda")
        self.lib.check(c.pb200_mul_mat_vec(t, C.c_void_p(W), hp["n_vocab"], hp["n_embd"], ptr(xn), ptr(y), ptr(act_ws(self.lib, hp["n_embd"])),
                                       None), "mul_mat_vec head")
        return y


# Views onto an engine's memory live only inside these helpers: a failing check's traceback is printed after the engine is freed,
# and printing a view of freed device memory would read it.
def nan_past(eng, tm, nl, comp, layers, start):
    """Cache rows from `start` on to f16 NaN: the engine's K / V of its nl layers and the composition's of the given layers."""
    for c in kv_tensors(eng, tm, 1, nl) + tuple(c for il in layers for c in (comp.kc[il], comp.vc[il])):
        c[..., start:, :] = F16_NAN


def engine_kv(eng, tm, nl):
    """Host copies of the engine's K / V caches, [layer][n_ctx][EK] int16 each."""
    return tuple(c[0].cpu().numpy() for c in kv_tensors(eng, tm, 1, nl))


def engine_hidden(ptr_dev, T, E):
    return _dev(ptr_dev, (T, E), "<f4").clone().cpu().numpy()


def check_cache(name, g, w, pos0, T):
    """Host arrays [n_ctx][EK]: rows [0, pos0 + T) bit-identical, rows past them still f16 NaN."""
    end = pos0 + T
    bad = np.nonzero((g[:end] != w[:end]).any(axis=1))[0]
    assert bad.size == 0, f"{name}: rows {bad[:16]} differ ({bad.size} rows; this call wrote [{pos0}, {end}))"
    assert np.all(g[end:] == F16_NAN), f"{name}: rows past {end} written: {np.nonzero((g[end:] != F16_NAN).any(axis=1))[0][:16] + end}"


def check_bits(name, got, want):
    g, w = got.view(np.uint32), want.view(np.uint32)
    bad = np.argwhere(g != w)
    assert bad.size == 0, f"{name}: {len(bad)} values differ, first at {tuple(bad[0])}: {got[tuple(bad[0])]!r} vs {want[tuple(bad[0])]!r}"


def check_logits(what, got, want):
    err = float(np.max(np.abs(got.astype(np.float64) - want.astype(np.float64))))
    same = np.array_equal(got.view(np.uint32), want.view(np.uint32))
    print(f"{what}: last-token logits {'bit-identical' if same else f'max |d| {err:.3e}'} (max |logit| {np.max(np.abs(want)):.3f})")
    assert np.isfinite(got).all() and err <= 4e-6 * float(np.max(np.abs(want))), (what, err)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(LAYER_CASES), ids=[case_id(n) for n in LAYER_CASES])
def test_prefill_layers_bit_identical_to_single_ops(cuda, lib, pkg, name):
    _, calls, _ = LAYER_CASES[name]
    tm = layer_model(name, seed=len(name))
    hp, nl, E, V = tm.hp, tm.hp["n_layer"], tm.hp["n_embd"], tm.hp["n_vocab"]
    shards = [tm.load_engine(pkg, layers=(il, il + 1), with_embd=il == 0, with_head=il == nl - 1) for il in range(nl)]
    comp = Compose(lib, tm, shards)
    outs, logits = [], []
    try:
        for pos0, T in calls:
            toks = [(i * 7919 + 13 * pos0 + 5) % V for i in range(T)]
            x = comp.embed(toks)
            for il, s in enumerate(shards):
                nan_past(s, tm, 1, comp, [il], pos0 + T)
                sync()
                lg = np.full(V, np.nan, np.float32) if il == nl - 1 else None
                before = lib.c.pb200_kernel_launches()
                hid = s.prefill_stage(toks if il == 0 else None, None if il == 0 else x.data_ptr(), T, pos0, lg, synchronize=True)
                n = lib.c.pb200_kernel_launches() - before
                assert lib.c.pb200_aborted() == 0
                plan = prefill_launches(layer_types(tm, il), hp, T, il == 0)
                if il < nl - 1:
                    assert n == plan.launches, (f"layer {il}: {n} launches, {plan_tag(plan)} makes {plan.launches}", plan)
                eng_out, (ek, ev) = engine_hidden(hid, T, E), engine_kv(s, tm, 1)
                y = comp.layer(il, x, pos0, T)
                sync()
                assert lib.c.pb200_aborted() == 0
                where = f"p{pos0}t{T} layer {il} ({plan_tag(plan)})"
                check_cache(f"{where} K", ek[0], comp.kc[il].cpu().numpy(), pos0, T)
                check_cache(f"{where} V", ev[0], comp.vc[il].cpu().numpy(), pos0, T)
                check_bits(f"{where} hidden out", eng_out, y.cpu().numpy())
                x = y
            outs.append(x.cpu().numpy())
            logits.append(lg)
            check_logits(f"p{pos0}t{T} head shard", lg, comp.head(x[T - 1]).cpu().numpy())
    finally:
        for s in shards:
            s.close()
    # the unsplit model through pb200_prefill: same calls, same caches, same hidden states, and the same logits as the head shard
    eng = tm.load_engine(pkg)
    try:
        for (pos0, T), want_out, want_lg in zip(calls, outs, logits):
            toks = [(i * 7919 + 13 * pos0 + 5) % V for i in range(T)]
            nan_past(eng, tm, nl, comp, [], pos0 + T)
            sync()
            lg = eng.prefill(toks, pos0).copy()
            assert lib.c.pb200_aborted() == 0
            ek, ev = engine_kv(eng, tm, nl)
            for il in range(nl):
                check_cache(f"unsplit p{pos0}t{T} layer {il} K", ek[il], comp.kc[il].cpu().numpy(), pos0, T)
                check_cache(f"unsplit p{pos0}t{T} layer {il} V", ev[il], comp.vc[il].cpu().numpy(), pos0, T)
            check_bits(f"unsplit p{pos0}t{T} hidden out", engine_hidden(lib.c.pb200_prefill_hidden_device(eng.h), T, E), want_out)
            check_bits(f"unsplit p{pos0}t{T} logits vs head shard", lg, want_lg)
    finally:
        eng.close()
