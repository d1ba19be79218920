"""The decode GEMV (k_gemv_kquant's bulk-copy ring, gemv.cu) at the shapes the served models launch and across the plans gemv_plan picks.

Faults of the ring (a stale stage, an mbarrier parity ABA, a split-row partial slot reused too early, an owner-only release count that
is off on a ragged last tile) only show once a CTA goes round its ring several times, i.e. at full matrix sizes.  So the weights are
U unique rows scattered over N rows by a seeded permutation: the oracle evaluates U rows while the device streams the whole matrix.
Every launch is checked three ways:
  * every row against its source row's oracle value, within 4e-6 max(1, |ref|) (fp32 summation order);
  * rows that share a source are bit-identical: the per-row arithmetic does not depend on the tile, stage, warp, sub-warp or the
    row's misalignment in the stage, so a stale stage or a row written to the wrong place shows up as a mismatch (biases and
    residuals are drawn per source as well, so the check covers the epilogue too);
  * y starts as NaN and pb200_aborted() is 0 after the synchronisation: a wait that gave up fails the test.
gemv_plan() below restates the launcher's arithmetic so that each case is named after the plan it reaches, and
test_sweep_cases_wrap_their_rings checks (without a GPU) that every sweep case makes each CTA go round its ring at least 3 times."""
import ctypes as C
import math
from collections import namedtuple

import numpy as np
import pytest
import torch

import legacy_types as L
import oracle_lib as O
from gpu_util import act_ws, act_ws_fields, dev_f32, ptr, sync
from test_gpu_fallbacks import GemvMat

KQ = [O.Q4_K, O.Q5_K, O.Q6_K]
BLK32 = [O.Q8_0, O.Q5_1, L.Q4_0, L.Q4_1, L.Q5_0]   # the 32-element block types (common.cuh is_blk32_type)
TN = O.TYPE_NAME | L.NAME
ENOTSUP = -3
U_ROWS = 2048              # unique rows per matrix
SWEEP_BYTES = 192 << 20    # weight bytes per sweep case: >= 3 turns of every CTA's ring whatever depth the plan picks
H100_SMS = 132

# ---- gemv_plan (gemv.cu) restated; constants from gemv.cuh / common.cuh ----
SMEM_LIMIT, CTL_BYTES, STAGE_TARGET, MAX_STAGE, ROWQ, NW, ACT_MAX_NBLK, CTAS_PER_SM = 113 * 1024, 768, 28 * 1024, 8, 8, 8, 116, 2
Plan = namedtuple("Plan", "wpr rpw rows nstage nstage_init owner_only ntiles")


def gemv_plan(types, Ns, K):
    """The ring geometry launch_gemv gives a group, or None where the group does not fit the ring kernel."""
    b32 = len(types) == 1 and types[0] in BLK32
    nblk = (K + 255) // 256
    if not (K % (32 if b32 else 256) == 0 and nblk <= ACT_MAX_NBLK):
        return None
    wpr = 1
    while wpr * 32 < nblk:
        wpr *= 2
    ngroups = NW // wpr
    nbp = 1
    while nbp < nblk and nbp < 32:
        nbp *= 2
    rpw = 1 if wpr > 1 else 32 // nbp
    rows, biggest = [], 0
    for t, N in zip(types, Ns):
        rb = L.row_size(t, K)
        if not (t in KQ or b32) or (b32 and rb % 8):           # the column dots read 64-bit words
            return None
        R = max(rpw, max(1, STAGE_TARGET // rb) // rpw * rpw)
        if wpr > 1:
            R = min(R, ngroups)
            while R > 1 and (SMEM_LIMIT - CTL_BYTES) // ((R * rb + 16 + 127) // 128 * 128) < 5:
                R -= 1
        if R > N:
            R = (N + rpw - 1) // rpw * rpw
        rows.append(R)
        biggest = max(biggest, R * rb)
    stage = (biggest + 16 + 127) // 128 * 128
    act_stages = -(-(nblk * (272 + 64) + 64) // stage)
    nstage = min(MAX_STAGE, (SMEM_LIMIT - CTL_BYTES) // stage, ROWQ - 1)
    owner = False
    slots = rows[0] // rpw
    if all(r == rows[0] for r in rows) and slots < ngroups:
        period = ngroups // math.gcd(slots, ngroups)
        ns = nstage // period * period
        if ns >= 3 and ns - act_stages >= 2:
            nstage, owner = ns, True
    if nstage - act_stages < (1 if b32 else 2):
        return None
    ntiles = sum(-(-N // R) for N, R in zip(Ns, rows))
    return Plan(wpr, rpw, rows, nstage, nstage - act_stages, owner, ntiles)


def plan_tag(p):
    rows = "+".join(map(str, sorted(set(p.rows))))
    return f"wpr{p.wpr}-rpw{p.rpw}-R{rows}-{p.nstage}st{p.nstage_init}pre" + ("-owner" if p.owner_only else "")


def ring_turns(p, sms):
    """Times the least loaded CTA goes round its ring (tile t goes to CTA t mod grid)."""
    grid = min(sms * CTAS_PER_SM, p.ntiles)
    return (p.ntiles // grid) / p.nstage


# ---- sweep cases: (weight types of the group, K, rows of each matrix) ----
def _n_for(t, K, n_min=1):
    return max(n_min, -(-SWEEP_BYTES // L.row_size(t, K)))


SWEEP_K = [768, 1280, 1536, 3072, 3584, 4096, 5120, 8192, 8448, 8960, 13824, 14336, 16384, 16640, 18944, 27648, 28672, 29696]
SWEEP = [((t,), K, (_n_for(t, K),)) for t in KQ for K in SWEEP_K]
SWEEP += [((t,), K, (_n_for(t, K, n),)) for t in (O.Q8_0, O.Q5_1) for n, K in ((8192, 29568), (16384, 4096))]
SWEEP += [((O.Q5_1,), 7392, (_n_for(O.Q5_1, 7392, 8192),))]
# q|k|v-like groups at K 8192: mixed types (the TYPE = 0 instantiation, unequal R), one type with R 5 and a 1-row last tile (owner_only off)
SWEEP += [((O.Q4_K, O.Q4_K, O.Q6_K), 8192, (24576, 8192, 8192)), ((O.Q5_K, O.Q5_K, O.Q5_K), 8192, (24576, 4096, 4101))]
# Q4_0 / Q4_1 / Q5_0 at Llama-3-8B's K, a Q4_1 K whose last 8-block column holds 2 blocks, and Qwen2.5-72B Q4_K_M's Q5_0 ffn_down
SWEEP += [((t,), K, (_n_for(t, K),)) for t in L.LEGACY_TYPES for K in (4096, 8192, 14336)]
SWEEP += [((L.Q4_1,), 4160, (_n_for(L.Q4_1, 4160),)), ((L.Q5_0,), 29568, (_n_for(L.Q5_0, 29568, 8192),))]


def sweep_id(case):
    types, K, Ns = case
    return f"{'+'.join(TN[t] for t in types)}-K{K}-{plan_tag(gemv_plan(types, Ns, K))}"


# the plan families of the launches the served models make (Llama-3-8B / 70B, Qwen2.5-72B), each reached by a sweep case above
FAMILIES = {
    ((O.Q4_K,), 4096): dict(rpw=2, rows=[12], nstage=4, owner_only=True),                       # Llama-3-8B gate|up, wo
    ((O.Q6_K,), 4096): dict(rpw=2, rows=[8]),                                                   # Llama-3-8B head
    ((O.Q4_K,), 14336): dict(wpr=2, rows=[2], nstage=6, owner_only=True),                       # Llama-3-8B ffn_down
    ((O.Q6_K,), 14336): dict(wpr=2, rows=[1], nstage=4, nstage_init=2, owner_only=True),
    ((O.Q5_K,), 8192): dict(wpr=1, rows=[5], owner_only=False),                                 # Qwen2.5-72B wo, gate|up
    ((O.Q6_K,), 8192): dict(rows=[4]),                                                          # the heads at K 8192
    ((O.Q8_0,), 29568): dict(wpr=4, rows=[1], nstage=3, nstage_init=1, owner_only=False),       # Qwen2.5-72B ffn_down
    ((O.Q5_1,), 29568): dict(wpr=4, nstage=4, owner_only=True),
    ((O.Q4_K,), 18944): dict(wpr=4, rows=[2]),
    ((O.Q4_K, O.Q4_K, O.Q6_K), 8192): dict(owner_only=False),
    ((O.Q5_K, O.Q5_K, O.Q5_K), 8192): dict(owner_only=False),
    ((L.Q4_0,), 4096): dict(wpr=1, rpw=2, rows=[12], nstage=4, owner_only=True),              # Llama-3-8B Q4_0 q, k, v, wo, gate, up
    ((L.Q4_0,), 14336): dict(wpr=2, rows=[2], nstage=6, nstage_init=4, owner_only=True),       # Llama-3-8B Q4_0 ffn_down
    ((L.Q5_0,), 29568): dict(wpr=4, rows=[1], nstage=4, nstage_init=2, owner_only=True),       # Qwen2.5-72B Q4_K_M ffn_down
}


def test_sweep_cases_wrap_their_rings():
    """No GPU: every sweep case fits the ring and, on an H100's 132 SMs, turns each CTA's ring at least 3 times; the plan families of
    the served models' launches are among them."""
    for case in SWEEP:
        p = gemv_plan(case[0], case[2], case[1])
        assert p is not None, case
        assert ring_turns(p, H100_SMS) >= 3, (sweep_id(case), ring_turns(p, H100_SMS))
    for (types, K), want in FAMILIES.items():
        case = next(c for c in SWEEP if c[0] == types and c[1] == K)
        p = gemv_plan(types, case[2], K)._asdict()
        assert {k: p[k] for k in want} == want, (sweep_id(case), p)
    # rows that are not 8-byte multiples leave the ring: Q8_0 at K 7392, Q4_0 / Q5_0 at K 4160 (130 blocks of 18 / 22 bytes)
    assert gemv_plan((O.Q8_0,), (4096,), 7392) is None and gemv_plan((O.Q5_1,), (4096,), 7392) is not None
    assert gemv_plan((L.Q4_0,), (4096,), 4160) is None and gemv_plan((L.Q5_0,), (4096,), 4160) is None
    assert gemv_plan((L.Q4_1,), (4096,), 4160) is not None
    # 32-element block types take the ring one matrix at a time
    assert gemv_plan((L.Q4_0, L.Q4_0), (4096, 1024), 4096) is None and gemv_plan((O.Q4_K, O.Q4_K), (4096, 1024), 4096) is not None


# ---- device helpers ----
def oracle_mul_mat(port, t, W, N, K, x):
    """The CPU's mat-vec for any weight type: the C port, or legacy_types' restatement for Q4_0 / Q4_1 / Q5_0."""
    return L.mul_mat(port, t, W, N, K, x) if t in L.LEGACY_TYPES else port.mul_mat(t, W, N, K, x)


def oracle_quantize_act(port, t, x):
    return L.quantize_act(port, t, x) if t in L.LEGACY_TYPES else port.quantize_act(t, x)


def _fused(lib):
    fn = lib.c.pb200_gemv_fused
    fn.argtypes = [C.c_int, C.POINTER(GemvMat), C.c_int64, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_int,
                   C.c_void_p]
    return fn


class Scattered:
    """U unique synth_blocks rows spread over N rows by a seeded permutation.  W: device [N][row_bytes] in a 16-byte aligned
    allocation padded by 64 bytes (the padding rule of prima_b200.h); src: each row's source row (host); y: NaN-filled output;
    add_u (optional): a bias / residual per source row, add its device image per row."""

    def __init__(self, t, N, K, seed, with_add=False, U=U_ROWS):
        self.t, self.N, self.K = t, N, K
        self.U = U = min(U, N)
        rb = L.row_size(t, K)
        self.Wu = L.synth_blocks(t, U, K, seed=seed)
        self.src = (torch.randperm(N, generator=torch.Generator().manual_seed(seed)) % U).numpy()
        Wud = torch.from_numpy(self.Wu.reshape(U, rb)).cuda()
        self.W = torch.zeros(N * rb + 64, dtype=torch.uint8, device="cuda")
        self.W[: N * rb].view(N, rb).copy_(Wud[torch.from_numpy(self.src).cuda()])
        assert self.W.data_ptr() % 16 == 0
        self.y = torch.full((N,), float("nan"), device="cuda")
        self.add_u = self.add = None
        if with_add:
            self.add_u = np.random.default_rng(seed + 1).standard_normal(U).astype(np.float32)
            self.add = dev_f32(self.add_u[self.src])

    def mat(self):
        return GemvMat(self.t, 0, self.W.data_ptr(), self.N, self.y.data_ptr(), self.add.data_ptr() if self.add is not None else None)

    def check(self, port, x, what, add_rows=None):
        """y against the oracle's mat-vec of the source rows on activation x (+ the per-source add, or add_rows per row)."""
        want_u = oracle_mul_mat(port, self.t, self.Wu, self.U, self.K, x)[0]
        if self.add_u is not None:
            want_u = want_u + self.add_u
        want = want_u[self.src]
        if add_rows is not None:
            want = want + add_rows
        got = self.y.cpu().numpy()
        bad = ~np.isfinite(got)
        assert not bad.any(), f"{what}: {int(bad.sum())} of {self.N} rows not written or not finite, first {np.flatnonzero(bad)[:8]}"
        err = np.abs(got - want)
        tol = 4e-6 * max(1.0, float(np.max(np.abs(want))))
        r = int(np.argmax(err))
        assert err[r] <= tol, f"{what}: row {r} (source {self.src[r]}) off by {err[r]:.3e} > {tol:.3e}; {int((err > tol).sum())} rows over"
        if add_rows is None:
            rep = np.empty(self.U, np.float32)
            rep[self.src] = got
            diff = np.flatnonzero(got.view(np.uint32) != rep[self.src].view(np.uint32))
            assert diff.size == 0, f"{what}: {diff.size} rows differ from another row of the same source, first {diff[:8]}"


def _no_abort(lib, what):
    sync()
    assert lib.c.pb200_aborted() == 0, f"{what}: an in-kernel wait gave up (watchdog)"


def _prologue_input(lib, port, prologue, K, eps, seed):
    """Device operands of a prologue and the f32 activation the oracle quantizes: rms_norm(a) * w, or silu(g) * u with the device's
    expf (the plain silu * mul ops, same arithmetic as the fused prologue), or a itself (prologue 0)."""
    rng = np.random.default_rng(seed)
    a = rng.standard_normal(K).astype(np.float32)
    b = (1.0 + 0.1 * rng.standard_normal(K)).astype(np.float32) if prologue == 1 else rng.standard_normal(K).astype(np.float32)
    ad, bd = dev_f32(a), dev_f32(b)
    if prologue == 1:
        return ad, bd, port.rms_norm(a, eps) * b
    if prologue == 0:
        return ad, bd, a
    return ad, bd, _silu_mul(lib, port, ad, bd)


def _silu_mul(lib, port, gd, ud):
    K = gd.numel()
    xd = torch.zeros(K, device="cuda")
    lib.check(lib.c.pb200_silu_mul(ptr(gd), ptr(ud), ptr(xd), K, None), "silu_mul")
    sync()
    x = xd.cpu().numpy()
    want = port.silu_mul(gd.cpu().numpy(), ud.cpu().numpy())
    assert np.max(np.abs(x - want)) <= 1e-6 * max(1.0, float(np.max(np.abs(x))))
    return x


def run_fused(lib, port, ms, K, prologue, eps=1e-5, seed=0, what=""):
    """One pb200_gemv_fused launch the way the engine makes it: barrier words, PDL on; prologue 0 quantizes the input first."""
    ad, bd, x = _prologue_input(lib, port, prologue, K, eps, seed)
    ws = act_ws(lib, K)
    sync_ws = torch.zeros(16, dtype=torch.uint8, device="cuda")
    if prologue == 0:
        lib.check(lib.c.pb200_quantize_act(O.Q4_K, ptr(ad), K, ptr(ws), None), "quantize_act")
    mats = (GemvMat * len(ms))(*[m.mat() for m in ms])
    lib.check(_fused(lib)(len(ms), mats, K, ws.data_ptr(), prologue, ad.data_ptr(), bd.data_ptr(), eps, sync_ws.data_ptr(), 1, None),
              f"gemv_fused {what}")
    _no_abort(lib, what)
    if prologue:
        assert np.array_equal(act_ws_fields(ws, K, "q8_K"), port.quantize_act(O.Q4_K, x)), f"{what}: act_ws differs from the oracle's q8_K"
    for i, m in enumerate(ms):
        m.check(port, x, f"{what} matrix {i}")


def run_blk32(lib, port, ms, K, prologue, eps=1e-5, seed=0, what=""):
    """32-element block type matrices, which pb200_gemv_fused does not take: the q8_0 / q8_1 producer of the prologue's f32 output, then
    one mat-vec per matrix (+ its residual).  A 32-element ffn_down comes from n_ff % 256 != 0 (Qwen2.5-72B: Q5_0 / Q8_0 in Q4_K_M,
    Q5_1 / Q8_0 in Q5_K_M); Q4_0 models have them everywhere but the head."""
    _, _, x = _prologue_input(lib, port, prologue, K, eps, seed)
    xd = dev_f32(x)
    ws = act_ws(lib, K)
    for i, m in enumerate(ms):
        lib.check(lib.c.pb200_quantize_act(m.t, ptr(xd), K, ptr(ws), None), "quantize_act")
        lib.check(lib.c.pb200_mul_mat_vec_q(m.t, ptr(m.W), m.N, K, ptr(ws), ptr(m.y), None, ptr(m.add) if m.add is not None else None, None),
                  "mul_mat_vec_q")
        _no_abort(lib, what)
        mode = "q8_1" if m.t in (O.Q5_1, L.Q4_1) else "q8_0"
        assert np.array_equal(act_ws_fields(ws, K, mode), oracle_quantize_act(port, m.t, x)), f"{what} matrix {i}: act_ws differs"
        m.check(port, x, f"{what} matrix {i}")


# ---- a. the launches of one decode step of each served model (engine.cu enqueue_step), at their real shapes ----
MODELS = {   # bench.py's hyper-parameters; default weight type of the mixture (Q4_K_M / Q5_K_M)
    "llama3-8b": dict(E=4096, QD=4096, EK=1024, F=14336, V=128256, t=O.Q4_K, eps=1e-5, qwen=False),
    "llama3-70b": dict(E=8192, QD=8192, EK=1024, F=28672, V=128256, t=O.Q4_K, eps=1e-5, qwen=False),
    "qwen2.5-72b": dict(E=8192, QD=8192, EK=1024, F=29568, V=152064, t=O.Q5_K, eps=1e-6, qwen=True),
    "llama3-8b-q4_0": dict(E=4096, QD=4096, EK=1024, F=14336, V=128256, t=L.Q4_0, eps=1e-5, qwen=False),
    "qwen2.5-72b-q4_K_M": dict(E=8192, QD=8192, EK=1024, F=29568, V=152064, t=O.Q4_K, eps=1e-6, qwen=True),
}
LAUNCHES = ["qkv-v_q5_K", "qkv-v_q6_K", "wo", "gate_up", "down-default", "down-q6_K", "head"]
# the Q4_0 mixture: every matrix Q4_0 but the Q6_K head, and with an imatrix Q4_1 ffn_down layers
Q4_0_LAUNCHES = ["qkv", "wo", "gate_up", "down-default", "down-q4_1", "head"]
# Qwen2.5-72B Q4_K_M adds only its 32-element ffn_down (Q5_0, and Q8_0 in the use_more_bits layers) to the k-quant launches above
MODEL_LAUNCH_LISTS = {"llama3-8b-q4_0": Q4_0_LAUNCHES, "qwen2.5-72b-q4_K_M": ["down-default", "down-q6_K"]}
MODEL_LAUNCHES = [(m, la) for m in MODELS for la in MODEL_LAUNCH_LISTS.get(m, LAUNCHES)]
ALL_LAUNCHES = LAUNCHES + ["qkv", "down-q4_1"]


@pytest.mark.gpu
@pytest.mark.parametrize("model,launch", MODEL_LAUNCHES, ids=[f"{m}-{la}" for m, la in MODEL_LAUNCHES])
def test_model_launch_vs_oracle(cuda, lib, port, model, launch):
    h = MODELS[model]
    E, t, eps, seed = h["E"], h["t"], h["eps"], 1000 * list(MODELS).index(model) + 10 * ALL_LAUNCHES.index(launch)
    what = f"{model} {launch}"
    if t == L.Q4_0 and launch != "head":
        K, ms, pro = {"qkv": (E, [(t, h["QD"]), (t, h["EK"]), (t, h["EK"])], 1), "wo": (h["QD"], [(t, E)], 0), "gate_up": (E, [(t, h["F"])] * 2, 1),
                      "down-default": (h["F"], [(t, E)], 2), "down-q4_1": (h["F"], [(L.Q4_1, E)], 2)}[launch]
        run_blk32(lib, port, [Scattered(tt, n, K, seed + i, with_add=pro != 1) for i, (tt, n) in enumerate(ms)], K, pro, eps, seed, what)
    elif launch.startswith("qkv"):
        tv = O.Q5_K if launch.endswith("q5_K") else O.Q6_K
        ms = [Scattered(tt, n, E, seed + i, with_add=h["qwen"]) for i, (tt, n) in enumerate(((t, h["QD"]), (t, h["EK"]), (tv, h["EK"])))]
        run_fused(lib, port, ms, E, 1, eps, seed, what)          # Qwen2's q / k / v biases ride in the epilogue
    elif launch == "wo":
        run_fused(lib, port, [Scattered(t, E, h["QD"], seed, with_add=True)], h["QD"], 0, eps, seed, what)
    elif launch == "gate_up":
        run_fused(lib, port, [Scattered(t, h["F"], E, seed + i) for i in range(2)], E, 1, eps, seed, what)
    elif launch.startswith("down"):
        td = O.Q6_K if launch.endswith("q6_K") else t
        if h["F"] % 256:
            td = {O.Q4_K: L.Q5_0, O.Q5_K: O.Q5_1, O.Q6_K: O.Q8_0}[td]   # the mixture's fallback types for n_ff % 256 != 0
            run_blk32(lib, port, [Scattered(td, E, h["F"], seed, with_add=True)], h["F"], 2, seed=seed, what=f"{what} ({TN[td]})")
        else:
            run_fused(lib, port, [Scattered(td, E, h["F"], seed, with_add=True)], h["F"], 2, eps, seed, what)
    else:
        run_fused(lib, port, [Scattered(O.Q6_K, h["V"], E, seed)], E, 1, eps, seed, what)   # the whole vocabulary


# ---- b. plan sweep ----
@pytest.mark.gpu
@pytest.mark.parametrize("case", SWEEP, ids=sweep_id)
def test_plan_sweep_vs_oracle(cuda, lib, port, case):
    types, K, Ns = case
    p = gemv_plan(types, Ns, K)
    assert ring_turns(p, lib.c.pb200_sm_count()) >= 3
    ms = [Scattered(t, n, K, seed=K + 7 * i + t) for i, (t, n) in enumerate(zip(types, Ns))]
    x = np.random.default_rng(K).standard_normal(K).astype(np.float32)
    ws = act_ws(lib, K)
    lib.check(lib.c.pb200_quantize_act(types[0], ptr(dev_f32(x)), K, ptr(ws), None), "quantize_act")
    def launch():
        if len(ms) == 1:
            m = ms[0]
            lib.check(lib.c.pb200_mul_mat_vec_q(m.t, ptr(m.W), m.N, K, ptr(ws), ptr(m.y), None, None, None), "mul_mat_vec_q")
        else:
            mats = (GemvMat * len(ms))(*[m.mat() for m in ms])
            lib.check(_fused(lib)(len(ms), mats, K, ws.data_ptr(), 0, None, None, 0.0, None, 1, None), "gemv_fused")

    n0 = lib.c.pb200_kernel_launches()
    launch()
    _no_abort(lib, sweep_id(case))
    assert lib.c.pb200_kernel_launches() - n0 == 1
    for i, m in enumerate(ms):
        m.check(port, x, f"{sweep_id(case)} matrix {i}")
    # the launch above ran the ring kernel on the grid the plan implies: its instrumented instantiation stamps one trace entry per CTA
    # (k_gemv_generic stamps nothing)
    trace = torch.zeros(4096, dtype=torch.int64, device="cuda")
    lib.c.pb200_debug_set_trace.argtypes = [C.c_void_p, C.c_int]
    lib.check(lib.c.pb200_debug_set_trace(trace.data_ptr(), 1), "trace")
    try:
        launch()
        _no_abort(lib, sweep_id(case) + " (traced)")
    finally:
        lib.c.pb200_debug_set_trace(None, 0)
    ctas = int((trace.view(512, 8)[:, 0] != 0).sum())
    assert ctas == min(p.ntiles, CTAS_PER_SM * lib.c.pb200_sm_count()), (ctas, p.ntiles)


# ---- c. tiny grids: only ntiles CTAs, so dist_prologue's loop over several super-blocks per warp and a grid barrier of 1-3 CTAs ----
@pytest.mark.gpu
@pytest.mark.parametrize("prologue", [1, 2], ids=["rms_norm", "silu_mul"])
@pytest.mark.parametrize("K", [8192, 28672])
@pytest.mark.parametrize("N", [1, 2, 3])
def test_tiny_grid_prologue_vs_oracle(cuda, lib, port, N, K, prologue):
    t = O.Q4_K if K == 8192 else O.Q6_K
    run_fused(lib, port, [Scattered(t, N, K, seed=N + K)], K, prologue, seed=N, what=f"N {N} K {K}")


@pytest.mark.gpu
def test_tiny_qkv_group_single_row_last_matrix(cuda, lib, port):
    ms = [Scattered(t, n, 8192, seed=40 + i) for i, (t, n) in enumerate(((O.Q4_K, 16), (O.Q4_K, 8), (O.Q6_K, 1)))]
    assert gemv_plan([m.t for m in ms], [m.N for m in ms], 8192).ntiles <= 8
    run_fused(lib, port, ms, 8192, 1, what="q|k|v 16/8/1")


# ---- d. one Llama-3-70B layer chained on one stream ----
@pytest.mark.gpu
def test_layer_chain_pdl_vs_oracle(cuda, lib, port):
    """The engine's order on one stream, every GEMV launch with PDL and one shared barrier word block, one synchronisation at the end:
    q|k|v (rms_norm) -> q8_K of a fixed attention vector -> wo (+ residual) -> gate|up (rms_norm of wo's output) -> ffn_down (silu * mul,
    + residual) -> the next layer's q|k|v (rms_norm of ffn_down's output).  Intermediate buffers start as NaN; each launch is checked
    against the oracle on the device's own copy of its input, so a launch that read its input before griddepcontrol.wait fails."""
    E, EK, F, eps = 8192, 1024, 28672, 1e-5
    fn = _fused(lib)
    rng = np.random.default_rng(70)
    x0 = rng.standard_normal(E).astype(np.float32)
    att = rng.standard_normal(E).astype(np.float32)
    n_attn, n_attn2, n_ffn = [(1.0 + 0.1 * rng.standard_normal(E)).astype(np.float32) for _ in range(3)]
    x0d, attd, n_attn_d, n_attn2_d, n_ffn_d = map(dev_f32, (x0, att, n_attn, n_attn2, n_ffn))
    qkv = [Scattered(t, n, E, seed=700 + i) for i, (t, n) in enumerate(((O.Q4_K, E), (O.Q4_K, EK), (O.Q6_K, EK)))]
    qkv2 = [Scattered(t, n, E, seed=700 + i) for i, (t, n) in enumerate(((O.Q4_K, E), (O.Q4_K, EK), (O.Q6_K, EK)))]
    wo = Scattered(O.Q4_K, E, E, seed=710)
    gate, up = Scattered(O.Q4_K, F, E, seed=720), Scattered(O.Q4_K, F, E, seed=721)
    down = Scattered(O.Q6_K, E, F, seed=730)
    actE, actQD, actF = act_ws(lib, E), act_ws(lib, E), act_ws(lib, F)
    sync_ws = torch.zeros(16, dtype=torch.uint8, device="cuda")
    wo_m, down_m = wo.mat(), down.mat()
    wo_m.add, down_m.add = x0d.data_ptr(), wo.y.data_ptr()       # residuals: the layer input, then ffn_inp
    sync()

    def launch(ms, K, act, prologue, in0, in1, what):
        mats = (GemvMat * len(ms))(*ms)
        lib.check(fn(len(ms), mats, K, act.data_ptr(), prologue, in0.data_ptr() if in0 is not None else None,
                     in1.data_ptr() if in1 is not None else None, eps, sync_ws.data_ptr(), 1, None), what)

    launch([m.mat() for m in qkv], E, actE, 1, x0d, n_attn_d, "qkv")
    lib.check(lib.c.pb200_quantize_act(O.Q4_K, ptr(attd), E, ptr(actQD), None), "quantize_act att")
    launch([wo_m], E, actQD, 0, None, None, "wo")
    launch([gate.mat(), up.mat()], E, actE, 1, wo.y, n_ffn_d, "gate|up")
    launch([down_m], F, actF, 2, gate.y, up.y, "down")
    launch([m.mat() for m in qkv2], E, actE, 1, down.y, n_attn2_d, "next qkv")
    _no_abort(lib, "layer chain")

    for i, m in enumerate(qkv):
        m.check(port, port.rms_norm(x0, eps) * n_attn, f"qkv matrix {i}")
    wo.check(port, att, "wo", add_rows=x0)
    x1 = wo.y.cpu().numpy()
    for m, name in ((gate, "gate"), (up, "up")):
        m.check(port, port.rms_norm(x1, eps) * n_ffn, name)
    down.check(port, _silu_mul(lib, port, gate.y, up.y), "down", add_rows=x1)
    x2 = down.y.cpu().numpy()
    for i, m in enumerate(qkv2):
        m.check(port, port.rms_norm(x2, eps) * n_attn2, f"next qkv matrix {i}")


# ---- e. the fused launch's K limit ----
@pytest.mark.gpu
def test_gemv_fused_k_limit(cuda, lib, port):
    """pb200_gemv_fused takes K up to 29 696 (116 super-blocks of activation in shared memory) and refuses 29 952 with PB200_ENOTSUP."""
    m = Scattered(O.Q4_K, 64, 29952, seed=3)
    ws = act_ws(lib, 29952)
    a = dev_f32(np.ones(29952, np.float32))
    mats = (GemvMat * 1)(m.mat())
    assert _fused(lib)(1, mats, 29952, ws.data_ptr(), 1, a.data_ptr(), a.data_ptr(), 1e-5, None, 0, None) == ENOTSUP
    for prologue in (1, 2):
        run_fused(lib, port, [Scattered(O.Q4_K, 300, 29696, seed=prologue)], 29696, prologue, seed=prologue, what=f"K 29696 prologue {prologue}")
