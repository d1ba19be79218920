// prima.cpp_b200/csrc/gemv.cuh — decode GEMV  y[N] = W[N,K] (GGUF k-quant blocks) . x[K]
//
// Replaces: ggml_cuda_mul_mat -> ggml_cuda_op_mul_mat_vec_q -> mul_mat_vec_q<type,1>
//           (ggml/src/ggml-cuda.cu:1883-1948, ggml-cuda/mmvq.cu:55-202, vecdotq.cuh:357-787).
// Numerics follow the CPU oracle instead (ggml_vec_dot_q{4,5,6}_K_q8_K, ggml-quants.c:7713-9566): the activation
// is q8_K, every integer sub-result is exact, only the order of the final fp32 adds differs.
//
// Design (memory-bound, no tensor cores):
//   * persistent grid of TWO 256-thread CTAs per SM (<= 113 KB of shared memory and 128 registers each).  Two CTAs per SM is
//     what lets consecutive kernels of the token overlap under programmatic dependent launch: when a CTA of launch A exits,
//     a CTA of launch B becomes resident on that SM and streams its first weight tiles (they never depend on A) while the
//     rest of A drains; a small kernel between two GEMVs (attention, silu-quant) runs while the next GEMV's rings fill.
//     a single 512-thread CTA per SM owning all of shared memory serialises every launch boundary instead (the next launch
//     cannot become resident before the previous one has left);
//   * row tiles of raw blocks stream HBM -> shared memory with cp.async.bulk (1-D TMA, SASS UBLKCP) into an nstage-deep ring
//     (4-8 stages of ~16-24 KB chosen per launch; ~185 KB in flight per SM).  There is no producer warp: the consumer warp
//     that finishes a stage last re-arms its mbarrier and issues the refill itself;
//   * 8 consumer warps; ONE LANE OWNS ONE SUPER-BLOCK COLUMN: lane l of sub-warp s keeps the 256 int8 activations of
//     super-block (32 s + l) plus its bsums and scale in registers for the whole kernel, so shared memory is read
//     exactly once per weight byte (128-bit LDS, conflict-free at 144/176-B strides) and the activation costs no
//     bandwidth at all after the prologue;
//   * rows of a stage are dealt to the warp groups round-robin ACROSS stages (row j of the CTA's sequence -> group j mod
//     ngroups), so any number of rows per stage keeps all warps busy and several stages are consumed concurrently;
//   * per row: integer dp4a/dp2a dot, one fp32 scale, a 5-step shuffle reduction; rows longer than 32 super-blocks
//     are split over 2/4 warps and combined through a few floats of shared memory in a fixed order
//     (deterministic, no atomics);
//   * several matrices that share one activation (q|k|v, gate|up) run as ONE launch (tile list over matrices).
#pragma once
#include "common.cuh"

namespace pb {

constexpr int GEMV_NW = 8;                        // consumer warps per CTA
constexpr int GEMV_THREADS = GEMV_NW * 32;
constexpr int GEMV_CTAS_PER_SM = 2;
constexpr int GEMV_MAX_STAGE = 8;
constexpr int GEMV_SMEM_LIMIT = 113 * 1024;       // 2 x (113 KB + 1 KB reserved per CTA) = the 228 KB of an SM
constexpr int GEMV_STAGE_TARGET = 28 * 1024;      // bytes per ring stage aimed for (rows per stage = target / row bytes)
constexpr int GEMV_ACT_MAX_NBLK = 116;            // K <= 29 696 on the fast path (Qwen2.5-72B's n_ff = 29 568)
constexpr int GEMV_MAX_MAT = 3;
__host__ __device__ inline int gemv_act_smem_bytes(int nblk) { return nblk * (ACT_SMEM_QS_STRIDE + 64) + 64; }   // padded qs | padded bsums + d (k-quants: 52 B per column) or d8 | s8 (32-element block types: 64 B)

struct GemvMat {
    const uint8_t * W;     // raw GGUF blocks, row-major [N][K/256 blocks]
    float * y;             // [N]
    const float * bias;    // optional [N]  (y = Wx + bias)                      -- Qwen2 q/k/v biases
    const float * resid;   // optional [N]  (y = Wx (+bias) + resid)             -- residual adds of the layer
    int64_t row_bytes;
    int64_t total_bytes;   // N * row_bytes
    int type;              // T_Q4_K / T_Q5_K / T_Q6_K
    int N;
    int rows_per_tile;
    int tile0;             // index of this matrix' first tile in the launch-wide tile list
};

// Prologue: how the launch gets its q8_K activation.
//   PRO_NONE          already quantized in HBM (`act`): one coalesced copy per CTA into shared memory, then registers
//   PRO_RMSNORM_DIST  act = q8_K( rms_norm(in0) * in1 )     llm_build_norm + quantize_row_q8_K   (in1 = norm weight)
//   PRO_SILU_DIST     act = q8_K( silu(in0) * in1 )         llm_build_ffn LLM_FFN_SILU / LLM_FFN_PAR -> ffn_down
//   Distributed: CTA c quantizes super-block c into `act` (HBM/L2), ONE grid barrier (all CTAs of the persistent grid are
//   co-resident), then every CTA stages the finished vector like PRO_NONE.  No tiny kernel + launch boundary in front of the GEMV,
//   and each CTA quantizes one super-block instead of every CTA recomputing the whole vector from L2.
enum : int { PRO_NONE = 0, PRO_RMSNORM_DIST = 4, PRO_SILU_DIST = 5 };

struct GemvParams {
    GemvMat mat[GEMV_MAX_MAT];
    int nmat;
    int ntiles;
    int K;
    int nblk;          // K / 256
    int wpr;           // warps per row: 1, 2 or 4
    int nblk_p2;       // lanes per row: nblk rounded up to a power of two, at most 32.  Short rows (K <= 4096) put 32 / nblk_p2 rows in one warp
    int nstage;        // ring depth of this launch
    int nstage_init;   // stages [nstage_init, nstage) overlay the activation staging area: they join the ring once the activation is in registers
    int rel_count;     // warps that hand a stage back before it is refilled: all 8, or only its owners (owner_only)
    int owner_only;    // a stage is always consumed by the same warps: the others skip it entirely (no wait, no release)
    int prefill;       // stages requested before griddepcontrol.wait; the other initial stages follow once the activation loads are out
    int stage_bytes;   // bytes reserved per stage (multiple of 128)
    ActQ act;          // q8_K activation (PRO_NONE)
    int prologue;
    const float * in0;
    const float * in1;
    float eps;
    unsigned int * gbar;           // distributed prologues: {arrivals, departures} of the grid barrier (self-resetting)
    int * abort_flag;              // host-mapped: set by the wait watchdog (never on a healthy run)
    unsigned long long * trace;    // per-CTA %globaltimer stamps (TRACE instantiation only)
};

// ---------------------------------------------------------------------------------------------------------------
// per-lane register-resident activation super-block
struct ActRegs {
    int a[64];      // 256 int8
    int bs[8];      // 16 x int16 bsums (pairs)
    int bs32[4];    // 8 x int16: bsums per 32 (pairs)
    float d;        // q8_K scale (0 for an out-of-range block => contributes nothing)
    // 32-element block weight types (Q8_0 / Q5_1): the column = 8 consecutive blocks, activation q8_0 / q8_1 with one scale (and one
    // d * sum) per block; nb = how many of the 8 blocks exist (the last column of a K % 256 != 0 row is short)
    float d8[8], s8[8];
    int nb;
};

__device__ __forceinline__ void load_act_regs(ActRegs & r, const ActQ & act, int blk, bool valid) {
    if (valid) {
        const int4 * q = reinterpret_cast<const int4 *>(act.qs + (int64_t) blk * act_qs_stride(act));
#pragma unroll
        for (int i = 0; i < 16; i++) {
            int4 v = q[i];
            r.a[4 * i + 0] = v.x; r.a[4 * i + 1] = v.y; r.a[4 * i + 2] = v.z; r.a[4 * i + 3] = v.w;
        }
        const int4 * b = reinterpret_cast<const int4 *>(act.bsums + (int64_t) blk * act_bs_stride(act));
        int4 b0 = b[0], b1 = b[1];
        r.bs[0] = b0.x; r.bs[1] = b0.y; r.bs[2] = b0.z; r.bs[3] = b0.w;
        r.bs[4] = b1.x; r.bs[5] = b1.y; r.bs[6] = b1.z; r.bs[7] = b1.w;
        r.d = act.d[blk];
    } else {
#pragma unroll
        for (int i = 0; i < 64; i++) r.a[i] = 0;
#pragma unroll
        for (int i = 0; i < 8; i++) r.bs[i] = 0;
        r.d = 0.f;
    }
}
// second half of load_act_regs, kept separate so that callers can put work between issuing the loads and using them
__device__ __forceinline__ void finish_act_regs(ActRegs & r) {
#pragma unroll
    for (int k = 0; k < 4; k++) {
        // per-32 sums: (bs16[4k]+bs16[4k+1], bs16[4k+2]+bs16[4k+3]) packed as int16x2
        int lo = (int)(short)(r.bs[2 * k] & 0xffff) + (r.bs[2 * k] >> 16);
        int hi = (int)(short)(r.bs[2 * k + 1] & 0xffff) + (r.bs[2 * k + 1] >> 16);
        r.bs32[k] = (lo & 0xffff) | (hi << 16);
    }
}

// scales/mins of a Q4_K/Q5_K super-block as packed bytes (get_scale_min_k4, ggml-quants.c:1898-1905)
__device__ __forceinline__ void unpack_scales_k4(uint32_t u0, uint32_t u1, uint32_t u2, uint32_t & sc_lo, uint32_t & sc_hi,
                                                 uint32_t & m_lo, uint32_t & m_hi) {
    sc_lo = u0 & 0x3f3f3f3fu;
    m_lo = u1 & 0x3f3f3f3fu;
    sc_hi = (u2 & 0x0f0f0f0fu) | (((u0 >> 6) & 0x03030303u) << 4);
    m_hi = ((u2 >> 4) & 0x0f0f0f0fu) | (((u1 >> 6) & 0x03030303u) << 4);
}
__device__ __forceinline__ int ubyte(uint32_t w, int i) { return (int) ((w >> (8 * i)) & 0xffu); }

// One Q4_K super-block (144 B, 16-B aligned in shared memory) against the lane's activation registers.
__device__ __forceinline__ float dot_q4K(const uint8_t * blk, const ActRegs & r) {
    const uint4 * p = reinterpret_cast<const uint4 *>(blk);
    const uint4 h = p[0];
    const __half2 dm = *reinterpret_cast<const __half2 *>(&h.x);
    uint32_t sc_lo, sc_hi, m_lo, m_hi;
    unpack_scales_k4(h.y, h.z, h.w, sc_lo, sc_hi, m_lo, m_hi);
    int sumi = 0;
#pragma unroll
    for (int c = 0; c < 4; c++) {
        const uint4 q0 = p[1 + 2 * c], q1 = p[2 + 2 * c];
        const uint32_t w[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
        // four dependency chains of 4 dp4a per chunk instead of two of 8 (integer sums: the regrouping is exact).  With 4 warps per
        // scheduler the kernel is bound by dependent-issue latency (~7 cycles between two instructions of a warp, 50-60 % issue slots used),
        // so instruction-level parallelism inside the dot is what the streaming rate of the issue-bound launches follows.
        int dlo0 = 0, dlo1 = 0, dhi0 = 0, dhi1 = 0;
#pragma unroll
        for (int i = 0; i < 8; i += 2) {
            dlo0 = dp4a_us(w[i] & 0x0f0f0f0fu, r.a[16 * c + i], dlo0);
            dlo1 = dp4a_us(w[i + 1] & 0x0f0f0f0fu, r.a[16 * c + i + 1], dlo1);
            dhi0 = dp4a_us(w[i] & 0xf0f0f0f0u, r.a[16 * c + 8 + i], dhi0);   // 16 x the high-nibble dot (exact)
            dhi1 = dp4a_us(w[i + 1] & 0xf0f0f0f0u, r.a[16 * c + 8 + i + 1], dhi1);
        }
        const int dlo = dlo0 + dlo1, dhi = dhi0 + dhi1;
        const uint32_t scw = c < 2 ? sc_lo : sc_hi;
        sumi += ubyte(scw, (2 * c) & 3) * dlo + ubyte(scw, (2 * c + 1) & 3) * (dhi >> 4);
    }
    int summ = dp2a_lo_su(r.bs32[0], m_lo, 0);
    summ = dp2a_hi_su(r.bs32[1], m_lo, summ);
    summ = dp2a_lo_su(r.bs32[2], m_hi, summ);
    summ = dp2a_hi_su(r.bs32[3], m_hi, summ);
    const float d = __low2float(dm) * r.d, dmin = __high2float(dm) * r.d;
    return d * (float) sumi - dmin * (float) summ;
}

// One Q5_K super-block (176 B, 16-B aligned): nibble dot + 16 x fifth-bit dot.
__device__ __forceinline__ float dot_q5K(const uint8_t * blk, const ActRegs & r) {
    const uint4 * p = reinterpret_cast<const uint4 *>(blk);
    const uint4 h = p[0];
    const __half2 dm = *reinterpret_cast<const __half2 *>(&h.x);
    uint32_t sc_lo, sc_hi, m_lo, m_hi;
    unpack_scales_k4(h.y, h.z, h.w, sc_lo, sc_hi, m_lo, m_hi);
    const uint4 h0 = p[1], h1 = p[2];
    const uint32_t qh[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
    int sumi = 0;
#pragma unroll
    for (int c = 0; c < 4; c++) {
        const uint4 q0 = p[3 + 2 * c], q1 = p[4 + 2 * c];
        const uint32_t w[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
        int dlo = 0, dhi = 0, blo = 0, bhi = 0;
#pragma unroll
        for (int i = 0; i < 8; i++) {
            dlo = dp4a_us(w[i] & 0x0f0f0f0fu, r.a[16 * c + i], dlo);
            dhi = dp4a_us(w[i] & 0xf0f0f0f0u, r.a[16 * c + 8 + i], dhi);
            blo = dp4a_us((qh[i] >> (2 * c)) & 0x01010101u, r.a[16 * c + i], blo);
            bhi = dp4a_us((qh[i] >> (2 * c + 1)) & 0x01010101u, r.a[16 * c + 8 + i], bhi);
        }
        const uint32_t scw = c < 2 ? sc_lo : sc_hi;
        sumi += ubyte(scw, (2 * c) & 3) * (dlo + 16 * blo) + ubyte(scw, (2 * c + 1) & 3) * ((dhi >> 4) + 16 * bhi);
    }
    int summ = dp2a_lo_su(r.bs32[0], m_lo, 0);
    summ = dp2a_hi_su(r.bs32[1], m_lo, summ);
    summ = dp2a_lo_su(r.bs32[2], m_hi, summ);
    summ = dp2a_hi_su(r.bs32[3], m_hi, summ);
    const float d = __low2float(dm) * r.d, dmin = __high2float(dm) * r.d;
    return d * (float) sumi - dmin * (float) summ;
}

// One Q6_K super-block (210 B, only 2-B aligned): aligned 32-bit loads + funnel shift by the misalignment.
__device__ __forceinline__ float dot_q6K(const uint8_t * blk, const ActRegs & r) {
    const uint32_t addr = smem_u32(blk);
    const uint32_t sh = (addr & 3u) * 8u;
    const uint32_t * base = reinterpret_cast<const uint32_t *>(blk - (addr & 3u));
    // scales (bytes 192..207) and d (bytes 208..209)
    uint32_t tail[6];
#pragma unroll
    for (int i = 0; i < 6; i++) tail[i] = base[48 + i];
    int scw[4];
#pragma unroll
    for (int i = 0; i < 4; i++) scw[i] = (int) __funnelshift_r(tail[i], tail[i + 1], sh);
    const uint32_t dword = __funnelshift_r(tail[4], tail[5], sh);
    const float dw = __half2float(__ushort_as_half((unsigned short) (dword & 0xffffu)));

    int sumi = 0;
#pragma unroll
    for (int n = 0; n < 2; n++) {
        uint32_t ql[17], qh[9];
#pragma unroll
        for (int i = 0; i < 17; i++) ql[i] = base[16 * n + i];
#pragma unroll
        for (int i = 0; i < 9; i++) qh[i] = base[32 + 8 * n + i];
        int acc[8];
#pragma unroll
        for (int j = 0; j < 8; j++) acc[j] = 0;
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const uint32_t A = __funnelshift_r(ql[i], ql[i + 1], sh);
            const uint32_t B = __funnelshift_r(ql[8 + i], ql[9 + i], sh);
            const uint32_t H = __funnelshift_r(qh[i], qh[i + 1], sh);
            const uint32_t v1 = (A & 0x0f0f0f0fu) | ((H << 4) & 0x30303030u);
            const uint32_t v2 = (B & 0x0f0f0f0fu) | ((H << 2) & 0x30303030u);
            const uint32_t v3 = ((A >> 4) & 0x0f0f0f0fu) | (H & 0x30303030u);
            const uint32_t v4 = ((B >> 4) & 0x0f0f0f0fu) | ((H >> 2) & 0x30303030u);
            const int g = i >> 2;   // which 16-element half of the 32-element run
            acc[0 + g] = dp4a_us(v1, r.a[32 * n + i], acc[0 + g]);
            acc[2 + g] = dp4a_us(v2, r.a[32 * n + 8 + i], acc[2 + g]);
            acc[4 + g] = dp4a_us(v3, r.a[32 * n + 16 + i], acc[4 + g]);
            acc[6 + g] = dp4a_us(v4, r.a[32 * n + 24 + i], acc[6 + g]);
        }
        // scales 8n .. 8n+7 are the signed bytes of scw[2n], scw[2n+1]
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const int s = (int) (signed char) ((scw[2 * n + (j >> 2)] >> (8 * (j & 3))) & 0xff);
            sumi += s * acc[j];
        }
    }
    // - 32 * sum_j scale_j * bsum16_j   (q6 = u6 - 32)
    int sb = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) {
        sb = (k & 1) ? dp2a_hi_ss(r.bs[k], scw[k >> 1], sb) : dp2a_lo_ss(r.bs[k], scw[k >> 1], sb);
    }
    return (dw * r.d) * (float) (sumi - 32 * sb);
}

// ---- 32-element block types on the same ring: a lane's column is 8 consecutive blocks (272 B of Q8_0, 192 B of Q5_1) ----
// Follows ggml_vec_dot_q8_0_q8_0 (ggml-quants.c:5518) and ggml_vec_dot_q5_1_q8_1 (:5144) block by block, like k_gemv_generic: the integer
// block sums are exact, the per-block fp32 scale products and the running fp32 sum are formed in the same order.
// Q8_0: rows are 8-byte aligned in the stage (row bytes = 34 * K/32; 31 416 for K = 29 568), so a column is read with 64-bit loads and
// the 2-byte phase of every block inside it is a compile-time constant (even blocks start on a word, odd ones in its upper half).
__device__ __forceinline__ float dot_q8_0x8(const uint8_t * col, const ActRegs & r) {
    const uint2 * c2 = reinterpret_cast<const uint2 *>(col);
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 8; j++) {
        if (j < r.nb) {
            const int wj = (34 * j) >> 2;            // first 32-bit word of the block inside the column
            const bool odd = (j & 1) != 0;           // block starts 2 bytes into that word
            uint32_t w[10];
#pragma unroll
            for (int i = 0; i < 5; i++) { const uint2 t = c2[(wj >> 1) + i]; w[2 * i] = t.x; w[2 * i + 1] = t.y; }
            const int o = wj & 1;
            const float d = __half2float(__ushort_as_half((unsigned short) (odd ? (w[o] >> 16) : (w[o] & 0xffffu))));
            int sumi = 0;
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const uint32_t q = odd ? w[o + 1 + i] : __byte_perm(w[o + i], w[o + i + 1], 0x5432);
                sumi = dp4a_ss((int) q, r.a[8 * j + i], sumi);
            }
            acc += (float) sumi * (d * r.d8[j]);
        }
    }
    return acc;
}
// Q5_1: 24-byte blocks [d f16][m f16][qh u32][16 x 2 nibbles]; rows are 16-byte aligned when K % 64 == 0, 8-byte otherwise.
__device__ __forceinline__ float dot_q5_1x8(const uint8_t * col, const ActRegs & r) {
    const uint2 * c2 = reinterpret_cast<const uint2 *>(col);
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 8; j++) {
        if (j < r.nb) {
            const uint2 hd = c2[3 * j], qa = c2[3 * j + 1], qb = c2[3 * j + 2];
            const float d = __half2float(__ushort_as_half((unsigned short) (hd.x & 0xffffu)));
            const float mm = __half2float(__ushort_as_half((unsigned short) (hd.x >> 16)));
            const uint32_t qh = hd.y;
            const uint32_t w[4] = {qa.x, qa.y, qb.x, qb.y};
            // sum (nibble + 16 * bit) * a  =  sum nibble * a  +  16 * sum bit * a: the fifth bits get their own dp4a instead of being merged into
            // the nibble bytes (13 instead of 18 instructions per 8 elements; integer sums, exact).  bit k of a nibble of qh -> bit 0 of byte k:
            // x * 0x00204081 puts bit k at 8k (no carries)
            int sumi = 0, sumb = 0;
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const uint32_t hb_lo = (((qh >> (4 * i)) & 0xFu) * 0x00204081u) & 0x01010101u;
                const uint32_t hb_hi = (((qh >> (4 * i + 16)) & 0xFu) * 0x00204081u) & 0x01010101u;
                sumi = dp4a_us(w[i] & 0x0f0f0f0fu, r.a[8 * j + i], sumi);
                sumb = dp4a_us(hb_lo, r.a[8 * j + i], sumb);
                sumi = dp4a_us((w[i] >> 4) & 0x0f0f0f0fu, r.a[8 * j + 4 + i], sumi);
                sumb = dp4a_us(hb_hi, r.a[8 * j + 4 + i], sumb);
            }
            sumi += 16 * sumb;
            acc += (d * r.d8[j]) * (float) sumi + mm * r.s8[j];
        }
    }
    return acc;
}

}  // namespace pb
