// prima.cpp_b200/csrc/common.cuh — shared device helpers for the sm_90a quantized-decode kernels.
//
// Wire formats are the reference's GGUF block layouts, read byte-for-byte from HBM
// (ggml/src/ggml-common.h:173-204, 286-335).  Nothing here is copied from ggml-cuda: the kernels use a
// different decomposition (one lane per super-block with the int8 activation resident in registers,
// weights staged through shared memory by cp.async.bulk / TMA), and a different activation format
// (q8_K, the CPU backend's, so results match the CPU oracle to fp32 summation order).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace pb {

// enum ggml_type values (ggml/include/ggml.h:356-395)
enum : int { T_F32 = 0, T_F16 = 1, T_Q4_0 = 2, T_Q4_1 = 3, T_Q5_0 = 6, T_Q5_1 = 7, T_Q8_0 = 8, T_Q4_K = 12, T_Q5_K = 13, T_Q6_K = 14 };

constexpr int QK_K = 256;
constexpr int BYTES_Q4_K = 144, BYTES_Q5_K = 176, BYTES_Q6_K = 210, BYTES_Q8_0 = 34, BYTES_Q5_1 = 24;
constexpr int BYTES_Q4_0 = 18, BYTES_Q4_1 = 20, BYTES_Q5_0 = 22;   // ggml-common.h:143-170

__host__ __device__ inline int64_t row_bytes(int type, int64_t k) {
    switch (type) {
        case T_F32: return k * 4;
        case T_F16: return k * 2;
        case T_Q4_K: return k / 256 * BYTES_Q4_K;
        case T_Q5_K: return k / 256 * BYTES_Q5_K;
        case T_Q6_K: return k / 256 * BYTES_Q6_K;
        case T_Q8_0: return k / 32 * BYTES_Q8_0;
        case T_Q5_1: return k / 32 * BYTES_Q5_1;
        case T_Q4_0: return k / 32 * BYTES_Q4_0;
        case T_Q4_1: return k / 32 * BYTES_Q4_1;
        case T_Q5_0: return k / 32 * BYTES_Q5_0;
    }
    return -1;
}
__host__ __device__ inline bool is_kquant(int t) { return t == T_Q4_K || t == T_Q5_K || t == T_Q6_K; }
// the 32-element block types: one fp16 scale (and offset) per 32 weights
__host__ __device__ inline bool is_blk32_type(int t) { return t == T_Q8_0 || t == T_Q5_1 || t == T_Q4_0 || t == T_Q4_1 || t == T_Q5_0; }
__host__ __device__ inline bool is_quant_type(int t) { return is_kquant(t) || is_blk32_type(t); }   // the quantized weight types
__host__ __device__ inline int block_elems(int t) { return is_kquant(t) ? 256 : (is_blk32_type(t) ? 32 : 1); }

// ---------------------------------------------------------------------------------------------
// Quantized activation vector in HBM (SoA so that a lane can pull its super-block with 128-bit loads).
//   mode Q8_K (for Q4_K/Q5_K/Q6_K weights; mirrors block_q8_K, ggml-common.h:330-335):
//       qs[K] int8, d[K/256] f32, bsums[K/16] int16
//   mode Q8_0 (for Q8_0 / Q4_0 / Q5_0 weights; block_q8_0): qs[K], d[K/32] = fp16-rounded scale widened to f32
//   mode Q8_1 (for Q5_1 / Q4_1 weights; block_q8_1): qs[K], d[K/32], s[K/32] (both fp16-rounded, widened)
struct ActQ {
    int8_t * qs;      // [K]           16-B aligned
    float * d;        // [K/256] or [K/32]
    int16_t * bsums;  // [K/16]        (Q8_K only)
    float * s;        // [K/32]        (Q8_1 only)
    // per-super-block strides (Q8_K mode): 0 = dense (256 B of qs, 16 bsums).  The shared-memory copy inside the GEMV uses
    // 272 B / 24 int16 so that 32 lanes reading 32 different super-blocks with 128-bit loads hit 32 different bank groups
    // (dense 256-B strides are a 32-way bank conflict).
    int qs_stride;    // bytes
    int bs_stride;    // int16 elements
};
__host__ __device__ inline int act_qs_stride(const ActQ & a) { return a.qs_stride ? a.qs_stride : 256; }
__host__ __device__ inline int act_bs_stride(const ActQ & a) { return a.bs_stride ? a.bs_stride : 16; }
constexpr int ACT_SMEM_QS_STRIDE = 272, ACT_SMEM_BS_STRIDE = 24;
enum : int { ACT_Q8_K = 0, ACT_Q8_0 = 1, ACT_Q8_1 = 2 };
// the weight type's vec_dot_type on the CPU (ggml/src/ggml.c:785-850): the offset types Q4_1 / Q5_1 take q8_1, whose s = d * sum(q)
// pays for the offset term
__host__ __device__ inline int act_mode_for(int wtype) {
    return is_kquant(wtype) ? ACT_Q8_K : ((wtype == T_Q5_1 || wtype == T_Q4_1) ? ACT_Q8_1 : ACT_Q8_0);
}

// ---------------------------------------------------------------------------------------------
// small PTX wrappers
__device__ __forceinline__ int dp4a_us(uint32_t a_u8x4, int b_s8x4, int c) {   // unsigned bytes x signed bytes
    int d;
    asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a_u8x4), "r"(b_s8x4), "r"(c));
    return d;
}
__device__ __forceinline__ int dp4a_ss(int a, int b, int c) { return __dp4a(a, b, c); }
// dp2a: two signed 16-bit values of a times the low / high two unsigned bytes of b
__device__ __forceinline__ int dp2a_lo_su(int a_s16x2, uint32_t b_u8x4, int c) {
    int d;
    asm("dp2a.lo.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a_s16x2), "r"(b_u8x4), "r"(c));
    return d;
}
__device__ __forceinline__ int dp2a_hi_su(int a_s16x2, uint32_t b_u8x4, int c) {
    int d;
    asm("dp2a.hi.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a_s16x2), "r"(b_u8x4), "r"(c));
    return d;
}
__device__ __forceinline__ int dp2a_lo_ss(int a_s16x2, int b_s8x4, int c) {
    int d;
    asm("dp2a.lo.s32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a_s16x2), "r"(b_s8x4), "r"(c));
    return d;
}
__device__ __forceinline__ int dp2a_hi_ss(int a_s16x2, int b_s8x4, int c) {
    int d;
    asm("dp2a.hi.s32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a_s16x2), "r"(b_s8x4), "r"(c));
    return d;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// First-occurrence arg-max, the CPU backend's rule (its loops compare with a strict '>'): a larger key wins, an equal key keeps the
// smaller index.  Folds the candidate (okey, oidx) into (key, idx); the optional payload *val travels with the winner.  Every
// arg-max that must agree bit for bit with the CPU (the q8_K scale, greedy sampling) decides here.
__device__ __forceinline__ void argmax_combine(float & key, int & idx, float okey, int oidx, float * val = nullptr, float oval = 0.f) {
    if (okey > key || (okey == key && oidx < idx)) {
        key = okey;
        idx = oidx;
        if (val) *val = oval;
    }
}
// the same over a warp: every lane ends with the warp's winner
__device__ __forceinline__ void warp_argmax(float & key, int & idx, float * val = nullptr) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float okey = __shfl_xor_sync(0xffffffffu, key, o);
        const float oval = val ? __shfl_xor_sync(0xffffffffu, *val, o) : 0.f;
        const int oidx = __shfl_xor_sync(0xffffffffu, idx, o);
        argmax_combine(key, idx, okey, oidx, val, oval);
    }
}

__device__ __forceinline__ uint32_t smem_u32(const void * p) { return (uint32_t) __cvta_generic_to_shared(p); }

// ---- mbarrier + bulk async copy (TMA 1-D, SASS UBLKCP) ----
__device__ __forceinline__ void mbar_init(uint64_t * bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t * bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t * bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Bounded waits.  A wait that exceeds ~1 s of SM clocks (a logic error, never load: the longest legitimate wait is one HBM
// round trip) raises the CTA-wide `cta_abort` word and the process-wide host-mapped `abort_flag`, after which every wait of
// the CTA returns at once: the launch terminates quickly with invalid results and the host reports PB200_EABORTED for the
// call that synchronises on it (engine.cu / api.cu check and clear the flag).  Nothing hangs, nothing fails silently.
constexpr long long PB_WAIT_TIMEOUT_CYCLES = 1ll << 31;
__device__ __forceinline__ bool mbar_try_parity(uint64_t * bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ bool mbar_try_token(uint64_t * bar, uint64_t token) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "l"(token)
        : "memory");
    return ok != 0;
}
static __device__ __noinline__ void wait_gave_up(volatile int * cta_abort, int * abort_flag) {
    *cta_abort = 1;
    if (abort_flag) { *(volatile int *) abort_flag = 1; __threadfence_system(); }
}
__device__ __forceinline__ void mbar_wait(uint64_t * bar, uint32_t parity, volatile int * cta_abort, int * abort_flag) {
    if (mbar_try_parity(bar, parity)) return;       // the common case costs one try_wait (which itself suspends for a while)
    const long long t0 = clock64();
    int spins = 0;
    while (!mbar_try_parity(bar, parity)) {
        if ((++spins & 63) == 0) {
            if (*cta_abort) return;
            if (clock64() - t0 > PB_WAIT_TIMEOUT_CYCLES) { wait_gave_up(cta_abort, abort_flag); return; }
        }
    }
}
// token flavour: the arriving thread gets the phase token and can wait for that phase without tracking a parity bit
__device__ __forceinline__ uint64_t mbar_arrive_token(uint64_t * bar) {
    uint64_t st;
    asm volatile("mbarrier.arrive.shared::cta.b64 %0, [%1];" : "=l"(st) : "r"(smem_u32(bar)) : "memory");
    return st;
}
__device__ __forceinline__ void mbar_wait_token(uint64_t * bar, uint64_t token, volatile int * cta_abort, int * abort_flag) {
    if (mbar_try_token(bar, token)) return;
    const long long t0 = clock64();
    int spins = 0;
    while (!mbar_try_token(bar, token)) {
        if ((++spins & 63) == 0) {
            if (*cta_abort) return;
            if (clock64() - t0 > PB_WAIT_TIMEOUT_CYCLES) { wait_gave_up(cta_abort, abort_flag); return; }
        }
    }
}
// L2 eviction policy for streamed-once weights
__device__ __forceinline__ uint64_t policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ void bulk_g2s(void * smem_dst, const void * gsrc, uint32_t bytes, uint64_t * bar, uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
            smem_u32(smem_dst)),
        "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
        : "memory");
}

// fire-and-forget prefetch of a 16-B-granular global range into L2 (no destination, no barrier)
__device__ __forceinline__ void bulk_prefetch_l2(const void * gsrc, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gsrc), "r"(bytes) : "memory");
}

// Programmatic dependent launch: wait for the producer grid's results / let the dependent grid start.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

}  // namespace pb
