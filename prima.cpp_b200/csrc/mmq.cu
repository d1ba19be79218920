// prima.cpp_b200/csrc/mmq.cu — batched (prefill) k-quant mat-mul on the Hopper tensor cores (wgmma, sm_90a).
//
// Replaces: ggml_cuda_op_mul_mat_q -> mul_mat_q<type,mmq_x,8,chk> (ggml-cuda/mmq.cu:3-98, mmq.cuh:2583-2650: int8 mma.sync
// tiles with __syncthreads ping-pong) and quantize_mmq_q8_1_cuda (quantize.cu:143-169), SURVEY §8 row a-4.
// Numerics follow the CPU backend the oracle restates: every activation row is quantized to q8_K exactly as
// quantize_row_q8_K_ref does (ggml-quants.c:3785-3822) and the weights are expanded with the dequantize_row_q{4,5,6}_K
// formulas (ggml-quants.c:2040-2065, 2390-2420, 2690-2725) evaluated in fp16 (exact integer q, fp16 sub-block scale and
// offset, one fused multiply-add); both operands are fp16 on the tensor pipe with fp32 accumulation.  The result differs
// from the integer-dot CPU value by a few fp16 roundings per product (NMSE ~1e-6; tests/test_gpu_mmq.py states the bound).
// Operand range: each activation row is scaled by a power of two into [2^14, 2^15) before its fp16 rounding (k_mmq_prep) and the
// epilogue undoes it, so any finite f32 activation works; the weights' sub-block scales d*sc below 2^-14 remain fp16 subnormals.
//
//   dst[t][n] = sum_k W[n][k] * X[t][k]        W: N x K k-quant rows, X: T x K f32, dst: T x N f32 (ggml layout)
// Also the 32-element block types Q8_0 / Q5_1 / Q4_0 / Q4_1 / Q5_0 (K % 64 == 0; activations quantized per 32 values like their CPU dot):
// Qwen2.5-72B's ffn_down, whose K = 29 568 rules the k-quants out (src/llama.cpp:19516-19551), and the Q4_0 files.
//
// Work decomposition (stream-K, persistent).  A work UNIT = one 256-element K group of one output tile (128 weight rows x one token
// tile of BN <= 128 columns).  The units of a launch, ordered tile by tile, are cut into one contiguous range per CTA (at most one CTA
// per SM), so every SM gets the same number of 64-element MMA steps whatever N, K and T are.  A CTA walks its range segment by segment
// (segment = its part of one tile); a segment that covers the tile's whole K stores its result, a partial one adds it into the
// pre-zeroed dst with fp32 atomics (one addend per CTA sharing the tile, up to ceil(ngrp / upc) + 1: 15 for K = 29 568, T = 24 on 132 SMs;
// the order of fp32 adds is the only non-determinism, below the kernel's own fp16 rounding).  Bias and residual ride on the K group 0
// segment only.  Inside a CTA the pipeline never drains between segments (raw-block ring, A and B stages and their
// barriers run on CTA-wide counters):
//   warps 0..7  two consumer warpgroups: warpgroup w issues 4 x wgmma.mma_async (M=64, N=BN, K=16, f16 in, f32 accumulators in
//               registers) per step for weight rows [64w, 64w + 64) of the tile, keeps one step in flight, and at the end of a segment
//               stores / adds its accumulators into dst
//   warp 8      activation producer: one cp.async.bulk per step of the pre-tiled fp16 chunk (BN x 128 B, already in the 128-byte
//               swizzle image wgmma reads), 2-4 stages deep
//   warps 9..16 (8 expansion warps, 2 threads per weight row) fetch their rows' raw quantized blocks (16-byte cp.async pieces, 3 K groups
//               deep, completion through cp.async.mbarrier.arrive) and expand 128 x 64 weights per step to fp16 straight into the swizzled A
//               stage (generic-proxy stores + fence.proxy.async), 2 stages
// Registers bound the tile: 17 warps leave 96 registers per thread (five warps share one SM sub-partition's register file), and a
// consumer thread holds BN / 2 fp32 accumulators; the epilogue therefore streams its residuals 16 columns at a time.
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>

#include "common.cuh"
#include "launch.h"
#include "quantize.cuh"

namespace pb {

constexpr int MMQ_BM = 128;
constexpr int MMQ_BK = 64;
constexpr int MMQ_BN_MAX = 128;   // token columns of a tile: 64 accumulator registers per consumer thread
constexpr int MMQ_A_MAX = 4;      // expanded-weight stages: P.a_nst = 2 or 4 (a power of two) of 16 KB, chosen at launch from the shared-memory budget
constexpr int MMQ_B_NST = 4;      // activation stages (L2 loads: the deep ring)
constexpr int MMQ_MIN_UNITS = 8;  // smallest stream-K share of a CTA, in K groups
constexpr int MMQ_MMA_WARPS = 8;  // two consumer warpgroups, 64 weight rows each
constexpr int MMQ_DQ_WARPS = 8;   // expansion warps: 2 threads per weight row, 32 weights per thread and step
constexpr int MMQ_DQ_WARP0 = MMQ_MMA_WARPS + 1;   // warp MMQ_MMA_WARPS = activation producer
constexpr int MMQ_THREADS = (MMQ_DQ_WARP0 + MMQ_DQ_WARPS) * 32;
constexpr int MMQ_A_BYTES = MMQ_BM * 128;   // one A stage: 128 rows x 64 fp16
constexpr int MMQ_CTL_BYTES = 256;

struct MmqParams {
    int * abort_flag;      // host-mapped, raised by the wait watchdog
    const uint8_t * W;
    const uint8_t * B;     // activations, fp16, tiled [T/BN][K/64][BN x 128 B swizzled]
    const float * rscale;  // [Tpad]: 2^-e_t, undoes the power-of-two row scale of the activation image (k_mmq_prep)
    float * dst;           // [T][N]
    const float * bias;    // [N] or null
    const float * resid;   // [T][N] or null: residual added in the epilogue
    int64_t row_bytes, total_bytes;
    int nraw, b_nst, a_nst;   // ring depths chosen at launch from the shared-memory budget (a_nst: 2 or 4)
    int ngrp, rtiles;      // 256-K groups per row (the last one may be short: 32-element block types), row tiles
    int upc, total_units;  // work units per CTA (CTA c owns units [c * upc, min((c + 1) * upc, total_units)) ), units of the launch
    int N, K, T, bpb, slot;   // slot: bytes reserved per row in a raw stage (16-B aligned window around one block)
};

struct MmqCtl {
    uint64_t raw_full[3], raw_empty[3];
    uint64_t a_ready[MMQ_A_MAX], b_full[MMQ_B_NST];
    uint64_t step_done[MMQ_B_NST];   // both consumer warpgroups arrive once step u's wgmma completed: step_done[u % 4] frees A stage u % a_nst and B stage u % b_nst
    volatile int abort;
};
static_assert(sizeof(MmqCtl) <= MMQ_CTL_BYTES, "ctl");


__device__ __forceinline__ bool mmq_try(uint64_t * bar, uint32_t parity) {
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
// bounded wait: a broken pipeline must end the launch (and report through pb200_mmq_aborted), never hang the device
__device__ __forceinline__ bool mmq_wait_(MmqCtl * ctl, uint64_t * bar, uint32_t parity, int * abort_flag) {
    if (mmq_try(bar, parity)) return true;          // the common case costs one try_wait
    const long long t0 = clock64();
    int spins = 0;
    while (!mmq_try(bar, parity)) {
        if ((++spins & 255) == 0) {
            if (ctl->abort) return false;
            if (clock64() - t0 > PB_WAIT_TIMEOUT_CYCLES) {
                ctl->abort = 1;                                          // inline on purpose: a call costs registers the kernel does not have
                if (abort_flag) *(volatile int *) abort_flag = 1;        // host-mapped; visible at the latest when the launch ends
                return false;
            }
        }
    }
    return true;
}
#define mmq_wait(ctl, bar, parity) mmq_wait_(ctl, bar, parity, P.abort_flag)
__device__ __forceinline__ void bulk_g2s_plain(void * smem_dst, const void * gsrc, uint32_t bytes, uint64_t * bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)), "l"(gsrc),
                 "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t saddr) {
    // wgmma matrix descriptor, K-major, 128-byte swizzle: rows of 128 B, 8-row groups 1024 B apart (the address must be 1024-B aligned
    // for a zero base offset; a K step of 16 fp16 inside the swizzle atom advances the start address by 32 B)
    uint64_t d = (uint64_t) ((saddr >> 4) & 0x3FFF);
    d |= (uint64_t) 1 << 16;               // leading byte offset: unused for swizzled K-major, canonical value 1
    d |= (uint64_t) (1024 >> 4) << 32;     // stride byte offset
    d |= (uint64_t) 1 << 62;               // 128-byte swizzle
    return d;
}
// D[64 x N] (+)= A[64 x 16] . B[N x 16]^T, both operands K-major in shared memory; accumulate == 0 overwrites D
template <int N>
__device__ __forceinline__ void wgmma_f16(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t accumulate);
template <> __device__ __forceinline__ void wgmma_f16<16>(float (&d)[8], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %10, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db), "r"(accumulate));
}
template <> __device__ __forceinline__ void wgmma_f16<32>(float (&d)[16], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %18, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(accumulate));
}
template <> __device__ __forceinline__ void wgmma_f16<64>(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(accumulate));
}
template <> __device__ __forceinline__ void wgmma_f16<128>(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int NPEND>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(NPEND) : "memory"); }
// keeps the compiler from touching accumulator registers across the asynchronous wgmma (reads before its wait_group)
__device__ __forceinline__ void reg_fence(float & r) { asm volatile("" : "+f"(r)::"memory"); }

__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t *>(&h);
}
// 32-bit load from shared memory at an address that is only 2-byte aligned
__device__ __forceinline__ uint32_t lds32_u2(const uint8_t * p) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    const uint32_t * w = reinterpret_cast<const uint32_t *>(a & ~(uintptr_t) 3);
    if ((a & 2) == 0) return w[0];
    return __funnelshift_r(w[0], w[1], 16);
}

// ---- weight expansion: thread (row, h) produces K elements [64c + 32h, 64c + 32h + 32) of its row as 16 half2 ----
// The integer q of every weight is made an EXACT fp16 with the exponent trick (0x6400 | q == 1024 + q, minus 1024 + zero),
// then one half2 FMA applies the sub-block scale and offset (both rounded to fp16).  A 32-bit word holds 4 consecutive-k
// bytes; the two half2 come out as (k0,k2) and (k1,k3): the activation tiles use the same within-4 order (k_mmq_prep).
__device__ __forceinline__ __half2 bits_h2(uint32_t v) { return *reinterpret_cast<__half2 *>(&v); }
__device__ __forceinline__ uint32_t h2_bits(__half2 v) { return *reinterpret_cast<uint32_t *>(&v); }
__device__ __forceinline__ uint32_t and_or(uint32_t a, uint32_t mask, uint32_t magic) {   // (a & mask) | magic in one LOP3
    uint32_t d;
    asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(d) : "r"(a), "r"(mask), "r"(magic));
    return d;
}
template <uint32_t MASK>
__device__ __forceinline__ void expand_word(uint32_t t, __half2 bias, __half2 scale, __half2 off, uint32_t & o02, uint32_t & o13) {
    const uint32_t p02 = and_or(t, MASK, 0x64006400u);
    const uint32_t p13 = and_or(t >> 8, MASK, 0x64006400u);
    o02 = h2_bits(__hfma2(__hadd2(bits_h2(p02), bias), scale, off));
    o13 = h2_bits(__hfma2(__hadd2(bits_h2(p13), bias), scale, off));
}
__device__ __forceinline__ void scale_min_k4(const uint8_t * sc, int j, int & s, int & m) {   // get_scale_min_k4, ggml-quants.c:1950-1958
    // branch-free: both packings are computed, j selects
    const int lo_s = sc[j & 3], lo_m = sc[(j & 3) + 4], hi = sc[(j & 3) + 8];
    const int s0 = lo_s & 63, m0 = lo_m & 63;
    const int s1 = (hi & 0xF) | ((lo_s >> 6) << 4), m1 = (hi >> 4) | ((lo_m >> 6) << 4);
    s = j < 4 ? s0 : s1;
    m = j < 4 ? m0 : m1;
}
// the 16 bytes at a 2-byte aligned shared-memory address as 4 words: 5 aligned loads, one funnel shift each
__device__ __forceinline__ void lds16_u2(const uint8_t * p, uint32_t (&w)[4]) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    const uint32_t * wp = reinterpret_cast<const uint32_t *>(a & ~(uintptr_t) 3);
    const uint32_t sh = (uint32_t) (a & 2) * 8;
    uint32_t x[5];
#pragma unroll
    for (int i = 0; i < 5; i++) x[i] = wp[i];
#pragma unroll
    for (int i = 0; i < 4; i++) w[i] = __funnelshift_r(x[i], x[i + 1], sh);
}

// thread (row, h, hh) produces K elements [64c + 32h + 16hh, 64c + 32h + 16hh + 16) of its row as 8 half2 (two 16-byte pieces of the A stage)
template <int TYPE>
__device__ __forceinline__ void expand(const uint8_t * blk, int c, int h, int hh, uint32_t (&out)[8]) {
    if (TYPE == T_Q4_0 || TYPE == T_Q4_1 || TYPE == T_Q5_0) {
        // Q4_0 [d f16][16 x 2 nibbles] (18 B, 2-byte aligned): d (q - 8); Q4_1 [d f16][m f16][nibbles] (20 B, word-aligned): d q + m;
        // Q5_0 [d f16][qh u32][nibbles] (22 B, 2-byte aligned): d ((q | h << 4) - 16).  Element j < 16 = low nibble of qs[j] (with bit j
        // of qh), element j + 16 = its high nibble (bit j + 16): hh = 0 takes the low nibbles, hh = 1 the high ones
        constexpr int BB = TYPE == T_Q4_0 ? BYTES_Q4_0 : TYPE == T_Q4_1 ? BYTES_Q4_1 : BYTES_Q5_0;
        constexpr int QOFF = TYPE == T_Q4_0 ? 2 : TYPE == T_Q4_1 ? 4 : 6;
        const uint8_t * bb = blk + (2 * c + h) * BB;
        const __half dh = *reinterpret_cast<const __half *>(bb);
        const __half2 scale = __half2half2(dh);
        const __half2 off = TYPE == T_Q4_1 ? __half2half2(*reinterpret_cast<const __half *>(bb + 2)) : __float2half2_rn(0.f);
        const __half2 bias = __float2half2_rn(TYPE == T_Q4_0 ? -1032.f : TYPE == T_Q4_1 ? -1024.f : -1040.f);
        uint32_t w[4];
        lds16_u2(bb + QOFF, w);
        if (TYPE == T_Q5_0) {
            const uint32_t qh = lds32_u2(bb + 2) >> (16 * hh);
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const uint32_t hb = ((((qh >> (4 * i)) & 0xFu) * 0x00204081u) & 0x01010101u) << 4;
                expand_word<0x001F001Fu>(((w[i] >> (4 * hh)) & 0x0F0F0F0Fu) | hb, bias, scale, off, out[2 * i], out[2 * i + 1]);
            }
        } else {
#pragma unroll
            for (int i = 0; i < 4; i++) expand_word<0x000F000Fu>(w[i] >> (4 * hh), bias, scale, off, out[2 * i], out[2 * i + 1]);
        }
    } else if (TYPE == T_Q8_0) {
        // 32-element blocks, 34 B each ([d f16][32 x i8]); blk = the group of 8 blocks covering 256 K, this thread's block is 2c + h.
        // Blocks are 2-byte aligned: qs (offset 2) is either word-aligned or straddles words -> one PRMT per word.
        const uint8_t * bb = blk + (2 * c + h) * BYTES_Q8_0;
        const uint32_t * wp = reinterpret_cast<const uint32_t *>(reinterpret_cast<uintptr_t>(bb) & ~(uintptr_t) 3);
        const bool odd = (reinterpret_cast<uintptr_t>(bb) & 2) != 0;
        const uint32_t sel = odd ? 0x7654u : 0x5432u;
        const uint32_t w0 = wp[0];
        uint32_t w[5];
#pragma unroll
        for (int i = 0; i < 5; i++) w[i] = wp[4 * hh + i];
        const __half dh = __ushort_as_half((unsigned short) ((w0 >> (odd ? 16 : 0)) & 0xffff));
        const __half2 scale = __half2half2(dh), bias = __float2half2_rn(-1152.f), zero = __float2half2_rn(0.f);
#pragma unroll
        for (int i = 0; i < 4; i++)   // q + 128 as an unsigned byte, 0x6400 | u = 1024 + u, minus 1152 = q exactly
            expand_word<0x00FF00FFu>(__byte_perm(w[i], w[i + 1], sel) ^ 0x80808080u, bias, scale, zero, out[2 * i], out[2 * i + 1]);
    } else if (TYPE == T_Q5_1) {
        // 24 B blocks ([d f16][m f16][qh u32][16 x 2 nibbles]), 8-byte aligned; element j < 16 = low nibble of qs[j] | bit j of qh << 4,
        // element j + 16 = high nibble | bit j + 16: hh = 0 takes the low nibbles, hh = 1 the high ones
        const uint8_t * bb = blk + (2 * c + h) * BYTES_Q5_1;
        const uint2 hd = *reinterpret_cast<const uint2 *>(bb);
        const __half2 dm = bits_h2(hd.x);
        const __half2 scale = __half2half2(__low2half(dm)), off = __half2half2(__high2half(dm)), bias = __float2half2_rn(-1024.f);
        const uint32_t qh = hd.y >> (16 * hh);
        const uint2 qa = *reinterpret_cast<const uint2 *>(bb + 8), qb = *reinterpret_cast<const uint2 *>(bb + 16);
        const uint32_t w[4] = {qa.x, qa.y, qb.x, qb.y};
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const uint32_t hb = ((((qh >> (4 * i)) & 0xFu) * 0x00204081u) & 0x01010101u) << 4;
            expand_word<0x001F001Fu>(((w[i] >> (4 * hh)) & 0x0F0F0F0Fu) | hb, bias, scale, off, out[2 * i], out[2 * i + 1]);
        }
    } else if (TYPE == T_Q4_K || TYPE == T_Q5_K) {
        const float d = __half2float(*reinterpret_cast<const __half *>(blk));
        const float dmin = __half2float(*reinterpret_cast<const __half *>(blk + 2));
        const int j = 2 * c + h;
        int s, m;
        scale_min_k4(blk + 4, j, s, m);
        const __half2 scale = __float2half2_rn(__fmul_rn(d, (float) s)), off = __float2half2_rn(-__fmul_rn(dmin, (float) m));
        const __half2 bias = __float2half2_rn(-1024.f);
        const uint4 qa = *reinterpret_cast<const uint4 *>(blk + (TYPE == T_Q4_K ? 16 : 48) + 32 * c + 16 * hh);
        const uint32_t w[4] = {qa.x, qa.y, qa.z, qa.w};
        if (TYPE == T_Q4_K) {
#pragma unroll
            for (int i = 0; i < 4; i++) expand_word<0x000F000Fu>(w[i] >> (4 * h), bias, scale, off, out[2 * i], out[2 * i + 1]);
        } else {
            const uint4 ha = *reinterpret_cast<const uint4 *>(blk + 16 + 16 * hh);
            const uint32_t hq[4] = {ha.x, ha.y, ha.z, ha.w};
#pragma unroll
            for (int i = 0; i < 4; i++)
                expand_word<0x001F001Fu>(((w[i] >> (4 * h)) & 0x0F0F0F0Fu) | (((hq[i] >> j) << 4) & 0x10101010u), bias, scale, off, out[2 * i],
                                         out[2 * i + 1]);
        }
    } else {
        // Q6_K: blk is 2-byte aligned only (210-byte blocks): words are fetched as aligned pairs and funnel-shifted
        const float d = __half2float(*reinterpret_cast<const __half *>(blk + 208));
        const int n = c >> 1, p = c & 1;
        const uint8_t * ql = blk + 64 * n + 32 * h + 16 * hh;
        const uint8_t * qh = blk + 128 + 32 * n + 16 * hh;
        const int8_t * sc = reinterpret_cast<const int8_t *>(blk + 192 + 8 * n + 2 * h + 4 * p);
        const __half2 sca = __float2half2_rn(__fmul_rn(d, (float) sc[hh]));
        const __half2 bias = __float2half2_rn(-1056.f), zero = __float2half2_rn(0.f);
        const uint32_t shl = (uint32_t) (reinterpret_cast<uintptr_t>(blk) & 2) * 8;     // 0 or 16 (ql and qh share blk's alignment)
        const uint32_t * lw = reinterpret_cast<const uint32_t *>(reinterpret_cast<uintptr_t>(ql) & ~(uintptr_t) 3);
        const uint32_t * hw = reinterpret_cast<const uint32_t *>(reinterpret_cast<uintptr_t>(qh) & ~(uintptr_t) 3);
        uint32_t lprev = lw[0], hprev = hw[0];
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const uint32_t lnext = lw[i + 1], hnext = hw[i + 1];
            const uint32_t l = __funnelshift_r(lprev, lnext, shl), hq = __funnelshift_r(hprev, hnext, shl);
            lprev = lnext; hprev = hnext;
            const uint32_t t = ((l >> (4 * p)) & 0x0F0F0F0Fu) | (((hq >> (4 * p + 2 * h)) << 4) & 0x30303030u);
            expand_word<0x003F003Fu>(t, bias, sca, zero, out[2 * i], out[2 * i + 1]);
        }
    }
}

__device__ __forceinline__ void cp_async16(void * smem_dst, const void * gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}


template <int TYPE, int BN>
__global__ void __launch_bounds__(MMQ_THREADS, 1) k_mmq_tc(const __grid_constant__ MmqParams P) {
    extern __shared__ uint8_t smem_raw[];
    // the swizzle-128B atoms (A and B stages) need 1024-byte alignment in the shared window
    uint8_t * smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    constexpr int b1 = BN * 128;                                 // one step of a token tile in the activation image = one B stage
    uint8_t * a_st = smem;                                       // [a_nst][16 KB]
    uint8_t * b_st = a_st + P.a_nst * MMQ_A_BYTES;               // [b_nst][BN * 128]
    const int amask = P.a_nst - 1, ashift = P.a_nst == 4 ? 2 : 1;
    uint8_t * raw = b_st + P.b_nst * b1;                         // [nraw][128 * slot]
    MmqCtl * ctl = reinterpret_cast<MmqCtl *>(raw + P.nraw * MMQ_BM * P.slot);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nstep_all = P.K / MMQ_BK;                          // 64-element steps of a whole row; group sb holds steps [4 sb, min(4 sb + 4, nstep_all))
    const int w0 = (int) blockIdx.x * P.upc, w1 = min(w0 + P.upc, P.total_units);   // this CTA's units

    if (threadIdx.x == 0) {
        for (int i = 0; i < 3; i++) { mbar_init(&ctl->raw_full[i], MMQ_DQ_WARPS * 32); mbar_init(&ctl->raw_empty[i], MMQ_DQ_WARPS); }
        for (int i = 0; i < MMQ_A_MAX; i++) mbar_init(&ctl->a_ready[i], MMQ_DQ_WARPS);
        for (int i = 0; i < MMQ_B_NST; i++) { mbar_init(&ctl->b_full[i], 1); mbar_init(&ctl->step_done[i], MMQ_MMA_WARPS / 4); }
        ctl->abort = 0;
        mbar_fence_init();
    }
    __syncthreads();

    // Every role walks the same segments: unit w -> tile w / ngrp (token tile tile / rtiles, row tile tile % rtiles), K group w % ngrp.
    if (warp < MMQ_MMA_WARPS) {
        // ================= consumers: warpgroup wg multiplies weight rows [64 wg, 64 wg + 64) of the tile =================
        const int wg = warp >> 2;
        const bool leader = (threadIdx.x & 127) == 0;
        float acc[BN / 2];
        int g = 0;                                               // CTA-wide step counter (barrier phases follow it)
        bool ok = true;
        for (int w = w0; w < w1 && ok;) {
            const int tile = w / P.ngrp, sbb = w - tile * P.ngrp, sbe = min(P.ngrp, sbb + (w1 - w));
            const int nsteps = min(4 * sbe, nstep_all) - 4 * sbb;
            for (int u = 0; u < nsteps; u++, g++) {
                const int sa = g & amask, sb = g % P.b_nst;
                if (!mmq_wait(ctl, &ctl->b_full[sb], (g / P.b_nst) & 1)) { ok = false; break; }
                if (!mmq_wait(ctl, &ctl->a_ready[sa], (g >> ashift) & 1)) { ok = false; break; }
                const uint64_t da = gmma_desc_sw128(smem_u32(a_st + (size_t) sa * MMQ_A_BYTES + wg * (MMQ_A_BYTES / 2)));
                const uint64_t db = gmma_desc_sw128(smem_u32(b_st + (size_t) sb * b1));
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < MMQ_BK / 16; k++) wgmma_f16<BN>(acc, da + 2 * k, db + 2 * k, (u | k) != 0);
                wgmma_commit();
                wgmma_wait<1>();                                 // step g - 1 has read its stages
                if (u > 0 && leader) mbar_arrive(&ctl->step_done[(g - 1) % MMQ_B_NST]);
            }
            wgmma_wait<0>();
#pragma unroll
            for (int i = 0; i < BN / 2; i++) reg_fence(acc[i]);
            if (!ok) break;
            if (leader) mbar_arrive(&ctl->step_done[(g - 1) % MMQ_B_NST]);
            // ================= epilogue of the segment, straight from the accumulator registers =================
            // wgmma's D fragment: acc[4 j + 2 i + e] = D[16 (warp % 4) + lane / 4 + 8 i][8 j + 2 (lane % 4) + e]
            const int t0 = (tile / P.rtiles) * BN + 2 * (lane & 3);
            const int nrow = (tile % P.rtiles) * MMQ_BM + wg * 64 + (warp & 3) * 16 + (lane >> 2);
            const bool first = sbb == 0, whole = first && sbe == P.ngrp;   // bias / residual ride on the K group 0 segment
            // undo the activation row scale (exact, a power of two) before bias and residual: t0 + 8 j + e < Tpad, rscale covers the padding
#pragma unroll
            for (int j = 0; j < BN / 8; j++)
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    const float s = __ldg(P.rscale + t0 + 8 * j + e);
                    acc[4 * j + e] = __fmul_rn(acc[4 * j + e], s);
                    acc[4 * j + 2 + e] = __fmul_rn(acc[4 * j + 2 + e], s);
                }
#pragma unroll
            for (int i = 0; i < 2; i++) {
                const int n = nrow + 8 * i;
                if (n >= P.N) continue;
                const float bias = (P.bias && first) ? P.bias[n] : 0.f;
                const float * __restrict__ rp = (P.resid && first) ? P.resid + n : nullptr;
                // a chunk's residuals are loaded before its stores: written as "load, add, store" per element the loads would serialise
                // behind the stores / atomics (dst and resid may alias as far as the compiler knows)
                constexpr int JC = 2;
#pragma unroll
                for (int j0 = 0; j0 < BN / 8; j0 += JC) {
                    float rv[2 * JC];
#pragma unroll
                    for (int j = 0; j < JC; j++)
#pragma unroll
                        for (int e = 0; e < 2; e++) {
                            const int t = t0 + 8 * (j0 + j) + e;
                            rv[2 * j + e] = (rp && t < P.T) ? __ldg(rp + (size_t) t * P.N) : 0.f;
                        }
#pragma unroll
                    for (int j = 0; j < JC; j++)
#pragma unroll
                        for (int e = 0; e < 2; e++) {
                            const int t = t0 + 8 * (j0 + j) + e;
                            if (t < P.T) {
                                const float y = __fadd_rn(__fadd_rn(acc[4 * (j0 + j) + 2 * i + e], bias), rv[2 * j + e]);
                                if (whole) P.dst[(size_t) t * P.N + n] = y;
                                else atomicAdd(&P.dst[(size_t) t * P.N + n], y);   // one addend per CTA sharing the tile, onto 0
                            }
                        }
                }
            }
            w += sbe - sbb;
        }
    } else if (warp == MMQ_MMA_WARPS) {
        // ================= activation producer: runs up to b_nst steps ahead of the tensor cores =================
        if (lane == 0) {
            const size_t tile_stride = (size_t) nstep_all * b1;
            int g = 0;
            bool ok = true;
            for (int w = w0; w < w1 && ok;) {
                const int tile = w / P.ngrp, sbb = w - tile * P.ngrp, sbe = min(P.ngrp, sbb + (w1 - w));
                const int nsteps = min(4 * sbe, nstep_all) - 4 * sbb;
                const uint8_t * Bt = P.B + (size_t) (tile / P.rtiles) * tile_stride + (size_t) sbb * 4 * b1;
                for (int u = 0; u < nsteps; u++, g++) {
                    const int sb = g % P.b_nst;
                    if (g >= P.b_nst) {   // step g - b_nst consumed this stage
                        const int f = g - P.b_nst;
                        if (!mmq_wait(ctl, &ctl->step_done[f % MMQ_B_NST], (f / MMQ_B_NST) & 1)) { ok = false; break; }
                    }
                    mbar_arrive_expect_tx(&ctl->b_full[sb], (uint32_t) b1);
                    bulk_g2s_plain(b_st + (size_t) sb * b1, Bt + (size_t) u * b1, (uint32_t) b1, &ctl->b_full[sb]);
                }
                w += sbe - sbb;
            }
        }
        __syncwarp();
    } else {
        // ================= weight expansion =================
        const int dt = threadIdx.x - MMQ_DQ_WARP0 * 32;        // 0..255
        const int r = dt >> 1, h = dt & 1;
        bool ok = true;
        // this thread fetches its own half of the row's block: 16-byte cp.async pieces of the 16-B aligned window around it
        const int64_t lim = (P.total_bytes + 15) & ~(int64_t) 15;
        const int cpr = P.slot >> 4, p_lo = cpr * h / 2, p_hi = cpr * (h + 1) / 2;
        const int nx = w1 - w0;                                 // groups this CTA walks, x = 0 .. nx-1 across its segments
        // fetch cursor: the group nraw-1 ahead of the one being expanded (tile / K group tracked incrementally: no divisions in the loop)
        int f_x = 0, f_sb, f_rt;
        { const int tile = w0 / P.ngrp; f_sb = w0 - tile * P.ngrp; f_rt = tile % P.rtiles; }
        auto fetch_next = [&](int slot) {                       // issues group f_x of this CTA into raw slot `slot`, advances the cursor
            const int gr = min(f_rt * MMQ_BM + r, P.N - 1);
            const int64_t src0 = ((int64_t) gr * P.row_bytes + (int64_t) f_sb * P.bpb) & ~(int64_t) 15;
            uint8_t * dst0 = raw + ((size_t) slot * MMQ_BM + r) * P.slot;
            for (int pc = p_lo; pc < p_hi; pc++)
                if (src0 + pc * 16 + 16 <= lim) cp_async16(dst0 + pc * 16, P.W + src0 + pc * 16);
            asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(&ctl->raw_full[slot])) : "memory");
            f_x++;
            if (++f_sb == P.ngrp) { f_sb = 0; if (++f_rt == P.rtiles) f_rt = 0; }
        };
        for (int i = 0; i < P.nraw - 1 && i < nx; i++) fetch_next(i);
        // the four 16-byte pieces (K elements 32h + 8q .. + 8, q = 0..3) this thread writes per step, already swizzled
        const uint32_t arow = r * 128;
        uint32_t o[4];
#pragma unroll
        for (int q = 0; q < 4; q++) o[q] = arow + (((4 * h + q) ^ (r & 7)) << 4);
        int g = 0;
        int rs = 0, rph = 0;                                    // raw slot / phase of the group being expanded
        int prs = P.nraw - 1, pph = 1;                          // ... of the group before it (the slot the next fetch goes into)
        for (int w = w0; w < w1 && ok;) {
            const int tile = w / P.ngrp, sbb = w - tile * P.ngrp, sbe = min(P.ngrp, sbb + (w1 - w));
            const int gr = min((tile % P.rtiles) * MMQ_BM + r, P.N - 1);
            for (int sb = sbb; sb < sbe && ok; sb++) {
                // refill the slot the previous group used, once every expansion warp has left it
                if (f_x < nx) {
                    if (f_x >= P.nraw && !mmq_wait(ctl, &ctl->raw_empty[prs], pph)) { ok = false; break; }
                    fetch_next(prs);
                }
                if (!mmq_wait(ctl, &ctl->raw_full[rs], rph)) { ok = false; break; }
                const int64_t g0 = (int64_t) gr * P.row_bytes + (int64_t) sb * P.bpb;
                const uint8_t * blk = raw + (size_t) (rs * MMQ_BM + r) * P.slot + (g0 & 15);
                const int nst = min(4, nstep_all - 4 * sb);      // the last group of a K % 256 != 0 row (32-element block types) is short
#pragma unroll
                for (int c = 0; c < 4; c++) {
                    if (c >= nst) break;
                    uint32_t v[2][8];
                    expand<TYPE>(blk, c, h, 0, v[0]);
                    expand<TYPE>(blk, c, h, 1, v[1]);
                    if (g >= P.a_nst) {     // step g - a_nst has consumed this A stage
                        const int f = g - P.a_nst;
                        if (!mmq_wait(ctl, &ctl->step_done[f % MMQ_B_NST], (f / MMQ_B_NST) & 1)) { ok = false; break; }
                    }
                    uint8_t * as = a_st + (size_t) (g & amask) * MMQ_A_BYTES;
#pragma unroll
                    for (int hh = 0; hh < 2; hh++) {
                        *reinterpret_cast<uint4 *>(as + o[2 * hh]) = make_uint4(v[hh][0], v[hh][1], v[hh][2], v[hh][3]);
                        *reinterpret_cast<uint4 *>(as + o[2 * hh + 1]) = make_uint4(v[hh][4], v[hh][5], v[hh][6], v[hh][7]);
                    }
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> visible to wgmma's async proxy
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&ctl->a_ready[g & amask]);
                    g++;
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&ctl->raw_empty[rs]);
                prs = rs; pph = rph;
                if (++rs == P.nraw) { rs = 0; rph ^= 1; }
            }
            w += sbe - sbb;
        }
    }
}

// ---- activation rows -> q8_K (exactly as the CPU backend quantizes them) -> fp16, written in the tiled 128-byte-swizzle image wgmma reads ----
// blk32: the weight type is Q8_0 / Q5_1, whose CPU dot quantizes the activation per 32 values (q8_0 / q8_1: d = amax / 127 stored
// as f16, q = round-half-even(x * 127 / amax), quantize_row_q8_0 ggml-quants.c:943-1010) instead of per 256 (q8_K).
// Fused producers of the activation (pre_kind): PRO_SILU_MUL = silu(x) * aux[t][k] (llm_build_ffn's SILU + MUL in front of ffn_down, the f32
// product never goes to HBM), PRO_RMSNORM = rms_norm(x) * aux[k] (llm_build_norm in front of q|k|v and gate|up): the same arithmetic, rounding for rounding, as
// k_silu_mul / k_rms_norm_rows followed by the plain pass (tests/test_gpu_prefill_layers.py checks it bit for bit).
// Operand range: the values d*q of row t are written as fp16 of d*q*2^e_t, e_t chosen so that the row's largest |d*q| lands in
// [2^14, 2^15) (e_t <= 126: rows whose largest value is below 2^-112 stay below that), and rscale[t] = 2^-e_t, which the consumers'
// epilogue applies to the fp32 accumulators.  So no activation overflows fp16 (|x| >= 65 520 was inf) or falls into its subnormals
// (rows with amax below ~1e-3 lost bits, below ~1e-7 were zero); where d*q was a normal fp16 already the scaled value is the old one
// times 2^e_t and the result is bit-identical.  The row's q and d wait in shared memory (mmq_prep_smem) while the CTA reduces the max.
static size_t mmq_prep_smem(int64_t K) { return (size_t) ((K + 255) / 256) * (256 + 8 * sizeof(float)); }   // int8 q[256] | f32 d[8] per 256 values

__global__ void __launch_bounds__(256) k_mmq_prep(const float * __restrict__ x, int64_t ldx, int T, int K, int BN, uint8_t * __restrict__ out,
                                                  float * __restrict__ rscale, int blk32, int pre_kind, const float * __restrict__ aux,
                                                  int64_t ld_aux, float eps) {
    extern __shared__ uint8_t prep_smem[];
    __shared__ float s_max[8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nblk = (K + 255) / 256;
    int8_t * sq = reinterpret_cast<int8_t *>(prep_smem);                    // [nblk][256]
    float * sd = reinterpret_cast<float *>(prep_smem + (size_t) nblk * 256);  // [nblk][8]: d of each 32 values
    const int t = blockIdx.x;                       // 0 .. Tpad-1
    const int b_bytes = BN * 128;
    const float nscale = pre_kind == PRO_RMSNORM && t < T ? block_rms_scale(x + (size_t) t * ldx, K, eps) : 1.f;   // k_rms_norm_rows' scale
    float rmax = 0.f;                               // largest |d * q| this thread quantized
    for (int b = warp; b < nblk; b += 8) {
        float v[8];
        const bool live = b * 256 + lane * 8 < K;   // K % 32 == 0: a 4-lane group (one 32-block) is live or dead as a whole
        if (t < T && live) {
            const float4 * p = reinterpret_cast<const float4 *>(x + (size_t) t * ldx + (size_t) b * 256 + lane * 8);
            const float4 a = p[0], c = p[1];
            v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = c.x; v[5] = c.y; v[6] = c.z; v[7] = c.w;
            if (pre_kind) {
                const float4 * q = reinterpret_cast<const float4 *>(aux + (pre_kind == PRO_SILU_MUL ? (size_t) t * ld_aux : (size_t) 0) + (size_t) b * 256 + lane * 8);
                const float4 e = q[0], f = q[1];
                const float w[8] = {e.x, e.y, e.z, e.w, f.x, f.y, f.z, f.w};
#pragma unroll
                for (int i = 0; i < 8; i++) v[i] = pre_kind == PRO_SILU_MUL ? __fmul_rn(silu_f(v[i]), w[i]) : __fmul_rn(__fmul_rn(v[i], nscale), w[i]);
            }
        } else {
#pragma unroll
            for (int i = 0; i < 8; i++) v[i] = 0.f;
        }
        int q[8];
        float d;
        if (blk32) {
            d = __half2float(__float2half_rn(q8_01_quant(v, q)));
        } else {
            float amax, vmax;
            int idx;
            q8K_lane_absmax(v, lane * 8, amax, vmax, idx);
            warp_argmax(amax, idx, &vmax);
            d = q8K_quant(v, amax, vmax, q);
        }
        uint32_t packed[2];
        int qsum;
        pack_q8(q, packed, qsum);
        *reinterpret_cast<uint2 *>(sq + (size_t) b * 256 + lane * 8) = make_uint2(packed[0], packed[1]);
        if ((lane & 3) == 0) sd[b * 8 + (lane >> 2)] = d;
#pragma unroll
        for (int i = 0; i < 8; i++) rmax = fmaxf(rmax, fabsf(__fmul_rn(d, (float) q[i])));
    }
    rmax = warp_max(rmax);
    if (lane == 0) s_max[warp] = rmax;
    __syncthreads();
    rmax = s_max[0];
#pragma unroll
    for (int i = 1; i < 8; i++) rmax = fmaxf(rmax, s_max[i]);
    // e = 14 - floor(log2(rmax)) from the exponent field (a zero row keeps e = 0)
    const int e = rmax > 0.f ? min(14 - (((__float_as_int(rmax) >> 23) & 0xff) - 127), 126) : 0;
    const float up = __int_as_float((127 + e) << 23);
    if (threadIdx.x == 0) rscale[t] = __int_as_float((127 - e) << 23);
    for (int b = warp; b < nblk; b += 8) {
        const bool live = b * 256 + lane * 8 < K;
        const uint2 pq = *reinterpret_cast<const uint2 *>(sq + (size_t) b * 256 + lane * 8);
        const float d = sd[b * 8 + (lane >> 2)];
        float f[8];
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const int qi = (int) (int8_t) (((i < 4 ? pq.x : pq.y) >> (8 * (i & 3))) & 0xff);
            f[i] = __fmul_rn(__fmul_rn(d, (float) qi), up);
        }
        // within every 4 consecutive k the order is (0,2,1,3): the weight expansion produces its half2 pairs that way
        const uint32_t h[4] = {pack_h2(f[0], f[2]), pack_h2(f[1], f[3]), pack_h2(f[4], f[6]), pack_h2(f[5], f[7])};
        const int k = b * 256 + lane * 8;
        const int kc = k >> 6, j = (k & 63) >> 3;
        const int tt = t / BN, tl = t % BN;
        uint8_t * dstp = out + ((size_t) tt * (K / 64) + kc) * b_bytes + (size_t) tl * 128 + (size_t) ((j ^ (tl & 7)) << 4);
        if (live) *reinterpret_cast<uint4 *>(dstp) = make_uint4(h[0], h[1], h[2], h[3]);
    }
}


static int mmq_pick_bn(int T) {   // a power of two: one kernel instance per width
    int bn = 16;
    while (bn < T && bn < MMQ_BN_MAX) bn <<= 1;
    return bn;
}
size_t mmq_workspace_bytes(int64_t K, int64_t T) {   // the fp16 activation image [Tpad][K], then rscale [Tpad] f32
    const int BN = mmq_pick_bn((int) T);
    const int64_t tpad = (T + BN - 1) / BN * BN;
    return (size_t) (tpad * K * 2 + tpad * 4);
}
bool mmq_supported(int type, int64_t K) {
    if (is_kquant(type)) return K % 256 == 0 && K >= 256;
    return is_blk32_type(type) && K % 64 == 0 && K >= 256;   // 32-element blocks: two per 64-element step
}

template <int TYPE, int BN>
static cudaError_t mmq_launch_bn(const MmqParams & P, dim3 grid, size_t smem, cudaStream_t st) {
    static FuncAttrCache attr_cache;
    cudaError_t e = ensure_dyn_smem(attr_cache, (const void *) k_mmq_tc<TYPE, BN>, smem, false);
    if (e != cudaSuccess) return e;
    k_mmq_tc<TYPE, BN><<<grid, MMQ_THREADS, smem, st>>>(P);
    return cudaGetLastError();
}
template <int TYPE>
static cudaError_t mmq_launch_typed(const MmqParams & P, int bn, dim3 grid, size_t smem, cudaStream_t st) {
    switch (bn) {
        case 16: return mmq_launch_bn<TYPE, 16>(P, grid, smem, st);
        case 32: return mmq_launch_bn<TYPE, 32>(P, grid, smem, st);
        case 64: return mmq_launch_bn<TYPE, 64>(P, grid, smem, st);
        default: return mmq_launch_bn<TYPE, 128>(P, grid, smem, st);
    }
}

cudaError_t launch_mmq(int type, const void * W, int64_t N, int64_t K, const float * x, int64_t ldx, int64_t T, float * dst, const float * bias,
                       const float * resid, void * ws, cudaStream_t st, bool reuse_prep, const MmqPre * pre) {
    if (pre && pre->kind != PRO_NONE && (!pre->aux || K % 256 != 0 || (pre->kind != PRO_RMSNORM && pre->kind != PRO_SILU_MUL))) return cudaErrorInvalidValue;
    if (!mmq_supported(type, K) || N <= 0 || T <= 0) return cudaErrorInvalidValue;
    const int BN = mmq_pick_bn((int) T);
    const int tpad = (int) ((T + BN - 1) / BN * BN);

    MmqParams P{};
    P.abort_flag = abort_flag();
    P.W = (const uint8_t *) W;
    P.B = (const uint8_t *) ws;
    float * rscale = reinterpret_cast<float *>((uint8_t *) ws + (size_t) tpad * (size_t) K * 2);   // behind the image (mmq_workspace_bytes)
    P.rscale = rscale;
    P.dst = dst;
    P.bias = bias;
    P.resid = resid;
    P.row_bytes = row_bytes(type, K);
    P.total_bytes = P.row_bytes * N;
    P.N = (int) N;
    P.K = (int) K;
    P.T = (int) T;
    // bytes of one 256-K group of a row, and the 16-byte aligned window reserved for it (Q6_K and Q8_0 rows are not 16-B aligned)
    // (Q4_0 / Q5_0 groups start 2-byte aligned, Q4_1 ones 8-byte aligned: their window is one 16-byte piece longer than the group)
    const bool legacy = type == T_Q4_0 || type == T_Q4_1 || type == T_Q5_0;
    P.bpb = legacy ? (int) row_bytes(type, 256)
                   : type == T_Q4_K ? BYTES_Q4_K : type == T_Q5_K ? BYTES_Q5_K : type == T_Q6_K ? BYTES_Q6_K : type == T_Q8_0 ? 8 * BYTES_Q8_0 : 8 * BYTES_Q5_1;
    P.slot = legacy ? P.bpb + 16 : type == T_Q6_K ? 240 : (type == T_Q8_0 ? 288 : P.bpb);
    P.rtiles = (int) ((N + MMQ_BM - 1) / MMQ_BM);
    const int ttiles = tpad / BN;
    P.ngrp = (int) ((K / MMQ_BK + 3) / 4);
    // stream-K: the tiles' K groups, tile after tile, in equal contiguous shares; a share is at least MMQ_MIN_UNITS groups (a segment's
    // pipeline fill + epilogue must stay small against its MMA steps) unless the whole launch is smaller than that
    const int64_t total = (int64_t) P.rtiles * ttiles * P.ngrp;
    if (total > 0x7fffffff) return cudaErrorInvalidValue;
    P.total_units = (int) total;
    const int nsm = sm_count();                // CTAs that can be resident: one CTA per SM
    int upc = (int) ((total + nsm - 1) / nsm);
    upc = std::max(upc, std::min(MMQ_MIN_UNITS, P.ngrp));
    P.upc = upc;
    const int grid_x = (int) ((total + upc - 1) / upc);
    const bool split = upc % P.ngrp != 0;      // some tile is shared by two CTAs: partial results meet in dst by atomic add
    if (!reuse_prep) {
        static FuncAttrCache prep_attr;
        const size_t prep_smem = mmq_prep_smem(K);
        cudaError_t e0 = ensure_dyn_smem(prep_attr, (const void *) k_mmq_prep, prep_smem, false);
        if (e0 != cudaSuccess) return e0;
        k_mmq_prep<<<tpad, 256, prep_smem, st>>>(x, ldx, (int) T, (int) K, BN, (uint8_t *) ws, rscale, is_kquant(type) ? 0 : 1, pre ? pre->kind : PRO_NONE,
                                                 pre ? pre->aux : nullptr, pre ? pre->ld_aux : 0, pre ? pre->eps : 0.f);
        e0 = cudaGetLastError();
        if (e0 != cudaSuccess) return e0;
    }
    if (split) {
        cudaError_t e0 = cudaMemsetAsync(dst, 0, (size_t) T * (size_t) N * sizeof(float), st);
        if (e0 != cudaSuccess) return e0;
    }
    auto smem_for = [&](int nraw, int b_nst) {
        return 1024 + (size_t) P.a_nst * MMQ_A_BYTES + (size_t) b_nst * BN * 128 + (size_t) nraw * MMQ_BM * P.slot + MMQ_CTL_BYTES;
    };
    // 2 expanded-weight stages, 3 raw slots if they fit, then as many activation stages (2..4) as the 227 KB budget leaves
    P.a_nst = 2;
    P.nraw = 3;
    if (smem_for(3, 2) > 232448) P.nraw = 2;
    P.b_nst = MMQ_B_NST;
    while (P.b_nst > 2 && smem_for(P.nraw, P.b_nst) > 232448) P.b_nst--;
    const size_t smem = smem_for(P.nraw, P.b_nst);
    if (smem > 232448) return cudaErrorInvalidConfiguration;
    dim3 grid((unsigned) grid_x, 1, 1);
    if (type == T_Q4_K) return mmq_launch_typed<T_Q4_K>(P, BN, grid, smem, st);
    if (type == T_Q5_K) return mmq_launch_typed<T_Q5_K>(P, BN, grid, smem, st);
    if (type == T_Q6_K) return mmq_launch_typed<T_Q6_K>(P, BN, grid, smem, st);
    if (type == T_Q8_0) return mmq_launch_typed<T_Q8_0>(P, BN, grid, smem, st);
    if (type == T_Q4_0) return mmq_launch_typed<T_Q4_0>(P, BN, grid, smem, st);
    if (type == T_Q4_1) return mmq_launch_typed<T_Q4_1>(P, BN, grid, smem, st);
    if (type == T_Q5_0) return mmq_launch_typed<T_Q5_0>(P, BN, grid, smem, st);
    return mmq_launch_typed<T_Q5_1>(P, BN, grid, smem, st);
}

}  // namespace pb
