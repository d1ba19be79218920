// prima.cpp_b200/csrc/quantize.cuh — activation quantization, bit-exact with the CPU backend's from_float.
//
// Replaces (different numerics on purpose, see SURVEY §0 trap #1): quantize_q8_1 ggml-cuda/quantize.cu:4-38.
// Follows: quantize_row_q8_K_ref ggml-quants.c:3785-3822 (Q8_K), quantize_row_q8_0 AVX2 branch ggml-quants.c:943-1010
// (Q8_0), quantize_row_q8_1 AVX2 branch ggml-quants.c:1260-1330 (Q8_1).
// One warp quantizes 256 consecutive values: lane l owns x[8l .. 8l+7].
#pragma once
#include "common.cuh"

namespace pb {

// v[8]: this lane's 8 values of super-block `blk` (values beyond K must be passed as 0 and K must be a multiple of 256).
__device__ __forceinline__ void quantize_warp_q8K(const float (&v)[8], int lane, int64_t blk, const ActQ & out) {
    // first-occurrence argmax of |x| (the CPU loop uses a strict '>' so ties keep the earlier element)
    float amax = 0.f, vmax = 0.f;
    int idx = 0x7fffffff;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        float ax = fabsf(v[i]);
        if (ax > amax) { amax = ax; vmax = v[i]; idx = lane * 8 + i; }
    }
    warp_argmax(amax, idx, &vmax);
    uint32_t packed[2] = {0u, 0u};
    int sum = 0;
    float d = 0.f;
    if (amax != 0.f) {
        const float iscale = __fdiv_rn(-127.f, vmax);
#pragma unroll
        for (int i = 0; i < 8; i++) {
            int q = nearest_int_magic(__fmul_rn(iscale, v[i]));
            q = q < 127 ? q : 127;
            sum += q;
            packed[i >> 2] |= (uint32_t)(q & 0xff) << (8 * (i & 3));
        }
        d = __fdiv_rn(1.f, iscale);
    }
    *reinterpret_cast<uint2 *>(out.qs + blk * act_qs_stride(out) + lane * 8) = make_uint2(packed[0], packed[1]);
    int other = __shfl_xor_sync(0xffffffffu, sum, 1);
    if ((lane & 1) == 0) out.bsums[blk * act_bs_stride(out) + (lane >> 1)] = (int16_t)(sum + other);
    if (lane == 0) out.d[blk] = d;
}

// Q8_0 / Q8_1: 32-value blocks = 4 lanes; `blk` indexes the 256-value group => 8 small blocks.
template <bool WITH_SUM>
__device__ __forceinline__ void quantize_warp_q8_01(const float (&v)[8], int lane, int64_t blk, const ActQ & out) {
    float amax = 0.f;
#pragma unroll
    for (int i = 0; i < 8; i++) amax = fmaxf(amax, fabsf(v[i]));
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
    const float d = __fdiv_rn(amax, 127.f);
    const float id = amax != 0.f ? __fdiv_rn(127.f, amax) : 0.f;
    uint32_t packed[2] = {0u, 0u};
    int sum = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        int q = __float2int_rn(__fmul_rn(v[i], id));   // round-half-even == _mm256_round_ps(_MM_ROUND_NEAREST)
        sum += q;
        packed[i >> 2] |= (uint32_t)(q & 0xff) << (8 * (i & 3));
    }
    *reinterpret_cast<uint2 *>(out.qs + blk * 256 + lane * 8) = make_uint2(packed[0], packed[1]);
    if (WITH_SUM) {
        sum += __shfl_xor_sync(0xffffffffu, sum, 1);
        sum += __shfl_xor_sync(0xffffffffu, sum, 2);
    }
    if ((lane & 3) == 0) {
        const int64_t sb = blk * 8 + (lane >> 2);
        out.d[sb] = __half2float(__float2half_rn(d));
        if (WITH_SUM) out.s[sb] = __half2float(__float2half_rn(__fmul_rn(d, (float) sum)));
    }
}

__device__ __forceinline__ void quantize_warp(int mode, const float (&v)[8], int lane, int64_t blk, const ActQ & out) {
    if (mode == ACT_Q8_K) quantize_warp_q8K(v, lane, blk, out);
    else if (mode == ACT_Q8_0) quantize_warp_q8_01<false>(v, lane, blk, out);
    else quantize_warp_q8_01<true>(v, lane, blk, out);
}

}  // namespace pb
