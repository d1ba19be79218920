// prima.cpp_b200/csrc/quantize.cuh — the activation producers' arithmetic (silu, the rms_norm scale, q8_K / q8_0 / q8_1),
// bit-exact with the CPU backend.  Every kernel that produces an activation calls these, so that arithmetic is written once.
//
// Replaces (different numerics on purpose, see SURVEY §0 trap #1): quantize_q8_1 ggml-cuda/quantize.cu:4-38.
// Follows: quantize_row_q8_K_ref ggml-quants.c:3785-3822 (Q8_K), quantize_row_q8_0 AVX2 branch ggml-quants.c:943-1010
// (Q8_0), quantize_row_q8_1 AVX2 branch ggml-quants.c:1260-1330 (Q8_1).
// One warp quantizes 256 consecutive values: lane l owns x[8l .. 8l+7].
#pragma once
#include "common.cuh"

namespace pb {

__device__ __forceinline__ float silu_f(float x) { return __fdiv_rn(x, 1.0f + expf(-x)); }   // ggml.c:2560

// rms_norm's scale from the double-precision sum of squares of its n values (ggml.c:11976-11984)
__device__ __forceinline__ float rms_scale(double sumsq, int n, float eps) {
    const float mean = (float) (sumsq / (double) n);
    return __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(mean, eps)));
}
// rms_scale of x[0..n) by a whole CTA of 256 threads: per-thread strided double sums, warp sums, thread 0 adds the 8 warps in order.
// Every thread calls it and gets the scale.
__device__ __forceinline__ float block_rms_scale(const float * __restrict__ x, int n, float eps) {
    __shared__ double red[8];
    __shared__ float s_scale;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double sum = 0.0;
    for (int i = threadIdx.x; i < n; i += 256) sum += (double) __fmul_rn(x[i], x[i]);
    sum = warp_sum_d(sum);
    if (lane == 0) red[warp] = sum;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0;
        for (int i = 0; i < 8; i++) t += red[i];
        s_scale = rms_scale(t, n, eps);
    }
    __syncthreads();
    return s_scale;
}

// nearest_int of ggml-quants.c:1639-1644 (round-half-even via the 1.5*2^23 magic add), bit-exact
__device__ __forceinline__ int nearest_int_magic(float f) {
    float v = __fadd_rn(f, 12582912.f);
    return (__float_as_int(v) & 0x007fffff) - 0x00400000;
}

// q8_K, first half: this lane's first-occurrence arg-max of |v| (the CPU loop uses a strict '>' so ties keep the earlier element);
// v[0] is element i0 of the super-block.  The caller folds the lanes with warp_argmax / argmax_combine.
template <int N>
__device__ __forceinline__ void q8K_lane_absmax(const float (&v)[N], int i0, float & amax, float & vmax, int & idx) {
    amax = 0.f; vmax = 0.f; idx = 0x7fffffff;
#pragma unroll
    for (int i = 0; i < N; i++) {
        const float ax = fabsf(v[i]);
        if (ax > amax) { amax = ax; vmax = v[i]; idx = i0 + i; }
    }
}
// q8_K, second half: from the super-block's arg-max (amax = |vmax|) each value's q = min(nearest_int(iscale * v), 127) with
// iscale = -127 / vmax; returns d = 1 / iscale.  An all-zero super-block gives q = 0 and d = 0.
template <int N>
__device__ __forceinline__ float q8K_quant(const float (&v)[N], float amax, float vmax, int (&q)[N]) {
    if (amax == 0.f) {
#pragma unroll
        for (int i = 0; i < N; i++) q[i] = 0;
        return 0.f;
    }
    const float iscale = __fdiv_rn(-127.f, vmax);
#pragma unroll
    for (int i = 0; i < N; i++) {
        const int t = nearest_int_magic(__fmul_rn(iscale, v[i]));
        q[i] = t < 127 ? t : 127;
    }
    return __fdiv_rn(1.f, iscale);
}

// q8_0 / q8_1 of the 32-value block of lanes 4j..4j+3 (this lane's 8 values are v): amax over the 4 lanes, q = round-half-even(v * 127 /
// amax) (== _mm256_round_ps(_MM_ROUND_NEAREST)).  Returns d = amax / 127 before its f16 rounding: the stored d is f16(d), q8_1's
// s = f16(d * sum).  Every lane of the warp calls it.
__device__ __forceinline__ float q8_01_quant(const float (&v)[8], int (&q)[8]) {
    float amax = 0.f;
#pragma unroll
    for (int i = 0; i < 8; i++) amax = fmaxf(amax, fabsf(v[i]));
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
    const float id = amax != 0.f ? __fdiv_rn(127.f, amax) : 0.f;
#pragma unroll
    for (int i = 0; i < 8; i++) q[i] = __float2int_rn(__fmul_rn(v[i], id));
    return __fdiv_rn(amax, 127.f);
}
// q[0..N) as int8 bytes: byte i & 3 of word i >> 2; sum = q[0] + ... + q[N-1]
template <int N>
__device__ __forceinline__ void pack_q8(const int (&q)[N], uint32_t (&packed)[N / 4], int & sum) {
    sum = 0;
#pragma unroll
    for (int i = 0; i < N / 4; i++) packed[i] = 0u;
#pragma unroll
    for (int i = 0; i < N; i++) {
        sum += q[i];
        packed[i >> 2] |= (uint32_t)(q[i] & 0xff) << (8 * (i & 3));
    }
}

// v[8]: this lane's 8 values of super-block `blk` (values beyond K must be passed as 0 and K must be a multiple of 256).
__device__ __forceinline__ void quantize_warp_q8K(const float (&v)[8], int lane, int64_t blk, const ActQ & out) {
    float amax, vmax;
    int idx;
    q8K_lane_absmax(v, lane * 8, amax, vmax, idx);
    warp_argmax(amax, idx, &vmax);
    int q[8];
    const float d = q8K_quant(v, amax, vmax, q);
    uint32_t packed[2];
    int sum;
    pack_q8(q, packed, sum);
    *reinterpret_cast<uint2 *>(out.qs + blk * act_qs_stride(out) + lane * 8) = make_uint2(packed[0], packed[1]);
    int other = __shfl_xor_sync(0xffffffffu, sum, 1);
    if ((lane & 1) == 0) out.bsums[blk * act_bs_stride(out) + (lane >> 1)] = (int16_t)(sum + other);
    if (lane == 0) out.d[blk] = d;
}

// Q8_0 / Q8_1: 32-value blocks = 4 lanes; `blk` indexes the 256-value group => 8 small blocks.
template <bool WITH_SUM>
__device__ __forceinline__ void quantize_warp_q8_01(const float (&v)[8], int lane, int64_t blk, const ActQ & out) {
    int q[8];
    const float d = q8_01_quant(v, q);
    uint32_t packed[2];
    int sum;
    pack_q8(q, packed, sum);
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
