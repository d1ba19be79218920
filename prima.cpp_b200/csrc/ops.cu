// prima.cpp_b200/csrc/ops.cu — the non-GEMV ops of the decode graph, fused the way the decode loop needs them.
//
// Reference ops replaced (file:line under the reference's ggml/src/ggml-cuda): quantize.cu:4-38 (activation quant),
// norm.cu:100-132 (rms_norm_f32) + binbcast.cu (MUL by the norm weight), rope.cu:32-109, cpy.cu:34 (f32->f16 KV store),
// softmax.cu:14-116, the FA-off attention chain ggml-cuda.cu:1737-1881 (batched cuBLAS KQ / KQV), unary.cu (silu),
// getrows.cu.  Numerics follow the CPU backend (ggml.c:11950, 14143, 13783, 12377), see each kernel.
#include "launch.h"
#include "quantize.cuh"
#include "rope.cuh"

#include <math.h>

#include <algorithm>

namespace pb {

// ------------------------------------------------------------------------------------------------
// activation quantization of x (u == nullptr) or of silu(x) * u: one warp per 256 values
__global__ void __launch_bounds__(256) k_quantize_act(const float * __restrict__ x, const float * __restrict__ u, int K, int mode, ActQ out) {
    pdl_trigger();   // dependents may launch now; they still wait for this grid's completion in their own pdl_wait()
    pdl_wait();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t blk = (int64_t) blockIdx.x * 8 + warp;
    const int64_t base = blk * 256 + lane * 8;
    if (blk * 256 >= K) return;
    float v[8];
    if (base + 8 <= K && ((((uintptr_t) x) | ((uintptr_t) u)) & 15) == 0) {   // both operands in flight before either is used
        const float4 x0 = __ldcg(reinterpret_cast<const float4 *>(x + base)), x1 = __ldcg(reinterpret_cast<const float4 *>(x + base + 4));
        v[0] = x0.x; v[1] = x0.y; v[2] = x0.z; v[3] = x0.w; v[4] = x1.x; v[5] = x1.y; v[6] = x1.z; v[7] = x1.w;
        if (u) {
            const float4 u0 = __ldcg(reinterpret_cast<const float4 *>(u + base)), u1 = __ldcg(reinterpret_cast<const float4 *>(u + base + 4));
            const float uv[8] = {u0.x, u0.y, u0.z, u0.w, u1.x, u1.y, u1.z, u1.w};
#pragma unroll
            for (int i = 0; i < 8; i++) v[i] = __fmul_rn(silu_f(v[i]), uv[i]);
        }
    } else {
#pragma unroll
        for (int i = 0; i < 8; i++) v[i] = base + i >= K ? 0.f : u ? __fmul_rn(silu_f(x[base + i]), u[base + i]) : x[base + i];
    }
    quantize_warp(mode, v, lane, blk, out);
}

// ------------------------------------------------------------------------------------------------
// y = rms_norm(x) * w, then quantize; single CTA (n <= 32 K), double-precision sum of squares like ggml.c:11976-11984
__global__ void __launch_bounds__(1024) k_rmsnorm_quant(const float * __restrict__ x, const float * __restrict__ w, int n, float eps, int mode,
                                                        ActQ out, float * __restrict__ f32_out) {
    __shared__ double red[32];
    __shared__ float s_scale;
    pdl_trigger();   // dependents may launch now; they still wait for this grid's completion in their own pdl_wait()
    pdl_wait();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double sum = 0.0;
    for (int i = threadIdx.x; i < n; i += 1024) {
        const float v = x[i];
        sum += (double) __fmul_rn(v, v);
    }
    sum = warp_sum_d(sum);
    if (lane == 0) red[warp] = sum;
    __syncthreads();
    if (warp == 0) {
        double t = red[lane];
        t = warp_sum_d(t);
        if (lane == 0) s_scale = rms_scale(t, n, eps);
    }
    __syncthreads();
    const float scale = s_scale;
    const int ngroups = (n + 255) / 256;
    for (int gidx = warp; gidx < ngroups; gidx += 32) {
        const int base = gidx * 256 + lane * 8;
        float v[8];
#pragma unroll
        for (int i = 0; i < 8; i++) {
            float t = 0.f;
            if (base + i < n) {
                t = __fmul_rn(x[base + i], scale);          // ggml_vec_scale_f32
                if (w) t = __fmul_rn(t, w[base + i]);       // ggml_mul by the norm weight
                if (f32_out) f32_out[base + i] = t;
            }
            v[i] = t;
        }
        if (out.qs) quantize_warp(mode, v, lane, gidx, out);
    }
}

// Decode-path variant: q8_K( rms_norm(x) * w ) of one vector, ONE CTA of 16 warps.  The vector is read once (128-bit loads, all
// issued before anything is used) and stays in registers between the sum of squares and the quantization.  Under PDL the GEMV
// that consumes the result is already resident and streaming its weights while this runs; doing the same work in the prologue
// of each of its CTAs would read the whole vector from L2 once per CTA.
constexpr int RQ_WARPS = 16;   // RQ_B super-blocks per warp in registers: 2 (n <= 8192, ~64 registers: fits beside a resident GEMV CTA) or 4
template <int RQ_B>
__global__ void __launch_bounds__(RQ_WARPS * 32) k_rmsnorm_q8K(const float * __restrict__ x, const float * __restrict__ w, int n, float eps, ActQ out) {
    __shared__ double red[RQ_WARPS];
    pdl_trigger();
    pdl_wait();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nblk = n / 256;
    float xv[RQ_B][8], wv[RQ_B][8];
#pragma unroll
    for (int j = 0; j < RQ_B; j++) {
        const int b = warp + j * RQ_WARPS;
        if (b < nblk) {
            const float4 a0 = __ldcg(reinterpret_cast<const float4 *>(x + b * 256 + lane * 8)), a1 = __ldcg(reinterpret_cast<const float4 *>(x + b * 256 + lane * 8 + 4));
            xv[j][0] = a0.x; xv[j][1] = a0.y; xv[j][2] = a0.z; xv[j][3] = a0.w; xv[j][4] = a1.x; xv[j][5] = a1.y; xv[j][6] = a1.z; xv[j][7] = a1.w;
            const float4 w0 = *reinterpret_cast<const float4 *>(w + b * 256 + lane * 8), w1 = *reinterpret_cast<const float4 *>(w + b * 256 + lane * 8 + 4);
            wv[j][0] = w0.x; wv[j][1] = w0.y; wv[j][2] = w0.z; wv[j][3] = w0.w; wv[j][4] = w1.x; wv[j][5] = w1.y; wv[j][6] = w1.z; wv[j][7] = w1.w;
        }
    }
    double sum = 0.0;   // float products widened to double: exact partial sums, grouping does not matter (ggml.c:11976-11984)
#pragma unroll
    for (int j = 0; j < RQ_B; j++) {
        if (warp + j * RQ_WARPS < nblk) {
#pragma unroll
            for (int i = 0; i < 8; i++) sum += (double) __fmul_rn(xv[j][i], xv[j][i]);
        }
    }
    sum = warp_sum_d(sum);
    if (lane == 0) red[warp] = sum;
    __syncthreads();
    double t = 0.0;
#pragma unroll
    for (int i = 0; i < RQ_WARPS; i++) t += red[i];
    const float scale = rms_scale(t, n, eps);
#pragma unroll
    for (int j = 0; j < RQ_B; j++) {
        const int b = warp + j * RQ_WARPS;
        if (b < nblk) {
#pragma unroll
            for (int i = 0; i < 8; i++) xv[j][i] = __fmul_rn(__fmul_rn(xv[j][i], scale), wv[j][i]);
            quantize_warp_q8K(xv[j], lane, b, out);
        }
    }
}

// plain row-wise rms_norm for the plugin (no weight): one CTA per row
__global__ void __launch_bounds__(256) k_rms_norm_rows(const float * __restrict__ x, float * __restrict__ y, int n, float eps,
                                                       const float * __restrict__ w) {
    const float * xr = x + (int64_t) blockIdx.x * n;
    float * yr = y + (int64_t) blockIdx.x * n;
    const float scale = block_rms_scale(xr, n, eps);
    if (w) {   // the following MUL node by the norm weight (src/llama.cpp:9772-9802), same two roundings as the separate kernels
        for (int i = threadIdx.x; i < n; i += 256) yr[i] = __fmul_rn(__fmul_rn(xr[i], scale), w[i]);
    } else {
        for (int i = threadIdx.x; i < n; i += 256) yr[i] = __fmul_rn(xr[i], scale);
    }
}

// ------------------------------------------------------------------------------------------------
// generic rope for the plugin: one CTA per (token, head)
__global__ void k_rope(const float * __restrict__ x, float * __restrict__ y, int n_head, int D, int64_t tok_stride, int64_t head_stride,
                       const int32_t * __restrict__ pos, RopeParams rp, const float * __restrict__ freq_factors) {
    const int tok = blockIdx.x / n_head, h = blockIdx.x % n_head;
    const float * xs = x + tok * tok_stride + h * head_stride;
    float * yd = y + ((int64_t) tok * n_head + h) * D;
    const int half_dims = rp.n_dims / 2;
    const bool neox = rp.mode & 2;
    for (int pair = threadIdx.x; pair < half_dims; pair += blockDim.x) {
        float c, s;
        rope_cos_sin(rp, pos[tok], pair, freq_factors, c, s);
        const int i0 = neox ? pair : 2 * pair, i1 = neox ? pair + half_dims : 2 * pair + 1;
        float y0, y1;
        rope_rotate(xs[i0], xs[i1], c, s, y0, y1);
        yd[i0] = y0; yd[i1] = y1;
    }
    for (int i = rp.n_dims + threadIdx.x; i < D; i += blockDim.x) yd[i] = xs[i];
}

// GGML_OP_ROPE on f16 rows (ggml_compute_forward_rope_f16, ggml.c:14269-14380): f16 -> f32, rotate, round to f16.  One CTA per
// (token, head); each element is read and written by the same thread, so y may equal x (the in-place K-shift of a KV cache).
__global__ void k_rope_f16(const __half * x, __half * y, int n_head, int D, const int32_t * __restrict__ pos, RopeParams rp,
                           const float * __restrict__ freq_factors) {
    const int tok = blockIdx.x / n_head;
    const __half * xs = x + (int64_t) blockIdx.x * D;
    __half * yd = y + (int64_t) blockIdx.x * D;
    const int half_dims = rp.n_dims / 2;
    const bool neox = rp.mode & 2;
    for (int pair = threadIdx.x; pair < half_dims; pair += blockDim.x) {
        float c, s;
        rope_cos_sin(rp, pos[tok], pair, freq_factors, c, s);
        const int i0 = neox ? pair : 2 * pair, i1 = neox ? pair + half_dims : 2 * pair + 1;
        float y0, y1;
        rope_rotate(__half2float(xs[i0]), __half2float(xs[i1]), c, s, y0, y1);
        yd[i0] = __float2half_rn(y0); yd[i1] = __float2half_rn(y1);
    }
    for (int i = rp.n_dims + threadIdx.x; i < D; i += blockDim.x) yd[i] = xs[i];
}

// Context shift of one sequence slot of the engine's cache (llama_kv_cache_seq_rm + llama_kv_cache_seq_add, src/llama.cpp:4378-4427,
// then the K-shift graph of build_k_shift, :10665-10719): every cell c in [p0, p1) moves to c + delta (delta < 0); its K row becomes
// f16(rope(f32(K), pos = delta)) with the rotation of k_rope_f16, its V row is copied bit for bit.  Per layer the caches are
// [cell][n_head_kv * 128] f16.  One warp owns one (layer, K|V, kv head) column and walks its cells upwards, so the destination of a
// move lies in cells the warp has already read: a launch never writes a cell another warp has yet to read.  Lanes 0-15 hold the
// sixteen 16-byte pieces of an even cell's row, lanes 16-31 those of the following cell; KS_U cell pairs are loaded before any is
// stored.  NORM pairs are lane-local, NEOX pairs (d, d + 64) sit 8 lanes apart and are exchanged with a shuffle.  head_dim == n_dims
// == 128.  Thread 0 also moves the slot's device position by delta when it is >= p0.
constexpr int KS_U = 8;
constexpr int KS_WARPS = 4;
__global__ void __launch_bounds__(KS_WARPS * 32) k_kv_shift(__half * kc, __half * vc, int n_cols, int n_head_kv, int64_t layer_stride, int p0,
                                                            int p1, int delta, RopeParams rp, const float * __restrict__ freq_factors,
                                                            int32_t * tokpos) {
    if (blockIdx.x == 0 && threadIdx.x == 0 && tokpos[1] >= p0) tokpos[1] += delta;
    const int col = blockIdx.x * KS_WARPS + (threadIdx.x >> 5);
    if (col >= n_cols) return;
    const int lane = threadIdx.x & 31, piece = lane & 15, odd = lane >> 4;
    const int layer = col / (2 * n_head_kv), rem = col % (2 * n_head_kv);
    const bool is_k = rem < n_head_kv;
    const int64_t EK = (int64_t) n_head_kv * 128;
    __half * base = (is_k ? kc : vc) + layer * layer_stride + (int64_t) (rem % n_head_kv) * 128 + piece * 8;
    const bool neox = rp.mode & 2;
    // this lane's dims 8 piece .. 8 piece + 7: NORM pairs 4 piece + j (j < 4), NEOX pairs 8 (piece % 8) + j (j < 8)
    float cs[8], sn[8];
#pragma unroll
    for (int j = 0; j < 8; j++) {
        cs[j] = 1.f; sn[j] = 0.f;
        if (is_k && (neox || j < 4)) rope_cos_sin(rp, delta, neox ? 8 * (piece & 7) + j : 4 * piece + j, freq_factors, cs[j], sn[j]);
    }
    for (int c0 = p0; c0 < p1; c0 += 2 * KS_U) {
        uint4 r[KS_U];
#pragma unroll
        for (int u = 0; u < KS_U; u++) {
            const int cell = c0 + 2 * u + odd;
            r[u] = cell < p1 ? __ldcs(reinterpret_cast<const uint4 *>(base + cell * EK)) : make_uint4(0, 0, 0, 0);
        }
        __syncwarp();   // every load of this batch is done before any lane stores into a cell of it
#pragma unroll
        for (int u = 0; u < KS_U; u++) {
            const int cell = c0 + 2 * u + odd;
            if (is_k) {   // warp-uniform
                __half2 * h = reinterpret_cast<__half2 *>(&r[u]);
                float x[8];
#pragma unroll
                for (int j = 0; j < 4; j++) { const float2 f = __half22float2(h[j]); x[2 * j] = f.x; x[2 * j + 1] = f.y; }
                float y[8];
                if (neox) {
                    const bool lo = piece < 8;
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        const float o = __shfl_xor_sync(0xffffffffu, x[j], 8);
                        float y0, y1;
                        rope_rotate(lo ? x[j] : o, lo ? o : x[j], cs[j], sn[j], y0, y1);
                        y[j] = lo ? y0 : y1;
                    }
                } else {
#pragma unroll
                    for (int j = 0; j < 4; j++) rope_rotate(x[2 * j], x[2 * j + 1], cs[j], sn[j], y[2 * j], y[2 * j + 1]);
                }
#pragma unroll
                for (int j = 0; j < 4; j++) h[j] = __halves2half2(__float2half_rn(y[2 * j]), __float2half_rn(y[2 * j + 1]));
            }
            if (cell < p1) __stcs(reinterpret_cast<uint4 *>(base + (cell + delta) * EK), r[u]);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Softmax of one row S[0..n) in shared memory by a CTA of WARPS warps, in the order of the FA-off chain's CPU soft_max
// (ggml.c:13783): per-thread strided fmaxf, warp max, thread 0 folds the warps in order; e = expf(s - max) written back in place
// (MASKED: a -inf score gives 0); per-thread double sum, warp sum, thread 0 adds the warps in order.  Returns inv = float(1 / sum)
// to every thread, S then holds e.  Every thread calls it; S may have been written by any of them.  red / redd hold WARPS values
// and bc one, all in shared memory.
template <int WARPS, bool MASKED>
__device__ __forceinline__ float block_softmax(float * S, int n, float * red, double * redd, float * bc) {
    constexpr int NT = WARPS * 32;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();
    float m = -INFINITY;
    for (int p = threadIdx.x; p < n; p += NT) m = fmaxf(m, S[p]);
    m = warp_max(m);
    if (lane == 0) red[warp] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = red[0];
        for (int i = 1; i < WARPS; i++) t = fmaxf(t, red[i]);
        *bc = t;
    }
    __syncthreads();
    const float mx = *bc;
    double dsum = 0.0;
    for (int p = threadIdx.x; p < n; p += NT) {
        const float s = S[p];
        const float e = (MASKED && s == -INFINITY) ? 0.f : expf(__fsub_rn(s, mx));
        S[p] = e;
        dsum += (double) e;
    }
    dsum = warp_sum_d(dsum);
    if (lane == 0) redd[warp] = dsum;
    __syncthreads();   // also: every thread has read the max, bc is free
    if (threadIdx.x == 0) {
        double t = 0;
        for (int i = 0; i < WARPS; i++) t += redd[i];
        *bc = (float) (1.0 / t);
    }
    __syncthreads();
    return *bc;
}

// ------------------------------------------------------------------------------------------------
// Attention over the engine's cache, one CTA (8 warps) per (q head, token).  D == 128 (4 values per lane).
//   s[p] = sum_d f32(K16[p][d]) * f32(f16(q[d]))            (CPU: mul_mat with f16 src0 rounds src1 to f16, ggml.c:12445)
//   w    = softmax(s * scale)                               (ggml.c:13783; double sum, p = e * float(1/sum))
//   o[d] = sum_p f32(V16[p][d]) * f32(f16(w[p]))            (second mul_mat, probabilities rounded to f16)
// Token blockIdx.y attends to cache rows [0, pos], pos = pos_dev[blockIdx.y]; its q and out rows are tok_stride floats after the
// previous token's.  Warp w visits rows w, w + 8, ... in that order, four rows' loads in flight before any is used.
// FRESH = false: q is already rotated and every row is in the cache.
// FRESH = true (one token, pre-RoPE q / k / v of it): RoPE (ggml.c:14087-14266) of the CTA's q head and its kv head's k into shared
// memory, k / v rounded to f16 exactly like the cache store; row pos is read from there, and the first q head of each GQA group
// writes it to the cache for later tokens.
template <bool FRESH>
__global__ void __launch_bounds__(256) k_attn_rows(const float * __restrict__ q, const float * __restrict__ k, const float * __restrict__ v,
                                                   __half * __restrict__ kc, __half * __restrict__ vc, float * __restrict__ out, int n_head,
                                                   int n_head_kv, const int32_t * __restrict__ pos_dev, RopeParams rp,
                                                   const float * __restrict__ freq_factors, float scale, int64_t tok_stride) {
    constexpr int D = 128;
    extern __shared__ float sm[];   // S[n_kv_pad] | red[8][128]
    __shared__ float q_s[D];
    __shared__ __align__(16) __half k_s[D];
    __shared__ __align__(16) __half v_s[D];
    __shared__ float s_red[8];
    __shared__ double s_redd[8];
    __shared__ float s_bc;
    pdl_trigger();   // dependents may launch now; they still wait for this grid's completion in their own pdl_wait()
    pdl_wait();
    const int pos = pos_dev[blockIdx.y];
    const int n_kv = pos + 1;
    const int gqa = n_head / n_head_kv;
    const int h = blockIdx.x, hk = h / gqa;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t EK = (int64_t) n_head_kv * D;
    q += (int64_t) blockIdx.y * tok_stride + (int64_t) h * D;
    out += (int64_t) blockIdx.y * tok_stride + (int64_t) h * D;
    float * S = sm;
    float * red = sm + ((n_kv + 31) & ~31);

    float q0, q1, q2, q3;
    if constexpr (FRESH) {
        // RoPE: threads 0..63 rotate q (pair = tid), threads 64..127 rotate k, threads 128..255 convert v
        const int half_dims = rp.n_dims / 2;
        const bool neox = rp.mode & 2;
        if (threadIdx.x < 128) {
            const int pair = threadIdx.x & 63;
            const bool is_q = threadIdx.x < 64;
            const float * src = is_q ? q : k + (int64_t) hk * D;
            if (pair < half_dims) {
                float c, s;
                rope_cos_sin(rp, pos, pair, freq_factors, c, s);
                const int i0 = neox ? pair : 2 * pair, i1 = neox ? pair + half_dims : 2 * pair + 1;
                float y0, y1;
                rope_rotate(src[i0], src[i1], c, s, y0, y1);
                if (is_q) { q_s[i0] = __half2float(__float2half_rn(y0)); q_s[i1] = __half2float(__float2half_rn(y1)); }
                else { k_s[i0] = __float2half_rn(y0); k_s[i1] = __float2half_rn(y1); }
            }
            for (int i = rp.n_dims + pair; i < D; i += 64) {   // un-rotated tail when n_dims < D
                if (is_q) q_s[i] = __half2float(__float2half_rn(src[i]));
                else k_s[i] = __float2half_rn(src[i]);
            }
        } else {
            const int i = threadIdx.x - 128;
            v_s[i] = __float2half_rn(v[(int64_t) hk * D + i]);
        }
        __syncthreads();
        if (h % gqa == 0 && threadIdx.x < 32) {   // one CTA per kv head publishes the fresh row (8 B per lane, coalesced)
            *reinterpret_cast<uint2 *>(kc + (int64_t) pos * EK + (int64_t) hk * D + 4 * lane) = *reinterpret_cast<const uint2 *>(k_s + 4 * lane);
            *reinterpret_cast<uint2 *>(vc + (int64_t) pos * EK + (int64_t) hk * D + 4 * lane) = *reinterpret_cast<const uint2 *>(v_s + 4 * lane);
        }
        q0 = q_s[4 * lane]; q1 = q_s[4 * lane + 1]; q2 = q_s[4 * lane + 2]; q3 = q_s[4 * lane + 3];
    } else {
        const float4 qv = *reinterpret_cast<const float4 *>(q + 4 * lane);
        q0 = __half2float(__float2half_rn(qv.x)); q1 = __half2float(__float2half_rn(qv.y));
        q2 = __half2float(__float2half_rn(qv.z)); q3 = __half2float(__float2half_rn(qv.w));
    }
    for (int p0 = warp; p0 < n_kv; p0 += 32) {     // 4 positions per warp in flight: all K rows requested before any is used
        uint2 kraw[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int p = p0 + 8 * j;
            if (p < n_kv) {
                const __half * krow = FRESH && p == pos ? k_s : kc + (int64_t) p * EK + (int64_t) hk * D;
                kraw[j] = *reinterpret_cast<const uint2 *>(krow + 4 * lane);
            }
        }
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int p = p0 + 8 * j;
            if (p < n_kv) {
                const float2 k01 = __half22float2(*reinterpret_cast<const __half2 *>(&kraw[j].x));
                const float2 k23 = __half22float2(*reinterpret_cast<const __half2 *>(&kraw[j].y));
                float s = k01.x * q0;
                s = fmaf(k01.y, q1, s);
                s = fmaf(k23.x, q2, s);
                s = fmaf(k23.y, q3, s);
                s = warp_sum(s);
                if (lane == 0) S[p] = __fmul_rn(s, scale);
            }
        }
    }
    const float inv = block_softmax<8, false>(S, n_kv, s_red, s_redd, &s_bc);
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    for (int p0 = warp; p0 < n_kv; p0 += 32) {
        uint2 vraw[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int p = p0 + 8 * j;
            if (p < n_kv) {
                const __half * vrow = FRESH && p == pos ? v_s : vc + (int64_t) p * EK + (int64_t) hk * D;
                vraw[j] = *reinterpret_cast<const uint2 *>(vrow + 4 * lane);
            }
        }
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int p = p0 + 8 * j;
            if (p < n_kv) {
                const float w = __half2float(__float2half_rn(__fmul_rn(S[p], inv)));
                const float2 v01 = __half22float2(*reinterpret_cast<const __half2 *>(&vraw[j].x));
                const float2 v23 = __half22float2(*reinterpret_cast<const __half2 *>(&vraw[j].y));
                a0 = fmaf(v01.x, w, a0); a1 = fmaf(v01.y, w, a1); a2 = fmaf(v23.x, w, a2); a3 = fmaf(v23.y, w, a3);
            }
        }
    }
    *reinterpret_cast<float4 *>(red + warp * 128 + 4 * lane) = make_float4(a0, a1, a2, a3);
    __syncthreads();
    if (threadIdx.x < 128) {
        float t = 0.f;
#pragma unroll
        for (int i = 0; i < 8; i++) t += red[i * 128 + threadIdx.x];
        out[threadIdx.x] = t;
    }
}

// ------------------------------------------------------------------------------------------------
// Tiled prompt-processing attention: one CTA per (kv head, ATT_TQ consecutive tokens; 4, or 2 / 1 for long contexts).  Warp w =
// q head w of the GQA group (loops when gqa > 8) for those tokens; K and V stream through shared memory in 32-position tiles and every tile is used by all
// gqa x 4 query rows (a per-(head, token) grid re-reads K/V for every row: measured L2-bound at 7 TB/s, 0.6 ms per 70B layer at T = 512).  Numerics are the CPU
// graph's (FA off): q and the probabilities rounded to f16, softmax sum in double; scores of all rows live in shared memory,
// so this kernel serves n_kv up to ATTN_TILED_MAX_KV and the launcher falls back beyond that.
constexpr int ATT_TK = 32, ATT_KSTRIDE = 130;   // halves per K row in smem: 65 words => conflict-free column walks
template <int ATT_TQ>
__global__ void __launch_bounds__(256) k_attn_prefill_tiled(const float * __restrict__ q, const __half * __restrict__ kc,
                                                            const __half * __restrict__ vc, float * __restrict__ out, int n_head, int n_head_kv,
                                                            const int32_t * __restrict__ pos_dev, int n_tok, float scale, int n_kv_pad) {
    constexpr int D = 128;
    extern __shared__ __align__(16) uint8_t att_smem[];
    const int gqa = n_head / n_head_kv;
    const int hk = blockIdx.x, t0 = blockIdx.y * ATT_TQ;
    const int ntq = min(ATT_TQ, n_tok - t0);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t EK = (int64_t) n_head_kv * D;
    float * S = reinterpret_cast<float *>(att_smem);                           // [gqa * TQ][n_kv_pad]
    float * q_s = S + (size_t) gqa * ATT_TQ * n_kv_pad;                        // [gqa * TQ][128]   f16-rounded q as f32
    __half * kv_s = reinterpret_cast<__half *>(q_s + (size_t) gqa * ATT_TQ * D);   // [TK][KSTRIDE]
    __shared__ int s_nkv[ATT_TQ];
    if (threadIdx.x < ATT_TQ) s_nkv[threadIdx.x] = threadIdx.x < ntq ? pos_dev[t0 + threadIdx.x] + 1 : 0;
    for (int i = threadIdx.x; i < gqa * ATT_TQ * D; i += 256) {
        const int row = i / D, d = i - row * D, hh = row / ATT_TQ, tq = row - hh * ATT_TQ;
        q_s[i] = tq < ntq ? __half2float(__float2half_rn(q[((int64_t) (t0 + tq) * n_head + hk * gqa + hh) * D + d])) : 0.f;
    }
    __syncthreads();
    int n_kv_max = 0;
#pragma unroll
    for (int i = 0; i < ATT_TQ; i++) n_kv_max = max(n_kv_max, s_nkv[i]);

    // ---- scores: S[row][p] = scale * q_row . K[p] ----
    for (int p0 = 0; p0 < n_kv_max; p0 += ATT_TK) {
        __syncthreads();
        for (int i = threadIdx.x; i < ATT_TK * (D / 8); i += 256) {            // 16-byte pieces: 32 rows x 16
            const int r = i >> 4, c = i & 15;
            uint4 v = make_uint4(0, 0, 0, 0);
            if (p0 + r < n_kv_max) v = *reinterpret_cast<const uint4 *>(kc + (int64_t) (p0 + r) * EK + (int64_t) hk * D + c * 8);
            uint32_t * dst = reinterpret_cast<uint32_t *>(kv_s + r * ATT_KSTRIDE + c * 8);   // rows are only 4-byte aligned (260 B stride)
            dst[0] = v.x; dst[1] = v.y; dst[2] = v.z; dst[3] = v.w;
        }
        __syncthreads();
        for (int hh = warp; hh < gqa; hh += 8) {
            const __half2 * krow = reinterpret_cast<const __half2 *>(kv_s + lane * ATT_KSTRIDE);   // lane = position p0 + lane
            const float * qh = q_s + (size_t) hh * ATT_TQ * D;
            float a[ATT_TQ];
#pragma unroll
            for (int tq = 0; tq < ATT_TQ; tq++) a[tq] = 0.f;
#pragma unroll 8
            for (int d2 = 0; d2 < D / 2; d2++) {
                const float2 k2 = __half22float2(krow[d2]);
#pragma unroll
                for (int tq = 0; tq < ATT_TQ; tq++) {
                    const float2 qq = *reinterpret_cast<const float2 *>(qh + tq * D + 2 * d2);
                    a[tq] = fmaf(k2.x, qq.x, a[tq]);
                    a[tq] = fmaf(k2.y, qq.y, a[tq]);
                }
            }
            float * Sr = S + (size_t) hh * ATT_TQ * n_kv_pad + p0 + lane;
#pragma unroll
            for (int tq = 0; tq < ATT_TQ; tq++) Sr[(size_t) tq * n_kv_pad] = __fmul_rn(a[tq], scale);
        }
    }
    __syncthreads();
    // ---- softmax per row (warp per row): p = f16(exp(s - max) * float(1 / double sum)), causal length per token ----
    for (int row = warp; row < gqa * ATT_TQ; row += 8) {
        const int n_kv = s_nkv[row % ATT_TQ];
        float * Sr = S + (size_t) row * n_kv_pad;
        float m = -INFINITY;
        for (int p = lane; p < n_kv; p += 32) m = fmaxf(m, Sr[p]);
        m = warp_max(m);
        double dsum = 0.0;
        for (int p = lane; p < n_kv; p += 32) {
            const float e = expf(__fsub_rn(Sr[p], m));
            Sr[p] = e;
            dsum += (double) e;
        }
        dsum = warp_sum_d(dsum);
        const float inv = n_kv > 0 ? (float) (1.0 / dsum) : 0.f;
        for (int p = lane; p < n_kv_pad; p += 32) Sr[p] = p < n_kv ? __half2float(__float2half_rn(__fmul_rn(Sr[p], inv))) : 0.f;
    }
    // ---- out[row][:] = sum_p P[row][p] * V[p][:]   (lane owns 4 of the 128 dims) ----
    float acc[1][ATT_TQ][4];
    for (int hbase = 0; hbase < gqa; hbase += 8) {
        const int hh = hbase + warp;
#pragma unroll
        for (int tq = 0; tq < ATT_TQ; tq++) { acc[0][tq][0] = acc[0][tq][1] = acc[0][tq][2] = acc[0][tq][3] = 0.f; }
        for (int p0 = 0; p0 < n_kv_max; p0 += ATT_TK) {
            __syncthreads();
            for (int i = threadIdx.x; i < ATT_TK * (D / 8); i += 256) {
                const int r = i >> 4, c = i & 15;
                uint4 v = make_uint4(0, 0, 0, 0);
                if (p0 + r < n_kv_max) v = *reinterpret_cast<const uint4 *>(vc + (int64_t) (p0 + r) * EK + (int64_t) hk * D + c * 8);
                *reinterpret_cast<uint4 *>(kv_s + r * D + c * 8) = v;             // V tile dense: rows of 256 B
            }
            __syncthreads();
            if (hh < gqa) {
                const float * Pr = S + (size_t) hh * ATT_TQ * n_kv_pad + p0;
                const int np = min(ATT_TK, n_kv_max - p0);
                for (int j = 0; j < np; j++) {
                    const uint2 vraw = *reinterpret_cast<const uint2 *>(kv_s + j * D + 4 * lane);
                    const float2 v01 = __half22float2(*reinterpret_cast<const __half2 *>(&vraw.x));
                    const float2 v23 = __half22float2(*reinterpret_cast<const __half2 *>(&vraw.y));
#pragma unroll
                    for (int tq = 0; tq < ATT_TQ; tq++) {
                        const float w = Pr[(size_t) tq * n_kv_pad + j];
                        acc[0][tq][0] = fmaf(v01.x, w, acc[0][tq][0]); acc[0][tq][1] = fmaf(v01.y, w, acc[0][tq][1]);
                        acc[0][tq][2] = fmaf(v23.x, w, acc[0][tq][2]); acc[0][tq][3] = fmaf(v23.y, w, acc[0][tq][3]);
                    }
                }
            }
        }
        if (hh < gqa) {
#pragma unroll
            for (int tq = 0; tq < ATT_TQ; tq++)
                if (tq < ntq)
                    *reinterpret_cast<float4 *>(out + ((int64_t) (t0 + tq) * n_head + hk * gqa + hh) * D + 4 * lane) =
                        make_float4(acc[0][tq][0], acc[0][tq][1], acc[0][tq][2], acc[0][tq][3]);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Decode attention v2 (the engine's per-token path): same arithmetic as k_attn_rows<true>, restructured for LATENCY — under PDL this
// kernel sits between the q|k|v GEMV and the wo GEMV, and every microsecond of it is a bubble in the weight stream:
//   * one CTA of 16 warps per q head, launched as CLUSTERS OF 2 (heads 2j, 2j+1 = one 256-value q8_K super-block of the output):
//     the pair agrees on the block's arg-max through distributed shared memory and writes the QUANTIZED activation itself,
//     so the wo GEMV needs no quantize prologue;
//   * everything that does not depend on the q|k|v GEMV happens BEFORE griddepcontrol.wait: the position, the RoPE angles and
//     the K/V cache rows [0, pos) (written by earlier tokens) — up to 256 rows each are in flight as cp.async copies into
//     shared memory (completion on mbarriers) while the GEMV drains.  Round 1's kernel chained ~10 dependent L2 round trips
//     (pos -> q -> K rows 4 at a time -> V rows 4 at a time);
//   * longer contexts stream further 128-row chunks through the same two buffers per tensor.
constexpr int A2_THREADS = 512, A2_WARPS = 16, A2_CHUNK = 128;
struct __align__(128) Attn2Smem {   // fixed part; dynamic tail: S[n_ctx padded to 32] floats
    uint64_t kbar[2], vbar[2];
    float cand[4];                 // this CTA's arg-max candidate {amax, vmax, idx, -} for the cluster exchange
    float s_bc;                    // block_softmax broadcast
    volatile int aborted;          // wait watchdog (common.cuh)
    float s_red[A2_WARPS];
    double s_redd[A2_WARPS];
    __align__(16) float q_s[128];
    __align__(16) float o_s[128];
    __align__(16) float cs[64][2];
    __align__(16) __half k_s[128];
    __align__(16) __half v_s[128];
    __align__(16) float red[A2_WARPS][128];
    __align__(128) __half kbuf[2][A2_CHUNK][128];
    __align__(128) __half vbuf[2][A2_CHUNK][128];
};
static_assert(offsetof(Attn2Smem, red) % 16 == 0 && offsetof(Attn2Smem, kbuf) % 128 == 0 && sizeof(Attn2Smem) % 128 == 0, "Attn2Smem layout");
// K (both layouts) and the engine's row-major V: 128 cells x 256 B, one 16-byte piece per cp.async
__device__ __forceinline__ void a2_issue_chunk(__half (*dst)[128], const __half * cache, int64_t EK, int hk, int c, int ncell, uint64_t * bar) {
    const int r0 = c * A2_CHUNK;
    const int nrows = min(A2_CHUNK, ncell - r0);
    const int pieces = nrows * 16;                      // 16-byte pieces: 16 per 256-byte row
    for (int i = threadIdx.x; i < pieces; i += A2_THREADS) {
        const int r = i >> 4, cpart = i & 15;
        const __half * src = cache + (int64_t) (r0 + r) * EK + (int64_t) hk * 128 + cpart * 8;
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(&dst[r][cpart * 8])), "l"(src) : "memory");
    }
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");   // fires when this thread's copies have landed
}
// ggml's FA-off V cache is TRANSPOSED (llm_build_kv_store, src/llama.cpp:9698-9716): channel-major [n_embd_v_gqa][n_ctx].
// The chunk is staged as dst[channel][cell in chunk]; ncell and the chunk start are multiples of 8 cells (16-byte pieces).
__device__ __forceinline__ void a2_issue_chunk_vt(__half (*dst)[128], const __half * cache, int64_t vt_stride, int hk, int c, int ncell, uint64_t * bar) {
    const int r0 = c * A2_CHUNK;
    const int ncol = min(A2_CHUNK, ncell - r0);
    const int ppc = ncol >> 3;                           // pieces per channel
    const int pieces = 128 * ppc;
    for (int i = threadIdx.x; i < pieces; i += A2_THREADS) {
        const int d = i / ppc, part = i - d * ppc;
        const __half * src = cache + (int64_t) (hk * 128 + d) * vt_stride + r0 + part * 8;
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(&dst[d][part * 8])), "l"(src) : "memory");
    }
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ float ld_dsmem_f32(const float * local_addr, uint32_t cta_rank) {
    uint32_t remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(local_addr)), "r"(cta_rank));
    float v;
    asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(remote) : "memory");
    return v;
}

struct Attn2Params {
    const float * q; const float * k; const float * v;   // this token's projections (f32, pre-RoPE)
    __half * kc;                  // K cache [cell][n_head_kv * 128]
    __half * vc;                  // V cache: engine [cell][n_head_kv * 128]; GGML: transposed [n_head_kv * 128][vt_stride]
    float * out;                  // [n_head * 128]
    ActQ outq;                    // optional q8_K of out (qs == nullptr: skip)
    int n_head, n_head_kv;
    const int32_t * pos_dev;      // the token's position (RoPE); engine layout: also the cell it is stored in
    RopeParams rp;
    const float * freq_factors;
    float scale;
    int * abort_flag;
    // GGML layout only (the FA-off chain of llm_build_kqv, src/llama.cpp:10032-10165)
    int n_cells;                  // cells attended: the graph's n_kv (multiple of 32)
    int kv_head;                  // cell this token's K / V are stored in (offset of the cache views of llm_build_kv_store)
    const int32_t * kv_head_dev;  // if set: the cell is read from device memory instead (a captured CUDA graph is replayed with a new cell)
    int64_t vt_stride;            // elements between two channels of the transposed V cache (n_ctx)
    const float * mask;           // [n_cells] additive f32 mask row of this token (0 / -inf), soft_max_ext src1
};

// GGML = false: the engine's cache (V row-major, cell == position, causal window [0, pos]).
// GGML = true: the tensors of the reference's graph: K cache row-major, V cache transposed, explicit mask row, explicit cell.
template <bool GGML>
__global__ void __launch_bounds__(A2_THREADS, 1) k_attn2(const __grid_constant__ Attn2Params P) {
    constexpr int D = 128;
    extern __shared__ __align__(128) uint8_t a2_raw[];
    Attn2Smem * sm = reinterpret_cast<Attn2Smem *>(a2_raw);
    float * S = reinterpret_cast<float *>(a2_raw + sizeof(Attn2Smem));
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n_head = P.n_head, n_head_kv = P.n_head_kv;
    const int gqa = n_head / n_head_kv;
    const int h = blockIdx.x, hk = h / gqa;
    const int64_t EK = (int64_t) n_head_kv * D;
    __half * const kc = P.kc;
    __half * const vc = P.vc;
    if (threadIdx.x == 0) {
        mbar_init(&sm->kbar[0], A2_THREADS); mbar_init(&sm->kbar[1], A2_THREADS);
        mbar_init(&sm->vbar[0], A2_THREADS); mbar_init(&sm->vbar[1], A2_THREADS);
        sm->aborted = 0;
        mbar_fence_init();
    }
    __syncthreads();
    pdl_trigger();
    // ---- independent of the producing GEMV: position (written before this token's first kernel), cache cells of earlier tokens
    const int pos = *P.pos_dev;
    const int ncell = GGML ? P.n_cells : pos + 1;              // cells attended
    const int fresh = GGML ? (P.kv_head_dev ? *P.kv_head_dev : P.kv_head) : pos;                  // this token's cell: its K / V come from shared memory, not from the cache
    const int nchunks = (ncell + A2_CHUNK - 1) / A2_CHUNK;
    a2_issue_chunk(sm->kbuf[0], kc, EK, hk, 0, ncell, &sm->kbar[0]);
    if (nchunks > 1) a2_issue_chunk(sm->kbuf[1], kc, EK, hk, 1, ncell, &sm->kbar[1]);
    if (GGML) {
        a2_issue_chunk_vt(sm->vbuf[0], vc, P.vt_stride, hk, 0, ncell, &sm->vbar[0]);
        if (nchunks > 1) a2_issue_chunk_vt(sm->vbuf[1], vc, P.vt_stride, hk, 1, ncell, &sm->vbar[1]);
    } else {
        a2_issue_chunk(sm->vbuf[0], vc, EK, hk, 0, ncell, &sm->vbar[0]);
        if (nchunks > 1) a2_issue_chunk(sm->vbuf[1], vc, EK, hk, 1, ncell, &sm->vbar[1]);
    }
    const RopeParams & rp = P.rp;
    const int half_dims = rp.n_dims / 2;
    const bool neox = rp.mode & 2;
    if (threadIdx.x < 64 && (int) threadIdx.x < half_dims) {
        float c, s;
        rope_cos_sin(rp, pos, threadIdx.x, P.freq_factors, c, s);
        sm->cs[threadIdx.x][0] = c; sm->cs[threadIdx.x][1] = s;
    }
    pdl_wait();
    // ---- q / k / v of this token (f32, just produced): RoPE in shared memory, f16 rounding identical to the cache store
    float x0 = 0.f, x1 = 0.f, vv = 0.f;
    {
        const int t = threadIdx.x;
        if (t < 128) {
            const int pair = t & 63;
            const float * src = t < 64 ? P.q + (int64_t) h * D : P.k + (int64_t) hk * D;
            if (pair < half_dims) {
                const int i0 = neox ? pair : 2 * pair, i1 = neox ? pair + half_dims : 2 * pair + 1;
                x0 = __ldcg(src + i0); x1 = __ldcg(src + i1);
            }
        } else if (t < 256) {
            vv = __ldcg(P.v + (int64_t) hk * D + (t - 128));
        }
    }
    __syncthreads();   // cs[] visible
    {
        const int t = threadIdx.x;
        if (t < 128) {
            const int pair = t & 63;
            const bool is_q = t < 64;
            const float * src = is_q ? P.q + (int64_t) h * D : P.k + (int64_t) hk * D;
            if (pair < half_dims) {
                const int i0 = neox ? pair : 2 * pair, i1 = neox ? pair + half_dims : 2 * pair + 1;
                float y0, y1;
                rope_rotate(x0, x1, sm->cs[pair][0], sm->cs[pair][1], y0, y1);
                if (is_q) { sm->q_s[i0] = __half2float(__float2half_rn(y0)); sm->q_s[i1] = __half2float(__float2half_rn(y1)); }
                else { sm->k_s[i0] = __float2half_rn(y0); sm->k_s[i1] = __float2half_rn(y1); }
            }
            for (int i = rp.n_dims + pair; i < D; i += 64) {   // un-rotated tail when n_dims < D
                if (is_q) sm->q_s[i] = __half2float(__float2half_rn(__ldcg(src + i)));
                else sm->k_s[i] = __float2half_rn(__ldcg(src + i));
            }
        } else if (t < 256) {
            sm->v_s[t - 128] = __float2half_rn(vv);
        }
    }
    __syncthreads();
    if (h % gqa == 0) {   // one CTA per kv head publishes the fresh K / V
        if (threadIdx.x < 32) *reinterpret_cast<uint2 *>(kc + (int64_t) fresh * EK + (int64_t) hk * D + 4 * lane) = *reinterpret_cast<const uint2 *>(sm->k_s + 4 * lane);
        if (GGML) {
            if (threadIdx.x >= 128 && threadIdx.x < 256) vc[(int64_t) (hk * D + (threadIdx.x - 128)) * P.vt_stride + fresh] = sm->v_s[threadIdx.x - 128];
        } else {
            if (threadIdx.x < 32) *reinterpret_cast<uint2 *>(vc + (int64_t) fresh * EK + (int64_t) hk * D + 4 * lane) = *reinterpret_cast<const uint2 *>(sm->v_s + 4 * lane);
        }
    }
    const float q0 = sm->q_s[4 * lane], q1 = sm->q_s[4 * lane + 1], q2 = sm->q_s[4 * lane + 2], q3 = sm->q_s[4 * lane + 3];
    auto score_row = [&](const __half * krow) -> float {
        const uint2 kraw = *reinterpret_cast<const uint2 *>(krow + 4 * lane);
        const float2 k01 = __half22float2(*reinterpret_cast<const __half2 *>(&kraw.x));
        const float2 k23 = __half22float2(*reinterpret_cast<const __half2 *>(&kraw.y));
        float s = k01.x * q0;
        s = fmaf(k01.y, q1, s);
        s = fmaf(k23.x, q2, s);
        s = fmaf(k23.y, q3, s);
        return warp_sum(s);
    };
    // ---- scores  (soft_max_ext: s * scale, then + mask; ggml.c ggml_compute_forward_soft_max_f32)
    for (int c = 0; c < nchunks; c++) {
        const int b = c & 1;
        mbar_wait(&sm->kbar[b], (uint32_t) ((c >> 1) & 1), &sm->aborted, P.abort_flag);
        const int r0 = c * A2_CHUNK, nrows = min(A2_CHUNK, ncell - r0);
        for (int r = warp; r < nrows; r += A2_WARPS) {
            const int p = r0 + r;
            const float s = score_row(p == fresh ? sm->k_s : sm->kbuf[b][r]);
            if (lane == 0) {
                float t = __fmul_rn(s, P.scale);
                if (GGML) t = __fadd_rn(t, P.mask[p]);
                S[p] = t;
            }
        }
        if (c + 2 < nchunks) {
            __syncthreads();   // every warp is done with this buffer
            a2_issue_chunk(sm->kbuf[b], kc, EK, hk, c + 2, ncell, &sm->kbar[b]);
        }
    }
    // ---- softmax (max, expf, double sum, p = e * float(1/sum)); the GGML mask's -inf cells get 0
    const float inv = block_softmax<A2_WARPS, GGML>(S, ncell, sm->s_red, sm->s_redd, &sm->s_bc);
    if (GGML) {
        // ---- P.V over the transposed cache: warp w owns channels w, w+16, ...; lane l owns cells 2l, 2l+1, 64+2l, 64+2l+1 of a chunk
        for (int p = threadIdx.x; p < ncell; p += A2_THREADS) S[p] = __half2float(__float2half_rn(__fmul_rn(S[p], inv)));   // f16-rounded probabilities
        __syncthreads();
        float acc[8];
#pragma unroll
        for (int i = 0; i < 8; i++) acc[i] = 0.f;
        for (int c = 0; c < nchunks; c++) {
            const int b = c & 1;
            mbar_wait(&sm->vbar[b], (uint32_t) ((c >> 1) & 1), &sm->aborted, P.abort_flag);
            const int r0 = c * A2_CHUNK, ncol = min(A2_CHUNK, ncell - r0);
#pragma unroll
            for (int j = 0; j < 2; j++) {
                const int cl = 2 * lane + 64 * j;
                if (cl < ncol) {
                    const float w0 = S[r0 + cl], w1 = S[r0 + cl + 1];
#pragma unroll
                    for (int i = 0; i < 8; i++) {
                        const int d = warp + A2_WARPS * i;
                        float2 vf = __half22float2(*reinterpret_cast<const __half2 *>(&sm->vbuf[b][d][cl]));
                        if (r0 + cl == fresh) vf.x = __half2float(sm->v_s[d]);
                        if (r0 + cl + 1 == fresh) vf.y = __half2float(sm->v_s[d]);
                        acc[i] = fmaf(vf.x, w0, acc[i]);
                        acc[i] = fmaf(vf.y, w1, acc[i]);
                    }
                }
            }
            if (c + 2 < nchunks) {
                __syncthreads();
                a2_issue_chunk_vt(sm->vbuf[b], vc, P.vt_stride, hk, c + 2, ncell, &sm->vbar[b]);
            }
        }
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const float t = warp_sum(acc[i]);
            if (lane == 0) {
                const int d = warp + A2_WARPS * i;
                P.out[(int64_t) h * D + d] = t;
                sm->o_s[d] = t;
            }
        }
    } else {
        // ---- P.V with f16-rounded probabilities, row-major V: lane owns 4 channels, warps split the cells
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
        auto pv_row = [&](const __half * vrow, int p) {
            const float w = __half2float(__float2half_rn(__fmul_rn(S[p], inv)));
            const uint2 vraw = *reinterpret_cast<const uint2 *>(vrow + 4 * lane);
            const float2 v01 = __half22float2(*reinterpret_cast<const __half2 *>(&vraw.x));
            const float2 v23 = __half22float2(*reinterpret_cast<const __half2 *>(&vraw.y));
            a0 = fmaf(v01.x, w, a0); a1 = fmaf(v01.y, w, a1); a2 = fmaf(v23.x, w, a2); a3 = fmaf(v23.y, w, a3);
        };
        for (int c = 0; c < nchunks; c++) {
            const int b = c & 1;
            mbar_wait(&sm->vbar[b], (uint32_t) ((c >> 1) & 1), &sm->aborted, P.abort_flag);
            const int r0 = c * A2_CHUNK, nrows = min(A2_CHUNK, ncell - r0);
            for (int r = warp; r < nrows; r += A2_WARPS) pv_row(r0 + r == fresh ? sm->v_s : sm->vbuf[b][r], r0 + r);
            if (c + 2 < nchunks) {
                __syncthreads();
                a2_issue_chunk(sm->vbuf[b], vc, EK, hk, c + 2, ncell, &sm->vbar[b]);
            }
        }
        *reinterpret_cast<float4 *>(&sm->red[warp][4 * lane]) = make_float4(a0, a1, a2, a3);
        __syncthreads();
        if (threadIdx.x < 128) {
            float t = 0.f;
#pragma unroll
            for (int i = 0; i < A2_WARPS; i++) t += sm->red[i][threadIdx.x];
            P.out[(int64_t) h * D + threadIdx.x] = t;
            sm->o_s[threadIdx.x] = t;
        }
    }
    // ---- q8_K of the output: heads (2j, 2j+1) = cluster ranks (0, 1) = super-block j  (quantize_row_q8_K_ref, ggml-quants.c:3785-3822)
    const ActQ & outq = P.outq;
    if (outq.qs) {
        __syncthreads();
        const uint32_t rank = h & 1u;
        float xv[4];
        float amax, vmax;
        int idx;
        if (warp == 0) {
#pragma unroll
            for (int i = 0; i < 4; i++) xv[i] = sm->o_s[4 * lane + i];
            q8K_lane_absmax(xv, (int) rank * 128 + 4 * lane, amax, vmax, idx);
            warp_argmax(amax, idx, &vmax);
            if (lane == 0) { sm->cand[0] = amax; sm->cand[1] = vmax; sm->cand[2] = __int_as_float(idx); }
        }
        cluster_sync_all();
        if (warp == 0) {
            const float oa = ld_dsmem_f32(&sm->cand[0], rank ^ 1u), ov = ld_dsmem_f32(&sm->cand[1], rank ^ 1u);
            const int oi = __float_as_int(ld_dsmem_f32(&sm->cand[2], rank ^ 1u));
            argmax_combine(amax, idx, oa, oi, &vmax, ov);
            const int64_t blk = h >> 1;
            int qv[4];
            const float d = q8K_quant(xv, amax, vmax, qv);
            uint32_t packed[1];
            int sum;
            pack_q8(qv, packed, sum);
            *reinterpret_cast<uint32_t *>(outq.qs + blk * act_qs_stride(outq) + rank * 128 + 4 * lane) = packed[0];
            sum += __shfl_xor_sync(0xffffffffu, sum, 1);
            sum += __shfl_xor_sync(0xffffffffu, sum, 2);
            if ((lane & 3) == 0) outq.bsums[blk * act_bs_stride(outq) + rank * 8 + (lane >> 2)] = (int16_t) sum;
            if (rank == 0 && lane == 0) outq.d[blk] = d;
        }
        cluster_sync_all();   // the partner may still be reading this CTA's candidate
    }
}

// ------------------------------------------------------------------------------------------------
// soft_max_ext rows (plugin): y = softmax(x*scale + mask).  The row is staged in shared memory when it fits (in_smem), otherwise the
// softmax runs in place on the output row in global memory: same arithmetic in the same order, any row length.
__global__ void __launch_bounds__(256) k_soft_max(const float * __restrict__ x, const float * __restrict__ mask, float * __restrict__ y, int ncols,
                                                  int64_t rows_per_mask_cycle, float scale, bool in_smem) {
    extern __shared__ float sm[];
    __shared__ float s_red[8];
    __shared__ double s_redd[8];
    __shared__ float s_b;
    const int64_t row = blockIdx.x;
    const float * xr = x + row * ncols;
    const float * mr = mask ? mask + (row % rows_per_mask_cycle) * ncols : nullptr;
    float * yr = y + row * ncols;
    float * S = in_smem ? sm : yr;
    for (int i = threadIdx.x; i < ncols; i += 256) {
        float v = __fmul_rn(xr[i], scale);
        if (mr) v = __fadd_rn(v, mr[i]);
        S[i] = v;
    }
    const float inv = block_softmax<8, true>(S, ncols, s_red, s_redd, &s_b);
    for (int i = threadIdx.x; i < ncols; i += 256) yr[i] = __fmul_rn(S[i], inv);   // element i: written and read by the same thread
}

// ------------------------------------------------------------------------------------------------
// get_rows: y[i][e] = dequant(table[ids[i]])[e]   (dequantize_row_q*_K, ggml-quants.c:2555-3006, 1589-1634)
__device__ float dequant_elem(int type, const uint8_t * row, int e) {
    switch (type) {
        case T_F32: return reinterpret_cast<const float *>(row)[e];
        case T_F16: return __half2float(reinterpret_cast<const __half *>(row)[e]);
        case T_Q8_0: {
            const uint8_t * b = row + (int64_t) (e / 32) * BYTES_Q8_0;
            const float d = __half2float(__ushort_as_half(*reinterpret_cast<const uint16_t *>(b)));
            return __fmul_rn((float) (int) (signed char) b[2 + (e & 31)], d);
        }
        case T_Q5_1: {
            const uint8_t * b = row + (int64_t) (e / 32) * BYTES_Q5_1;
            const float d = __half2float(__ushort_as_half(*reinterpret_cast<const uint16_t *>(b)));
            const float m = __half2float(__ushort_as_half(*reinterpret_cast<const uint16_t *>(b + 2)));
            const uint32_t qh = *reinterpret_cast<const uint32_t *>(b + 4);
            const int j = e & 31;
            const int q = j < 16 ? ((b[8 + j] & 0xF) | (((qh >> j) & 1) << 4)) : ((b[8 + j - 16] >> 4) | (((qh >> j) & 1) << 4));
            return __fadd_rn(__fmul_rn((float) q, d), m);
        }
        case T_Q4_0:
        case T_Q4_1:
        case T_Q5_0: {   // dequantize_row_q4_0 / _q4_1 / _q5_0, ggml-quants.c:1522-1580
            const int bb = type == T_Q4_0 ? BYTES_Q4_0 : type == T_Q4_1 ? BYTES_Q4_1 : BYTES_Q5_0;
            const uint8_t * b = row + (int64_t) (e / 32) * bb;
            const float d = __half2float(__ushort_as_half((uint16_t) (b[0] | (b[1] << 8))));
            const int j = e & 31;
            const uint8_t * qs = b + (type == T_Q4_0 ? 2 : type == T_Q4_1 ? 4 : 6);
            int q = j < 16 ? (qs[j] & 0xF) : (qs[j - 16] >> 4);
            if (type == T_Q4_1) return __fadd_rn(__fmul_rn((float) q, d), __half2float(__ushort_as_half((uint16_t) (b[2] | (b[3] << 8)))));
            if (type == T_Q5_0) q = (q | (((b[2 + j / 8] >> (j & 7)) & 1) << 4)) - 16;
            else q -= 8;
            return __fmul_rn((float) q, d);
        }
        case T_Q4_K:
        case T_Q5_K: {
            const bool q5 = type == T_Q5_K;
            const uint8_t * b = row + (int64_t) (e / 256) * (q5 ? BYTES_Q5_K : BYTES_Q4_K);
            const int i = e & 255, j = i / 32, l = i & 31;
            const float d = __half2float(__ushort_as_half(*reinterpret_cast<const uint16_t *>(b)));
            const float dmin = __half2float(__ushort_as_half(*reinterpret_cast<const uint16_t *>(b + 2)));
            const uint8_t * scb = b + 4;
            int sc, mn;
            if (j < 4) { sc = scb[j] & 63; mn = scb[j + 4] & 63; }
            else { sc = (scb[j + 4] & 0xF) | ((scb[j - 4] >> 6) << 4); mn = (scb[j + 4] >> 4) | ((scb[j] >> 6) << 4); }
            const uint8_t * qs = b + (q5 ? 48 : 16);
            const uint8_t byte = qs[32 * (j / 2) + l];
            int qv = (j & 1) ? (byte >> 4) : (byte & 0xF);
            if (q5 && ((b[16 + l] >> j) & 1)) qv += 16;
            return __fsub_rn(__fmul_rn(__fmul_rn(d, (float) sc), (float) qv), __fmul_rn(dmin, (float) mn));
        }
        case T_Q6_K: {
            const uint8_t * b = row + (int64_t) (e / 256) * BYTES_Q6_K;
            const int i = e & 255, n = i / 128, r = i & 127, quarter = r / 32, l = r & 31;
            const uint8_t * ql = b + 64 * n, * qh = b + 128 + 32 * n;
            const int8_t * sc = reinterpret_cast<const int8_t *>(b + 192) + 8 * n;
            const float d = __half2float(__ushort_as_half(*reinterpret_cast<const uint16_t *>(b + 208)));
            const uint8_t lo = (quarter & 1) ? ql[l + 32] : ql[l];
            const int nib = (quarter & 2) ? (lo >> 4) : (lo & 0xF);
            const int qv = (nib | (((qh[l] >> (2 * quarter)) & 3) << 4)) - 32;
            return __fmul_rn(__fmul_rn(d, (float) sc[l / 16 + 2 * quarter]), (float) qv);
        }
    }
    return 0.f;
}

// Ids on grid.y, which is capped at 65 535: a CTA row takes ids blockIdx.y, blockIdx.y + gridDim.y, ...
__global__ void __launch_bounds__(256) k_get_rows(const uint8_t * __restrict__ table, int type, int K, int64_t row_bytes_,
                                                  const int32_t * __restrict__ ids, int n_ids, float * __restrict__ y) {
    pdl_trigger();   // dependents may launch now; they still wait for this grid's completion in their own pdl_wait()
    pdl_wait();
    const int e = blockIdx.x * 256 + threadIdx.x;
    if (e >= K) return;
    for (int64_t i = blockIdx.y; i < n_ids; i += gridDim.y) y[i * K + e] = dequant_elem(type, table + (int64_t) ids[i] * row_bytes_, e);
}

// ------------------------------------------------------------------------------------------------
__global__ void k_binary(int op, const float * __restrict__ a, const float * __restrict__ b, float * __restrict__ y, int64_t n, int64_t nb) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float bv = b[i % nb];
    y[i] = op == 0 ? __fadd_rn(a[i], bv) : __fmul_rn(a[i], bv);
}
__global__ void k_silu(const float * __restrict__ x, float * __restrict__ y, int64_t n) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] = silu_f(x[i]);
}
__global__ void k_silu_mul(const float * __restrict__ g, const float * __restrict__ u, float * __restrict__ y, int64_t n) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] = __fmul_rn(silu_f(g[i]), u[i]);
}
__global__ void k_cpy_f32_f16(const float * __restrict__ x, __half * __restrict__ y, int64_t n) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] = __float2half_rn(x[i]);
}

// ------------------------------------------------------------------------------------------------
// generic 4-D strided copy f32 -> f32 / f16 (CPY, CONT, DUP of views: K store, transposed V store, kqv merge)
struct Copy4 { int64_t ne[4]; int64_t sb[4]; int64_t db[4]; };   // element counts, src / dst BYTE strides
template <typename T>
__global__ void k_copy_strided(const char * __restrict__ src, char * __restrict__ dst, Copy4 c, int64_t n) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    // dst index space is enumerated in dst logical order; src may have a different shape with the same element count
    int64_t r = i;
    const int64_t i0 = r % c.ne[0]; r /= c.ne[0];
    const int64_t i1 = r % c.ne[1]; r /= c.ne[1];
    const int64_t i2 = r % c.ne[2]; r /= c.ne[2];
    const int64_t i3 = r;
    const float v = *reinterpret_cast<const float *>(src + i0 * c.sb[0] + i1 * c.sb[1] + i2 * c.sb[2] + i3 * c.sb[3]);
    T * d = reinterpret_cast<T *>(dst + i0 * c.db[0] + i1 * c.db[1] + i2 * c.db[2] + i3 * c.db[3]);
    if constexpr (sizeof(T) == 2) *d = __float2half_rn(v); else *d = v;
}

// dst[i0,i1,i2,i3] = sum_k src0_f16[k,i0,i2/r2,i3/r3] * f16(src1_f32[k,i1,i2,i3])   (ggml mul_mat with F16 src0: the CPU backend
// rounds src1 to f16 and accumulates in f32, ggml.c:12445-12473).  One warp per output element; byte strides.
struct MM16 { int64_t K, ne0, ne1, ne2, ne3, r2, r3; int64_t a[4]; int64_t b[4]; int64_t d[4]; };
__global__ void __launch_bounds__(256) k_mul_mat_f16(const char * __restrict__ A, const char * __restrict__ B, char * __restrict__ D, MM16 m) {
    const int64_t w = (int64_t) blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    const int64_t total = m.ne0 * m.ne1 * m.ne2 * m.ne3;
    if (w >= total) return;
    int64_t r = w;
    const int64_t i0 = r % m.ne0; r /= m.ne0;
    const int64_t i1 = r % m.ne1; r /= m.ne1;
    const int64_t i2 = r % m.ne2; r /= m.ne2;
    const int64_t i3 = r;
    const char * a = A + i0 * m.a[1] + (i2 / m.r2) * m.a[2] + (i3 / m.r3) * m.a[3];
    const char * b = B + i1 * m.b[1] + i2 * m.b[2] + i3 * m.b[3];
    float acc = 0.f;
    for (int64_t k = lane; k < m.K; k += 32) {
        const float av = __half2float(*reinterpret_cast<const __half *>(a + k * m.a[0]));
        const float bv = __half2float(__float2half_rn(*reinterpret_cast<const float *>(b + k * m.b[0])));
        acc = fmaf(av, bv, acc);
    }
    acc = warp_sum(acc);
    if (lane == 0) *reinterpret_cast<float *>(D + i0 * m.d[0] + i1 * m.d[1] + i2 * m.d[2] + i3 * m.d[3]) = acc;
}

// ------------------------------------------------------------------------------------------------
// GGML_OP_FLASH_ATTN_EXT (ggml_cuda_flash_attn_ext, ggml-cuda/fattn.cu:298-345; CPU: ggml_compute_forward_flash_attn_ext_f16,
// ggml.c:15538-15748): out[h][t] = softmax(scale * K q + slope * mask) . V with f16 K / V, one CTA per (token, head).
// The 8 warps split the KV range and each runs the online softmax (running max M, sum S, f32 accumulator: one lane owns the
// dimensions lane, lane + 32, ...), then the partial results are merged like the reference's split-KV combine
// (flash_attn_combine_results, fattn-common.cuh:519-561).  Cells whose mask is -inf are skipped as on the CPU; ALiBi slope and
// logit soft-cap follow ggml.c:15601-15605, 15652-15656.  Any head size up to 256 (64 / 80 / 128 / 256 in the reference's tests).
constexpr int FA_WARPS = 8, FA_MAXD = 256;
struct FlashParams {
    const float * q; const __half * k; const __half * v; const __half * mask; float * dst;
    int D, n_tok, n_head, n_head_kv, n_kv;
    int64_t q_nb1, q_nb2, k_nb1, k_nb2, v_nb1, v_nb2, mask_nb1;    // bytes
    float scale, max_bias, softcap, m0, m1;
    int n_head_log2;
};
__global__ void __launch_bounds__(FA_WARPS * 32) k_flash_attn_ext(const __grid_constant__ FlashParams P) {
    __shared__ float s_q[FA_MAXD];
    __shared__ float s_acc[FA_WARPS][FA_MAXD];
    __shared__ float s_M[FA_WARPS], s_S[FA_WARPS];
    const int t = blockIdx.x, h = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int D = P.D;
    const int hk = h / (P.n_head / P.n_head_kv);
    const float * q = reinterpret_cast<const float *>(reinterpret_cast<const char *>(P.q) + t * P.q_nb1 + h * P.q_nb2);
    // the CPU converts q to f16 before the dot (q_to_vec_dot, ggml.c:15630): same rounding here
    for (int d = threadIdx.x; d < D; d += FA_WARPS * 32) s_q[d] = __half2float(__float2half_rn(q[d]));
    __syncthreads();
    const float slope = P.max_bias > 0.0f ? (h < P.n_head_log2 ? powf(P.m0, (float) (h + 1)) : powf(P.m1, (float) (2 * (h - P.n_head_log2) + 1))) : 1.0f;
    const __half * mp = P.mask ? reinterpret_cast<const __half *>(reinterpret_cast<const char *>(P.mask) + t * P.mask_nb1) : nullptr;
    constexpr int NPL = FA_MAXD / 32;
    float qr[NPL], acc[NPL];
#pragma unroll
    for (int i = 0; i < NPL; i++) { const int d = lane + 32 * i; qr[i] = d < D ? s_q[d] : 0.f; acc[i] = 0.f; }
    float M = -INFINITY, S = 0.f;
    float scale = P.scale;
    if (P.softcap != 0.0f) scale /= P.softcap;
    for (int c = warp; c < P.n_kv; c += FA_WARPS) {
        const float mv = mp ? slope * __half2float(mp[c]) : 0.0f;
        if (mv == -INFINITY) continue;
        const __half * kr = reinterpret_cast<const __half *>(reinterpret_cast<const char *>(P.k) + c * P.k_nb1 + hk * P.k_nb2);
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < NPL; i++) { const int d = lane + 32 * i; if (d < D) s = fmaf(__half2float(kr[d]), qr[i], s); }
        s = warp_sum(s);
        s *= scale;
        if (P.softcap != 0.0f) s = P.softcap * tanhf(s);
        s += mv;
        float ms = 1.0f, vs = 1.0f;
        if (s > M) { ms = expf(M - s); M = s; } else { vs = expf(s - M); }
        const __half * vr = reinterpret_cast<const __half *>(reinterpret_cast<const char *>(P.v) + c * P.v_nb1 + hk * P.v_nb2);
#pragma unroll
        for (int i = 0; i < NPL; i++) { const int d = lane + 32 * i; if (d < D) acc[i] = fmaf(__half2float(vr[d]), vs, acc[i] * ms); }
        S = S * ms + vs;
    }
    if (lane == 0) { s_M[warp] = M; s_S[warp] = S; }
#pragma unroll
    for (int i = 0; i < NPL; i++) { const int d = lane + 32 * i; if (d < D) s_acc[warp][d] = acc[i]; }
    __syncthreads();
    float Mg = -INFINITY;
#pragma unroll
    for (int w = 0; w < FA_WARPS; w++) Mg = fmaxf(Mg, s_M[w]);
    float Sg = 0.f;
#pragma unroll
    for (int w = 0; w < FA_WARPS; w++) Sg += s_M[w] == -INFINITY ? 0.f : s_S[w] * expf(s_M[w] - Mg);
    const float inv = 1.0f / Sg;
    float * out = P.dst + ((int64_t) t * P.n_head + h) * D;      // dst is [D, n_head, n_tok] (the op writes the permuted result)
    for (int d = threadIdx.x; d < D; d += FA_WARPS * 32) {
        float a = 0.f;
#pragma unroll
        for (int w = 0; w < FA_WARPS; w++) a += s_M[w] == -INFINITY ? 0.f : s_acc[w][d] * expf(s_M[w] - Mg);
        out[d] = a * inv;
    }
}

// ================================================================================================ launchers
int launch_copy_strided(const void * src, void * dst, int dst_is_f16, const int64_t ne[4], const int64_t sb[4], const int64_t db[4], cudaStream_t stream) {
    Copy4 c;
    int64_t n = 1;
    for (int i = 0; i < 4; i++) { c.ne[i] = ne[i]; c.sb[i] = sb[i]; c.db[i] = db[i]; n *= ne[i]; }
    if (n == 0) return 0;
    if (dst_is_f16) k_copy_strided<__half><<<(unsigned) ((n + 255) / 256), 256, 0, stream>>>((const char *) src, (char *) dst, c, n);
    else k_copy_strided<float><<<(unsigned) ((n + 255) / 256), 256, 0, stream>>>((const char *) src, (char *) dst, c, n);
    return (int) cudaGetLastError();
}
int launch_mul_mat_f16(const void * A, const void * B, void * D, int64_t K, const int64_t ne[4], int64_t r2, int64_t r3, const int64_t ab[4],
                       const int64_t bb[4], const int64_t db[4], cudaStream_t stream) {
    MM16 m;
    m.K = K; m.ne0 = ne[0]; m.ne1 = ne[1]; m.ne2 = ne[2]; m.ne3 = ne[3]; m.r2 = r2; m.r3 = r3;
    for (int i = 0; i < 4; i++) { m.a[i] = ab[i]; m.b[i] = bb[i]; m.d[i] = db[i]; }
    const int64_t total = ne[0] * ne[1] * ne[2] * ne[3];
    if (total == 0) return 0;
    k_mul_mat_f16<<<(unsigned) ((total + 7) / 8), 256, 0, stream>>>((const char *) A, (const char *) B, (char *) D, m);
    return (int) cudaGetLastError();
}

int launch_quantize_act(const float * x, const float * up, int K, int mode, const ActQ & out, cudaStream_t stream, bool pdl) {
    const int ngroups = (K + 255) / 256;
    LaunchCfg lc(dim3((ngroups + 7) / 8), dim3(256), 0, stream, pdl);
    return (int) cudaLaunchKernelEx(&lc.cfg, k_quantize_act, x, up, K, mode, out);
}
int launch_rmsnorm_quant(const float * x, const float * w, int n, float eps, int mode, const ActQ & out, float * f32_out, cudaStream_t stream, bool pdl) {
    if (mode == ACT_Q8_K && w && !f32_out && out.qs && n % 256 == 0 && n / 256 <= RQ_WARPS * 4 && ((uintptr_t) x & 15) == 0 && ((uintptr_t) w & 15) == 0) {
        LaunchCfg lc(dim3(1), dim3(RQ_WARPS * 32), 0, stream, pdl);
        if (n / 256 <= RQ_WARPS * 2) return (int) cudaLaunchKernelEx(&lc.cfg, k_rmsnorm_q8K<2>, x, w, n, eps, out);
        return (int) cudaLaunchKernelEx(&lc.cfg, k_rmsnorm_q8K<4>, x, w, n, eps, out);
    }
    LaunchCfg lc(dim3(1), dim3(1024), 0, stream, pdl);
    return (int) cudaLaunchKernelEx(&lc.cfg, k_rmsnorm_quant, x, w, n, eps, mode, out, f32_out);
}
int launch_rms_norm(const float * x, float * y, int n, int64_t nrows, float eps, cudaStream_t stream, const float * w) {
    k_rms_norm_rows<<<(unsigned) nrows, 256, 0, stream>>>(x, y, n, eps, w);
    return (int) cudaGetLastError();
}

static float rope_yarn_corr_dim(int n_dims, int n_ctx_orig, float n_rot, float base) {
    return n_dims * logf(n_ctx_orig / (n_rot * 2 * (float) M_PI)) / (2 * logf(base));
}
void rope_params_init(RopeParams & rp, int n_dims, int mode, int n_ctx_orig, float freq_base, float freq_scale, float ext_factor, float attn_factor,
                      float beta_fast, float beta_slow) {
    rp.n_dims = n_dims; rp.mode = mode; rp.n_ctx_orig = n_ctx_orig;
    rp.freq_base = freq_base; rp.freq_scale = freq_scale; rp.ext_factor = ext_factor; rp.attn_factor = attn_factor;
    rp.beta_fast = beta_fast; rp.beta_slow = beta_slow;
    rp.theta_scale = powf(freq_base, -2.0f / n_dims);
    const float start = floorf(rope_yarn_corr_dim(n_dims, n_ctx_orig, beta_fast, freq_base));
    const float end = ceilf(rope_yarn_corr_dim(n_dims, n_ctx_orig, beta_slow, freq_base));
    rp.corr_dims[0] = fmaxf(0.f, start);
    rp.corr_dims[1] = fminf((float) n_dims - 1, end);
}

int launch_rope(const float * x, float * y, int64_t ntok, int n_head, int D, int64_t tok_stride, int64_t head_stride, const int32_t * pos,
                const RopeParams & rp, const float * freq_factors, cudaStream_t stream) {
    k_rope<<<(unsigned) (ntok * n_head), 64, 0, stream>>>(x, y, n_head, D, tok_stride, head_stride, pos, rp, freq_factors);
    return (int) cudaGetLastError();
}

int launch_rope_f16(const __half * x, __half * y, int64_t ntok, int n_head, int D, const int32_t * pos, const RopeParams & rp, const float * freq_factors,
                    cudaStream_t stream) {
    k_rope_f16<<<(unsigned) (ntok * n_head), 64, 0, stream>>>(x, y, n_head, D, pos, rp, freq_factors);
    return (int) cudaGetLastError();
}

int launch_kv_shift(__half * kc, __half * vc, int n_layer, int n_head_kv, int n_ctx, int p0, int p1, int delta, const RopeParams & rp,
                    const float * freq_factors, int32_t * tokpos, cudaStream_t stream) {
    const int n_cols = n_layer * 2 * n_head_kv;
    const int grid = std::max(1, (n_cols + KS_WARPS - 1) / KS_WARPS);   // at least one CTA: the slot position moves on shards without layers too
    k_kv_shift<<<grid, KS_WARPS * 32, 0, stream>>>(kc, vc, n_cols, n_head_kv, (int64_t) n_ctx * n_head_kv * 128, p0, p1, delta, rp, freq_factors, tokpos);
    return (int) cudaGetLastError();
}

// k_attn_rows<FRESH> for n_head heads x n_tok tokens (q / out rows tok_stride floats apart), scores of up to n_kv_max cells.
// Dynamic shared memory: the score row padded to 32 plus red[8][128]; cudaErrorNotSupported when that exceeds the device's limit.
static FuncAttrCache attn_rows_attr[2];
static size_t attn_rows_smem(int n_kv_max) { return ((size_t) ((n_kv_max + 31) & ~31) + 8 * 128) * sizeof(float); }
int attn_rows_max_kv() {
    const size_t lim = std::min(dyn_smem_limit(attn_rows_attr[0], (const void *) k_attn_rows<false>),
                                dyn_smem_limit(attn_rows_attr[1], (const void *) k_attn_rows<true>));
    const int64_t n = (int64_t) (lim / sizeof(float)) - 8 * 128;   // largest padded row with attn_rows_smem(n) <= lim
    return n > 0 ? (int) (n & ~31) : 0;
}
template <bool FRESH>
static int launch_attn_rows(const float * q, const float * k, const float * v, __half * kc, __half * vc, float * out, int n_head, int n_head_kv,
                            const int32_t * pos_dev, const RopeParams & rp, const float * freq_factors, float scale, int n_tok, int64_t tok_stride,
                            int n_kv_max, cudaStream_t stream, bool pdl) {
    const size_t smem = attn_rows_smem(n_kv_max);
    {
        cudaError_t e = ensure_dyn_smem(attn_rows_attr[FRESH], (const void *) k_attn_rows<FRESH>, smem, false);
        if (e != cudaSuccess) return (int) e;
    }
    LaunchCfg lc(dim3(n_head, n_tok), dim3(256), smem, stream, pdl);
    return (int) cudaLaunchKernelEx(&lc.cfg, k_attn_rows<FRESH>, q, k, v, kc, vc, out, n_head, n_head_kv, pos_dev, rp, freq_factors, scale, tok_stride);
}
// k_attn_rows<false> only reads the caches
int launch_attn_decode(const float * q, const __half * kcache, const __half * vcache, float * out, int n_head, int n_head_kv, int D,
                       const int32_t * pos_dev, int n_ctx, float scale, cudaStream_t stream, bool pdl) {
    if (D != 128) return (int) cudaErrorInvalidValue;
    return launch_attn_rows<false>(q, nullptr, nullptr, const_cast<__half *>(kcache), const_cast<__half *>(vcache), out, n_head, n_head_kv, pos_dev,
                                   RopeParams{}, nullptr, scale, 1, 0, n_ctx, stream, pdl);
}
// prefill: n_tok query rows (strides in floats), token t attends to cache rows [0, pos_dev[t]]
int launch_attn_batch(const float * q, const __half * kcache, const __half * vcache, float * out, int n_head, int n_head_kv, int D,
                      const int32_t * pos_dev, int n_tok, int n_kv_max, float scale, cudaStream_t stream) {
    if (D != 128 || n_tok <= 0 || n_tok > 65535) return (int) cudaErrorInvalidValue;
    if (n_head % n_head_kv == 0) {   // tiled kernel: all score rows of gqa x TQ queries in shared memory
        const int gqa = n_head / n_head_kv;
        const int n_kv_pad = (n_kv_max + 31) & ~31;
        auto smem_for = [&](int tq) { return (size_t) gqa * tq * n_kv_pad * 4 + (size_t) gqa * tq * D * 4 + (size_t) ATT_TK * ATT_KSTRIDE * 2; };
        const int tq = smem_for(4) <= 200 * 1024 ? 4 : (smem_for(2) <= 200 * 1024 ? 2 : (smem_for(1) <= 200 * 1024 ? 1 : 0));
        if (tq) {
            const size_t smem_t = smem_for(tq);
            static FuncAttrCache attr_t[5];
            const void * fn = tq == 4 ? (const void *) k_attn_prefill_tiled<4> : (tq == 2 ? (const void *) k_attn_prefill_tiled<2> : (const void *) k_attn_prefill_tiled<1>);
            {
                cudaError_t e = ensure_dyn_smem(attr_t[tq], fn, smem_t, false);
                if (e != cudaSuccess) return (int) e;
            }
            const dim3 grid(n_head_kv, (n_tok + tq - 1) / tq);
            if (tq == 4) k_attn_prefill_tiled<4><<<grid, 256, smem_t, stream>>>(q, kcache, vcache, out, n_head, n_head_kv, pos_dev, n_tok, scale, n_kv_pad);
            else if (tq == 2) k_attn_prefill_tiled<2><<<grid, 256, smem_t, stream>>>(q, kcache, vcache, out, n_head, n_head_kv, pos_dev, n_tok, scale, n_kv_pad);
            else k_attn_prefill_tiled<1><<<grid, 256, smem_t, stream>>>(q, kcache, vcache, out, n_head, n_head_kv, pos_dev, n_tok, scale, n_kv_pad);
            return (int) cudaGetLastError();
        }
    }
    return launch_attn_rows<false>(q, nullptr, nullptr, const_cast<__half *>(kcache), const_cast<__half *>(vcache), out, n_head, n_head_kv, pos_dev,
                                   RopeParams{}, nullptr, scale, n_tok, (int64_t) n_head * D, n_kv_max, stream, false);
}

static FuncAttrCache attn2_attr[2];   // k_attn2<false>, k_attn2<true>
int attn2_max_cells() {
    const size_t lim = std::min({(size_t) 200 * 1024, dyn_smem_limit(attn2_attr[0], (const void *) k_attn2<false>),
                                 dyn_smem_limit(attn2_attr[1], (const void *) k_attn2<true>)});
    return lim > sizeof(Attn2Smem) ? (int) (((lim - sizeof(Attn2Smem)) / sizeof(float)) & ~(size_t) 31) : 0;
}
// k_attn2: cudaErrorNotSupported for shapes the clustered kernel does not take (odd n_head, scores beyond attn2_max_cells())
template <bool GGML>
static int launch_attn2(Attn2Params & P, int n_score_slots, cudaStream_t stream, bool pdl) {
    if ((P.n_head & 1) || P.n_head_kv <= 0 || P.n_head % P.n_head_kv || n_score_slots > attn2_max_cells()) return (int) cudaErrorNotSupported;
    const size_t smem = sizeof(Attn2Smem) + (size_t) ((n_score_slots + 31) & ~31) * sizeof(float);
    {
        cudaError_t e = ensure_dyn_smem(attn2_attr[GGML], (const void *) k_attn2<GGML>, smem, false);
        if (e != cudaSuccess) return (int) e;
    }
    P.abort_flag = abort_flag();
    LaunchCfg lc(dim3(P.n_head), dim3(A2_THREADS), smem, stream, pdl, 2);
    return (int) cudaLaunchKernelEx(&lc.cfg, k_attn2<GGML>, P);
}
int launch_attn_step(const float * q, const float * k, const float * v, __half * kcache, __half * vcache, float * out, const ActQ & outq,
                     int outq_mode, int n_head, int n_head_kv, int D, const int32_t * pos_dev, int n_ctx, const RopeParams & rp,
                     const float * freq_factors, float scale, cudaStream_t stream, bool pdl, bool & quantized) {
    quantized = false;
    if (D != 128) return (int) cudaErrorInvalidValue;
    // k_attn2 when the output feeds a q8_K GEMV whose ring kernel can stage it
    if (outq_mode == ACT_Q8_K && gemv_fused_prologue_ok(n_head * D)) {
        Attn2Params P{};
        P.q = q; P.k = k; P.v = v; P.kc = kcache; P.vc = vcache; P.out = out; P.outq = outq; P.n_head = n_head; P.n_head_kv = n_head_kv;
        P.pos_dev = pos_dev; P.rp = rp; P.freq_factors = freq_factors; P.scale = scale;
        const int rc = launch_attn2<false>(P, n_ctx, stream, pdl);
        if (rc != (int) cudaErrorNotSupported) {
            quantized = rc == 0;
            return rc;
        }
    }
    return launch_attn_rows<true>(q, k, v, kcache, vcache, out, n_head, n_head_kv, pos_dev, rp, freq_factors, scale, 1, 0, n_ctx, stream, pdl);
}
// the reference graph's tensors (FA off): K cache rows, transposed V cache, explicit mask row and destination cell
int launch_attn_ggml(const float * q, const float * k, const float * v, __half * kcache, __half * vcache_t, int64_t vt_stride, float * out, const ActQ & outq,
                     int n_head, int n_head_kv, int D, const int32_t * pos_dev, int n_cells, int kv_head, const int32_t * kv_head_dev, const float * mask,
                     const RopeParams & rp, const float * freq_factors, float scale, cudaStream_t stream, bool pdl) {
    if (D != 128 || n_cells <= 0 || (n_cells & 7) || kv_head < 0 || kv_head >= n_cells || (vt_stride & 7) || ((uintptr_t) vcache_t & 15) || ((uintptr_t) kcache & 15) || !mask)
        return (int) cudaErrorNotSupported;
    Attn2Params P{};
    P.q = q; P.k = k; P.v = v; P.kc = kcache; P.vc = vcache_t; P.out = out; P.outq = outq; P.n_head = n_head; P.n_head_kv = n_head_kv;
    P.pos_dev = pos_dev; P.rp = rp; P.freq_factors = freq_factors; P.scale = scale;
    P.n_cells = n_cells; P.kv_head = kv_head; P.kv_head_dev = kv_head_dev; P.vt_stride = vt_stride; P.mask = mask;
    return launch_attn2<true>(P, n_cells, stream, pdl);
}

int launch_flash_attn_ext(const float * q, const void * k, const void * v, const void * mask, float * dst, int D, int n_tok, int n_head, int n_head_kv,
                          int n_kv, const int64_t * q_nb, const int64_t * k_nb, const int64_t * v_nb, int64_t mask_nb1, float scale, float max_bias,
                          float softcap, cudaStream_t stream) {
    if (D <= 0 || D > FA_MAXD || n_tok <= 0 || n_head <= 0 || n_head_kv <= 0 || n_head % n_head_kv || n_tok > 2147483647 || n_head > 65535)
        return (int) cudaErrorInvalidValue;
    FlashParams P{};
    P.q = q; P.k = (const __half *) k; P.v = (const __half *) v; P.mask = (const __half *) mask; P.dst = dst;
    P.D = D; P.n_tok = n_tok; P.n_head = n_head; P.n_head_kv = n_head_kv; P.n_kv = n_kv;
    P.q_nb1 = q_nb[0]; P.q_nb2 = q_nb[1]; P.k_nb1 = k_nb[0]; P.k_nb2 = k_nb[1]; P.v_nb1 = v_nb[0]; P.v_nb2 = v_nb[1]; P.mask_nb1 = mask_nb1;
    P.scale = scale; P.max_bias = max_bias; P.softcap = softcap;
    P.n_head_log2 = 1;
    while (P.n_head_log2 * 2 <= n_head) P.n_head_log2 *= 2;
    P.m0 = powf(2.0f, -max_bias / P.n_head_log2);
    P.m1 = powf(2.0f, -(max_bias / 2.0f) / P.n_head_log2);
    k_flash_attn_ext<<<dim3(n_tok, n_head), FA_WARPS * 32, 0, stream>>>(P);
    return (int) cudaGetLastError();
}

static FuncAttrCache sm_attr;   // k_soft_max
size_t soft_max_smem(int ncols, size_t * static_bytes) {
    const size_t bytes = (size_t) ncols * sizeof(float);
    const size_t limit = dyn_smem_limit(sm_attr, (const void *) k_soft_max);
    if (static_bytes) *static_bytes = sm_attr.stat[cur_device()];
    return limit && bytes > limit ? 0 : bytes;   // 0: the row does not fit, softmax in place in y
}
int launch_soft_max(const float * x, const float * mask, float * y, int ncols, int64_t nrows, int64_t rows_per_mask_cycle, float scale,
                    cudaStream_t stream) {
    const size_t smem = soft_max_smem(ncols, nullptr);
    if (smem) {
        cudaError_t e = ensure_dyn_smem(sm_attr, (const void *) k_soft_max, smem, false);
        if (e != cudaSuccess) return (int) e;
    }
    k_soft_max<<<(unsigned) nrows, 256, smem, stream>>>(x, mask, y, ncols, rows_per_mask_cycle, scale, smem != 0);
    return (int) cudaGetLastError();
}

int launch_get_rows(const void * table, int type, int K, const int32_t * ids, int n_ids, float * y, cudaStream_t stream, bool pdl) {
    LaunchCfg lc(dim3((K + 255) / 256, std::min(n_ids, 65535)), dim3(256), 0, stream, pdl);
    return (int) cudaLaunchKernelEx(&lc.cfg, k_get_rows, (const uint8_t *) table, type, K, row_bytes(type, K), ids, n_ids, y);
}

int launch_binary(int op, const float * a, const float * b, float * y, int64_t n, int64_t nb, cudaStream_t stream) {
    k_binary<<<(unsigned) ((n + 255) / 256), 256, 0, stream>>>(op, a, b, y, n, nb);
    return (int) cudaGetLastError();
}
int launch_silu(const float * x, float * y, int64_t n, cudaStream_t stream) {
    k_silu<<<(unsigned) ((n + 255) / 256), 256, 0, stream>>>(x, y, n);
    return (int) cudaGetLastError();
}
int launch_silu_mul(const float * g, const float * u, float * y, int64_t n, cudaStream_t stream) {
    k_silu_mul<<<(unsigned) ((n + 255) / 256), 256, 0, stream>>>(g, u, y, n);
    return (int) cudaGetLastError();
}
int launch_cpy_f32_f16(const float * x, __half * y, int64_t n, cudaStream_t stream) {
    k_cpy_f32_f16<<<(unsigned) ((n + 255) / 256), 256, 0, stream>>>(x, y, n);
    return (int) cudaGetLastError();
}

}  // namespace pb
