// prima.cpp_b200/csrc/launch.h — host-side launchers of the sm_90a kernels (internal C++ API; the public C ABI is
// include/prima_b200.h).  Every launcher enqueues on `stream` and returns a cudaError_t as int (0 = success).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/prima_b200.h"
#include "common.cuh"

namespace pb {

struct GemvDesc {
    const void * W;        // raw GGUF blocks [N][K]
    float * y;             // [N]
    const float * bias;    // optional
    const float * resid;   // optional
    int type;
    int N;
};

// Activation workspace of K values (pb200_act_workspace_bytes): qs[kp] | d[kp/32] f32 | s[kp/32] f32 | bsums[kp/16] i16, kp = K rounded
// up to 256 (every part 16-B aligned)
inline size_t act_ws_bytes(int64_t k) {
    const int64_t kp = (k + 255) / 256 * 256;
    return (size_t) kp + (size_t) kp / 32 * 8 + (size_t) kp / 16 * 2;
}
inline ActQ act_from_ws(void * ws, int64_t k) {
    const int64_t kp = (k + 255) / 256 * 256;
    ActQ a{};
    uint8_t * p = (uint8_t *) ws;
    a.qs = (int8_t *) p;
    a.d = (float *) (p + kp);
    a.s = (float *) (p + kp + kp / 32 * 4);
    a.bsums = (int16_t *) (p + kp + kp / 32 * 8);
    return a;
}

// Where a mat-mul's activation comes from: the GEMV launcher, the GEMV kernel's distributed prologue and the tensor-core mat-mul's
// activation pass (MmqPre) share this numbering.
enum Prologue : int {
    PRO_NONE = 0,       // already quantized in `act`
    PRO_QUANTIZE = 1,   // act = quant(in0)
    PRO_RMSNORM = 2,    // act = quant(rms_norm(in0, eps) * in1)   llm_build_norm (in1 = norm weight)
    PRO_SILU_MUL = 3,   // act = quant(silu(in0) * in1)            llm_build_ffn LLM_FFN_SILU / LLM_FFN_PAR
};
struct GemvPrologue {
    int kind = PRO_NONE;
    const float * in0 = nullptr;
    const float * in1 = nullptr;
    float eps = 0.f;
    unsigned int * gbar = nullptr;   // two zero-initialised words of device memory owned by the caller (grid barrier state): lets
                                     // PRO_RMSNORM / PRO_SILU_MUL run distributed inside the k-quant GEMV instead of in a kernel in front
    float * f32 = nullptr;           // [K] scratch for PRO_RMSNORM when the matrices need different activation modes
};

// Launch configuration for cudaLaunchKernelEx: programmatic dependent launch as requested, clusters of cluster_x CTAs when > 1.
struct LaunchCfg {
    cudaLaunchConfig_t cfg{};
    cudaLaunchAttribute attr[2];
    LaunchCfg(dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool pdl, int cluster_x = 1) {
        cfg.gridDim = grid;
        cfg.blockDim = block;
        cfg.dynamicSmemBytes = smem;
        cfg.stream = stream;
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = pdl ? 1 : 0;
        attr[1].id = cudaLaunchAttributeClusterDimension;
        attr[1].val.clusterDim.x = cluster_x; attr[1].val.clusterDim.y = 1; attr[1].val.clusterDim.z = 1;
        cfg.attrs = attr;
        cfg.numAttrs = cluster_x > 1 ? 2 : 1;
    }
    LaunchCfg(const LaunchCfg &) = delete;   // cfg.attrs points into this object
};

// ---- per-device host state (gemv.cu): cudaFuncSetAttribute / SM count are per device, one process may drive several ----
constexpr int PB_MAX_DEV = 64;
struct FuncAttrCache { size_t bytes[PB_MAX_DEV] = {0}; size_t limit[PB_MAX_DEV] = {0}; };
int cur_device();
int sm_count();                       // of the current device
// the most dynamic shared memory a launch of fn may request on the current device: the opt-in limit per block minus fn's static
// shared memory (0 if the device cannot be queried)
size_t dyn_smem_limit(FuncAttrCache & c, const void * fn);
// raise a kernel's dynamic shared-memory limit on the current device if needed (max_carveout: also prefer the full 228 KB carve-out);
// cudaErrorNotSupported, with nothing changed, when bytes exceed dyn_smem_limit
cudaError_t ensure_dyn_smem(FuncAttrCache & c, const void * fn, size_t bytes, bool max_carveout);
// wait watchdogs (common.cuh): host-mapped flag every kernel with a bounded wait gets a pointer to; check_clear_abort() returns 1
// once per abort and re-arms — the C ABI reports PB200_EABORTED for the call that synchronised on the aborted launch
int * abort_flag();
int check_clear_abort();

int gemv_set_trace(unsigned long long * dev_buf, int slots);   // profiling: per-CTA stamps of k_gemv_kquant, launch i -> row i % slots of u64[4096]; NULL = off

// y_i = W_i . act (+ bias_i) (+ resid_i) for 1..3 matrices sharing one input vector of K values, `pro` says where the activation comes
// from.  Enqueues, in order:
//   1. the activation: with PRO_RMSNORM / PRO_SILU_MUL, k-quant matrices on the ring kernel, a barrier and a co-resident grid, CTA c of
//      the GEMV produces super-block c itself (no kernel in front); otherwise one producer kernel per activation mode the matrices need
//      (one mode: written straight into `act`; several: PRO_RMSNORM materialises the vector in pro.f32 first, then quantize + matrices
//      per mode);
//   2. the GEMV: the bulk-copy ring kernel when the group fits it (gemv_plan), else per matrix: the ring for a 32-element block type
//      matrix (Q8_0 / Q5_1 / Q4_0 / Q4_1 / Q5_0) that fits it on its own, k_gemv_blk32 (such rows that fit its activation stage) or
//      k_gemv_generic.
// The first kernel gets `pdl`, every later one is chained to its predecessor by programmatic dependent launch.  Adds the number of
// kernels enqueued to nlaunch.  start (optional, profiling): an event recorded just before the first GEMV kernel, i.e. after any
// producer kernel.
int launch_gemv(const GemvDesc * d, int nmat, int K, const ActQ & act, const GemvPrologue & pro, cudaStream_t stream, bool pdl, uint64_t & nlaunch,
                cudaEvent_t start = nullptr);
bool gemv_fused_prologue_ok(int K);   // K fits the ring kernel's activation staging (K % 256 == 0, K <= 29 696)

// activation quantization (mode = ACT_Q8_K / ACT_Q8_0 / ACT_Q8_1); K padded to 256 in the ActQ buffers
//   out = quant( x ), or with up: out = quant( silu(x) * up )   [llm_build_ffn LLM_FFN_SILU/PAR, src/llama.cpp:9858-9907]
int launch_quantize_act(const float * x, const float * up, int K, int mode, const ActQ & out, cudaStream_t stream, bool pdl);
// out = quant( rms_norm(x) * w ), optional f32 copy  [llm_build_norm, src/llama.cpp:9772-9802; ggml.c:11950-11996]
int launch_rmsnorm_quant(const float * x, const float * w, int n, float eps, int mode, const ActQ & out, float * f32_out, cudaStream_t stream, bool pdl);
// plain ops for the ggml-backend plugin (rows x n)
int launch_rms_norm(const float * x, float * y, int n, int64_t nrows, float eps, cudaStream_t stream, const float * w = nullptr);   // w: fused MUL by the norm weight

struct RopeParams {
    int n_dims, mode, n_ctx_orig;
    float freq_base, freq_scale, ext_factor, attn_factor, beta_fast, beta_slow;
    float theta_scale;      // powf(freq_base, -2/n_dims), computed on the host like ggml.c:14193
    float corr_dims[2];     // ggml_rope_yarn_corr_dims, ggml.c:14133-14141
};
void rope_params_init(RopeParams & rp, int n_dims, int mode, int n_ctx_orig, float freq_base, float freq_scale, float ext_factor,
                      float attn_factor, float beta_fast, float beta_slow);

// generic rope for the plugin: x [ntok][n_head][D] -> y, positions pos[ntok]
int launch_rope(const float * x, float * y, int64_t ntok, int n_head, int D, int64_t tok_stride, int64_t head_stride, const int32_t * pos,
                const RopeParams & rp, const float * freq_factors, cudaStream_t stream);
// GGML_OP_ROPE on contiguous f16 rows x [ntok][n_head][D] -> y (y may equal x), positions pos[ntok]
int launch_rope_f16(const __half * x, __half * y, int64_t ntok, int n_head, int D, const int32_t * pos, const RopeParams & rp, const float * freq_factors,
                    cudaStream_t stream);
// context shift of one slot's caches kc / vc ([n_layer][n_ctx][n_head_kv*128] f16 each): cells [p0, p1) -> c + delta (delta < 0), K rows
// re-rotated by delta like launch_rope_f16 (rp.n_dims == 128), V rows copied; tokpos[1] += delta when it is >= p0.  One launch.
int launch_kv_shift(__half * kc, __half * vc, int n_layer, int n_head_kv, int n_ctx, int p0, int p1, int delta, const RopeParams & rp,
                    const float * freq_factors, int32_t * tokpos, cudaStream_t stream);

// decode attention (k_attn_rows), FA-off numerics of the CPU backend (f16-rounded q and probabilities, f32 accumulation):
//   out[h][:] = softmax(scale * K[0..n_kv) . q_h) . V   — GQA-aware, K/V read once per kv head.  n_kv = *pos_dev + 1.
int launch_attn_decode(const float * q, const __half * kcache, const __half * vcache, float * out, int n_head, int n_head_kv, int D,
                       const int32_t * pos_dev, int n_ctx, float scale, cudaStream_t stream, bool pdl);
// k_attn_rows keeps a whole score row in shared memory: the longest row (a multiple of 32) it takes on the current device.  Longer
// n_ctx / n_kv_max make launch_attn_decode, launch_attn_batch's per-row form and launch_attn_step's fallback return cudaErrorNotSupported.
int attn_rows_max_kv();
// k_attn2 keeps a score row of n cells (padded to 32) in shared memory behind its fixed part, at most 200 KB: the largest n (a multiple of
// 32) it takes on the current device.  launch_attn_step / launch_attn_ggml refuse more (pb200_attn_ggml_max_cells).
int attn2_max_cells();
// batched form for prompt processing: token t (q row t, out row t) attends to cache rows [0, pos_dev[t]].  The tiled kernel when its
// scores fit shared memory, else k_attn_rows per (head, token)
int launch_attn_batch(const float * q, const __half * kcache, const __half * vcache, float * out, int n_head, int n_head_kv, int D,
                      const int32_t * pos_dev, int n_tok, int n_kv_max, float scale, cudaStream_t stream);
// The engine's per-token attention, one launch: rope(q), rope(k) -> f16 K row, v -> f16 V row, cache store and attention.  When the
// consumer of `out` wants it in mode ACT_Q8_K (outq_mode) and the shape allows, the clustered k_attn2 also writes that activation
// into outq and `quantized` is set; otherwise (odd n_head, scores beyond its shared memory at long n_ctx, other modes)
// k_attn_rows<true> writes `out` only and `quantized` is cleared.
int launch_attn_step(const float * q, const float * k, const float * v, __half * kcache, __half * vcache, float * out, const ActQ & outq,
                     int outq_mode, int n_head, int n_head_kv, int D, const int32_t * pos_dev, int n_ctx, const RopeParams & rp,
                     const float * freq_factors, float scale, cudaStream_t stream, bool pdl, bool & quantized);

// k_attn2 on the reference graph's tensors (FA off, one token): K cache [cell][n_head_kv*128] f16, V cache TRANSPOSED
// [n_head_kv*128][vt_stride] f16, additive f32 mask row over n_cells (multiple of 32) cells, this token stored in cell kv_head
int launch_attn_ggml(const float * q, const float * k, const float * v, __half * kcache, __half * vcache_t, int64_t vt_stride, float * out, const ActQ & outq,
                     int n_head, int n_head_kv, int D, const int32_t * pos_dev, int n_cells, int kv_head, const int32_t * kv_head_dev, const float * mask,
                     const RopeParams & rp, const float * freq_factors, float scale, cudaStream_t stream, bool pdl);

// GGML_OP_FLASH_ATTN_EXT with f16 K / V (byte strides {nb1, nb2}; mask f16 rows of mask_nb1 bytes or NULL); dst [D][n_head][n_tok]
int launch_flash_attn_ext(const float * q, const void * k, const void * v, const void * mask, float * dst, int D, int n_tok, int n_head, int n_head_kv,
                          int n_kv, const int64_t * q_nb, const int64_t * k_nb, const int64_t * v_nb, int64_t mask_nb1, float scale, float max_bias,
                          float softcap, cudaStream_t stream);

// soft_max_ext for the plugin: y[r][:] = softmax(x[r][:]*scale + mask[r % mask_rows][:])  (softmax.cu:14-116)
int launch_soft_max(const float * x, const float * mask, float * y, int ncols, int64_t nrows, int64_t rows_per_mask_cycle, float scale,
                    cudaStream_t stream);

// get_rows on a quantized / f16 / f32 table: y[i][:] = dequant(table[ids[i]])   (getrows.cu; ggml.c get_rows_q)
// batched k-quant mat-mul on the wgmma tensor cores (mmq.cu): dst[T][N] = X[T][K] . W[N][K]^T (+ bias[N]); ws from mmq_workspace_bytes
size_t mmq_workspace_bytes(int64_t K, int64_t T);
bool mmq_supported(int type, int64_t K);
struct MmqPre {            // producer fused into the activation pass: PRO_SILU_MUL: x <- silu(x) * aux[t][k] (ld_aux floats per row), PRO_RMSNORM: x <- rms_norm(x, eps) * aux[k]
    int kind = PRO_NONE;
    const float * aux = nullptr;
    int64_t ld_aux = 0;
    float eps = 0.f;
};
cudaError_t launch_mmq(int type, const void * W, int64_t N, int64_t K, const float * x, int64_t ldx, int64_t T, float * dst, const float * bias,
                       const float * resid, void * ws, cudaStream_t st, bool reuse_prep = false, const MmqPre * pre = nullptr);
// resid: [T][N] added in the epilogue (must not alias dst).  reuse_prep: ws already holds this x (same K, T) from the previous launch_mmq
// on the stream (q|k|v and gate|up share one activation: the q8_K -> fp16 tiling pass runs once)
int launch_get_rows(const void * table, int type, int K, const int32_t * ids, int n_ids, float * y, cudaStream_t stream, bool pdl);

// greedy token: first index of the maximum of x[n] -> *out (and *out2 if set); the engine's k_argmax
int launch_argmax(const float * x, int n, int32_t * out, int32_t * out2, cudaStream_t stream, bool pdl);
// seeded sampling (sample.cu): the reference's top-k / top-p / min-p / temperature / dist chain over x[n] -> *out (and *out2 if set),
// one clustered launch; temp <= 0 launches launch_argmax.  state: sampler_state_bytes() of device memory seeded by launch_sampler_seed.
// cudaErrorNotSupported when a slice of n / 16 logits exceeds the device's shared memory.
size_t sampler_state_bytes();
bool sampling_params_ok(const pb200_sampling * p);   // finite, top_p in (0, 1], min_p in [0, 1), min_keep >= 0
int launch_sampler_seed(void * state, uint32_t seed, cudaStream_t stream);
int launch_sample(const float * x, int n, const pb200_sampling & p, void * state, int32_t * out, int32_t * out2, cudaStream_t stream, bool pdl);
// logit bias + penalties (sample.cu): state = header, bias list, history ring of penalty_state_bytes(last_n, n_bias) device bytes.
// launch_penalty_init enqueues max(1, ceil(n_bias / 256)) launches (the list travels in their arguments) and adds them to nlaunch;
// launch_penalize writes the penalised copy of x[n] into out (k_penalize, one launch); launch_penalty_accept pushes tokens[n] (device)
// into the history (one launch; nothing happens on the device when last_n is 0).
size_t penalty_state_bytes(int last_n, int n_bias);
bool penalties_ok(const pb200_penalties * p);   // repeat finite and > 0, freq / present finite, no NaN bias, a list where n_logit_bias > 0
int launch_penalty_init(void * state, int n_vocab, const pb200_penalties & p, cudaStream_t stream, uint64_t & nlaunch);
int launch_penalize(const float * x, int n, const void * state, float * out, cudaStream_t stream, bool pdl);
int launch_penalty_accept(void * state, const int32_t * tokens, int n, cudaStream_t stream, bool pdl);

// element-wise helpers for the plugin
int launch_binary(int op /*0 add, 1 mul*/, const float * a, const float * b, float * y, int64_t n, int64_t nb /*b broadcast period*/, cudaStream_t stream);
int launch_silu(const float * x, float * y, int64_t n, cudaStream_t stream);
int launch_silu_mul(const float * g, const float * u, float * y, int64_t n, cudaStream_t stream);   // y = silu(g) * u
int launch_cpy_f32_f16(const float * x, __half * y, int64_t n, cudaStream_t stream);
int launch_copy_strided(const void * src, void * dst, int dst_is_f16, const int64_t ne[4], const int64_t sb[4], const int64_t db[4], cudaStream_t stream);
int launch_mul_mat_f16(const void * A, const void * B, void * D, int64_t K, const int64_t ne[4], int64_t r2, int64_t r3, const int64_t ab[4],
                       const int64_t bb[4], const int64_t db[4], cudaStream_t stream);

}  // namespace pb
