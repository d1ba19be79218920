// prima.cpp_b200/csrc/launch.h — host-side launchers of the sm_90a kernels (internal C++ API; the public C ABI is
// include/prima_b200.h).  Every launcher enqueues on `stream` and returns a cudaError_t as int (0 = success).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

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

struct GemvFused {       // fused activation prologue of the k-quant GEMV (PRO_* in gemv.cuh)
    int kind = 0;        // 0 none (activation already quantized), 4 rms_norm(in0)*in1, 5 silu(in0)*in1 — distributed over the grid (PRO_* in gemv.cuh)
    const float * in0 = nullptr;
    const float * in1 = nullptr;
    float eps = 0.f;
    unsigned int * gbar = nullptr;   // kinds 4, 5: two zero-initialised words of device memory owned by the caller (grid barrier state)
};

// ---- per-device host state (gemv.cu): cudaFuncSetAttribute / SM count are per device, one process may drive several ----
constexpr int PB_MAX_DEV = 64;
struct FuncAttrCache { size_t bytes[PB_MAX_DEV] = {0}; };
int cur_device();
int sm_count();                       // of the current device
// raise a kernel's dynamic shared-memory limit on the current device if needed (max_carveout: also prefer the full 228 KB carve-out)
cudaError_t ensure_dyn_smem(FuncAttrCache & c, const void * fn, size_t bytes, bool max_carveout);
// wait watchdogs (common.cuh): host-mapped flag every kernel with a bounded wait gets a pointer to; check_clear_abort() returns 1
// once per abort and re-arms — the C ABI reports PB200_EABORTED for the call that synchronised on the aborted launch
int * abort_flag();
int check_clear_abort();

int gemv_set_trace(unsigned long long * dev_buf, int slots);   // profiling: per-CTA stamps of k_gemv_kquant, launch i -> row i % slots of u64[4096]; NULL = off
int gemv_smem_bytes(int type, int K, int N);        // dynamic shared memory of the fast kernel for this shape (0: generic kernel)

// y_i = W_i . act  for up to 3 k-quant matrices sharing one q8_K activation (TMA-staged persistent kernel)
int launch_gemv_kquant(const GemvDesc * d, int nmat, int K, const ActQ & act, cudaStream_t stream, bool pdl);
int launch_gemv_kquant_fused(const GemvDesc * d, int nmat, int K, const ActQ & act, const GemvFused & pro, cudaStream_t stream, bool pdl);
bool gemv_fused_prologue_ok(int K);
bool gemv_dist_prologue_ok();   // the full persistent grid is co-resident on the current device (needed by the in-kernel grid barrier)
// any supported type / any K, one warp per row, direct global loads
int launch_gemv_generic(const GemvDesc & d, int K, const ActQ & act, cudaStream_t stream, bool pdl);
// picks the right kernel per weight type (all matrices must need the same activation mode)
int launch_gemv(const GemvDesc * d, int nmat, int K, const ActQ & act, cudaStream_t stream, bool pdl);

// activation quantization (mode = ACT_Q8_K / ACT_Q8_0 / ACT_Q8_1); K padded to 256 in the ActQ buffers
int launch_quantize_act(const float * x, int K, int mode, const ActQ & out, cudaStream_t stream, bool pdl);
// out = quant( silu(gate) * up )           [llm_build_ffn LLM_FFN_SILU/PAR, src/llama.cpp:9858-9907]
int launch_silu_mul_quant(const float * gate, const float * up, int K, int mode, const ActQ & out, float * f32_out, cudaStream_t stream, bool pdl);
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

// RoPE on q [n_head][D] in place and on k [n_head_kv][D]; stores rope(k) and v as f16 rows `pos` of the KV cache
// (rope.cu:188-271 + cpy_f32_f16 cpy.cu:34 + llm_build_kv_store src/llama.cpp:9673-9718).  pos is read from device memory.
int launch_rope_kvstore(float * q, const float * k, const float * v, __half * kcache, __half * vcache, int n_head, int n_head_kv, int D,
                        const int32_t * pos_dev, const RopeParams & rp, const float * freq_factors, cudaStream_t stream, bool pdl);
// generic rope for the plugin: x [ntok][n_head][D] -> y, positions pos[ntok]
int launch_rope(const float * x, float * y, int64_t ntok, int n_head, int D, int64_t tok_stride, int64_t head_stride, const int32_t * pos,
                const RopeParams & rp, const float * freq_factors, cudaStream_t stream);

// decode attention, FA-off numerics of the CPU backend (f16-rounded q and probabilities, f32 accumulation):
//   out[h][:] = softmax(scale * K[0..n_kv) . q_h) . V   — GQA-aware, K/V read once per kv head.  n_kv = *pos_dev + 1.
// Optionally quantizes out (n_head*D values) for the following wo GEMV.
int launch_attn_decode(const float * q, const __half * kcache, const __half * vcache, float * out, int n_head, int n_head_kv, int D,
                       const int32_t * pos_dev, int n_ctx, float scale, float * scratch, cudaStream_t stream, bool pdl);
int attn_scratch_floats(int n_head, int n_ctx);
// batched form for prompt processing: token t (q row t, out row t) attends to cache rows [0, pos_dev[t]]
int launch_attn_batch(const float * q, const __half * kcache, const __half * vcache, float * out, int n_head, int n_head_kv, int D,
                      const int32_t * pos_dev, int n_tok, int n_kv_max, float scale, cudaStream_t stream);
// rope(q), rope(k) -> f16 K row, v -> f16 V row, cache store and attention in one launch (the engine's per-token path)
int launch_attn_fused(const float * q, const float * k, const float * v, __half * kcache, __half * vcache, float * out, int n_head, int n_head_kv,
                      int D, const int32_t * pos_dev, int n_ctx, const RopeParams & rp, const float * freq_factors, float scale, cudaStream_t stream,
                      bool pdl);

// latency-restructured version that also writes the q8_K-quantized output (clusters of 2 CTAs = one super-block); returns
// cudaErrorNotSupported for shapes it does not handle (odd n_head, very long n_ctx): fall back to launch_attn_fused
int launch_attn_fused2(const float * q, const float * k, const float * v, __half * kcache, __half * vcache, float * out, const ActQ & outq, int n_head,
                       int n_head_kv, int D, const int32_t * pos_dev, int n_ctx, const RopeParams & rp, const float * freq_factors, float scale,
                       cudaStream_t stream, bool pdl);

// the same kernel on the reference graph's tensors (FA off, one token): K cache [cell][n_head_kv*128] f16, V cache TRANSPOSED
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
struct MmqPre {            // producer fused into the activation pass: 1: x <- silu(x) * aux[t][k] (ld_aux floats per row), 2: x <- rms_norm(x, eps) * aux[k]
    int kind = 0;
    const float * aux = nullptr;
    int64_t ld_aux = 0;
    float eps = 0.f;
};
cudaError_t launch_mmq(int type, const void * W, int64_t N, int64_t K, const float * x, int64_t ldx, int64_t T, float * dst, const float * bias,
                       const float * resid, void * ws, cudaStream_t st, bool reuse_prep = false, const MmqPre * pre = nullptr);
// resid: [T][N] added in the epilogue (must not alias dst).  reuse_prep: ws already holds this x (same K, T) from the previous launch_mmq
// on the stream (q|k|v and gate|up share one activation: the q8_K -> fp16 tiling pass runs once)
int launch_get_rows(const void * table, int type, int K, const int32_t * ids, int n_ids, float * y, cudaStream_t stream, bool pdl);

// element-wise helpers for the plugin
int launch_binary(int op /*0 add, 1 mul*/, const float * a, const float * b, float * y, int64_t n, int64_t nb /*b broadcast period*/, cudaStream_t stream);
int launch_silu(const float * x, float * y, int64_t n, cudaStream_t stream);
int launch_silu_mul(const float * g, const float * u, float * y, int64_t n, cudaStream_t stream);   // y = silu(g) * u
int launch_cpy_f32_f16(const float * x, __half * y, int64_t n, cudaStream_t stream);
int launch_copy_strided(const void * src, void * dst, int dst_is_f16, const int64_t ne[4], const int64_t sb[4], const int64_t db[4], cudaStream_t stream);
int launch_mul_mat_f16(const void * A, const void * B, void * D, int64_t K, const int64_t ne[4], int64_t r2, int64_t r3, const int64_t ab[4],
                       const int64_t bb[4], const int64_t db[4], cudaStream_t stream);

}  // namespace pb
