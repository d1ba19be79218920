// prima.cpp_b200/csrc/api.cu — single-op entry points of the C ABI (include/prima_b200.h).
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <atomic>
#include <cstdint>
#include <cstring>
#include <mutex>

#include "../../include/prima_b200.h"
#include "launch.h"

using namespace pb;

extern std::atomic<uint64_t> g_launches;

extern "C" {

const char * pb200_version(void) { return "prima.cpp_b200 0.1 (sm_90a)"; }

const char * pb200_error_string(int code) {
    switch (code) {
        case 0: return "success";
        case PB200_EINVAL: return "invalid argument";
        case PB200_ENOMEM: return "out of memory";
        case PB200_ENOTSUP: return "unsupported tensor type or shape on this path";
        case PB200_ESTATE: return "model not in the right state (missing tensors / not finalized)";
        case PB200_EABORTED: return "a kernel's wait watchdog gave up: the results of this call are invalid (later calls are unaffected)";
    }
    return code > 0 ? cudaGetErrorString((cudaError_t) code) : "unknown error";
}

int pb200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}
int pb200_sm_count(void) { return sm_count(); }
int64_t pb200_row_bytes(int type, int64_t k) { return row_bytes(type, k); }
uint64_t pb200_kernel_launches(void) { return g_launches.load(); }
void pb200_kernel_launches_add(uint64_t n) { g_launches += n; }

size_t pb200_act_workspace_bytes(int64_t k) { return act_ws_bytes(k); }

int pb200_quantize_act(int wtype, const float * x, int64_t k, void * act_ws, void * stream) {
    if (!is_quant_type(wtype) || !x || !act_ws || k <= 0 || k % block_elems(wtype) != 0) return PB200_EINVAL;
    g_launches++;
    return launch_quantize_act(x, nullptr, (int) k, act_mode_for(wtype), act_from_ws(act_ws, k), (cudaStream_t) stream, false);
}

int pb200_mul_mat_vec_q(int type, const void * W, int64_t n, int64_t k, const void * act_ws, float * y, const float * bias, const float * resid,
                        void * stream) {
    if (!is_quant_type(type) || !W || !act_ws || !y || n <= 0 || k <= 0 || k % block_elems(type) != 0) return PB200_EINVAL;
    GemvDesc d = {W, y, bias, resid, type, (int) n};
    uint64_t nl = 0;
    const int rc = launch_gemv(&d, 1, (int) k, act_from_ws(const_cast<void *>(act_ws), k), GemvPrologue{}, (cudaStream_t) stream, false, nl);
    g_launches += nl;
    return rc;
}

int pb200_mul_mat_vec(int type, const void * W, int64_t n, int64_t k, const float * x, float * y, void * act_ws, void * stream) {
    int e = pb200_quantize_act(type, x, k, act_ws, stream);
    if (e) return e;
    return pb200_mul_mat_vec_q(type, W, n, k, act_ws, y, nullptr, nullptr, stream);
}

int pb200_mul_mat_vec_fused(int nmat, const int * types, const void * const * W, const int64_t * n, int64_t k, const void * act_ws,
                            float * const * y, void * stream) {
    if (nmat < 1 || nmat > 3 || !types || !W || !n || !y || !act_ws) return PB200_EINVAL;
    GemvDesc d[3];
    for (int i = 0; i < nmat; i++) {
        if (!is_quant_type(types[i]) || k % block_elems(types[i]) != 0) return PB200_EINVAL;
        if (act_mode_for(types[i]) != act_mode_for(types[0])) return PB200_EINVAL;   // one activation: one quantization format
        d[i] = GemvDesc{W[i], y[i], nullptr, nullptr, types[i], (int) n[i]};
    }
    uint64_t nl = 0;
    const int rc = launch_gemv(d, nmat, (int) k, act_from_ws(const_cast<void *>(act_ws), k), GemvPrologue{}, (cudaStream_t) stream, false, nl);
    g_launches += nl;
    return rc;
}

int pb200_mul_mat_vec_host(int type, const void * W_dev, int64_t n, int64_t k, const float * x_host, float * y_host) {
    if (!is_quant_type(type) || !W_dev || !x_host || !y_host) return PB200_EINVAL;
    // per-thread cached staging buffers (pinned host + device), grown on demand
    struct Stage { float * hx = nullptr, * hy = nullptr, * dx = nullptr, * dy = nullptr; void * ws = nullptr; int64_t n = 0, k = 0; cudaStream_t st = nullptr; };
    static thread_local Stage S;
    if (!S.st && cudaStreamCreateWithFlags(&S.st, cudaStreamNonBlocking) != cudaSuccess) return (int) cudaGetLastError();
    if (k > S.k) {
        if (S.hx) cudaFreeHost(S.hx);
        if (S.dx) cudaFree(S.dx);
        if (S.ws) cudaFree(S.ws);
        S.hx = S.dx = nullptr; S.ws = nullptr; S.k = 0;     // a failed re-allocation below must not leave dangling pointers behind
        cudaError_t e;
        if ((e = cudaMallocHost((void **) &S.hx, (size_t) k * 4)) != cudaSuccess) return (int) e;
        if ((e = cudaMalloc((void **) &S.dx, (size_t) k * 4)) != cudaSuccess) return (int) e;
        if ((e = cudaMalloc(&S.ws, pb200_act_workspace_bytes(k))) != cudaSuccess) return (int) e;
        S.k = k;
    }
    if (n > S.n) {
        if (S.hy) cudaFreeHost(S.hy);
        if (S.dy) cudaFree(S.dy);
        S.hy = S.dy = nullptr; S.n = 0;
        cudaError_t e;
        if ((e = cudaMallocHost((void **) &S.hy, (size_t) n * 4)) != cudaSuccess) return (int) e;
        if ((e = cudaMalloc((void **) &S.dy, (size_t) n * 4)) != cudaSuccess) return (int) e;
        S.n = n;
    }
    memcpy(S.hx, x_host, (size_t) k * 4);
    cudaError_t e;
    if ((e = cudaMemcpyAsync(S.dx, S.hx, (size_t) k * 4, cudaMemcpyHostToDevice, S.st)) != cudaSuccess) return (int) e;
    int rc = pb200_mul_mat_vec(type, W_dev, n, k, S.dx, S.dy, S.ws, S.st);
    if (rc) return rc;
    if ((e = cudaMemcpyAsync(S.hy, S.dy, (size_t) n * 4, cudaMemcpyDeviceToHost, S.st)) != cudaSuccess) return (int) e;
    if ((e = cudaStreamSynchronize(S.st)) != cudaSuccess) return (int) e;
    memcpy(y_host, S.hy, (size_t) n * 4);
    return 0;
}

int pb200_debug_set_trace(void * dev_buf, int slots) { return gemv_set_trace((unsigned long long *) dev_buf, slots); }

int pb200_rms_norm(const float * x, float * y, int64_t n, int64_t nrows, float eps, void * stream) {
    if (!x || !y || n <= 0 || nrows <= 0) return PB200_EINVAL;
    g_launches++;
    return launch_rms_norm(x, y, (int) n, nrows, eps, (cudaStream_t) stream);
}

int pb200_rope(const float * x, float * y, int64_t n_tokens, int n_head, int head_dim, int n_dims, int mode, const int32_t * pos, float freq_base,
               float freq_scale, float ext_factor, float attn_factor, float beta_fast, float beta_slow, int n_ctx_orig, const float * freq_factors,
               void * stream) {
    if (!x || !y || !pos || n_dims > head_dim || (n_dims & 1)) return PB200_EINVAL;
    RopeParams rp;
    rope_params_init(rp, n_dims, mode, n_ctx_orig, freq_base, freq_scale, ext_factor, attn_factor, beta_fast, beta_slow);
    g_launches++;
    return launch_rope(x, y, n_tokens, n_head, head_dim, (int64_t) n_head * head_dim, head_dim, pos, rp, freq_factors, (cudaStream_t) stream);
}

int pb200_rope_f16(const void * x, void * y, int64_t n_rows, int n_head, int head_dim, int n_dims, int mode, const int32_t * pos, float freq_base,
                   float freq_scale, float ext_factor, float attn_factor, float beta_fast, float beta_slow, int n_ctx_orig, const float * freq_factors,
                   void * stream) {
    if (!x || !y || !pos || n_rows <= 0 || n_head <= 0 || n_dims <= 0 || n_dims > head_dim || (n_dims & 1) || n_rows * n_head > INT32_MAX) return PB200_EINVAL;
    RopeParams rp;
    rope_params_init(rp, n_dims, mode, n_ctx_orig, freq_base, freq_scale, ext_factor, attn_factor, beta_fast, beta_slow);
    g_launches++;
    return launch_rope_f16((const __half *) x, (__half *) y, n_rows, n_head, head_dim, pos, rp, freq_factors, (cudaStream_t) stream);
}

int pb200_soft_max(const float * x, const float * mask, float * y, int64_t ncols, int64_t nrows, int64_t mask_rows, float scale, void * stream) {
    if (!x || !y || ncols <= 0 || nrows <= 0) return PB200_EINVAL;
    g_launches++;
    return launch_soft_max(x, mask, y, (int) ncols, nrows, mask_rows > 0 ? mask_rows : 1, scale, (cudaStream_t) stream);
}

int pb200_silu_mul(const float * gate, const float * up, float * y, int64_t n, void * stream) {
    if (!gate || !up || !y || n <= 0) return PB200_EINVAL;
    g_launches++;
    int e = launch_silu(gate, y, n, (cudaStream_t) stream);
    if (e) return e;
    g_launches++;
    return launch_binary(1, y, up, y, n, n, (cudaStream_t) stream);
}

int pb200_binary(int op, const float * a, const float * b, float * y, int64_t n, int64_t nb, void * stream) {
    if (!a || !b || !y || n <= 0 || nb <= 0 || (op != 0 && op != 1)) return PB200_EINVAL;
    g_launches++;
    return launch_binary(op, a, b, y, n, nb, (cudaStream_t) stream);
}
int pb200_silu(const float * x, float * y, int64_t n, void * stream) {
    if (!x || !y || n <= 0) return PB200_EINVAL;
    g_launches++;
    return launch_silu(x, y, n, (cudaStream_t) stream);
}
int pb200_copy_strided(const void * src_f32, void * dst, int dst_is_f16, const int64_t * ne, const int64_t * src_strides, const int64_t * dst_strides,
                       void * stream) {
    if (!src_f32 || !dst || !ne || !src_strides || !dst_strides) return PB200_EINVAL;
    g_launches++;
    return launch_copy_strided(src_f32, dst, dst_is_f16, ne, src_strides, dst_strides, (cudaStream_t) stream);
}
int pb200_mul_mat_f16(const void * a_f16, const float * b_f32, float * d, int64_t k, const int64_t * ne, int64_t r2, int64_t r3,
                      const int64_t * a_strides, const int64_t * b_strides, const int64_t * d_strides, void * stream) {
    if (!a_f16 || !b_f32 || !d || !ne || !a_strides || !b_strides || !d_strides || k <= 0 || r2 <= 0 || r3 <= 0) return PB200_EINVAL;
    g_launches++;
    return launch_mul_mat_f16(a_f16, b_f32, d, k, ne, r2, r3, a_strides, b_strides, d_strides, (cudaStream_t) stream);
}

size_t pb200_mul_mat_q_workspace_bytes(int64_t k, int64_t t) { return (k > 0 && t > 0) ? mmq_workspace_bytes(k, t) : 0; }
int pb200_mul_mat_q_supported(int type, int64_t k) { return mmq_supported(type, k); }
int pb200_mul_mat_q(int type, const void * W, int64_t n, int64_t k, const float * x, int64_t ldx, int64_t t, float * dst, const float * bias,
                    const float * resid, void * ws, void * stream) {
    if (!W || !x || !dst || !ws || n <= 0 || t <= 0 || ldx < k || resid == dst) return PB200_EINVAL;
    if (((uintptr_t) x & 15) || (ldx & 3) || ((uintptr_t) W & 15)) return PB200_EINVAL;   // rows are read as float4, weights as 16-byte pieces
    if (!mmq_supported(type, k)) return PB200_ENOTSUP;
    g_launches += 2;
    return (int) launch_mmq(type, W, n, k, x, ldx, t, dst, bias, resid, ws, (cudaStream_t) stream);
}
int pb200_aborted(void) { return check_clear_abort(); }

int pb200_get_rows(int type, const void * table, int64_t k, const int32_t * ids, int64_t n_ids, float * y, void * stream) {
    if (!table || !ids || !y || k <= 0 || n_ids <= 0) return PB200_EINVAL;
    if (!(is_quant_type(type) || type == T_F32 || type == T_F16)) return PB200_ENOTSUP;
    g_launches++;
    return launch_get_rows(table, type, (int) k, ids, (int) n_ids, y, (cudaStream_t) stream, false);
}

int pb200_attn_decode(const float * q, const void * k_cache_f16, const void * v_cache_f16, float * out, int n_head, int n_head_kv, int head_dim,
                      const int32_t * pos_dev, int n_ctx, float scale, void * stream) {
    if (!q || !k_cache_f16 || !v_cache_f16 || !out || !pos_dev || head_dim != 128 || n_head_kv <= 0 || n_head <= 0 || n_head % n_head_kv) return PB200_EINVAL;
    const int rc = launch_attn_decode(q, (const __half *) k_cache_f16, (const __half *) v_cache_f16, out, n_head, n_head_kv, head_dim, pos_dev, n_ctx,
                                      scale, (cudaStream_t) stream, false);
    if (rc == (int) cudaErrorNotSupported) return PB200_ENOTSUP;   // n_ctx above the score row k_attn_rows keeps in shared memory
    if (rc == 0) g_launches++;
    return rc;
}

int pb200_gemv_fused_supported(int type, int64_t k) { return is_kquant(type) && k <= INT32_MAX && gemv_fused_prologue_ok((int) k); }
int pb200_gemv_fused(int nmat, const pb200_gemv_mat * mats, int64_t k, void * act_ws, int prologue, const float * in0, const float * in1, float eps,
                     void * sync_ws, int pdl, void * stream) {
    if (nmat < 1 || nmat > 3 || !mats || !act_ws || k <= 0 || prologue < 0 || prologue > 2) return PB200_EINVAL;
    if (prologue != 0 && (!in0 || !in1)) return PB200_EINVAL;
    if (!gemv_fused_prologue_ok((int) k)) return PB200_ENOTSUP;
    GemvDesc d[3];
    for (int i = 0; i < nmat; i++) {
        if (!mats[i].W || !mats[i].y || mats[i].n <= 0) return PB200_EINVAL;
        if (!pb200_gemv_fused_supported(mats[i].type, k) || ((uintptr_t) mats[i].W & 15)) return PB200_ENOTSUP;
        d[i] = GemvDesc{mats[i].W, mats[i].y, nullptr, mats[i].add, mats[i].type, (int) mats[i].n};
    }
    static const int kind[3] = {PRO_NONE, PRO_RMSNORM, PRO_SILU_MUL};   // the ABI's prologue codes
    const GemvPrologue pro{kind[prologue], in0, in1, eps, (unsigned int *) sync_ws, nullptr};
    uint64_t nl = 0;
    const int rc = launch_gemv(d, nmat, (int) k, act_from_ws(act_ws, k), pro, (cudaStream_t) stream, pdl != 0, nl);
    g_launches += nl;
    return rc;
}

int pb200_attn_ggml_max_cells(void) { return attn2_max_cells(); }
int pb200_attn_ggml(const float * q, const float * k, const float * v, void * k_cache_f16, void * v_cache_t_f16, int64_t vt_stride, float * out,
                    void * act_ws_out, int n_head, int n_head_kv, int head_dim, const int32_t * pos_dev, int n_cells, int kv_head,
                    const int32_t * kv_head_dev, const float * mask, int n_dims, int mode, float freq_base, float freq_scale, float ext_factor, float attn_factor, float beta_fast, float beta_slow,
                    int n_ctx_orig, const float * freq_factors, float scale, int pdl, void * stream) {
    if (!q || !k || !v || !k_cache_f16 || !v_cache_t_f16 || !out || !pos_dev || !mask || n_head <= 0 || n_head_kv <= 0) return PB200_EINVAL;
    if (head_dim != 128 || n_dims > head_dim || (n_dims & 1) || (mode != 0 && mode != 2)) return PB200_ENOTSUP;
    RopeParams rp;
    rope_params_init(rp, n_dims, mode, n_ctx_orig, freq_base, freq_scale, ext_factor, attn_factor, beta_fast, beta_slow);
    ActQ outq{};
    if (act_ws_out) {
        if (((int64_t) n_head * head_dim) % 256 != 0) return PB200_ENOTSUP;
        outq = act_from_ws(act_ws_out, (int64_t) n_head * head_dim);
    }
    const int rc = launch_attn_ggml(q, k, v, (__half *) k_cache_f16, (__half *) v_cache_t_f16, vt_stride, out, outq, n_head, n_head_kv, head_dim, pos_dev,
                                    n_cells, kv_head, kv_head_dev, mask, rp, freq_factors, scale, (cudaStream_t) stream, pdl != 0);
    if (rc == (int) cudaErrorNotSupported) return PB200_ENOTSUP;
    if (rc == 0) g_launches++;
    return rc;
}

int pb200_flash_attn_ext(const float * q, const void * k_f16, const void * v_f16, const void * mask_f16, float * dst, int head_dim, int n_tokens, int n_head,
                         int n_head_kv, int n_kv, const int64_t * q_nb, const int64_t * k_nb, const int64_t * v_nb, int64_t mask_nb1, float scale,
                         float max_bias, float logit_softcap, void * stream) {
    if (!q || !k_f16 || !v_f16 || !dst || !q_nb || !k_nb || !v_nb || n_kv <= 0) return PB200_EINVAL;
    if (head_dim > 256) return PB200_ENOTSUP;
    g_launches++;
    return launch_flash_attn_ext(q, k_f16, v_f16, mask_f16, dst, head_dim, n_tokens, n_head, n_head_kv, n_kv, q_nb, k_nb, v_nb, mask_nb1, scale, max_bias,
                                 logit_softcap, (cudaStream_t) stream);
}

int pb200_attn_prefill(const float * q, const void * k_cache_f16, const void * v_cache_f16, float * out, int n_head, int n_head_kv, int head_dim,
                       const int32_t * pos_dev, int n_tok, int n_kv_max, float scale, void * stream) {
    if (!q || !k_cache_f16 || !v_cache_f16 || !out || !pos_dev || head_dim != 128 || n_head_kv <= 0 || n_head % n_head_kv || n_tok <= 0 || n_kv_max <= 0)
        return PB200_EINVAL;
    const int rc = launch_attn_batch(q, (const __half *) k_cache_f16, (const __half *) v_cache_f16, out, n_head, n_head_kv, head_dim, pos_dev, n_tok,
                                     n_kv_max, scale, (cudaStream_t) stream);
    if (rc == (int) cudaErrorNotSupported) return PB200_ENOTSUP;
    if (rc == 0) g_launches++;
    return rc;
}

size_t pb200_sampler_state_bytes(void) { return sampler_state_bytes(); }
int pb200_sampler_seed(void * state_dev, uint32_t seed, void * stream) {
    if (!state_dev) return PB200_EINVAL;
    return launch_sampler_seed(state_dev, seed, (cudaStream_t) stream);
}
int pb200_sample(const float * logits, int n_vocab, const pb200_sampling * p, void * state_dev, int32_t * token_dev, void * stream) {
    if (!logits || n_vocab <= 0 || !state_dev || !token_dev || !sampling_params_ok(p)) return PB200_EINVAL;
    const int rc = launch_sample(logits, n_vocab, *p, state_dev, token_dev, nullptr, (cudaStream_t) stream, false);
    if (rc == (int) cudaErrorNotSupported) return PB200_ENOTSUP;
    if (rc == 0) g_launches++;
    return rc;
}

size_t pb200_penalty_state_bytes(int n_vocab, int last_n, int n_logit_bias) { (void) n_vocab; return penalty_state_bytes(last_n, n_logit_bias); }
int pb200_penalty_init(void * state_dev, int n_vocab, const pb200_penalties * p, void * stream) {
    if (!state_dev || n_vocab <= 0 || !penalties_ok(p)) return PB200_EINVAL;
    uint64_t nl = 0;
    const int rc = launch_penalty_init(state_dev, n_vocab, *p, (cudaStream_t) stream, nl);
    g_launches += nl;
    return rc;
}
int pb200_penalty_accept(void * state_dev, const int32_t * tokens_dev, int n, void * stream) {
    if (!state_dev || n < 0 || (n > 0 && !tokens_dev)) return PB200_EINVAL;
    if (n == 0) return 0;
    const int rc = launch_penalty_accept(state_dev, tokens_dev, n, (cudaStream_t) stream, false);
    if (rc == 0) g_launches++;
    return rc;
}
int pb200_penalty_apply(const float * logits, int n_vocab, const void * state_dev, float * out, void * stream) {
    if (!logits || n_vocab <= 0 || !state_dev || !out || out == logits) return PB200_EINVAL;
    const int rc = launch_penalize(logits, n_vocab, state_dev, out, (cudaStream_t) stream, false);
    if (rc == 0) g_launches++;
    return rc;
}

}  // extern "C"
