// prima.cpp_b200/ggml_backend/ggml_b200.cpp — ggml backend "B200": the reference's plugin vtables (ggml-backend-impl.h:15-220)
// implemented on top of the C ABI of libprima_b200.so.  Written against the interface, not against ggml-cuda.cu: buffers are
// plain cudaMalloc regions, there is one stream per backend instance, graph_compute maps each node to one or two pb200_* calls.
//
// supports_op is exact (SURVEY §7.3 H6): only what the Llama / Qwen2 decode graph needs (build_llama / build_qwen2,
// src/llama.cpp:11000-11216, 12736-12916, FA off); everything else returns false so the scheduler keeps it on the CPU.
#include "ggml-backend-impl.h"
#include "ggml-backend.h"
#include "ggml.h"

#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/ggml_b200.h"
#include "../../include/prima_b200.h"

#define B200_MAX_DEVICES 16

static std::atomic<unsigned long long> g_nodes{0};
static std::atomic<unsigned long long> g_fused_steps{0};
static std::atomic<unsigned long long> g_graph_replays{0};

#define CUDA_OK(expr)                                                                                   \
    do {                                                                                                \
        cudaError_t e_ = (expr);                                                                        \
        if (e_ != cudaSuccess) {                                                                        \
            fprintf(stderr, "ggml-b200: %s failed: %s (%s:%d)\n", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); \
            GGML_ABORT("CUDA error");   /* same convention as ggml_cuda_error, ggml-cuda.cu:62-72 */    \
        }                                                                                               \
    } while (0)

// ---------------------------------------------------------------------------------------------------- contexts
struct b200_device_ctx {
    int device;
    std::string name, description;
};
// ---- execution plan of the fused decode path (see graph_compute) ----
struct b200_step {
    int kind;                 // 0 = single node, 1 = fused GEMV group, 2 = fused attention
    int node;                 // kind 0: node index
    // kind 1
    int nmat, mm[3], out[3], add_vec[3];   // MUL_MAT node, node whose buffer receives y, node/leaf supplying the added vector (-1 none; see add_src)
    int add_src[3];                        // which src of the ADD node is the vector
    int prologue;                          // 0 quantize src1 with a separate kernel, 1 rms-norm, 2 silu, 3 activation left quantized by the attention step
    int p0, p1;                            // prologue 1: RMS_NORM node, MUL node; prologue 2: UNARY node, MUL node
    int ws;                                // workspace role
    int out_scratch[3];                    // >= 0: the result never leaves the fused steps (q, k, v, gate, up): it goes to this private buffer
    int in_scratch[2];                     // prologue 2: gate / up come from these private buffers
    // kind 2
    int rope_q, rope_k, cpy_k, cpy_v, kq, soft, kqv, cont, quant_out;
    int q_scratch, k_scratch, v_scratch;   // private buffers holding this token's q / k / v (see out_scratch)
    int out_private;                       // the f32 attention output is read by nobody (wo takes the quantized copy): keep it private
};
struct b200_plan {
    uint64_t key;
    int n_nodes;
    std::vector<b200_step> steps;
    // CUDA graph of the whole step sequence, valid while every tensor keeps its address (`bind`); the destination cell of the
    // attention launches is read from device memory so that the same graph serves token after token
    // (the reference captures node by node and patches the cpy nodes: ggml-cuda.cu:2602-2617, 2640, 2741-2771)
    cudaGraphExec_t exec = nullptr;
    std::vector<int> store_nodes;      // cache-store nodes and their destination views: their address IS the destination cell
    bool has_attn = false;
    uint64_t bind = 0;
    int seen = 0;
    uint64_t launches = 0, nodes = 0, fused = 0;
    ~b200_plan() { if (exec) cudaGraphExecDestroy(exec); }
};
// Why private buffers: the graph allocator (ggml_gallocr) recycles a tensor's memory right after its last consumer IN GRAPH ORDER.
// A fused step reads q / k / v (or gate / up) later than the nodes it replaces would have, by which time the allocator may have handed
// their memory to another tensor of the same size (measured: Vcur lands exactly on Kcur).  Results that are consumed only inside
// fused steps therefore never touch the graph's buffers; results that escape (ffn_inp, l_out, logits) are written at their own
// node's position like the unfused path would.
enum { SCR_Q = 0, SCR_K = 1, SCR_V = 2, SCR_G = 3, SCR_U = 4, SCR_ATT = 5, SCR_COUNT = 6 };

struct b200_backend_ctx {
    int device;
    cudaStream_t stream = nullptr;
    void * act_ws = nullptr;       // quantized-activation workspace (grown on demand)
    size_t act_ws_bytes = 0;
    // fused decode path (graph_compute): one activation workspace per role so that a producer never overwrites what the
    // previous launch may still be reading under programmatic dependent launch; barrier state of pb200_gemv_fused; plan cache
    void * fact_ws[3] = {nullptr, nullptr, nullptr};   // 0: norm prologue (K = n_embd), 1: attention output, 2: silu prologue (K = n_ff)
    size_t fact_bytes[3] = {0, 0, 0};
    void * sync_ws = nullptr;
    float * attn_tmp = nullptr;
    size_t attn_tmp_floats = 0;
    float * scratch[SCR_COUNT] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    size_t scratch_floats[SCR_COUNT] = {0, 0, 0, 0, 0, 0};
    cudaEvent_t copy_event = nullptr;
    int32_t * kvh_dev = nullptr;       // destination cell of the current token (device word read by the captured attention launches)
    int32_t * kvh_host = nullptr;      // pinned staging words for it
    unsigned kvh_idx = 0;
    bool capturing = false, capture_failed = false;
    std::vector<char> skip;
    std::vector<b200_plan *> plans;
    void * mmq_ws = nullptr;       // fp16 activation tiles for the tensor-core path (grown on demand)
    size_t mmq_ws_bytes = 0;
    // generation of the plugin-owned device buffers a captured launch can hold by value (act_ws, mmq_ws, fact_ws, scratch,
    // attn_tmp, sync_ws, kvh_dev): bumped at every (re)allocation and folded into each plan's `bind`, so that a CUDA graph
    // captured before a buffer moved is recaptured instead of replayed.  Buffers only grow, so it changes a bounded number of times.
    uint64_t ws_gen = 0;
    std::string name;
};
struct b200_buffer_ctx {
    int device;
    void * base;
};

static const int64_t MMQ_MIN_COLS = 8;
static bool mmq_ok(enum ggml_type t, int64_t k) {   // mirrors mmq_supported() of the library
    if (t == GGML_TYPE_Q4_K || t == GGML_TYPE_Q5_K || t == GGML_TYPE_Q6_K) return k % 256 == 0;
    return (t == GGML_TYPE_Q8_0 || t == GGML_TYPE_Q5_1) && k % 64 == 0 && k >= 256;
}
static bool type_is_quant(enum ggml_type t) {
    return t == GGML_TYPE_Q4_K || t == GGML_TYPE_Q5_K || t == GGML_TYPE_Q6_K || t == GGML_TYPE_Q8_0 || t == GGML_TYPE_Q5_1;
}

// ---------------------------------------------------------------------------------------------------- buffer
static const char * b200_buffer_get_name(ggml_backend_buffer_t) { return "B200"; }
static void b200_buffer_free(ggml_backend_buffer_t buffer) {
    b200_buffer_ctx * ctx = (b200_buffer_ctx *) buffer->context;
    cudaSetDevice(ctx->device);
    cudaFree(ctx->base);
    delete ctx;
}
static void * b200_buffer_get_base(ggml_backend_buffer_t buffer) { return ((b200_buffer_ctx *) buffer->context)->base; }
static void b200_buffer_init_tensor(ggml_backend_buffer_t buffer, ggml_tensor * tensor) {
    // like ggml-cuda.cu:444-462: zero the padding behind quantized rows so that over-reads see defined bytes
    if (tensor->view_src == nullptr && ggml_is_quantized(tensor->type)) {
        b200_buffer_ctx * ctx = (b200_buffer_ctx *) buffer->context;
        const size_t sz = ggml_nbytes(tensor);
        const size_t padded = ggml_backend_buft_get_alloc_size(buffer->buft, tensor);
        if (padded > sz) {
            cudaSetDevice(ctx->device);
            CUDA_OK(cudaMemset((char *) tensor->data + sz, 0, padded - sz));
        }
    }
}
static void b200_buffer_memset_tensor(ggml_backend_buffer_t buffer, ggml_tensor * tensor, uint8_t value, size_t offset, size_t size) {
    cudaSetDevice(((b200_buffer_ctx *) buffer->context)->device);
    CUDA_OK(cudaMemset((char *) tensor->data + offset, value, size));
}
static void b200_buffer_set_tensor(ggml_backend_buffer_t buffer, ggml_tensor * tensor, const void * data, size_t offset, size_t size) {
    cudaSetDevice(((b200_buffer_ctx *) buffer->context)->device);
    CUDA_OK(cudaMemcpy((char *) tensor->data + offset, data, size, cudaMemcpyHostToDevice));   // synchronous w.r.t. the caller
}
static void b200_buffer_get_tensor(ggml_backend_buffer_t buffer, const ggml_tensor * tensor, void * data, size_t offset, size_t size) {
    cudaSetDevice(((b200_buffer_ctx *) buffer->context)->device);
    CUDA_OK(cudaDeviceSynchronize());
    CUDA_OK(cudaMemcpy(data, (const char *) tensor->data + offset, size, cudaMemcpyDeviceToHost));
}
static bool b200_buffer_cpy_tensor(ggml_backend_buffer_t buffer, const ggml_tensor * src, ggml_tensor * dst) {
    if (src->buffer && src->buffer->iface.get_name == b200_buffer_get_name && ggml_is_contiguous(src) && ggml_is_contiguous(dst)) {
        cudaSetDevice(((b200_buffer_ctx *) buffer->context)->device);
        CUDA_OK(cudaDeviceSynchronize());
        CUDA_OK(cudaMemcpy(dst->data, src->data, ggml_nbytes(src), cudaMemcpyDeviceToDevice));
        return true;
    }
    return false;
}
static void b200_buffer_clear(ggml_backend_buffer_t buffer, uint8_t value) {
    b200_buffer_ctx * ctx = (b200_buffer_ctx *) buffer->context;
    cudaSetDevice(ctx->device);
    CUDA_OK(cudaDeviceSynchronize());
    CUDA_OK(cudaMemset(ctx->base, value, buffer->size));
}
static const ggml_backend_buffer_i b200_buffer_iface = {
    /* .get_name      = */ b200_buffer_get_name,
    /* .free_buffer   = */ b200_buffer_free,
    /* .get_base      = */ b200_buffer_get_base,
    /* .init_tensor   = */ b200_buffer_init_tensor,
    /* .memset_tensor = */ b200_buffer_memset_tensor,
    /* .set_tensor    = */ b200_buffer_set_tensor,
    /* .get_tensor    = */ b200_buffer_get_tensor,
    /* .cpy_tensor    = */ b200_buffer_cpy_tensor,
    /* .clear         = */ b200_buffer_clear,
    /* .reset         = */ nullptr,
};

// ---------------------------------------------------------------------------------------------------- buffer type
static const char * b200_buft_get_name(ggml_backend_buffer_type_t buft) { return ((b200_device_ctx *) buft->device->context)->name.c_str(); }
static ggml_backend_buffer_t b200_buft_alloc(ggml_backend_buffer_type_t buft, size_t size) {
    b200_device_ctx * dctx = (b200_device_ctx *) buft->device->context;
    cudaSetDevice(dctx->device);
    void * p = nullptr;
    size = size > 0 ? size : 1;
    if (cudaMalloc(&p, size + 256) != cudaSuccess) {   // allocation failure -> NULL (ggml-cuda.cu:556-561), no abort
        cudaGetLastError();
        return nullptr;
    }
    return ggml_backend_buffer_init(buft, b200_buffer_iface, new b200_buffer_ctx{dctx->device, p}, size);
}
static size_t b200_buft_alignment(ggml_backend_buffer_type_t) { return 128; }
static size_t b200_buft_alloc_size(ggml_backend_buffer_type_t, const ggml_tensor * tensor) {
    size_t size = ggml_nbytes(tensor);
    if (ggml_is_quantized(tensor->type)) size = (size + 15) / 16 * 16 + 16;   // the GEMV's bulk copies move whole 16-B units
    return size;
}
static const ggml_backend_buffer_type_i b200_buft_iface = {
    /* .get_name       = */ b200_buft_get_name,
    /* .alloc_buffer   = */ b200_buft_alloc,
    /* .get_alignment  = */ b200_buft_alignment,
    /* .get_max_size   = */ nullptr,
    /* .get_alloc_size = */ b200_buft_alloc_size,
    /* .is_host        = */ nullptr,
};

// ---------------------------------------------------------------------------------------------------- op support
static bool is_noop(enum ggml_op op) {
    return op == GGML_OP_NONE || op == GGML_OP_RESHAPE || op == GGML_OP_VIEW || op == GGML_OP_PERMUTE || op == GGML_OP_TRANSPOSE;
}
// b is broadcast over a by plain repetition of its contiguous data (bias / norm weight / same shape)
static bool bcast_ok(const ggml_tensor * a, const ggml_tensor * b) {
    if (!ggml_is_contiguous(a) || !ggml_is_contiguous(b)) return false;
    bool tail = false;
    for (int d = 0; d < GGML_MAX_DIMS; d++) {
        if (b->ne[d] == a->ne[d] && !tail) continue;
        if (b->ne[d] == 1) { tail = true; continue; }
        return false;
    }
    return true;
}
static bool b200_supports_op(ggml_backend_dev_t, const ggml_tensor * op) {
    const ggml_tensor * a = op->src[0], * b = op->src[1];
    if (is_noop(op->op)) return true;
    switch (op->op) {
        case GGML_OP_RMS_NORM:
            return a->type == GGML_TYPE_F32 && op->type == GGML_TYPE_F32 && ggml_is_contiguous(a) && ggml_is_contiguous(op);
        case GGML_OP_ADD:
        case GGML_OP_MUL:
            return a->type == GGML_TYPE_F32 && b->type == GGML_TYPE_F32 && op->type == GGML_TYPE_F32 && ggml_is_contiguous(op) && bcast_ok(a, b);
        case GGML_OP_UNARY:
            return ggml_get_unary_op(op) == GGML_UNARY_OP_SILU && a->type == GGML_TYPE_F32 && ggml_is_contiguous(a) && ggml_is_contiguous(op);
        case GGML_OP_MUL_MAT: {
            if (b->type != GGML_TYPE_F32 || op->type != GGML_TYPE_F32) return false;
            if (a->ne[2] == 0 || a->ne[3] == 0 || b->ne[2] % a->ne[2] || b->ne[3] % a->ne[3]) return false;
            if (a->type == GGML_TYPE_F16) return a->nb[0] == sizeof(ggml_fp16_t) && b->nb[0] == sizeof(float) && op->nb[0] == sizeof(float);
            if (!type_is_quant(a->type)) return false;
            // quantized weights: rows of src1 must be dense.  The decode GEMV handles one activation column per launch; k-quant
            // weights with K % 256 == 0 take the tensor-core path (pb200_mul_mat_q) for any number of columns.
            if (!(ggml_is_contiguous(a) && b->nb[0] == sizeof(float) && ggml_is_contiguous(op) && a->ne[0] % ggml_blck_size(a->type) == 0)) return false;
            if (mmq_ok(a->type, a->ne[0]) && b->nb[1] % 16 == 0) return true;
            return b->ne[1] * b->ne[2] * b->ne[3] <= 64;
        }
        case GGML_OP_ROPE: {
            // f32 (q / k of the forward graph) or f16 -> f16 (the in-place K-shift of the f16 K cache, build_k_shift src/llama.cpp:10665-10719)
            const int mode = ((const int32_t *) op->op_params)[2];
            const bool f32 = a->type == GGML_TYPE_F32 && op->type == GGML_TYPE_F32, f16 = a->type == GGML_TYPE_F16 && op->type == GGML_TYPE_F16;
            return (f32 || f16) && ggml_is_contiguous(a) && ggml_is_contiguous(op) && (mode == 0 || mode == 2) &&
                   a->ne[3] == 1 && (op->src[2] == nullptr || op->src[2]->type == GGML_TYPE_F32);
        }
        case GGML_OP_SOFT_MAX: {
            float max_bias;
            memcpy(&max_bias, (const float *) op->op_params + 1, sizeof(float));
            return a->type == GGML_TYPE_F32 && ggml_is_contiguous(a) && ggml_is_contiguous(op) && max_bias == 0.0f &&
                   (b == nullptr || (b->type == GGML_TYPE_F32 && ggml_is_contiguous(b) && b->ne[0] == a->ne[0] && b->ne[1] >= a->ne[1]));
        }
        case GGML_OP_CPY:
        case GGML_OP_DUP:
        case GGML_OP_CONT:
            return a->type == GGML_TYPE_F32 && (op->type == GGML_TYPE_F32 || op->type == GGML_TYPE_F16) && ggml_nelements(a) == ggml_nelements(op);
        case GGML_OP_FLASH_ATTN_EXT: {   // f16 K / V (the KV cache types this backend runs with), any head size up to 256, one batch
            const ggml_tensor * k = op->src[1], * v = op->src[2], * m = op->src[3];
            return a->type == GGML_TYPE_F32 && k->type == GGML_TYPE_F16 && v->type == GGML_TYPE_F16 && op->type == GGML_TYPE_F32 && a->ne[0] <= 256 &&
                   a->ne[0] == k->ne[0] && a->ne[0] == v->ne[0] && a->ne[3] == 1 && k->ne[3] == 1 && v->ne[3] == 1 && k->ne[2] == v->ne[2] && k->ne[1] == v->ne[1] &&
                   k->ne[2] > 0 && a->ne[2] % k->ne[2] == 0 && a->nb[0] == sizeof(float) && k->nb[0] == 2 && v->nb[0] == 2 && ggml_is_contiguous(op) &&
                   (m == nullptr || (m->type == GGML_TYPE_F16 && m->ne[0] == k->ne[1] && m->ne[1] >= a->ne[1] && m->nb[0] == 2));
        }
        case GGML_OP_GET_ROWS:
            return (a->type == GGML_TYPE_F32 || a->type == GGML_TYPE_F16 || type_is_quant(a->type)) && b->type == GGML_TYPE_I32 && op->type == GGML_TYPE_F32 &&
                   ggml_is_contiguous(a) && ggml_is_contiguous(b) && ggml_is_contiguous(op) && a->ne[2] == 1 && a->ne[3] == 1 && b->ne[2] == 1 && b->ne[3] == 1;
        default:
            return false;
    }
}

// ---------------------------------------------------------------------------------------------------- compute
#define PB_OK(expr)                                                                          \
    do {                                                                                     \
        int rc_ = (expr);                                                                    \
        if (rc_ != 0) {                                                                      \
            fprintf(stderr, "ggml-b200: %s -> %s (%d)\n", #expr, pb200_error_string(rc_), rc_); \
            return false;                                                                    \
        }                                                                                    \
    } while (0)

static bool b200_compute_node(b200_backend_ctx * ctx, ggml_tensor * dst) {
    const ggml_tensor * a = dst->src[0], * b = dst->src[1];
    void * st = ctx->stream;
    switch (dst->op) {
        case GGML_OP_RMS_NORM: {
            float eps;
            memcpy(&eps, dst->op_params, sizeof(float));
            PB_OK(pb200_rms_norm((const float *) a->data, (float *) dst->data, a->ne[0], ggml_nrows(a), eps, st));
            return true;
        }
        case GGML_OP_ADD:
        case GGML_OP_MUL:
            PB_OK(pb200_binary(dst->op == GGML_OP_ADD ? 0 : 1, (const float *) a->data, (const float *) b->data, (float *) dst->data, ggml_nelements(dst),
                               ggml_nelements(b), st));
            return true;
        case GGML_OP_UNARY:
            PB_OK(pb200_silu((const float *) a->data, (float *) dst->data, ggml_nelements(dst), st));
            return true;
        case GGML_OP_MUL_MAT: {
            if (a->type == GGML_TYPE_F16) {
                const int64_t ne[4] = {dst->ne[0], dst->ne[1], dst->ne[2], dst->ne[3]};
                const int64_t as[4] = {(int64_t) a->nb[0], (int64_t) a->nb[1], (int64_t) a->nb[2], (int64_t) a->nb[3]};
                const int64_t bs[4] = {(int64_t) b->nb[0], (int64_t) b->nb[1], (int64_t) b->nb[2], (int64_t) b->nb[3]};
                const int64_t ds[4] = {(int64_t) dst->nb[0], (int64_t) dst->nb[1], (int64_t) dst->nb[2], (int64_t) dst->nb[3]};
                PB_OK(pb200_mul_mat_f16(a->data, (const float *) b->data, (float *) dst->data, a->ne[0], ne, b->ne[2] / a->ne[2], b->ne[3] / a->ne[3], as, bs,
                                        ds, st));
                return true;
            }
            const int64_t K = a->ne[0], N = a->ne[1];
            const size_t need = pb200_act_workspace_bytes(K);
            // no allocation inside a capture (as grow_ws): enqueue nothing, the capture is discarded and the call runs directly
            if (need > ctx->act_ws_bytes && ctx->capturing) { ctx->capture_failed = true; return true; }
            if (need > ctx->act_ws_bytes) {
                if (ctx->act_ws) { CUDA_OK(cudaStreamSynchronize(ctx->stream)); cudaFree(ctx->act_ws); }
                CUDA_OK(cudaMalloc(&ctx->act_ws, need + 256));
                ctx->act_ws_bytes = need;
                ctx->ws_gen++;
            }
            const int64_t r2 = b->ne[2] / a->ne[2], r3 = b->ne[3] / a->ne[3];
            if (b->ne[1] >= MMQ_MIN_COLS && mmq_ok(a->type, K) && b->nb[1] % 16 == 0 && (uintptr_t) b->data % 16 == 0 && b->nb[2] % 16 == 0 && b->nb[3] % 16 == 0 &&
                (uintptr_t) a->data % 16 == 0 && a->nb[2] % 16 == 0 && a->nb[3] % 16 == 0) {   // the prep kernel reads rows as float4
                // batched / prefill: the reference switches to mul_mat_q above 8 columns as well (ggml-cuda/mmq.cu:137-139)
                const size_t need_q = pb200_mul_mat_q_workspace_bytes(K, b->ne[1]);
                if (need_q > ctx->mmq_ws_bytes && ctx->capturing) { ctx->capture_failed = true; return true; }
                if (need_q > ctx->mmq_ws_bytes) {
                    if (ctx->mmq_ws) { CUDA_OK(cudaStreamSynchronize(ctx->stream)); cudaFree(ctx->mmq_ws); }
                    CUDA_OK(cudaMalloc(&ctx->mmq_ws, need_q + 256));
                    ctx->mmq_ws_bytes = need_q;
                    ctx->ws_gen++;
                }
                for (int64_t i3 = 0; i3 < b->ne[3]; i3++)
                    for (int64_t i2 = 0; i2 < b->ne[2]; i2++) {
                        const char * w = (const char *) a->data + (i2 / r2) * a->nb[2] + (i3 / r3) * a->nb[3];
                        const float * x = (const float *) ((const char *) b->data + i2 * b->nb[2] + i3 * b->nb[3]);
                        float * y = (float *) ((char *) dst->data + i2 * dst->nb[2] + i3 * dst->nb[3]);
                        PB_OK(pb200_mul_mat_q((int) a->type, w, N, K, x, (int64_t) (b->nb[1] / sizeof(float)), b->ne[1], y, nullptr, nullptr, ctx->mmq_ws, st));
                    }
                return true;
            }
            for (int64_t i3 = 0; i3 < b->ne[3]; i3++)
                for (int64_t i2 = 0; i2 < b->ne[2]; i2++)
                    for (int64_t i1 = 0; i1 < b->ne[1]; i1++) {
                        const char * w = (const char *) a->data + (i2 / r2) * a->nb[2] + (i3 / r3) * a->nb[3];
                        const float * x = (const float *) ((const char *) b->data + i1 * b->nb[1] + i2 * b->nb[2] + i3 * b->nb[3]);
                        float * y = (float *) ((char *) dst->data + i1 * dst->nb[1] + i2 * dst->nb[2] + i3 * dst->nb[3]);
                        PB_OK(pb200_mul_mat_vec((int) a->type, w, N, K, x, y, ctx->act_ws, st));
                    }
            return true;
        }
        case GGML_OP_ROPE: {
            const int32_t * p = (const int32_t *) dst->op_params;
            float fb, fs, ef, af, bf, bsl;
            memcpy(&fb, p + 5, 4); memcpy(&fs, p + 6, 4); memcpy(&ef, p + 7, 4); memcpy(&af, p + 8, 4); memcpy(&bf, p + 9, 4); memcpy(&bsl, p + 10, 4);
            if (a->type == GGML_TYPE_F16) {
                PB_OK(pb200_rope_f16(a->data, dst->data, a->ne[2], (int) a->ne[1], (int) a->ne[0], p[1], p[2], (const int32_t *) b->data, fb, fs, ef, af, bf,
                                     bsl, p[4], dst->src[2] ? (const float *) dst->src[2]->data : nullptr, st));
                return true;
            }
            PB_OK(pb200_rope((const float *) a->data, (float *) dst->data, a->ne[2], (int) a->ne[1], (int) a->ne[0], p[1], p[2], (const int32_t *) b->data, fb, fs,
                             ef, af, bf, bsl, p[4], dst->src[2] ? (const float *) dst->src[2]->data : nullptr, st));
            return true;
        }
        case GGML_OP_SOFT_MAX: {
            float scale;
            memcpy(&scale, dst->op_params, sizeof(float));
            PB_OK(pb200_soft_max((const float *) a->data, b ? (const float *) b->data : nullptr, (float *) dst->data, a->ne[0], ggml_nrows(a), a->ne[1], scale, st));
            return true;
        }
        case GGML_OP_CPY:
        case GGML_OP_DUP:
        case GGML_OP_CONT: {
            // enumerate in the SOURCE's logical order when shapes agree, else both sides must be contiguous-compatible
            const ggml_tensor * d = dst->op == GGML_OP_CPY ? dst->src[1] : dst;
            void * out = dst->data;   // a CPY node is a view of its destination (ggml_cpy_impl): same address, and what the CPU backend writes to
            int64_t ne[4], sb[4], db[4];
            if (ggml_are_same_shape(a, d)) {
                for (int i = 0; i < 4; i++) { ne[i] = a->ne[i]; sb[i] = a->nb[i]; db[i] = d->nb[i]; }
            } else if (ggml_is_contiguous(d)) {          // e.g. cont_2d of a permuted tensor, or cpy into a flat cache view
                const int64_t es = (int64_t) ggml_type_size(d->type);
                for (int i = 0; i < 4; i++) { ne[i] = a->ne[i]; sb[i] = a->nb[i]; }
                db[0] = es; db[1] = es * ne[0]; db[2] = db[1] * ne[1]; db[3] = db[2] * ne[2];
            } else if (ggml_is_contiguous(a)) {
                for (int i = 0; i < 4; i++) { ne[i] = d->ne[i]; db[i] = d->nb[i]; }
                sb[0] = 4; sb[1] = 4 * ne[0]; sb[2] = sb[1] * ne[1]; sb[3] = sb[2] * ne[2];
            } else {
                return false;
            }
            PB_OK(pb200_copy_strided(a->data, out, d->type == GGML_TYPE_F16, ne, sb, db, st));
            return true;
        }
        case GGML_OP_FLASH_ATTN_EXT: {
            const ggml_tensor * k = dst->src[1], * v = dst->src[2], * m = dst->src[3];
            float scale, max_bias, softcap;
            memcpy(&scale, (const float *) dst->op_params + 0, 4); memcpy(&max_bias, (const float *) dst->op_params + 1, 4); memcpy(&softcap, (const float *) dst->op_params + 2, 4);
            const int64_t qnb[2] = {(int64_t) a->nb[1], (int64_t) a->nb[2]}, knb[2] = {(int64_t) k->nb[1], (int64_t) k->nb[2]}, vnb[2] = {(int64_t) v->nb[1], (int64_t) v->nb[2]};
            PB_OK(pb200_flash_attn_ext((const float *) a->data, k->data, v->data, m ? m->data : nullptr, (float *) dst->data, (int) a->ne[0], (int) a->ne[1], (int) a->ne[2],
                                       (int) k->ne[2], (int) k->ne[1], qnb, knb, vnb, m ? (int64_t) m->nb[1] : 0, scale, max_bias, softcap, st));
            return true;
        }
        case GGML_OP_GET_ROWS:
            PB_OK(pb200_get_rows((int) a->type, a->data, a->ne[0], (const int32_t *) b->data, ggml_nelements(b), (float *) dst->data, st));
            return true;
        default:
            return false;
    }
}

// ---------------------------------------------------------------------------------------------------- backend
static ggml_guid_t b200_guid() {
    static ggml_guid guid = {0xb2, 0x00, 0x5e, 0x10, 0x0a, 0x47, 0x4d, 0x41, 0x9c, 0x21, 0x70, 0x72, 0x69, 0x6d, 0x61, 0x01};
    return &guid;
}
static const char * b200_backend_get_name(ggml_backend_t backend) { return ((b200_backend_ctx *) backend->context)->name.c_str(); }
static void b200_backend_free(ggml_backend_t backend) {
    b200_backend_ctx * ctx = (b200_backend_ctx *) backend->context;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    if (ctx->act_ws) cudaFree(ctx->act_ws);
    if (ctx->mmq_ws) cudaFree(ctx->mmq_ws);
    for (void * p : ctx->fact_ws) if (p) cudaFree(p);
    if (ctx->sync_ws) cudaFree(ctx->sync_ws);
    if (ctx->attn_tmp) cudaFree(ctx->attn_tmp);
    for (float * p : ctx->scratch) if (p) cudaFree(p);
    if (ctx->copy_event) cudaEventDestroy(ctx->copy_event);
    if (ctx->kvh_dev) cudaFree(ctx->kvh_dev);
    if (ctx->kvh_host) cudaFreeHost(ctx->kvh_host);
    for (b200_plan * p : ctx->plans) delete p;
    cudaStreamDestroy(ctx->stream);
    delete ctx;
    delete backend;
}
static ggml_backend_buffer_type_t b200_backend_get_default_buft(ggml_backend_t backend) {
    return ggml_backend_b200_buffer_type(((b200_backend_ctx *) backend->context)->device);
}
static void b200_backend_set_tensor_async(ggml_backend_t backend, ggml_tensor * tensor, const void * data, size_t offset, size_t size) {
    b200_backend_ctx * ctx = (b200_backend_ctx *) backend->context;
    cudaSetDevice(ctx->device);
    CUDA_OK(cudaMemcpyAsync((char *) tensor->data + offset, data, size, cudaMemcpyHostToDevice, ctx->stream));
}
static void b200_backend_get_tensor_async(ggml_backend_t backend, const ggml_tensor * tensor, void * data, size_t offset, size_t size) {
    b200_backend_ctx * ctx = (b200_backend_ctx *) backend->context;
    cudaSetDevice(ctx->device);
    CUDA_OK(cudaMemcpyAsync(data, (const char *) tensor->data + offset, size, cudaMemcpyDeviceToHost, ctx->stream));
}
static void b200_backend_synchronize(ggml_backend_t backend) {
    b200_backend_ctx * ctx = (b200_backend_ctx *) backend->context;
    cudaSetDevice(ctx->device);
    CUDA_OK(cudaStreamSynchronize(ctx->stream));
}
// ====================================================================================================================
// graph_compute.  The reference dispatches node by node and hides the launch overhead behind a CUDA graph
// (ggml_backend_cuda_graph_compute, ggml-cuda.cu:2508-2778).  Here the decode graph (one token) of build_llama / build_qwen2
// (src/llama.cpp:11000-11216, 12736-12916, FA off) is pattern-matched into the fused launches of the engine:
//     RMS_NORM -> MUL(norm weight) -> {MUL_MAT k-quant}x1..3 [-> ADD bias]            => ONE pb200_gemv_fused (rms-norm prologue)
//     ROPE q, ROPE k, CPY k -> cache, CPY v^T -> cache, MUL_MAT(K,q), SOFT_MAX, MUL_MAT(V,p), CONT  => ONE pb200_attn_ggml
//     MUL_MAT(wo) -> ADD residual                                                     => ONE pb200_gemv_fused (activation quantized by the attention launch)
//     UNARY(SILU) -> MUL -> MUL_MAT(down) -> ADD residual                             => ONE pb200_gemv_fused (silu prologue)
// i.e. 5 launches per layer instead of ~25, every launch chained with programmatic dependent launch so that the next kernel's
// weight stream starts while the previous one drains.  Anything that does not match runs 1:1 as before.  The plan is derived once
// per graph topology (llama.cpp rebuilds the same topology every token; n_kv changes it every 32 tokens) and re-bound to the
// tensors' current addresses / view offsets on every call — the reference patches its captured graph for the same reason
// (ggml-cuda.cu:2602-2617, 2741-2752).  No CUDA graph is needed on top: the host enqueues ~5 launches per layer (~1 ms per 70B token)
// while the device needs ~9 ms, so the stream never runs dry.
static uint64_t fnv(uint64_t h, uint64_t v) { h ^= v; return h * 0x100000001b3ull; }
static int node_index_of(const ggml_cgraph * g, const ggml_tensor * t, int hint_end) {
    for (int i = hint_end - 1; i >= 0; i--) if (ggml_graph_node((ggml_cgraph *) g, i) == t) return i;
    return -1;
}
// topology signature of a graph: ops, types, shapes, strides that matter, op parameters, what each node reads.  Computed on every
// graph_compute call (the host may rebuild a different graph in the same memory), so it is kept to three multiplies per node.
static uint64_t graph_key(ggml_cgraph * g) {
    const int n = ggml_graph_n_nodes(g);
    uint64_t h = fnv(0xcbf29ce484222325ull, (uint64_t) n);
    for (int i = 0; i < n; i++) {
        const ggml_tensor * t = ggml_graph_node(g, i);
        const uint64_t w0 = (uint64_t) t->op | ((uint64_t) t->type << 8) | ((uint64_t) t->ne[0] << 16) ^ ((uint64_t) t->ne[1] << 40);
        const uint64_t w1 = (uint64_t) t->ne[2] ^ ((uint64_t) t->nb[1] << 12) ^ ((uint64_t) t->nb[2] << 36) ^ (uint64_t) (uint32_t) t->op_params[0] ^
                            ((uint64_t) (uint32_t) t->op_params[1] << 32) ^ ((uint64_t) (uint32_t) t->op_params[2] << 17) ^ ((uint64_t) (uint32_t) t->op_params[5] << 7);
        uint64_t w2 = 0;
        for (int k = 0; k < 3; k++) {
            const ggml_tensor * sN = t->src[k];
            w2 = w2 * 1315423911ull + (sN ? (uint64_t) sN->op * 131 + (uint64_t) sN->type * 7 + (uint64_t) sN->ne[0] * 3 + (uint64_t) sN->ne[1] : 0x9e37ull);
        }
        h = fnv(fnv(fnv(h, w0), w1), w2);
    }
    return h;
}
static bool is_kq(enum ggml_type t) { return t == GGML_TYPE_Q4_K || t == GGML_TYPE_Q5_K || t == GGML_TYPE_Q6_K; }
static bool is_vec_f32(const ggml_tensor * t, int64_t n) {
    return t && t->type == GGML_TYPE_F32 && t->ne[0] == n && t->ne[1] == 1 && t->ne[2] == 1 && t->ne[3] == 1 && t->nb[0] == sizeof(float);
}
// a MUL_MAT the fused GEMV takes: k-quant weights, one contiguous f32 activation column, K % 256 == 0, K <= 28672
static bool gemv_fusable(const ggml_tensor * t) {
    if (t->op != GGML_OP_MUL_MAT) return false;
    const ggml_tensor * W = t->src[0], * X = t->src[1];
    if (!is_kq(W->type) || !ggml_is_contiguous(W) || W->ne[2] != 1 || W->ne[3] != 1) return false;
    const int64_t K = W->ne[0];
    return is_vec_f32(X, K) && K % 256 == 0 && K <= 28672 && t->type == GGML_TYPE_F32 && ggml_is_contiguous(t);
}
static const ggml_tensor * strip_views(const ggml_tensor * t) {   // RESHAPE / PERMUTE / TRANSPOSE / VIEW of a COMPUTED tensor
    while (t && (t->op == GGML_OP_RESHAPE || t->op == GGML_OP_PERMUTE || t->op == GGML_OP_TRANSPOSE || t->op == GGML_OP_VIEW) && t->src[0]) t = t->src[0];
    return t;
}

struct graph_info {
    ggml_cgraph * g;
    int n;
    std::vector<std::vector<int>> cons;   // consumers of node i (direct src references, views included as nodes)
    std::unordered_map<const ggml_tensor *, int> index;
    int idx(const ggml_tensor * t) const { auto it = index.find(t); return it == index.end() ? -1 : it->second; }
};
// consumers of a node "through" no-op views: the real ops that eventually read it
static void real_consumers(const graph_info & G, int i, std::vector<int> & out) {
    for (int c : G.cons[i]) {
        const ggml_tensor * t = ggml_graph_node(G.g, c);
        if (is_noop(t->op)) real_consumers(G, c, out); else out.push_back(c);
    }
}

static bool plan_attention(const graph_info & G, int soft, std::vector<char> & taken, b200_step & st) {
    ggml_cgraph * g = G.g;
    const ggml_tensor * sm = ggml_graph_node(g, soft);
    const ggml_tensor * kq = sm->src[0], * mask = sm->src[1];
    if (!kq || kq->op != GGML_OP_MUL_MAT || !mask || mask->type != GGML_TYPE_F32) return false;
    float scale, max_bias;
    memcpy(&scale, sm->op_params, 4); memcpy(&max_bias, (const float *) sm->op_params + 1, 4);
    if (max_bias != 0.0f) return false;
    const ggml_tensor * kview = kq->src[0], * qp = kq->src[1];
    if (!kview || kview->type != GGML_TYPE_F16 || kview->op != GGML_OP_VIEW || !kview->view_src) return false;
    const ggml_tensor * ropeq = strip_views(qp);
    if (!ropeq || ropeq->op != GGML_OP_ROPE || qp->ne[0] != 128 || qp->ne[1] != 1 || qp->ne[3] != 1) return false;   // [D, n_tokens = 1, H]
    const int64_t D = 128, H = qp->ne[2], n_kv = kview->ne[1], HK = kview->ne[2];
    if (kview->ne[0] != D || HK <= 0 || H % HK || (H & 1) || (n_kv & 31)) return false;
    if (kview->nb[1] != (size_t) (HK * D * 2) || kview->nb[2] != (size_t) (D * 2) || kview->view_offs != 0) return false;
    if (mask->ne[0] != n_kv || !ggml_is_contiguous(mask)) return false;
    // the single consumer chain soft_max -> mul_mat(v, p) -> permute -> cont
    std::vector<int> c1; real_consumers(G, soft, c1);
    if (c1.size() != 1) return false;
    const int kqv_i = c1[0];
    const ggml_tensor * kqv = ggml_graph_node(g, kqv_i);
    if (kqv->op != GGML_OP_MUL_MAT || kqv->src[1] != sm) return false;
    const ggml_tensor * vview = kqv->src[0];
    if (!vview || vview->type != GGML_TYPE_F16 || vview->op != GGML_OP_VIEW || !vview->view_src || vview->view_offs != 0) return false;
    if (vview->ne[0] != n_kv || vview->ne[1] != D || vview->ne[2] != HK || vview->nb[0] != 2 || vview->nb[2] != vview->nb[1] * (size_t) D) return false;
    std::vector<int> c2; real_consumers(G, kqv_i, c2);
    if (c2.size() != 1) return false;
    const int cont_i = c2[0];
    const ggml_tensor * cont = ggml_graph_node(g, cont_i);
    if (cont->op != GGML_OP_CONT || cont->type != GGML_TYPE_F32 || ggml_nelements(cont) != D * H || !ggml_is_contiguous(cont)) return false;
    // q side: rope(reshape(Qcur)) consumed only by kq
    const int ropeq_i = G.idx(ropeq), kq_i = G.idx(kq);
    if (ropeq_i < 0 || kq_i < 0) return false;
    { std::vector<int> c; real_consumers(G, ropeq_i, c); if (c.size() != 1 || c[0] != kq_i) return false; }
    { std::vector<int> c; real_consumers(G, kq_i, c); if (c.size() != 1 || c[0] != soft) return false; }
    // k side: a ROPE node with the same parameters whose only consumer is a CPY into a view of the same K cache tensor
    int ropek_i = -1, cpyk_i = -1;
    const int w0 = std::max(0, soft - 96), w1 = std::min(G.n, soft + 16);   // the chain of one layer sits within a few dozen nodes
    for (int i = w0; i < w1; i++) {
        const ggml_tensor * t = ggml_graph_node(g, i);
        if (t->op != GGML_OP_CPY || !t->src[1] || t->src[1]->view_src != kview->view_src || taken[i]) continue;
        const ggml_tensor * rk = strip_views(t->src[0]);
        if (!rk || rk->op != GGML_OP_ROPE) continue;
        ropek_i = G.idx(rk); cpyk_i = i;
    }
    if (ropek_i < 0) return false;
    const ggml_tensor * ropek = ggml_graph_node(g, ropek_i), * cpyk = ggml_graph_node(g, cpyk_i);
    { std::vector<int> c; real_consumers(G, ropek_i, c); if (c.size() != 1 || c[0] != cpyk_i) return false; }
    if (memcmp(ropeq->op_params, ropek->op_params, sizeof(int32_t) * 11) != 0 || ropeq->src[1] != ropek->src[1] || ropeq->src[2] != ropek->src[2]) return false;
    const int32_t * rp = (const int32_t *) ropeq->op_params;
    if ((rp[2] != 0 && rp[2] != 2) || rp[1] > D || (rp[1] & 1)) return false;
    if (ropeq->src[1]->type != GGML_TYPE_I32 || (ropeq->src[2] && ropeq->src[2]->type != GGML_TYPE_F32)) return false;
    if (!ropeq->src[0] || !ropek->src[0] || ggml_nelements(ropek->src[0]) != HK * D || ropek->src[0]->type != GGML_TYPE_F32) return false;
    if (cpyk->src[1]->type != GGML_TYPE_F16 || ggml_nelements(cpyk->src[1]) != HK * D) return false;
    // v side: CPY(transpose(Vcur)) into a [1, HK*D] strided view of the same V cache tensor
    int cpyv_i = -1;
    for (int i = w0; i < w1; i++) {
        const ggml_tensor * t = ggml_graph_node(g, i);
        if (t->op == GGML_OP_CPY && t->src[1] && t->src[1]->view_src == vview->view_src && !taken[i]) cpyv_i = i;
    }
    if (cpyv_i < 0) return false;
    const ggml_tensor * cpyv = ggml_graph_node(g, cpyv_i);
    const ggml_tensor * vdst = cpyv->src[1], * vsrc = strip_views(cpyv->src[0]);
    if (vdst->type != GGML_TYPE_F16 || vdst->ne[0] != 1 || vdst->ne[1] != HK * D || vdst->nb[1] != vview->nb[1]) return false;
    if (!vsrc || vsrc->type != GGML_TYPE_F32 || ggml_nelements(vsrc) != HK * D || !ggml_is_contiguous(vsrc)) return false;
    if (!ggml_is_contiguous(ropeq->src[0]) || !ggml_is_contiguous(ropek->src[0])) return false;
    const int nodes[8] = {ropeq_i, ropek_i, cpyk_i, cpyv_i, kq_i, soft, kqv_i, cont_i};
    for (int i : nodes) if (taken[i]) return false;
    // everything the launch reads must be computed before the CONT position (where the step runs), its output after
    if (G.idx(vsrc) > cont_i) return false;
    for (int i : nodes) taken[i] = 1;
    st = b200_step{};
    st.kind = 2; st.rope_q = ropeq_i; st.rope_k = ropek_i; st.cpy_k = cpyk_i; st.cpy_v = cpyv_i; st.kq = kq_i; st.soft = soft; st.kqv = kqv_i; st.cont = cont_i;
    st.node = cont_i; st.quant_out = 0;
    return true;
}

// vector added to a mul_mat result by the single consumer ADD (bias or residual): returns the ADD node index or -1
static int find_add(const graph_info & G, int mm_i, int & vec_src) {
    std::vector<int> c; real_consumers(G, mm_i, c);
    if (c.size() != 1) return -1;
    const ggml_tensor * a = ggml_graph_node(G.g, c[0]), * mm = ggml_graph_node(G.g, mm_i);
    if (a->op != GGML_OP_ADD || a->type != GGML_TYPE_F32 || !ggml_is_contiguous(a)) return -1;
    for (int k = 0; k < 2; k++) {
        if (a->src[k] == mm && is_vec_f32(a->src[1 - k], mm->ne[0]) && ggml_is_contiguous(a->src[1 - k])) { vec_src = 1 - k; return c[0]; }
    }
    return -1;
}

static b200_plan * build_plan(ggml_cgraph * g, uint64_t key) {
    graph_info G;
    G.g = g; G.n = ggml_graph_n_nodes(g);
    G.cons.assign(G.n, {});
    G.index.reserve((size_t) G.n * 2);
    for (int i = 0; i < G.n; i++) G.index[ggml_graph_node(g, i)] = i;
    for (int i = 0; i < G.n; i++) {
        const ggml_tensor * t = ggml_graph_node(g, i);
        for (int k = 0; k < GGML_MAX_SRC; k++) {
            if (!t->src[k]) continue;
            const int j = G.idx(t->src[k]);
            if (j >= 0 && j < i) G.cons[j].push_back(i);
        }
    }
    std::vector<char> taken(G.n, 0);
    std::vector<b200_step> at(G.n);          // fused step anchored at node i (kind != 0)
    std::vector<char> has(G.n, 0);
    static const bool no_fuse = getenv("GGML_B200_NO_FUSE") != nullptr;
    bool fused_ok = !no_fuse;
    std::vector<int> attn_anchor;
    if (fused_ok) {
        // 1) attention chains (anchor: SOFT_MAX; the step runs at its CONT node)
        for (int i = 0; i < G.n; i++) {
            const ggml_tensor * t = ggml_graph_node(g, i);
            if (t->op != GGML_OP_SOFT_MAX || taken[i]) continue;
            b200_step st;
            if (plan_attention(G, i, taken, st)) {
                st.q_scratch = st.k_scratch = st.v_scratch = -1; st.out_private = 0;
                at[st.node] = st; has[st.node] = 1; attn_anchor.push_back(st.node);
            }
        }
        // 2) mat-vec groups (anchor: the activation shared by k-quant MUL_MATs with one column)
        for (int i = 0; i < G.n; i++) {
            const ggml_tensor * t = ggml_graph_node(g, i);
            if (taken[i] || !gemv_fusable(t)) continue;
            const ggml_tensor * W = t->src[0], * X = t->src[1];
            const int64_t K = W->ne[0];
            b200_step st{};
            st.kind = 1; st.prologue = 0; st.p0 = st.p1 = -1; st.ws = 0;
            for (int j = 0; j < 3; j++) st.out_scratch[j] = -1;
            st.in_scratch[0] = st.in_scratch[1] = -1;
            const int xi = G.idx(X);
            if (xi >= 0 && X->op == GGML_OP_MUL && !taken[xi]) {
                // prologue candidates: MUL(RMS_NORM(x), w) or MUL(SILU(g), u), intermediate results read by nobody else
                for (int k = 0; k < 2; k++) {
                    const ggml_tensor * a = X->src[k], * b = X->src[1 - k];
                    const int ai = G.idx(a);
                    if (ai < 0 || taken[ai]) continue;
                    std::vector<int> ca; real_consumers(G, ai, ca);
                    if (ca.size() != 1 || ca[0] != xi) continue;
                    if (a->op == GGML_OP_RMS_NORM && is_vec_f32(b, K) && ggml_is_contiguous(b) && is_vec_f32(a->src[0], K) && ggml_is_contiguous(a->src[0])) {
                        st.prologue = 1; st.p0 = ai; st.p1 = xi; st.ws = 0; break;
                    }
                    if (a->op == GGML_OP_UNARY && ggml_get_unary_op(a) == GGML_UNARY_OP_SILU && is_vec_f32(b, K) && ggml_is_contiguous(b) &&
                        is_vec_f32(a->src[0], K) && ggml_is_contiguous(a->src[0])) {
                        // gate and up must have been redirected to private buffers by the group that produced them (liveness, see above)
                        const int gi = G.idx(a->src[0]), ui = G.idx(b);
                        int sg = -1, su = -1;
                        for (int q = std::max(0, i - 64); q < i; q++) {
                            if (!has[q] || at[q].kind != 1) continue;
                            for (int j = 0; j < at[q].nmat; j++) {
                                if (at[q].out[j] == gi) sg = at[q].out_scratch[j];
                                if (at[q].out[j] == ui) su = at[q].out_scratch[j];
                            }
                        }
                        if (sg >= 0 && su >= 0) { st.prologue = 2; st.p0 = ai; st.p1 = xi; st.ws = 2; st.in_scratch[0] = sg; st.in_scratch[1] = su; }
                        break;
                    }
                }
            } else if (xi >= 0 && has[xi] && at[xi].kind == 2) {
                st.prologue = 3; st.ws = 1;                                   // X is the CONT of a fused attention step
            }
            // all k-quant mat-vecs fed by X
            std::vector<int> cx, group;
            if (xi >= 0) real_consumers(G, xi, cx); else cx.push_back(i);
            bool all_mm = true;
            for (int c : cx) {
                const ggml_tensor * m = ggml_graph_node(g, c);
                if (m->op != GGML_OP_MUL_MAT || m->src[1] != X || !is_kq(m->src[0]->type) || m->src[0]->ne[0] != K || !ggml_is_contiguous(m->src[0]) ||
                    m->src[0]->ne[2] != 1 || m->src[0]->ne[3] != 1 || !ggml_is_contiguous(m) || taken[c]) { all_mm = false; break; }
            }
            if (!all_mm || cx.size() > 3) {
                // somebody else reads the activation (or too many matrices): keep it materialised, one launch per matrix
                if (st.prologue == 1 || st.prologue == 2) { st.prologue = 0; st.p0 = st.p1 = -1; st.in_scratch[0] = st.in_scratch[1] = -1; }
                if (st.prologue == 3 && cx.size() != 1) st.prologue = 0;
                group.push_back(i);
            } else {
                group = cx;
                std::sort(group.begin(), group.end());
            }
            st.nmat = (int) group.size();
            int last = 0;
            bool need_graph_buffers = false;
            for (int j = 0; j < st.nmat; j++) {
                st.mm[j] = group[j]; st.out[j] = group[j]; st.add_vec[j] = -1; st.add_src[j] = 0;
                int vs = 0;
                const int ad = find_add(G, group[j], vs);
                // with several matrices the step runs later than some of its ADDs: only fold vectors that cannot have been recycled
                // by the graph allocator in between (leafs: biases)
                if (ad >= 0 && !taken[ad] && (st.nmat == 1 || ggml_graph_node(g, ad)->src[vs]->op == GGML_OP_NONE)) { st.out[j] = ad; st.add_vec[j] = ad; st.add_src[j] = vs; }
                last = std::max(last, st.out[j]);
            }
            if (st.nmat > 1) {
                // results of a multi-matrix group are produced at ONE point in time: each must be consumed only inside fused steps
                // (attention: q / k / v; silu prologue: gate / up) so that it can live in a private buffer
                for (int j = 0; j < st.nmat; j++) {
                    std::vector<int> co; real_consumers(G, st.out[j], co);
                    int slot = -1;
                    for (int anchor : attn_anchor) {
                        if (anchor < i || anchor > i + 96) continue;
                        const b200_step & A = at[anchor];
                        const ggml_tensor * o = ggml_graph_node(g, st.out[j]);
                        if (co.size() == 1 && co[0] == A.rope_q && strip_views(ggml_graph_node(g, A.rope_q)->src[0]) == o) slot = SCR_Q;
                        if (co.size() == 1 && co[0] == A.rope_k && strip_views(ggml_graph_node(g, A.rope_k)->src[0]) == o) slot = SCR_K;
                        if (co.size() == 1 && co[0] == A.cpy_v && strip_views(ggml_graph_node(g, A.cpy_v)->src[0]) == o) slot = SCR_V;
                    }
                    if (slot < 0 && co.size() == 1) {
                        const ggml_tensor * c0 = ggml_graph_node(g, co[0]);
                        int mul_i = -1;
                        if (c0->op == GGML_OP_UNARY && ggml_get_unary_op(c0) == GGML_UNARY_OP_SILU) {
                            std::vector<int> cs; real_consumers(G, co[0], cs);
                            if (cs.size() == 1) { slot = SCR_G; mul_i = cs[0]; }
                        } else if (c0->op == GGML_OP_MUL) {
                            const ggml_tensor * other = c0->src[0] == ggml_graph_node(g, st.out[j]) ? c0->src[1] : c0->src[0];
                            if (other && other->op == GGML_OP_UNARY && ggml_get_unary_op(other) == GGML_UNARY_OP_SILU) { slot = SCR_U; mul_i = co[0]; }
                        }
                        // gate / up may only stay private if silu(gate) * up feeds a down projection the silu-prologue GEMV takes
                        // (an ffn_down of Q5_1 / Q8_0, as for n_ff % 256 != 0, runs 1:1 and reads gate / up from the graph)
                        if (slot >= 0) {
                            std::vector<int> cm; real_consumers(G, mul_i, cm);
                            if (cm.size() != 1 || !gemv_fusable(ggml_graph_node(g, cm[0]))) slot = -1;
                        }
                    }
                    st.out_scratch[j] = slot;
                    if (slot < 0) need_graph_buffers = true;
                }
                if (need_graph_buffers) {   // not the llama / qwen2 motif: one launch per matrix at its own position, activation materialised
                    if (st.prologue == 1 || st.prologue == 2) { st.prologue = 0; st.p0 = st.p1 = -1; }
                    st.nmat = 1; st.mm[0] = i; st.out[0] = i; st.add_vec[0] = -1; st.out_scratch[0] = -1;
                    int vs = 0;
                    const int ad = find_add(G, i, vs);
                    if (ad >= 0 && !taken[ad]) { st.out[0] = ad; st.add_vec[0] = ad; st.add_src[0] = vs; }
                    last = st.out[0];
                }
            }
            if (st.prologue == 3) at[xi].quant_out = 1;
            for (int j = 0; j < st.nmat; j++) { taken[st.mm[j]] = 1; taken[st.out[j]] = 1; }
            if (st.p0 >= 0) { taken[st.p0] = 1; taken[st.p1] = 1; }
            st.node = last;
            at[last] = st; has[last] = 1;
        }
        // 3) every fused attention must take q / k / v from private buffers filled by a fused group, and its f32 result is private when
        //    wo consumes the quantized copy; a SILU prologue needs its producer likewise.  Anything else: no fusion for this graph.
        for (int anchor : attn_anchor) {
            b200_step & A = at[anchor];
            const ggml_tensor * qs = strip_views(ggml_graph_node(g, A.rope_q)->src[0]), * ks = strip_views(ggml_graph_node(g, A.rope_k)->src[0]);
            const ggml_tensor * vs = strip_views(ggml_graph_node(g, A.cpy_v)->src[0]);
            for (int q = std::max(0, anchor - 96); q < anchor; q++) {
                if (!has[q] || at[q].kind != 1) continue;
                for (int j = 0; j < at[q].nmat; j++) {
                    const ggml_tensor * o = ggml_graph_node(g, at[q].out[j]);
                    if (o == qs && at[q].out_scratch[j] == SCR_Q) A.q_scratch = SCR_Q;
                    if (o == ks && at[q].out_scratch[j] == SCR_K) A.k_scratch = SCR_K;
                    if (o == vs && at[q].out_scratch[j] == SCR_V) A.v_scratch = SCR_V;
                }
            }
            if (A.q_scratch < 0 || A.k_scratch < 0 || A.v_scratch < 0) fused_ok = false;
            std::vector<int> co; real_consumers(G, A.cont, co);
            A.out_private = (A.quant_out && co.size() == 1) ? 1 : 0;
        }
        // and every gate / up kept private must be read by a silu-prologue step: nothing else sees the private buffers
        for (int q = 0; q < G.n; q++) {
            if (!has[q] || at[q].kind != 1) continue;
            for (int j = 0; j < at[q].nmat; j++) {
                const int slot = at[q].out_scratch[j];
                if (slot != SCR_G && slot != SCR_U) continue;
                const ggml_tensor * o = ggml_graph_node(g, at[q].out[j]);
                bool read = false;
                for (int r = 0; r < G.n && !read; r++) {
                    if (!has[r] || at[r].kind != 1 || at[r].prologue != 2) continue;
                    const ggml_tensor * un = ggml_graph_node(g, at[r].p0), * mul = ggml_graph_node(g, at[r].p1);
                    const ggml_tensor * up = mul->src[0] == un ? mul->src[1] : mul->src[0];
                    read = slot == SCR_G ? (un->src[0] == o && at[r].in_scratch[0] == SCR_G) : (up == o && at[r].in_scratch[1] == SCR_U);
                }
                if (!read) fused_ok = false;
            }
        }
    }
    b200_plan * plan = new b200_plan();
    plan->key = key; plan->n_nodes = G.n;
    if (fused_ok) {
        for (int anchor : attn_anchor) {
            plan->has_attn = true;
            for (int i : {at[anchor].cpy_k, at[anchor].cpy_v}) {
                plan->store_nodes.push_back(i);
                const int v = G.idx(ggml_graph_node(g, i)->src[1]);
                if (v >= 0) plan->store_nodes.push_back(v);
            }
        }
    }
    for (int i = 0; i < G.n; i++) {
        if (fused_ok && has[i]) { plan->steps.push_back(at[i]); continue; }
        if (fused_ok && taken[i]) continue;
        const ggml_tensor * t = ggml_graph_node(g, i);
        if (ggml_is_empty(t) || is_noop(t->op)) continue;
        b200_step st{};
        st.kind = 0; st.node = i;
        plan->steps.push_back(st);
    }
    return plan;
}

static float * grow_scratch(b200_backend_ctx * ctx, int slot, size_t floats) {
    if (floats > ctx->scratch_floats[slot] && ctx->capturing) { ctx->capture_failed = true; return ctx->scratch[slot]; }
    if (floats > ctx->scratch_floats[slot]) {
        if (ctx->scratch[slot]) { CUDA_OK(cudaStreamSynchronize(ctx->stream)); cudaFree(ctx->scratch[slot]); }
        CUDA_OK(cudaMalloc((void **) &ctx->scratch[slot], floats * 4 + 256));
        ctx->scratch_floats[slot] = floats;
        ctx->ws_gen++;
    }
    return ctx->scratch[slot];
}
static void * grow_ws(b200_backend_ctx * ctx, int role, size_t need) {
    if (need > ctx->fact_bytes[role] && ctx->capturing) { ctx->capture_failed = true; return ctx->fact_ws[role]; }   // no allocation inside a capture
    if (need > ctx->fact_bytes[role]) {
        if (ctx->fact_ws[role]) { CUDA_OK(cudaStreamSynchronize(ctx->stream)); cudaFree(ctx->fact_ws[role]); }
        CUDA_OK(cudaMalloc(&ctx->fact_ws[role], need + 256));
        ctx->fact_bytes[role] = need;
        ctx->ws_gen++;
    }
    return ctx->fact_ws[role];
}
static bool overlaps(const void * a, size_t na, const void * b, size_t nb) {
    const char * pa = (const char *) a, * pb = (const char *) b;
    return pa < pb + nb && pb < pa + na;
}

static bool run_gemv_step(b200_backend_ctx * ctx, ggml_cgraph * g, const b200_step & st) {
    const ggml_tensor * m0 = ggml_graph_node(g, st.mm[0]);
    const int64_t K = m0->src[0]->ne[0];
    pb200_gemv_mat mats[3];
    for (int j = 0; j < st.nmat; j++) {
        const ggml_tensor * mm = ggml_graph_node(g, st.mm[j]);
        const ggml_tensor * out = ggml_graph_node(g, st.out[j]);
        mats[j].type = (int32_t) mm->src[0]->type; mats[j]._pad = 0;
        mats[j].W = mm->src[0]->data; mats[j].n = mm->src[0]->ne[1];
        mats[j].y = st.out_scratch[j] >= 0 ? grow_scratch(ctx, st.out_scratch[j], (size_t) mm->src[0]->ne[1]) : (float *) out->data;
        mats[j].add = st.add_vec[j] >= 0 ? (const float *) out->src[st.add_src[j]]->data : nullptr;
    }
    void * ws = grow_ws(ctx, st.ws, pb200_act_workspace_bytes(K));
    if (!ctx->sync_ws && ctx->capturing) { ctx->capture_failed = true; return true; }
    if (!ctx->sync_ws) { CUDA_OK(cudaMalloc(&ctx->sync_ws, 256)); CUDA_OK(cudaMemsetAsync(ctx->sync_ws, 0, 256, ctx->stream)); ctx->ws_gen++; }
    int rc;
    if (st.prologue == 1) {
        const ggml_tensor * nrm = ggml_graph_node(g, st.p0), * mul = ggml_graph_node(g, st.p1);
        float eps; memcpy(&eps, nrm->op_params, 4);
        const ggml_tensor * w = mul->src[0] == nrm ? mul->src[1] : mul->src[0];
        rc = pb200_gemv_fused(st.nmat, mats, K, ws, 1, (const float *) nrm->src[0]->data, (const float *) w->data, eps, ctx->sync_ws, 1, ctx->stream);
    } else if (st.prologue == 2) {
        const ggml_tensor * un = ggml_graph_node(g, st.p0), * mul = ggml_graph_node(g, st.p1);
        const ggml_tensor * u = mul->src[0] == un ? mul->src[1] : mul->src[0];
        (void) un; (void) mul; (void) u;
        rc = pb200_gemv_fused(st.nmat, mats, K, ws, 2, ctx->scratch[st.in_scratch[0]], ctx->scratch[st.in_scratch[1]], 0.f, ctx->sync_ws, 1, ctx->stream);
    } else {
        if (st.prologue == 0) {
            PB_OK(pb200_quantize_act((int) m0->src[0]->type, (const float *) m0->src[1]->data, K, ws, ctx->stream));
        }
        rc = pb200_gemv_fused(st.nmat, mats, K, ws, 0, nullptr, nullptr, 0.f, ctx->sync_ws, 1, ctx->stream);
    }
    if (rc == PB200_ENOTSUP) return false;
    PB_OK(rc);
    return true;
}

static bool run_attn_step(b200_backend_ctx * ctx, ggml_cgraph * g, const b200_step & st) {
    const ggml_tensor * ropeq = ggml_graph_node(g, st.rope_q), * ropek = ggml_graph_node(g, st.rope_k);
    const ggml_tensor * cpyk = ggml_graph_node(g, st.cpy_k), * cpyv = ggml_graph_node(g, st.cpy_v);
    const ggml_tensor * kq = ggml_graph_node(g, st.kq), * sm = ggml_graph_node(g, st.soft), * kqv = ggml_graph_node(g, st.kqv);
    ggml_tensor * cont = ggml_graph_node(g, st.cont);
    const ggml_tensor * kview = kq->src[0], * vview = kqv->src[0], * mask = sm->src[1];
    const int64_t D = 128, H = kq->src[1]->ne[2], HK = kview->ne[2], n_kv = kview->ne[1];
    const int64_t vt_stride = (int64_t) (vview->nb[1] / 2);
    const int64_t k_off = (const char *) cpyk->data - (const char *) kview->data;   // the CPY nodes are views of their destinations
    const int64_t v_off = (const char *) cpyv->data - (const char *) vview->data;
    if (k_off < 0 || k_off % (HK * D * 2) != 0 || v_off != (k_off / (HK * D * 2)) * 2) return false;
    const int kv_head = (int) (k_off / (HK * D * 2));
    if (kv_head >= n_kv) return false;
    const int32_t * p = (const int32_t *) ropeq->op_params;
    float fb, fs, ef, af, bf, bsl, scale;
    memcpy(&fb, p + 5, 4); memcpy(&fs, p + 6, 4); memcpy(&ef, p + 7, 4); memcpy(&af, p + 8, 4); memcpy(&bf, p + 9, 4); memcpy(&bsl, p + 10, 4);
    memcpy(&scale, sm->op_params, 4);
    const float * q = ctx->scratch[st.q_scratch], * k = ctx->scratch[st.k_scratch], * v = ctx->scratch[st.v_scratch];   // filled by the fused q|k|v group
    float * out = st.out_private ? grow_scratch(ctx, SCR_ATT, (size_t) (H * D)) : (float *) cont->data;
    const size_t out_bytes = (size_t) (H * D) * 4;
    // the graph allocator may have placed the CONT result on top of q / k / v (their last readers are folded into this launch):
    // heads finish at different times, so only the exact q <-> out aliasing (head h reads and writes its own slice) is safe
    // q / k / v are private; the only graph tensor read while heads finish at different times is the mask row
    bool via_tmp = !st.out_private && overlaps(out, out_bytes, mask->data, (size_t) n_kv * 4);
    if (via_tmp) {
        if (ctx->attn_tmp_floats < (size_t) (H * D) && ctx->capturing) { ctx->capture_failed = true; return false; }
        if (ctx->attn_tmp_floats < (size_t) (H * D)) {
            if (ctx->attn_tmp) { CUDA_OK(cudaStreamSynchronize(ctx->stream)); cudaFree(ctx->attn_tmp); }
            CUDA_OK(cudaMalloc((void **) &ctx->attn_tmp, out_bytes + 256));
            ctx->attn_tmp_floats = (size_t) (H * D);
            ctx->ws_gen++;
        }
        out = ctx->attn_tmp;
    }
    void * ws = st.quant_out ? grow_ws(ctx, 1, pb200_act_workspace_bytes(H * D)) : nullptr;
    const int rc = pb200_attn_ggml(q, k, v, (void *) kview->data, (void *) vview->data, vt_stride, out, ws, (int) H, (int) HK, (int) D,
                                   (const int32_t *) ropeq->src[1]->data, (int) n_kv, kv_head, ctx->capturing ? ctx->kvh_dev : nullptr, (const float *) mask->data, p[1], p[2],
                                   fb, fs, ef, af, bf, bsl, p[4],
                                   ropeq->src[2] ? (const float *) ropeq->src[2]->data : nullptr, scale, 1, ctx->stream);
    if (rc == PB200_ENOTSUP) return false;
    PB_OK(rc);
    if (via_tmp) CUDA_OK(cudaMemcpyAsync(cont->data, out, out_bytes, cudaMemcpyDeviceToDevice, ctx->stream));
    return true;
}

static void run_nodes_unfused(b200_backend_ctx * ctx, ggml_cgraph * g, const int * idx, int n) {
    for (int k = 0; k < n; k++) {
        if (idx[k] < 0) continue;
        ggml_tensor * node = ggml_graph_node(g, idx[k]);
        if (ggml_is_empty(node) || is_noop(node->op)) continue;
        if (!b200_compute_node(ctx, node)) {
            fprintf(stderr, "ggml-b200: op %s not supported inside graph_compute (supports_op must be consulted)\n", ggml_op_name(node->op));
            GGML_ABORT("unsupported op");   // ggml-cuda.cu:2671-2675
        }
        g_nodes++;
    }
}

static void run_plan(b200_backend_ctx * ctx, ggml_cgraph * cgraph, b200_plan * plan) {
    for (const b200_step & st : plan->steps) {
        if (st.kind == 0) {
            run_nodes_unfused(ctx, cgraph, &st.node, 1);
        } else if (st.kind == 1) {
            if (run_gemv_step(ctx, cgraph, st)) { g_nodes += st.nmat; g_fused_steps++; continue; }
            // shape outside the fused kernel: the nodes of the group, in graph order
            std::vector<int> nodes;
            if (st.p0 >= 0) { nodes.push_back(st.p0); nodes.push_back(st.p1); }
            for (int j = 0; j < st.nmat; j++) { nodes.push_back(st.mm[j]); if (st.out[j] != st.mm[j]) nodes.push_back(st.out[j]); }
            std::sort(nodes.begin(), nodes.end());
            run_nodes_unfused(ctx, cgraph, nodes.data(), (int) nodes.size());
        } else {
            if (run_attn_step(ctx, cgraph, st)) { g_nodes += 8; g_fused_steps++; continue; }
            int nodes[8] = {st.rope_q, st.rope_k, st.cpy_k, st.cpy_v, st.kq, st.soft, st.kqv, st.cont};
            std::sort(nodes, nodes + 8);
            run_nodes_unfused(ctx, cgraph, nodes, 8);
        }
    }
}

// destination cell of this call (-1: the plan has no fused attention, -2: the layers disagree)
static int plan_kv_head(ggml_cgraph * g, const b200_plan * plan) {
    int kvh = -1;
    for (const b200_step & st : plan->steps) {
        if (st.kind != 2) continue;
        const ggml_tensor * cpyk = ggml_graph_node(g, st.cpy_k), * kq = ggml_graph_node(g, st.kq);
        const ggml_tensor * kview = kq->src[0];
        const int64_t row = kview->ne[2] * 128 * 2;
        const int64_t off = (const char *) cpyk->data - (const char *) kview->data;
        const int v = (off >= 0 && off % row == 0) ? (int) (off / row) : -2;
        if (kvh == -1) kvh = v; else if (kvh != v) return -2;
        if (v < 0 || v >= kview->ne[1]) return -2;
    }
    return kvh;
}

static enum ggml_status b200_backend_graph_compute(ggml_backend_t backend, ggml_cgraph * cgraph) {
    b200_backend_ctx * ctx = (b200_backend_ctx *) backend->context;
    cudaSetDevice(ctx->device);
    const uint64_t key = graph_key(cgraph);
    b200_plan * plan = nullptr;
    for (b200_plan * p : ctx->plans) if (p->key == key && p->n_nodes == ggml_graph_n_nodes(cgraph)) { plan = p; break; }
    if (!plan) {
        plan = build_plan(cgraph, key);
        if (ctx->plans.size() >= 16) { CUDA_OK(cudaStreamSynchronize(ctx->stream)); delete ctx->plans.front(); ctx->plans.erase(ctx->plans.begin()); }
        ctx->plans.push_back(plan);
    }
    static const bool use_graphs = getenv("GGML_B200_NO_GRAPHS") == nullptr;
    // which addresses this call binds: every node's data except the cache-store nodes (their address IS the destination cell)
    const bool has_attn = plan->has_attn;
    ctx->skip.assign((size_t) plan->n_nodes, 0);
    for (int i : plan->store_nodes) ctx->skip[(size_t) i] = 1;
    uint64_t addr_bind = 0xcbf29ce484222325ull;
    for (int i = 0; i < plan->n_nodes; i++) {
        if (ctx->skip[(size_t) i]) continue;
        const ggml_tensor * t = ggml_graph_node(cgraph, i);
        uint64_t w = (uint64_t) (uintptr_t) t->data;
        for (int k = 0; k < 3; k++) if (t->src[k]) w = w * 1315423911ull + (uint64_t) (uintptr_t) t->src[k]->data;   // leafs (weights, inputs) included
        addr_bind = fnv(addr_bind, w);
    }
    const uint64_t bind = fnv(addr_bind, ctx->ws_gen);   // an exec captured before a workspace moved must not be replayed
    const int kvh = has_attn ? plan_kv_head(cgraph, plan) : -1;
    const bool graphable = use_graphs && kvh != -2 && plan->steps.size() >= 8;
    if (graphable && !ctx->kvh_dev) {
        CUDA_OK(cudaMalloc((void **) &ctx->kvh_dev, 256));
        CUDA_OK(cudaMallocHost((void **) &ctx->kvh_host, 64 * sizeof(int32_t)));
        ctx->ws_gen++;
    }
    auto push_cell = [&]() {
        if (kvh >= 0) {   // a ring of pinned words: the host may run several calls ahead of the copies
            int32_t * w = ctx->kvh_host + (ctx->kvh_idx++ & 63);
            *w = kvh;
            CUDA_OK(cudaMemcpyAsync(ctx->kvh_dev, w, 4, cudaMemcpyHostToDevice, ctx->stream));
        }
    };
    if (graphable && plan->exec && plan->bind == bind) {
        // replay: same topology, same addresses; only the destination cell (and the input tensors' contents) changed
        push_cell();
        CUDA_OK(cudaGraphLaunch(plan->exec, ctx->stream));
        g_nodes += plan->nodes; g_fused_steps += plan->fused; g_graph_replays++;
        pb200_kernel_launches_add(plan->launches);
        return GGML_STATUS_SUCCESS;
    }
    if (plan->exec) { CUDA_OK(cudaStreamSynchronize(ctx->stream)); cudaGraphExecDestroy(plan->exec); plan->exec = nullptr; }
    if (graphable && plan->bind == bind && plan->seen >= 1) {
        // second call with these addresses: every workspace has its final size, capture the whole step sequence once
        const unsigned long long n0 = g_nodes.load(), f0 = g_fused_steps.load();
        const uint64_t l0 = pb200_kernel_launches();
        ctx->capturing = true; ctx->capture_failed = false;
        cudaGraph_t graph = nullptr;
        push_cell();
        if (cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
            run_plan(ctx, cgraph, plan);
            cudaError_t e = cudaStreamEndCapture(ctx->stream, &graph);
            ctx->capturing = false;
            if (e == cudaSuccess && graph && !ctx->capture_failed && cudaGraphInstantiate(&plan->exec, graph, 0) == cudaSuccess) {
                plan->nodes = g_nodes.load() - n0; plan->fused = g_fused_steps.load() - f0; plan->launches = pb200_kernel_launches() - l0;
                cudaGraphDestroy(graph);
                CUDA_OK(cudaGraphLaunch(plan->exec, ctx->stream));
                return GGML_STATUS_SUCCESS;
            }
            if (graph) cudaGraphDestroy(graph);
            plan->exec = nullptr;
            cudaGetLastError();
        }
        ctx->capturing = false;
        plan->seen = -1000000;          // this plan cannot be captured: direct launches from now on
    }
    run_plan(ctx, cgraph, plan);
    // keyed with the generation this call leaves behind: a call that grew a workspace does not delay its own plan's capture
    const uint64_t bind_end = fnv(addr_bind, ctx->ws_gen);
    if (plan->bind == bind_end) plan->seen++; else { plan->bind = bind_end; plan->seen = 1; }
    return GGML_STATUS_SUCCESS;   // asynchronous: work is enqueued on the backend stream
}

// ---- the entries the scheduler uses to move tensors between backends and to order their streams (ggml-cuda.cu:2392-2445, 2780-2823) ----
static bool b200_backend_cpy_tensor_async(ggml_backend_t backend_src, ggml_backend_t backend_dst, const ggml_tensor * src, ggml_tensor * dst) {
    if (!ggml_backend_is_b200(backend_src) || !ggml_backend_is_b200(backend_dst)) return false;
    ggml_backend_buffer_t bs = src->view_src ? src->view_src->buffer : src->buffer, bd = dst->view_src ? dst->view_src->buffer : dst->buffer;
    if (!bs || !bd || bs->iface.get_name != b200_buffer_get_name || bd->iface.get_name != b200_buffer_get_name) return false;
    if (!ggml_is_contiguous(src) || !ggml_is_contiguous(dst) || ggml_nbytes(src) != ggml_nbytes(dst)) return false;
    b200_backend_ctx * cs = (b200_backend_ctx *) backend_src->context, * cd = (b200_backend_ctx *) backend_dst->context;
    const int dev_s = ((b200_buffer_ctx *) bs->context)->device, dev_d = ((b200_buffer_ctx *) bd->context)->device;
    if (cs->device != dev_s || cd->device != dev_d) return false;
    cudaSetDevice(cs->device);
    if (backend_src == backend_dst) {
        CUDA_OK(cudaMemcpyAsync(dst->data, src->data, ggml_nbytes(dst), cudaMemcpyDeviceToDevice, cs->stream));
        return true;
    }
    // copy on the source stream (peer copy over NVLink between devices), then make the destination stream wait for it
    if (dev_s == dev_d) CUDA_OK(cudaMemcpyAsync(dst->data, src->data, ggml_nbytes(dst), cudaMemcpyDeviceToDevice, cs->stream));
    else CUDA_OK(cudaMemcpyPeerAsync(dst->data, dev_d, src->data, dev_s, ggml_nbytes(dst), cs->stream));
    if (!cs->copy_event) CUDA_OK(cudaEventCreateWithFlags(&cs->copy_event, cudaEventDisableTiming));
    CUDA_OK(cudaEventRecord(cs->copy_event, cs->stream));
    cudaSetDevice(cd->device);
    CUDA_OK(cudaStreamWaitEvent(cd->stream, cs->copy_event, 0));
    return true;
}
static void b200_backend_event_record(ggml_backend_t backend, ggml_backend_event_t event) {
    b200_backend_ctx * ctx = (b200_backend_ctx *) backend->context;
    cudaSetDevice(ctx->device);
    CUDA_OK(cudaEventRecord((cudaEvent_t) event->context, ctx->stream));
}
static void b200_backend_event_wait(ggml_backend_t backend, ggml_backend_event_t event) {
    if (ggml_backend_is_b200(backend)) {
        b200_backend_ctx * ctx = (b200_backend_ctx *) backend->context;
        cudaSetDevice(ctx->device);
        CUDA_OK(cudaStreamWaitEvent(ctx->stream, (cudaEvent_t) event->context, 0));
    } else {
        CUDA_OK(cudaEventSynchronize((cudaEvent_t) event->context));   // a foreign backend: block the host instead
    }
}

static const ggml_backend_i b200_backend_iface = {
    /* .get_name                = */ b200_backend_get_name,
    /* .free                    = */ b200_backend_free,
    /* .get_default_buffer_type = */ b200_backend_get_default_buft,
    /* .set_tensor_async        = */ b200_backend_set_tensor_async,
    /* .get_tensor_async        = */ b200_backend_get_tensor_async,
    /* .cpy_tensor_async        = */ b200_backend_cpy_tensor_async,
    /* .synchronize             = */ b200_backend_synchronize,
    /* .graph_plan_create       = */ nullptr,
    /* .graph_plan_free         = */ nullptr,
    /* .graph_plan_update       = */ nullptr,
    /* .graph_plan_compute      = */ nullptr,
    /* .graph_compute           = */ b200_backend_graph_compute,
    /* .supports_op             = */ nullptr,
    /* .supports_buft           = */ nullptr,
    /* .offload_op              = */ nullptr,
    /* .event_record            = */ b200_backend_event_record,
    /* .event_wait              = */ b200_backend_event_wait,
};

// ---------------------------------------------------------------------------------------------------- device + reg
static const char * b200_dev_get_name(ggml_backend_dev_t dev) { return ((b200_device_ctx *) dev->context)->name.c_str(); }
static const char * b200_dev_get_description(ggml_backend_dev_t dev) { return ((b200_device_ctx *) dev->context)->description.c_str(); }
static void b200_dev_get_memory(ggml_backend_dev_t dev, size_t * free, size_t * total) {
    cudaSetDevice(((b200_device_ctx *) dev->context)->device);
    CUDA_OK(cudaMemGetInfo(free, total));
}
static enum ggml_backend_dev_type b200_dev_get_type(ggml_backend_dev_t) { return GGML_BACKEND_DEVICE_TYPE_GPU_FULL; }
static void b200_dev_get_props(ggml_backend_dev_t dev, ggml_backend_dev_props * props) {
    props->name = b200_dev_get_name(dev);
    props->description = b200_dev_get_description(dev);
    props->type = b200_dev_get_type(dev);
    b200_dev_get_memory(dev, &props->memory_free, &props->memory_total);
    props->caps = { /* async */ true, /* host_buffer */ true, /* buffer_from_host_ptr */ false, /* events */ true };
}
static ggml_backend_t b200_dev_init_backend(ggml_backend_dev_t dev, const char *) { return ggml_backend_b200_init(((b200_device_ctx *) dev->context)->device); }
static ggml_backend_buffer_type_t b200_dev_get_buft(ggml_backend_dev_t dev) { return ggml_backend_b200_buffer_type(((b200_device_ctx *) dev->context)->device); }
static bool b200_dev_supports_buft(ggml_backend_dev_t dev, ggml_backend_buffer_type_t buft) {
    return buft->iface.get_name == b200_buft_get_name && buft->device == dev;
}
static bool b200_dev_offload_op(ggml_backend_dev_t, const ggml_tensor *) { return false; }   // never pull CPU-resident weights over PCIe (App. B)

// ---- events (ggml-cuda.cu:3210-3256) and the pinned host buffer type (ggml-cuda.cu:1008-1080): what ggml_backend_sched uses to
// overlap the copies of a split's inputs with the previous split's compute ----
static ggml_backend_event_t b200_dev_event_new(ggml_backend_dev_t dev) {
    cudaSetDevice(((b200_device_ctx *) dev->context)->device);
    cudaEvent_t ev = nullptr;
    if (cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return new ggml_backend_event{dev, ev};
}
static void b200_dev_event_free(ggml_backend_dev_t dev, ggml_backend_event_t event) {
    cudaSetDevice(((b200_device_ctx *) dev->context)->device);
    cudaEventDestroy((cudaEvent_t) event->context);
    delete event;
}
static void b200_dev_event_synchronize(ggml_backend_dev_t dev, ggml_backend_event_t event) {
    cudaSetDevice(((b200_device_ctx *) dev->context)->device);
    CUDA_OK(cudaEventSynchronize((cudaEvent_t) event->context));
}
static const char * b200_host_buft_name(ggml_backend_buffer_type_t) { return "B200_Host"; }
static const char * b200_host_buffer_name(ggml_backend_buffer_t) { return "B200_Host"; }
static void b200_host_buffer_free(ggml_backend_buffer_t buffer) { cudaFreeHost(buffer->context); }
static ggml_backend_buffer_t b200_host_buft_alloc(ggml_backend_buffer_type_t buft, size_t size) {
    void * ptr = nullptr;
    if (cudaMallocHost(&ptr, size > 0 ? size : 1) != cudaSuccess) {   // no pinned memory left: plain host memory still works, only slower
        cudaGetLastError();
        return ggml_backend_buft_alloc_buffer(ggml_backend_cpu_buffer_type(), size);
    }
    // a CPU buffer over pinned pages: the CPU backend computes in it, H2D / D2H copies from it are asynchronous DMA
    ggml_backend_buffer_t buffer = ggml_backend_cpu_buffer_from_ptr(ptr, size);
    buffer->buft = buft;
    buffer->iface.get_name = b200_host_buffer_name;
    buffer->iface.free_buffer = b200_host_buffer_free;
    return buffer;
}
static ggml_backend_buffer_type_t b200_dev_get_host_buft(ggml_backend_dev_t dev) {
    static ggml_backend_buffer_type host_buft;
    static std::once_flag once;
    std::call_once(once, [dev] {
        ggml_backend_buffer_type_t cpu = ggml_backend_cpu_buffer_type();
        host_buft.iface = cpu->iface;            // alignment / alloc size / is_host as for any CPU buffer
        host_buft.iface.get_name = b200_host_buft_name;
        host_buft.iface.alloc_buffer = b200_host_buft_alloc;
        host_buft.device = dev->reg->iface.get_device(dev->reg, 0);
        host_buft.context = nullptr;
    });
    return &host_buft;
}

static const ggml_backend_device_i b200_device_iface = {
    /* .get_name             = */ b200_dev_get_name,
    /* .get_description      = */ b200_dev_get_description,
    /* .get_memory           = */ b200_dev_get_memory,
    /* .get_type             = */ b200_dev_get_type,
    /* .get_props            = */ b200_dev_get_props,
    /* .init_backend         = */ b200_dev_init_backend,
    /* .get_buffer_type      = */ b200_dev_get_buft,
    /* .get_host_buffer_type = */ b200_dev_get_host_buft,
    /* .buffer_from_host_ptr = */ nullptr,
    /* .supports_op          = */ b200_supports_op,
    /* .supports_buft        = */ b200_dev_supports_buft,
    /* .offload_op           = */ b200_dev_offload_op,
    /* .event_new            = */ b200_dev_event_new,
    /* .event_free           = */ b200_dev_event_free,
    /* .event_synchronize    = */ b200_dev_event_synchronize,
};

struct b200_reg_ctx {
    std::vector<ggml_backend_device> devices;
    std::vector<ggml_backend_buffer_type> bufts;
};
static const char * b200_reg_get_name(ggml_backend_reg_t) { return "B200"; }
static size_t b200_reg_device_count(ggml_backend_reg_t reg) { return ((b200_reg_ctx *) reg->context)->devices.size(); }
static ggml_backend_dev_t b200_reg_get_device(ggml_backend_reg_t reg, size_t i) {
    b200_reg_ctx * ctx = (b200_reg_ctx *) reg->context;
    GGML_ASSERT(i < ctx->devices.size());
    return &ctx->devices[i];
}
// names llama.cpp looks up (src/llama.cpp:3772, 21261; ggml-cuda.cu:3280-3292).  Row-split buffers are not provided (prima disables
// tensor split, src/llama.cpp:21106-21107); host-memory registration maps to cudaHostRegister like the reference's.
static bool b200_register_host_buffer(void * buffer, size_t size) {
    if (cudaHostRegister(buffer, size, cudaHostRegisterPortable | cudaHostRegisterReadOnly) != cudaSuccess) { cudaGetLastError(); return false; }
    return true;
}
static void b200_unregister_host_buffer(void * buffer) { if (cudaHostUnregister(buffer) != cudaSuccess) cudaGetLastError(); }
static void * b200_reg_get_proc_address(ggml_backend_reg_t, const char * name) {
    if (strcmp(name, "ggml_backend_register_host_buffer") == 0) return (void *) b200_register_host_buffer;
    if (strcmp(name, "ggml_backend_unregister_host_buffer") == 0) return (void *) b200_unregister_host_buffer;
    return nullptr;   // "ggml_backend_split_buffer_type", "ggml_backend_set_n_threads": not applicable
}
static const ggml_backend_reg_i b200_reg_iface = {
    /* .get_name         = */ b200_reg_get_name,
    /* .get_device_count = */ b200_reg_device_count,
    /* .get_device       = */ b200_reg_get_device,
    /* .get_proc_address = */ b200_reg_get_proc_address,
};

extern "C" {

ggml_backend_reg_t ggml_backend_b200_reg(void) {
    static ggml_backend_reg reg;
    static std::once_flag once;
    std::call_once(once, [] {
        b200_reg_ctx * ctx = new b200_reg_ctx();
        int n = pb200_device_count();
        if (n > B200_MAX_DEVICES) n = B200_MAX_DEVICES;
        ctx->devices.resize(n);
        ctx->bufts.resize(n);
        reg.iface = b200_reg_iface;
        reg.context = ctx;
        for (int i = 0; i < n; i++) {
            cudaDeviceProp prop;
            std::string desc = "CUDA device";
            if (cudaGetDeviceProperties(&prop, i) == cudaSuccess) desc = prop.name;
            ctx->devices[i].iface = b200_device_iface;
            ctx->devices[i].reg = &reg;
            ctx->devices[i].context = new b200_device_ctx{i, "B200_" + std::to_string(i), desc};
            ctx->bufts[i].iface = b200_buft_iface;
            ctx->bufts[i].device = &ctx->devices[i];
            ctx->bufts[i].context = nullptr;
        }
    });
    return &reg;
}

ggml_backend_buffer_type_t ggml_backend_b200_buffer_type(int device) {
    b200_reg_ctx * ctx = (b200_reg_ctx *) ggml_backend_b200_reg()->context;
    if (device < 0 || device >= (int) ctx->bufts.size()) return nullptr;
    return &ctx->bufts[device];
}

ggml_backend_t ggml_backend_b200_init(int device) {
    b200_reg_ctx * rctx = (b200_reg_ctx *) ggml_backend_b200_reg()->context;
    if (device < 0 || device >= (int) rctx->devices.size()) return nullptr;
    if (cudaSetDevice(device) != cudaSuccess) return nullptr;
    b200_backend_ctx * ctx = new b200_backend_ctx();
    ctx->device = device;
    ctx->name = "B200_" + std::to_string(device);
    if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) { delete ctx; return nullptr; }
    return new ggml_backend{b200_guid(), b200_backend_iface, &rctx->devices[device], ctx};
}

int ggml_backend_is_b200(ggml_backend_t backend) { return backend != nullptr && ggml_guid_matches(backend->guid, b200_guid()); }
unsigned long long ggml_backend_b200_nodes_computed(void) { return g_nodes.load(); }
unsigned long long ggml_backend_b200_fused_steps(void) { return g_fused_steps.load(); }
unsigned long long ggml_backend_b200_graph_replays(void) { return g_graph_replays.load(); }

}  // extern "C"

// loading the plugin registers it with the host's registry (ggml_backend_register, ggml-backend-impl.h:220)
__attribute__((constructor)) static void ggml_b200_autoregister() {
    if (getenv("GGML_B200_NO_AUTOREG")) return;
    // only when the host process really carries a ggml registry (LD_PRELOAD also reaches unrelated helper processes)
    typedef void (*register_fn)(ggml_backend_reg_t);
    register_fn reg_fn = (register_fn) dlsym(RTLD_DEFAULT, "ggml_backend_register");
    if (!reg_fn) return;
    ggml_backend_reg_t reg = ggml_backend_b200_reg();
    if (b200_reg_device_count(reg) > 0) reg_fn(reg);
}
