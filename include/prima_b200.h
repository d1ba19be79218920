/*
 * include/prima_b200.h — C ABI of libprima_b200.so, the H100-native (sm_90a) quantized-decode hot path of prima.cpp.
 *
 * Plain pointers and sizes only; no torch / ggml types.  All functions return 0 on success, a cudaError_t (>0) for
 * CUDA failures or a negative PB200_E* code for argument errors; nothing throws or aborts across the ABI.
 * Device pointers are raw CUDA device addresses, `stream` is a cudaStream_t passed as void* (NULL = default stream).
 *
 * What each entry point replaces in the reference (paths relative to the reference source tree):
 *   pb200_mul_mat_vec*      ggml_cuda_mul_mat -> ggml_cuda_op_mul_mat_vec_q -> mul_mat_vec_q<type,1>
 *                           ggml/src/ggml-cuda.cu:1883-1948, ggml-cuda/mmvq.cu:55-202, vecdotq.cuh:357-787
 *                           (+ the per-call quantize_row_q8_1_cuda, quantize.cu:129-141); CPU semantics:
 *                           ggml_compute_forward_mul_mat ggml/src/ggml.c:12377-12600
 *   pb200_quantize_act      quantize_q8_1 quantize.cu:4-38; CPU: quantize_row_q8_K_ref ggml-quants.c:3785-3822
 *   pb200_rms_norm          ggml_cuda_op_rms_norm norm.cu:206-224; CPU ggml.c:11950-11996
 *   pb200_rope              ggml_cuda_op_rope rope.cu:188-271; CPU ggml.c:14143-14266
 *   pb200_rope_f16          the same on f16 rows (rope.cu:200-262); CPU ggml.c:14269-14380
 *   pb200_kv_seq_shift      llama_kv_cache_seq_rm + seq_add (src/llama.cpp:4378-4427) and the K-shift graph of build_k_shift
 *                           (:10665-10719) that llama_kv_cache_update_internal runs at the next decode (:19102-19134)
 *   pb200_soft_max          ggml_cuda_op_soft_max softmax.cu:170-206; CPU ggml.c:13783-13880
 *   pb200_attn_decode       FA-off attention chain: ggml_cuda_mul_mat_batched_cublas x2 + soft_max + cont,
 *                           ggml-cuda.cu:1737-1881; graph src/llama.cpp:10032-10165
 *   pb200_mul_mat_q         ggml_cuda_op_mul_mat_q mmq.cu:3-98 -> mul_mat_q<type,...> mmq.cuh:2583-2650 (+ quantize_mmq_q8_1_cuda
 *                           quantize.cu:143-169): the batched / prefill product, here on wgmma tensor cores
 *   pb200_get_rows          ggml_cuda_op_get_rows getrows.cu (k-quant rows are unsupported there, ggml-cuda.cu:3033-3047)
 *   pb200_model_* / pb200_decode*   the per-token loop ggml_backend_cuda_graph_compute ggml-cuda.cu:2508-2778 over the
 *                           graph of build_llama / build_qwen2 (src/llama.cpp:11000-11216, 12736-12916) — one fused,
 *                           CUDA-graph-replayed launch sequence instead of ~30 launches per layer
 *   (the ggml-backend plugin that exposes the same kernels through ggml_backend_reg/device/buffer vtables is
 *    include/ggml_b200.h)
 */
#ifndef PRIMA_B200_H
#define PRIMA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PB200_API __attribute__((visibility("default")))

/* enum ggml_type values used on this path (ggml/include/ggml.h:356-395) */
enum { PB200_TYPE_F32 = 0, PB200_TYPE_F16 = 1, PB200_TYPE_Q4_0 = 2, PB200_TYPE_Q4_1 = 3, PB200_TYPE_Q5_0 = 6, PB200_TYPE_Q5_1 = 7, PB200_TYPE_Q8_0 = 8,
       PB200_TYPE_Q4_K = 12, PB200_TYPE_Q5_K = 13, PB200_TYPE_Q6_K = 14 };

enum { PB200_EINVAL = -1, PB200_ENOMEM = -2, PB200_ENOTSUP = -3, PB200_ESTATE = -4, PB200_EABORTED = -5 };

/* ---- library ---- */
PB200_API const char * pb200_version(void);
PB200_API const char * pb200_error_string(int code);
PB200_API int          pb200_device_count(void);
PB200_API int          pb200_sm_count(void);              /* of the current device */
PB200_API int64_t      pb200_row_bytes(int type, int64_t k);   /* ggml_row_size */
PB200_API uint64_t     pb200_kernel_launches(void);       /* kernels launched by this library since load (bench `gpu_launches`) */
PB200_API void         pb200_kernel_launches_add(uint64_t n);   /* a host that replays a CUDA graph of this library's launches accounts for them here */

/* ---- single ops, device buffers ---- */
/* workspace for the quantized activation of length k (any mode): bytes to allocate */
PB200_API size_t pb200_act_workspace_bytes(int64_t k);
/* x[k] f32 -> activation workspace in the format the CPU backend uses for weight type wtype (q8_K / q8_0 / q8_1) */
PB200_API int pb200_quantize_act(int wtype, const float * x, int64_t k, void * act_ws, void * stream);
/* y[n] = W[n][k] . x   with W raw GGUF blocks of `type`; act_ws from pb200_quantize_act(type, x, k).
 * W must be 16-byte aligned and its allocation padded to a multiple of 16 bytes (+16): the kernel moves whole 16-byte units and
 * may read up to 15 bytes past the last row (Q6_K / Q8_0 / Q4_0 / Q4_1 / Q5_0 rows need not be multiples of 16 bytes).  ggml-backend buffers of the B200
 * plugin and pb200_model_set_tensor pad for you. */
PB200_API int pb200_mul_mat_vec_q(int type, const void * W, int64_t n, int64_t k, const void * act_ws, float * y,
                                  const float * bias, const float * resid, void * stream);
/* convenience: quantize + mul_mat_vec in one call (what ggml_cuda_mul_mat does for ne11 == 1) */
PB200_API int pb200_mul_mat_vec(int type, const void * W, int64_t n, int64_t k, const float * x, float * y, void * act_ws, void * stream);
/* up to 3 matrices sharing one activation, one fused launch (q|k|v, gate|up) */
PB200_API int pb200_mul_mat_vec_fused(int nmat, const int * types, const void * const * W, const int64_t * n, int64_t k,
                                      const void * act_ws, float * const * y, void * stream);
/* HOST buffers end to end (H2D of x, quantize, GEMV, D2H of y, synchronised): W must already be on the device */
PB200_API int pb200_mul_mat_vec_host(int type, const void * W_dev, int64_t n, int64_t k, const float * x_host, float * y_host);

/* profiling: while a buffer is set, k_gemv_kquant runs its instrumented instantiation: launch i writes row (i % slots) of
 * dev_buf (rows of 4096 u64), CTA c its 8 entries [8c .. 8c+7]: [0..5] %globaltimer (ns) at CTA start / ring fill issued /
 * dependency resolved (griddepcontrol.wait returned) / activation in registers / first tile landed / done, [6], [7] clock64 at
 * the first and last stamp.  NULL or slots = 0 switches back to the uninstrumented kernel. */
PB200_API int pb200_debug_set_trace(void * dev_buf, int slots);
/* Every in-kernel wait is bounded (~1 s of SM clocks).  A wait that gives up ends its launch quickly with invalid results and
 * the call that synchronises on it (pb200_decode, pb200_synchronize, pb200_prefill) returns PB200_EABORTED once; the flag
 * re-arms, later calls are unaffected.  Callers that only use the single-op entry points on their own streams poll this after
 * synchronising: returns 1 (and clears the flag) if any launch of this process gave up since the last call. */
PB200_API int pb200_aborted(void);

PB200_API int pb200_rms_norm(const float * x, float * y, int64_t n, int64_t nrows, float eps, void * stream);
PB200_API int pb200_rope(const float * x, float * y, int64_t n_tokens, int n_head, int head_dim, int n_dims, int mode, const int32_t * pos,
                         float freq_base, float freq_scale, float ext_factor, float attn_factor, float beta_fast, float beta_slow,
                         int n_ctx_orig, const float * freq_factors, void * stream);
/* GGML_OP_ROPE on f16 rows (ggml_compute_forward_rope_f16, ggml.c:14269-14380): x, y contiguous f16 [n_rows][n_head][head_dim], row t
 * rotated by pos[t] (device int32), f16 -> f32, rotate, round to f16; y may equal x (the in-place K-shift of a KV cache).  Modes 0 (NORM)
 * and 2 (NEOX), n_dims <= head_dim (the tail is copied), YaRN and freq factors; other parameters as in pb200_rope. */
PB200_API int pb200_rope_f16(const void * x, void * y, int64_t n_rows, int n_head, int head_dim, int n_dims, int mode, const int32_t * pos,
                             float freq_base, float freq_scale, float ext_factor, float attn_factor, float beta_fast, float beta_slow,
                             int n_ctx_orig, const float * freq_factors, void * stream);
PB200_API int pb200_soft_max(const float * x, const float * mask, float * y, int64_t ncols, int64_t nrows, int64_t mask_rows, float scale, void * stream);
PB200_API int pb200_silu_mul(const float * gate, const float * up, float * y, int64_t n, void * stream);
/* element-wise glue of the graph (binbcast.cu / unary.cu / cpy.cu): y = a (+|*) b[i % nb]  (op 0 add, 1 mul); y = silu(x);
 * 4-D strided copy f32 -> f32|f16 (byte strides; dst logical order) — CPY / CONT / DUP incl. the transposed V-cache store */
PB200_API int pb200_binary(int op, const float * a, const float * b, float * y, int64_t n, int64_t nb, void * stream);
PB200_API int pb200_silu(const float * x, float * y, int64_t n, void * stream);
PB200_API int pb200_copy_strided(const void * src_f32, void * dst, int dst_is_f16, const int64_t * ne, const int64_t * src_strides,
                                 const int64_t * dst_strides, void * stream);
/* d[i0,i1,i2,i3] = sum_k a_f16[k,i0,i2/r2,i3/r3] * f16(b[k,i1,i2,i3]) — the FA-off KQ / KQV products (ggml-cuda.cu:1737-1881), byte strides */
PB200_API int pb200_mul_mat_f16(const void * a_f16, const float * b_f32, float * d, int64_t k, const int64_t * ne, int64_t r2, int64_t r3,
                                const int64_t * a_strides, const int64_t * b_strides, const int64_t * d_strides, void * stream);
/* batched (prefill) product: dst[t][n] = sum_k W[n][k] * x[t][k] (+ bias[n]) (+ resid[t][n]); W: n rows of k-quant blocks
 * (Q4_K/Q5_K/Q6_K with k % 256 == 0, or Q8_0/Q5_1/Q4_0/Q4_1/Q5_0 with k % 64 == 0), x: t rows of ldx floats, dst / resid: t rows of n floats, resid must not alias dst; W and x 16-byte aligned, ldx % 4 == 0.  Activations are quantized like the CPU backend does for that weight type (q8_K, or q8_0/q8_1 per 32 values: q8_1 for Q5_1/Q4_1),
 * then both operands run as fp16 on the tensor cores with fp32 accumulation.  ws: pb200_mul_mat_q_workspace_bytes(k, t) = tpad * (2 k + 4)
 * bytes, tpad = t rounded up to the token tile: the fp16 activation image, then one f32 power-of-two scale per padded row that keeps
 * every activation magnitude inside fp16's normal range. */
PB200_API size_t pb200_mul_mat_q_workspace_bytes(int64_t k, int64_t t);
/* 1 when pb200_mul_mat_q takes weights of this type with k columns (the type and k rule above), else 0 */
PB200_API int pb200_mul_mat_q_supported(int type, int64_t k);
PB200_API int pb200_mul_mat_q(int type, const void * W, int64_t n, int64_t k, const float * x, int64_t ldx, int64_t t, float * dst,
                              const float * bias, const float * resid, void * ws, void * stream);
PB200_API int pb200_get_rows(int type, const void * table, int64_t k, const int32_t * ids, int64_t n_ids, float * y, void * stream);
/* decode attention over an f16 KV cache laid out [n_ctx][n_head_kv*head_dim]; n_kv = *pos_dev + 1.  The kernel keeps a score row of
 * n_ctx floats in shared memory: PB200_ENOTSUP when that exceeds the device's limit (n_ctx above 57 056 on an H100); likewise
 * pb200_attn_prefill for n_kv_max. */
PB200_API int pb200_attn_decode(const float * q, const void * k_cache_f16, const void * v_cache_f16, float * out, int n_head, int n_head_kv,
                                int head_dim, const int32_t * pos_dev, int n_ctx, float scale, void * stream);
/* prompt-processing attention: n_tok query rows q[t][n_head][head_dim]; token t attends to cache rows [0, pos_dev[t]] (its own
 * K/V row already stored); n_kv_max >= max(pos_dev) + 1.  Same FA-off arithmetic per row as pb200_attn_decode. */
PB200_API int pb200_attn_prefill(const float * q, const void * k_cache_f16, const void * v_cache_f16, float * out, int n_head, int n_head_kv,
                                 int head_dim, const int32_t * pos_dev, int n_tok, int n_kv_max, float scale, void * stream);

/* GGML_OP_FLASH_ATTN_EXT (ggml_cuda_flash_attn_ext, ggml-cuda/fattn.cu:298-345; CPU ggml.c:15538-15748) with f16 K / V:
 * dst[D][n_head][n_tokens] = softmax(scale * K q + slope * mask) . V per (token, head); online softmax split over the KV range and
 * merged (flash_attn_combine_results, fattn-common.cuh:519-561).  Byte strides: q_nb = {nb1 (token), nb2 (head)}, k_nb / v_nb =
 * {nb1 (cell), nb2 (kv head)}; mask f16 [n_kv] rows of mask_nb1 bytes or NULL; max_bias = ALiBi, logit_softcap = Gemma-2 style cap. */
PB200_API int pb200_flash_attn_ext(const float * q, const void * k_f16, const void * v_f16, const void * mask_f16, float * dst, int head_dim, int n_tokens,
                                   int n_head, int n_head_kv, int n_kv, const int64_t * q_nb, const int64_t * k_nb, const int64_t * v_nb, int64_t mask_nb1,
                                   float scale, float max_bias, float logit_softcap, void * stream);

/* ---- seeded sampling on the device: the chain gpt_sampler_init builds for temp > 0 without mirostat (common/sampling.cpp:140-224):
 *   top-k -> top-p -> min-p -> temperature -> softmax -> dist (src/llama-sampling.cpp:91-165, 557-588, 624-684, 913-918, 66-89, 18-46)
 * top_k <= 0: the whole vocabulary; top_p 1: off; min_p 0: off; min_keep as in the reference; temp <= 0: greedy (first index of
 * the maximum, the same kernel as pb200_argmax_seq).  The draw is std::mt19937(seed) through std::discrete_distribution (two 32-bit
 * outputs per draw; nothing is drawn when one token survives), so a sequence of draws follows the reference's generator.  Equal
 * logits are ordered by ascending token id.  Logit bias and the repeat / frequency / presence penalties, the two samplers the
 * reference puts in front of every chain, are pb200_penalty_apply below: a penalised copy of the row that this call then reads.
 * Tail-free, typical, dynamic temperature, mirostat and grammars are not provided.  Invalid parameters (NaN / inf, top_p outside (0, 1], min_p outside [0, 1), min_keep < 0) return
 * PB200_EINVAL.  Where every softmax weight vanishes (a temperature so small that logit / temp overflows, a row of -inf) the token
 * is the top one.  Top-p is cut where the exact running mass reaches p; the reference's float running sum over a whole vocabulary
 * (top_k <= 0) can stop a little earlier (up to about 5e-4 of mass measured, a few dozen tokens of 130 000). */
typedef struct pb200_sampling {
    int32_t top_k;
    float   top_p, min_p, temp;
    int32_t min_keep;
    uint32_t seed;             /* explicit: choosing a random seed (LLAMA_DEFAULT_SEED) is the host's business */
} pb200_sampling;
/* device memory one generator state takes (624 words + index, padded) */
PB200_API size_t pb200_sampler_state_bytes(void);
/* state_dev = std::mt19937(seed), enqueued on stream */
PB200_API int pb200_sampler_seed(void * state_dev, uint32_t seed, void * stream);
/* one token from logits[n_vocab] (device) -> *token_dev; advances state_dev.  One launch, no host synchronisation or allocation:
 * capturable in a CUDA graph.  p->seed is not used here (pb200_sampler_seed seeds).  PB200_ENOTSUP when n_vocab / 16 logits exceed
 * the device's shared memory per block (n_vocab above about 880 000 on an H100). */
PB200_API int pb200_sample(const float * logits, int n_vocab, const pb200_sampling * p, void * state_dev, int32_t * token_dev, void * stream);

/* ---- logit bias and repeat / frequency / presence penalties: llama_sampler_init_logit_bias (src/llama-sampling.cpp:1568-1645) and
 * llama_sampler_init_penalties (:1373-1566), which gpt_sampler_init puts ahead of every chain, greedy included (common/sampling.cpp:156-172).
 * pb200_penalty_apply writes a penalised COPY of the row, in the reference's order:
 *   1. logit[token] += bias for each list entry in list order (one rounded f32 add each; ids outside [0, n_vocab) are ignored);
 *   2. ignore_eos with eos_token >= 0: logit[eos] = -inf;
 *   3. stop here when last_n == 0 or repeat == 1 && freq == 0 && present == 0;
 *   4. for every id occurring count > 0 times among the last min(last_n, accepted) accepted tokens (ids outside [0, n_vocab) ignored):
 *      logit = logit <= 0 ? logit * repeat : logit / repeat, then logit -= count * freq + present, each operation rounded separately;
 *      with !penalize_nl the newline keeps the logit it had after step 2.
 * last_n < 0 behaves as 0 (llama_sampler_init_penalties clamps it; it is not "context size").  eos_token / nl_token -1: the vocabulary
 * has none (ignore_eos off / penalize_nl on).  Then pb200_sample (or, greedy, its temp <= 0 form) on the copy, then
 * pb200_penalty_accept of the token: that is gpt_sampler_sample + gpt_sampler_accept. */
typedef struct pb200_logit_bias { int32_t token; float bias; } pb200_logit_bias;          /* llama_logit_bias */
typedef struct pb200_penalties {
    int32_t last_n;                     /* penalty_last_n; < 0 behaves as 0, like the reference */
    float   repeat, freq, present;      /* 1 / 0 / 0: off */
    int32_t penalize_nl, ignore_eos;
    int32_t nl_token, eos_token;        /* -1: the vocabulary has none */
    int32_t n_logit_bias;
    const pb200_logit_bias * logit_bias;   /* host array, copied by the call */
} pb200_penalties;
/* device bytes of one penalty state: configuration, bias list, a history ring of last_n tokens and its count */
PB200_API size_t pb200_penalty_state_bytes(int n_vocab, int last_n, int n_logit_bias);
/* a fresh penalties sampler in state_dev (pb200_penalty_state_bytes(n_vocab, p->last_n, p->n_logit_bias) bytes): configuration and bias
 * list uploaded, history cleared.  The list travels in the launches' arguments (one launch per 256 entries, at least one), so p may be
 * freed when the call returns.  PB200_EINVAL: repeat not finite or <= 0, freq / present not finite, a NaN bias, n_logit_bias < 0, or
 * a NULL list with n_logit_bias > 0. */
PB200_API int pb200_penalty_init(void * state_dev, int n_vocab, const pb200_penalties * p, void * stream);
/* llama_sampler_accept for n tokens in device memory: only the last last_n of them are kept.  One launch. */
PB200_API int pb200_penalty_accept(void * state_dev, const int32_t * tokens_dev, int n, void * stream);
/* steps 1-4 above: out[n_vocab] = the penalised copy of logits[n_vocab]; out must not alias logits.  One launch. */
PB200_API int pb200_penalty_apply(const float * logits, int n_vocab, const void * state_dev, float * out, void * stream);
/* All three only enqueue on stream: no host synchronisation, no allocation, capturable in a CUDA graph. */

/* ---- fused decode launches (what the engine is made of), for graph-level fusion in a host such as the ggml-backend plugin ---- */
typedef struct pb200_gemv_mat {
    int32_t type;          /* k-quant type of W (Q4_K / Q5_K / Q6_K) */
    int32_t _pad;
    const void * W;        /* [n][k] raw GGUF blocks, 16-byte aligned (padding rule above) */
    int64_t n;
    float * y;             /* [n]  y = W . act (+ add[row]) */
    const float * add;     /* optional [n]: bias or residual added in the epilogue (ggml ADD node folded in) */
} pb200_gemv_mat;
/* Up to 3 matrices sharing one activation of length k (k % 256 == 0, k <= 29696), ONE launch.  prologue:
 *   0  act_ws already holds the q8_K activation (pb200_quantize_act, or pb200_attn_ggml with act_ws_out)
 *   1  act = q8_K( rms_norm(in0, eps) * in1 )     ggml RMS_NORM + MUL by the norm weight   (llm_build_norm, src/llama.cpp:9772-9802)
 *   2  act = q8_K( silu(in0) * in1 )              ggml UNARY(SILU) + MUL                    (llm_build_ffn, src/llama.cpp:9858-9907)
 * computed once, distributed over the launch's CTAs (one in-kernel grid barrier), left in act_ws.  sync_ws: 16 bytes of zero-initialised
 * device memory owned by the caller (barrier state, self-resetting; one per stream).  pdl != 0: the launch may start while the
 * previous kernel of the stream drains (programmatic dependent launch); its inputs are read only after that kernel has completed.
 * Returns PB200_ENOTSUP for types / shapes outside the fast kernel: pb200_gemv_fused_supported tells them apart before the call. */
PB200_API int pb200_gemv_fused(int nmat, const pb200_gemv_mat * mats, int64_t k, void * act_ws, int prologue, const float * in0, const float * in1,
                               float eps, void * sync_ws, int pdl, void * stream);
/* 1 when pb200_gemv_fused takes a matrix of this type with k columns (a k-quant type, k % 256 == 0, k <= 29696), else 0.  W's
 * 16-byte alignment is a precondition on top of it. */
PB200_API int pb200_gemv_fused_supported(int type, int64_t k);
/* One token of the reference graph's FA-off attention chain as ONE launch (llm_build_kv_store + llm_build_kqv, src/llama.cpp:9673-9718,
 * 10032-10165): rope(q), rope(k) -> f16 K row into cell kv_head of k_cache [cell][n_head_kv*128]; v -> f16 into column kv_head of the
 * TRANSPOSED v cache [n_head_kv*128][vt_stride]; out[h] = softmax(scale * K q_h + mask) . V over n_cells cells (multiple of 32, mask f32
 * [n_cells], -inf = not visible).  head_dim 128, n_head even.  act_ws_out (optional): also leaves q8_K(out) there for the following
 * mat-vec.  kv_head_dev (optional): the cell is read from this device word instead of kv_head, so a CUDA graph that captured the launch can
 * be replayed for the next token.  rope op parameters as in pb200_rope.  Returns PB200_ENOTSUP for shapes it does not handle, among
 * them n_cells above pb200_attn_ggml_max_cells(). */
PB200_API int pb200_attn_ggml(const float * q, const float * k, const float * v, void * k_cache_f16, void * v_cache_t_f16, int64_t vt_stride, float * out,
                              void * act_ws_out, int n_head, int n_head_kv, int head_dim, const int32_t * pos_dev, int n_cells, int kv_head,
                              const int32_t * kv_head_dev, const float * mask, int n_dims, int mode, float freq_base, float freq_scale, float ext_factor, float attn_factor,
                              float beta_fast, float beta_slow, int n_ctx_orig, const float * freq_factors, float scale, int pdl, void * stream);
/* the largest n_cells pb200_attn_ggml takes on the current device (a multiple of 32): the score row lives in shared memory */
PB200_API int pb200_attn_ggml_max_cells(void);

/* ---- decode engine (one model shard per process / GPU) ---- */
typedef struct pb200_hparams {
    int32_t n_layer, n_embd, n_head, n_head_kv, head_dim, n_ff, n_vocab, n_ctx;
    int32_t rope_mode;        /* 0 = NORM (llama), 2 = NEOX (qwen2) */
    int32_t n_ctx_orig;
    float   rope_freq_base, rope_freq_scale, rms_eps;
} pb200_hparams;

typedef struct pb200_model pb200_model;

/* layers [layer_begin, layer_end) live on this device (prima's layer window, src/llama.cpp:3838-3883);
 * with_embd / with_head: whether token_embd and output_norm+output live here (first / last pipeline stage).
 * NULL for an n_ctx longer than the attention kernels can hold: beyond about 15k cells the decode step keeps a whole score row of
 * n_ctx floats in shared memory, which limits n_ctx to 56 800 on an H100 (the device's opt-in shared memory per block). */
PB200_API pb200_model * pb200_model_create(const pb200_hparams * hp, int device, int layer_begin, int layer_end, int with_embd, int with_head);
PB200_API void          pb200_model_free(pb200_model * m);
/* tensor names follow GGUF: "token_embd.weight", "output_norm.weight", "output.weight", "rope_freqs.weight",
 * "blk.%d.{attn_norm,attn_q,attn_k,attn_v,attn_output,ffn_norm,ffn_gate,ffn_up,ffn_down}.weight", "blk.%d.attn_{q,k,v}.bias".
 * data: HOST pointer to raw GGUF bytes (exactly ggml_nbytes) — the same bytes llm_load_tensors hands to set_tensor. */
PB200_API int pb200_model_set_tensor(pb200_model * m, const char * name, int type, const void * host_data, size_t nbytes);
/* The same without the copy: reserves the tensor's device memory and returns its address in *dev_ptr (NULL with return 0: the tensor
 * belongs to another stage) for hosts that stream the bytes themselves (pb200_model_load_gguf does). */
PB200_API int pb200_model_tensor_alloc(pb200_model * m, const char * name, int type, size_t nbytes, void ** dev_ptr);
/* GGUF file -> finalized model shard (SURVEY N2; replaces gguf_init_from_file + llm_load_hparams + llm_load_tensors' per-tensor
 * synchronous set_tensor, ggml-cuda.cu:464-487, for this path): v2 / v3 containers, architectures "llama" and "qwen2", tensors kept in
 * their raw block layout; the file is streamed through two pinned 64-MiB buffers with cudaMemcpyAsync so reading chunk i+1 overlaps the
 * PCIe copy of chunk i.  layer_end < 0: to the last layer; with_embd / with_head < 0: derived from the window; n_ctx <= 0:
 * min(trained context, 4096).  seconds / bytes_loaded (optional) report the load.  pb200_gguf_probe only parses (no CUDA): hyper-parameters,
 * tensor count, bytes of the data section, architecture string (16 bytes). */
PB200_API int pb200_model_load_gguf(const char * path, int device, int layer_begin, int layer_end, int n_ctx, int with_embd, int with_head,
                                    pb200_model ** out, double * seconds, int64_t * bytes_loaded);
PB200_API int pb200_gguf_probe(const char * path, pb200_hparams * hp, int32_t * n_tensors, int64_t * data_bytes, char * arch_out16);
/* random-init weights generated on the device with the Q4_K_M (ftype 0), Q5_K_M (ftype 1) or Q4_0 (ftype 2) type mixture of
 * llama_tensor_get_type (src/llama.cpp:19271-19556), fallbacks for rows that are not a multiple of 256 included (Q4_K -> Q5_0,
 * Q5_K -> Q5_1, Q6_K -> Q8_0: Qwen2.5-72B's ffn_down).  Q4_0 is the no-imatrix mixture: every matrix and the embedding Q4_0, the
 * output head Q6_K.  Types: Q4_K, Q5_K, Q6_K, Q8_0, Q5_1, Q5_0, Q4_0.  For benchmarking without a checkpoint */
PB200_API int pb200_model_synth(pb200_model * m, int ftype, uint64_t seed);
PB200_API int pb200_model_finalize(pb200_model * m);     /* allocate KV cache + activations, capture the CUDA graph */
/* device address, size and ggml type of a tensor this shard holds (GGUF names as in pb200_model_set_tensor): lets a host copy
 * weights device-to-device, e.g. bench.py moving the synthetic model into the ggml-backend buffers of the plugin */
PB200_API int pb200_model_tensor_device(pb200_model * m, const char * name, const void ** dev_ptr, size_t * nbytes, int * type);
PB200_API int64_t pb200_model_weight_bytes(const pb200_model * m);    /* algorithmic bytes read per decoded token on this shard */
/* Prompt processing (prefill): n_tokens tokens at positions pos0 .. pos0+n_tokens-1 through all layers as one batch — the
 * reference's llama_decode with a multi-token ubatch (ne11 > 1: ggml_cuda_op_mul_mat_q, mmq.cu:3-98; attention
 * ggml-cuda.cu:1737-1881).  Mat-muls on the tensor cores (pb200_mul_mat_q), attention over the K/V rows just stored.  The KV
 * cache is left exactly as n_tokens pb200_decode calls would leave it up to fp16-rounding differences in the mat-muls;
 * logits of the LAST token go to logits_host (may be NULL).  Models created with with_embd and first_layer == 0 only. */
PB200_API int pb200_prefill(pb200_model * m, const int32_t * tokens_host, int32_t n_tokens, int32_t pos0, float * logits_host);
/* Prompt processing on a pipeline shard (prima's layer windows, src/llama.cpp:3838-3883, 17825-18029): ONE ubatch of n_tokens <= 512 through
 * the layers of this model object.  The stage that holds the embedding takes tokens_host (hidden_in_dev ignored); every other stage takes
 * the previous stage's hidden states hidden_in_dev [n_tokens][n_embd] f32 in device memory (not modified).  The stage's output hidden
 * states stay on the device at pb200_prefill_hidden_device(m) until the next prefill call (the caller ships them to the next stage, e.g.
 * with ncclSend on the model stream); the stage with the head also computes the last token's logits.  synchronize = 0: everything is
 * only enqueued on the model stream (micro-batched pipelines keep several ubatches in flight across the stages); logits_host requires
 * synchronize != 0.  K/V rows pos0 .. pos0+n_tokens-1 of this shard's layers are written like pb200_prefill writes them. */
PB200_API int pb200_prefill_stage(pb200_model * m, const int32_t * tokens_host, const float * hidden_in_dev, int32_t n_tokens, int32_t pos0,
                                  float * logits_host, int32_t synchronize);
PB200_API float * pb200_prefill_hidden_device(pb200_model * m);
PB200_API int pb200_kv_clear(pb200_model * m);
/* prima's context shift on this shard's cache for slot seq (what llama-cli does when the context fills, examples/main/main.cpp:578-608):
 *   llama_kv_cache_seq_rm(seq, p0 + delta, p0) + llama_kv_cache_seq_add(seq, p0, p1, delta)
 * (src/llama.cpp:4378-4427; K rotated like build_k_shift, :10665-10719).  The engine keeps cell == position, so the cells are
 * compacted: cell c in [p0, p1) moves to c + delta, for every layer of this shard (any pipeline shard, with or without embedding / head).
 *   - Arguments: delta < 0, p0 + delta >= 0, p0 < p1 <= n_ctx, 0 <= seq < n_seq, else PB200_EINVAL; NULL / unfinalized model: PB200_ESTATE
 *     (the three conditions on delta, p0 and p1 alone are checked first, before the model).
 *   - The moved K row is f16(rope(f32(K), pos = delta)), V rows are copied bit for bit.  That is what the reference's K-shift computes; it
 *     is NOT K computed directly at the new position (the row was rounded to f16 at its old position and is rounded again here).
 *     Equality with the reference holds for one shift between two decodes, which is what llama-cli does.  The reference adds up the deltas of several
 *     seq_add calls and rotates once at the next decode; this call rotates and rounds every time, so two shifts with no decode in
 *     between are rounded twice where the reference rounds once.
 *   - Cells below p0 + delta and all other slots stay bit-identical; cells [p1 + delta, p1) are unspecified afterwards.
 *   - The slot's device position (pb200_token_device(m, seq)[1]) moves by delta when it is >= p0; its token is kept.  A device-resident
 *     loop (pb200_step_seq_dev + pb200_argmax_seq / pb200_sample_seq with feed_back) continues without a host round trip, and the captured
 *     per-slot CUDA graphs stay valid (they read the position from device memory).
 *   - One launch enqueued on the model stream, no host synchronisation; call it outside any stream capture, like pb200_sampling_set_seq. */
PB200_API int pb200_kv_seq_shift(pb200_model * m, int seq, int32_t p0, int32_t p1, int32_t delta);
/* device address of the f16 K (v == 0) or V (v != 0) cache of this shard: [n_seq][layer_end - layer_begin][n_ctx][n_head_kv * head_dim]
 * (white-box tests and hosts that inspect the cache; NULL before finalize or on a shard without layers) */
PB200_API void * pb200_kv_device(pb200_model * m, int v);

/* one decode step, HOST in/out (the llama_decode-equivalent call): token id + position in, n_vocab logits out.
 * On a pipeline stage without the embedding / head the hidden state is exchanged through pb200_hidden_* instead. */
PB200_API int pb200_decode(pb200_model * m, int32_t token, int32_t pos, float * logits_host);
/* device-resident variant: enqueue one step on the model stream, no host copies, no synchronisation */
PB200_API int pb200_decode_async(pb200_model * m, int32_t token, int32_t pos);
PB200_API int pb200_synchronize(pb200_model * m);
/* Several independent sequences per shard (each with its own KV cache, token and position slot): what keeps every stage of the layer
 * pipeline busy — prima's piped ring with one token per stage in flight (src/llama.cpp:17825-18029, 18299-18387).  Set before finalize. */
PB200_API int pb200_model_set_n_seq(pb200_model * m, int n_seq);
PB200_API int pb200_decode_seq_async(pb200_model * m, int seq, int32_t token, int32_t pos);   /* pb200_decode_async on slot seq */
/* one step of slot seq with token id and position taken from device memory (written by a hand-off, pb200_set_tokpos_seq or
 * pb200_argmax_seq); nothing crosses the host.  advance_pos != 0: the slot's position is incremented afterwards. */
PB200_API int pb200_step_seq_dev(pb200_model * m, int seq, int advance_pos);
PB200_API int pb200_set_tokpos_seq(pb200_model * m, int seq, int32_t token, int32_t pos);
/* greedy sampling on the device (ggml-cuda/argmax.cu:7): argmax of the slot's logits -> pb200_sample_device(m, seq); feed_back != 0 on a
 * shard that also holds the embedding writes it into the slot's token as well (single-GPU generation without a host round trip) */
PB200_API int pb200_argmax_seq(pb200_model * m, int seq, int feed_back);
/* seeded sampling per slot (the chain of pb200_sample): pb200_sampling_set_seq stores the parameters and seeds the slot's own generator
 * with p->seed (on the model stream; call it outside any capture); pb200_sample_seq then works like pb200_argmax_seq with those
 * parameters -> pb200_sample_device(m, seq), and with feed_back the slot's token.  PB200_ESTATE for a slot without parameters. */
PB200_API int pb200_sampling_set_seq(pb200_model * m, int seq, const pb200_sampling * p);
PB200_API int pb200_sample_seq(pb200_model * m, int seq, int feed_back);
/* logit bias and penalties per slot (pb200_penalty_apply's semantics): pb200_penalties_set_seq configures slot seq and clears its
 * history (NULL removes them); it allocates the slot's state on first use, so call it outside any capture.  It does not touch the
 * sampling parameters or the generator.  With penalties set, pb200_sample_seq is apply -> the slot's chain on the penalised row (greedy
 * for temp <= 0) -> accept of the token: three launches, the last left out when last_n is 0.  pb200_logits_device keeps the raw
 * logits.  pb200_argmax_seq stays a plain argmax: greedy with penalties is pb200_sample_seq with temp <= 0.  pb200_sampler_accept_seq
 * accepts n host tokens into the slot's history (the prompt, as llama-cli accepts it); PB200_ESTATE for a slot without penalties.
 * pb200_kv_clear and pb200_kv_seq_shift leave the history alone, as the reference's sampler is independent of the KV cache.
 * PB200_ESTATE on a shard without the head. */
PB200_API int pb200_penalties_set_seq(pb200_model * m, int seq, const pb200_penalties * p);
PB200_API int pb200_sampler_accept_seq(pb200_model * m, int seq, const int32_t * tokens_host, int n);
PB200_API int32_t * pb200_token_device(pb200_model * m, int seq);    /* int32[2]: {token, position} of the slot */
PB200_API int32_t * pb200_sample_device(pb200_model * m, int seq);   /* int32: the slot's last sample (pb200_argmax_seq or pb200_sample_seq) */
PB200_API float * pb200_logits_device(pb200_model * m);      /* [n_vocab] f32 */
PB200_API float * pb200_hidden_in_device(pb200_model * m);   /* [n_embd] f32: input of layer_begin (written by the previous stage) */
PB200_API float * pb200_hidden_out_device(pb200_model * m);  /* [n_embd] f32: output of layer_end-1 */
PB200_API void *  pb200_stream(pb200_model * m);
PB200_API int pb200_get_hidden(pb200_model * m, float * hidden_host);   /* copies hidden_out to the host (tests) */
/* one step with CUDA events around every GEMV launch (direct launches): summed GEMV device time, the algorithmic
 * weight bytes those launches read, their count and the whole-step time — the live roofline measurement of bench.py */
PB200_API int pb200_profile_step(pb200_model * m, int32_t token, int32_t pos, double * gemv_ms, int64_t * gemv_bytes, int32_t * gemv_launches, double * step_ms);
PB200_API int pb200_set_hidden(pb200_model * m, const float * hidden_host);   /* host -> hidden_in (tests, host-staged hand-off) */
PB200_API int pb200_debug_read(pb200_model * m, const char * name, float * host, int64_t n);   /* white-box tests: q,k,v,att,g,u,x_a,x_b,xn,logits */
PB200_API int pb200_set_use_graph(pb200_model * m, int on);             /* CUDA-graph replay on/off (default on) */

#ifdef __cplusplus
}
#endif
#endif /* PRIMA_B200_H */
