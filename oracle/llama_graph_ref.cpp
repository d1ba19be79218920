// oracle/llama_graph_ref.cpp — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// End-to-end oracle: a restatement of the reference's graph builders build_llama / build_qwen2
// (src/llama.cpp:11000-11216, 12736-12916; helpers llm_build_norm :9772, llm_build_ffn :9804,
// llm_build_kv_store :9673, llm_build_kqv :10032, KQ mask :10838 + llama_set_inputs :17276, KV padding
// :4485) that is EXECUTED BY THE UNMODIFIED REFERENCE CPU ggml BACKEND (oracle/_ref/*/libggml_ref.so,
// compiled from the reference's ggml/src).  libllama itself cannot be built here (needs <zmq.h>,
// src/llama.cpp:1), so only the op sequence is restated; every kernel that runs is the reference's.
// FA off, KV cache f16, V cache transposed — the reference defaults (common/common.h:275).
//
// C ABI (ctypes): gref_create / gref_decode / gref_free, model description identical to
// oracle/kquants_port.c's port_model so the same weight blobs feed both oracles.
#include "ggml.h"
#include "ggml-backend.h"

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

extern "C" {

typedef struct {
    int32_t n_layer, n_embd, n_head, n_head_kv, head_dim, n_ff, n_vocab, n_ctx;
    int32_t rope_mode, n_ctx_orig;
    float rope_freq_base, rope_freq_scale, rms_eps;
} gref_hparams;
typedef struct { int32_t type; int32_t _pad; const void * data; } gref_weight;
typedef struct {
    const float *attn_norm, *ffn_norm;
    gref_weight wq, wk, wv, wo, gate, up, down;
    const float *bq, *bk, *bv;
} gref_layer;
typedef struct {
    gref_hparams hp;
    gref_weight tok_embd;
    const float * output_norm;
    gref_weight output;
    const gref_layer * layers;
    const float * rope_freq_factors;
    uint16_t *k_cache, *v_cache;   // [n_layer][n_ctx*n_embd_kv] f16; V is used TRANSPOSED per layer: [n_embd_kv][n_ctx]
} gref_model;

struct gref_ctx {
    gref_model m;
    std::vector<gref_layer> layers;
    int n_threads;
    ggml_context * wctx = nullptr;   // weight tensor headers (no_alloc, data -> caller memory)
    ggml_tensor *tok_embd, *output_norm, *output, *rope_ff = nullptr;
    struct L { ggml_tensor *attn_norm, *ffn_norm, *wq, *wk, *wv, *wo, *gate, *up, *down, *bq, *bk, *bv, *k, *v; };
    std::vector<L> L_;
};

static ggml_tensor * wrap2d(ggml_context * c, int type, const void * data, int64_t ne0, int64_t ne1) {
    ggml_tensor * t = ggml_new_tensor_2d(c, (ggml_type) type, ne0, ne1);
    t->data = const_cast<void *>(data);
    return t;
}
static ggml_tensor * wrap1d(ggml_context * c, int type, const void * data, int64_t ne0) {
    if (!data) return nullptr;
    ggml_tensor * t = ggml_new_tensor_1d(c, (ggml_type) type, ne0);
    t->data = const_cast<void *>(data);
    return t;
}

void * gref_create(const gref_model * model, int n_threads) {
    gref_ctx * g = new gref_ctx();
    g->m = *model;
    g->layers.assign(model->layers, model->layers + model->hp.n_layer);
    g->m.layers = g->layers.data();
    g->n_threads = n_threads;
    const gref_hparams & hp = g->m.hp;
    ggml_init_params ip = { (size_t) ggml_tensor_overhead() * (size_t)(16 + 16 * hp.n_layer) + 4096, nullptr, true };
    g->wctx = ggml_init(ip);
    ggml_context * c = g->wctx;
    const int64_t E = hp.n_embd, QD = (int64_t) hp.n_head * hp.head_dim, EK = (int64_t) hp.n_head_kv * hp.head_dim, F = hp.n_ff;
    g->tok_embd = wrap2d(c, g->m.tok_embd.type, g->m.tok_embd.data, E, hp.n_vocab);
    g->output_norm = wrap1d(c, GGML_TYPE_F32, g->m.output_norm, E);
    g->output = wrap2d(c, g->m.output.type, g->m.output.data, E, hp.n_vocab);
    g->rope_ff = wrap1d(c, GGML_TYPE_F32, g->m.rope_freq_factors, hp.head_dim / 2);
    g->L_.resize(hp.n_layer);
    for (int il = 0; il < hp.n_layer; il++) {
        const gref_layer & s = g->layers[il];
        gref_ctx::L & d = g->L_[il];
        d.attn_norm = wrap1d(c, GGML_TYPE_F32, s.attn_norm, E);
        d.ffn_norm = wrap1d(c, GGML_TYPE_F32, s.ffn_norm, E);
        d.wq = wrap2d(c, s.wq.type, s.wq.data, E, QD);
        d.wk = wrap2d(c, s.wk.type, s.wk.data, E, EK);
        d.wv = wrap2d(c, s.wv.type, s.wv.data, E, EK);
        d.wo = wrap2d(c, s.wo.type, s.wo.data, QD, E);
        d.gate = wrap2d(c, s.gate.type, s.gate.data, E, F);
        d.up = wrap2d(c, s.up.type, s.up.data, E, F);
        d.down = wrap2d(c, s.down.type, s.down.data, F, E);
        d.bq = wrap1d(c, GGML_TYPE_F32, s.bq, QD);
        d.bk = wrap1d(c, GGML_TYPE_F32, s.bk, EK);
        d.bv = wrap1d(c, GGML_TYPE_F32, s.bv, EK);
        // llama_kv_cache_init (src/llama.cpp:3955-3975): 1-D f16 tensors of n_embd_k_gqa*kv_size per layer
        d.k = wrap1d(c, GGML_TYPE_F16, g->m.k_cache + (size_t) il * hp.n_ctx * EK, EK * hp.n_ctx);
        d.v = wrap1d(c, GGML_TYPE_F16, g->m.v_cache + (size_t) il * hp.n_ctx * EK, EK * hp.n_ctx);
    }
    return g;
}

void gref_free(void * p) {
    gref_ctx * g = (gref_ctx *) p;
    if (!g) return;
    ggml_free(g->wctx);
    delete g;
}

// Processes n_tokens tokens at positions pos0..pos0+n_tokens-1 (kv_head = pos0).  logits: [n_tokens][n_vocab]
// (all rows; the reference gathers output rows with inp_out_ids, equivalent for the rows kept).
// hidden_out (optional): [n_tokens][n_embd] last-layer output (l_out).  Returns 0 on success.
int gref_decode(void * p, const int32_t * tokens, int n_tokens, int pos0, float * logits, float * hidden_out, size_t mem_bytes) {
    gref_ctx * g = (gref_ctx *) p;
    const gref_hparams & hp = g->m.hp;
    const int64_t E = hp.n_embd, H = hp.n_head, HK = hp.n_head_kv, D = hp.head_dim;
    const int64_t EK = HK * D;
    const int64_t n_ctx = hp.n_ctx;
    const int64_t kv_head = pos0;
    // kv_self.n = min(size, max(pad, GGML_PAD(cell_max, pad))), pad = 32 when FA off (src/llama.cpp:4485, 18442-18451)
    int64_t n_kv = ((pos0 + n_tokens + 31) / 32) * 32;
    if (n_kv < 32) n_kv = 32;
    if (n_kv > n_ctx) n_kv = n_ctx;

    ggml_init_params ip = { mem_bytes, nullptr, false };
    ggml_context * c = ggml_init(ip);
    if (!c) return -1;
    ggml_cgraph * gf = ggml_new_graph_custom(c, 65536, false);

    ggml_tensor * inp_tokens = ggml_new_tensor_1d(c, GGML_TYPE_I32, n_tokens);
    memcpy(inp_tokens->data, tokens, sizeof(int32_t) * n_tokens);
    ggml_tensor * inp_pos = ggml_new_tensor_1d(c, GGML_TYPE_I32, n_tokens);
    for (int i = 0; i < n_tokens; i++) ((int32_t *) inp_pos->data)[i] = pos0 + i;
    const int64_t n_tok_pad = GGML_PAD(n_tokens, GGML_KQ_MASK_PAD);
    ggml_tensor * KQ_mask = ggml_new_tensor_2d(c, GGML_TYPE_F32, n_kv, n_tok_pad);
    {   // llama_set_inputs causal mask (src/llama.cpp:17330-17380): -inf where cell pos > token pos; padded rows -inf
        float * md = (float *) KQ_mask->data;
        for (int64_t j = 0; j < n_tok_pad; j++)
            for (int64_t i = 0; i < n_kv; i++)
                md[j * n_kv + i] = (j < n_tokens && i <= pos0 + j) ? 0.0f : -INFINITY;
    }

    // llm_build_inp_embd (:9640-9671)
    ggml_tensor * inpL = ggml_get_rows(c, g->tok_embd, inp_tokens);
    const float kq_scale = 1.0f / sqrtf((float) D);
    ggml_tensor * cur = nullptr;
    for (int il = 0; il < hp.n_layer; il++) {
        gref_ctx::L & L = g->L_[il];
        ggml_tensor * inpSA = inpL;
        cur = ggml_rms_norm(c, inpL, hp.rms_eps);
        cur = ggml_mul(c, cur, L.attn_norm);
        ggml_tensor * Qcur = ggml_mul_mat(c, L.wq, cur);
        if (L.bq) Qcur = ggml_add(c, Qcur, L.bq);
        ggml_tensor * Kcur = ggml_mul_mat(c, L.wk, cur);
        if (L.bk) Kcur = ggml_add(c, Kcur, L.bk);
        ggml_tensor * Vcur = ggml_mul_mat(c, L.wv, cur);
        if (L.bv) Vcur = ggml_add(c, Vcur, L.bv);
        Qcur = ggml_rope_ext(c, ggml_reshape_3d(c, Qcur, D, H, n_tokens), inp_pos, g->rope_ff, (int) D, hp.rope_mode,
                             hp.n_ctx_orig, hp.rope_freq_base, hp.rope_freq_scale, 0.0f, 1.0f, 32.0f, 1.0f);
        Kcur = ggml_rope_ext(c, ggml_reshape_3d(c, Kcur, D, HK, n_tokens), inp_pos, g->rope_ff, (int) D, hp.rope_mode,
                             hp.n_ctx_orig, hp.rope_freq_base, hp.rope_freq_scale, 0.0f, 1.0f, 32.0f, 1.0f);
        // llm_build_kv_store (:9673-9718), FA off: V cache transposed
        {
            ggml_tensor * k_view = ggml_view_1d(c, L.k, n_tokens * EK, ggml_row_size(L.k->type, EK) * kv_head);
            ggml_build_forward_expand(gf, ggml_cpy(c, Kcur, k_view));
            ggml_tensor * v_view = ggml_view_2d(c, L.v, n_tokens, EK, n_ctx * ggml_element_size(L.v), kv_head * ggml_element_size(L.v));
            ggml_tensor * v_cur_t = ggml_transpose(c, Vcur);
            ggml_build_forward_expand(gf, ggml_cpy(c, v_cur_t, v_view));
        }
        // llm_build_kqv (:10032-10165), FA off
        {
            ggml_tensor * q = ggml_permute(c, Qcur, 0, 2, 1, 3);
            ggml_tensor * k = ggml_view_3d(c, L.k, D, n_kv, HK, ggml_row_size(L.k->type, EK), ggml_row_size(L.k->type, D), 0);
            ggml_tensor * kq = ggml_mul_mat(c, k, q);
            if (hp.rope_mode == 2) ggml_mul_mat_set_prec(kq, GGML_PREC_F32);   // LLM_ARCH_QWEN2 (:10100-10104); no-op on CPU
            kq = ggml_soft_max_ext(c, kq, KQ_mask, kq_scale, 0.0f);
            ggml_tensor * v = ggml_view_3d(c, L.v, n_kv, D, HK, ggml_element_size(L.v) * n_ctx, ggml_element_size(L.v) * n_ctx * D, 0);
            ggml_tensor * kqv = ggml_mul_mat(c, v, kq);
            ggml_tensor * kqv_merged = ggml_permute(c, kqv, 0, 2, 1, 3);
            cur = ggml_cont_2d(c, kqv_merged, D * H, n_tokens);
            ggml_build_forward_expand(gf, cur);
            cur = ggml_mul_mat(c, L.wo, cur);
        }
        ggml_tensor * ffn_inp = ggml_add(c, cur, inpSA);
        cur = ggml_rms_norm(c, ffn_inp, hp.rms_eps);
        cur = ggml_mul(c, cur, L.ffn_norm);
        {   // llm_build_ffn LLM_FFN_SILU / LLM_FFN_PAR (:9804-9929)
            ggml_tensor * tmp = ggml_mul_mat(c, L.up, cur);
            cur = ggml_mul_mat(c, L.gate, cur);
            cur = ggml_silu(c, cur);
            cur = ggml_mul(c, cur, tmp);
            cur = ggml_mul_mat(c, L.down, cur);
        }
        cur = ggml_add(c, cur, ffn_inp);
        inpL = cur;
    }
    ggml_tensor * l_out = cur;
    cur = ggml_rms_norm(c, cur, hp.rms_eps);
    cur = ggml_mul(c, cur, g->output_norm);
    cur = ggml_mul_mat(c, g->output, cur);
    ggml_build_forward_expand(gf, cur);

    ggml_status st = ggml_graph_compute_with_ctx(c, gf, g->n_threads);
    if (st == GGML_STATUS_SUCCESS) {
        if (logits) memcpy(logits, cur->data, sizeof(float) * (size_t) hp.n_vocab * n_tokens);
        if (hidden_out) memcpy(hidden_out, l_out->data, sizeof(float) * (size_t) E * n_tokens);
    }
    ggml_free(c);
    return st == GGML_STATUS_SUCCESS ? 0 : -2;
}

// Single reference mul_mat on the CPU backend: dst[T][N] = W[N][K] (type) x X[T][K] f32 — used to pin the port and
// as the CPU baseline for the GEMV micro-benchmark (ggml_compute_forward_mul_mat, ggml.c:12377).
int gref_mul_mat(int type, const void * W, int64_t N, int64_t K, const float * X, int64_t T, float * dst, int n_threads) {
    size_t mem = (size_t)(N * T * 4 + K * T * 8) + (64u << 20);
    ggml_init_params ip = { mem, nullptr, false };
    ggml_context * c = ggml_init(ip);
    if (!c) return -1;
    ggml_set_no_alloc(c, true);                                        // headers only: data stays in caller memory
    ggml_tensor * w = ggml_new_tensor_2d(c, (ggml_type) type, K, N);
    w->data = const_cast<void *>(W);
    ggml_tensor * x = ggml_new_tensor_2d(c, GGML_TYPE_F32, K, T);
    x->data = const_cast<float *>(X);
    ggml_set_no_alloc(c, false);
    ggml_tensor * y = ggml_mul_mat(c, w, x);
    ggml_cgraph * gf = ggml_new_graph(c);
    ggml_build_forward_expand(gf, y);
    ggml_status st = ggml_graph_compute_with_ctx(c, gf, n_threads);
    if (st == GGML_STATUS_SUCCESS) memcpy(dst, y->data, sizeof(float) * (size_t)(N * T));
    ggml_free(c);
    return st == GGML_STATUS_SUCCESS ? 0 : -2;
}

}  // extern "C"
