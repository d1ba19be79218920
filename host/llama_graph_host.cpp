// host/llama_graph_host.cpp — a stand-in for the part of libllama that the drop-in boundary talks to.
//
// libllama (src/llama.cpp) cannot be built in this environment (it needs <zmq.h>, src/llama.cpp:1), so the tests and
// bench.py's end-to-end leg need something that plays its role: own the weights and the KV cache in ggml BACKEND BUFFERS,
// build the decode graph of build_llama / build_qwen2 (src/llama.cpp:11000-11216, 12736-12916; llm_build_norm :9772,
// llm_build_ffn :9804, llm_build_kv_store :9673, llm_build_kqv :10032, KQ mask :10838 + llama_set_inputs :17276, KV padding
// :4485) with the host's ggml, hand it to ANY registered ggml backend through the public ggml-backend API
// (ggml_backend_graph_compute, ggml_backend_tensor_set / _get) and read the logits back.  Run against "CPU" it is the
// reference path; run against "B200_0" it exercises exactly what llama_decode would exercise in the plugin: buffer
// allocation, set_tensor, graph_compute (with its graph-level fusion), get_tensor.
//
// This file is host-application code.  It links the host's ggml only (host/Makefile builds one from the reference tree,
// unmodified) and knows nothing about libprima_b200.so.  FA off, KV cache f16, V cache transposed — the reference defaults.
//
// Compute buffer: like llama_new_context_with_model (src/llama.cpp:21361-21402), one ggml_gallocr per context reserves the
// worst-case graph (n_tokens_max tokens, n_kv = n_ctx) once and keeps its buffer for the life of the context; each graph rebuild
// frees only the graph's ggml_context.  Graphs that fit the reservation therefore land at the same addresses every time their
// topology comes back, which is what lets a backend replay work it captured for that topology.
#include "ggml.h"
#include "ggml-alloc.h"
#include "ggml-backend.h"

#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

extern "C" {

typedef struct {
    int32_t n_layer, n_embd, n_head, n_head_kv, head_dim, n_ff, n_vocab, n_ctx;
    int32_t rope_mode, n_ctx_orig;
    float rope_freq_base, rope_freq_scale, rms_eps;
    int32_t has_bias, has_freq_factors;
    int32_t type_default, type_v_even, type_v_odd, type_down_even, type_down_odd, type_output;   // unused by the builder: informational
} lgh_hparams;

struct lgh_layer { ggml_tensor *attn_norm, *ffn_norm, *wq, *wk, *wv, *wo, *gate, *up, *down, *bq, *bk, *bv, *k, *v; };

struct lgh_ctx {
    lgh_hparams hp;
    ggml_backend_t backend = nullptr;
    bool is_cpu = false;
    ggml_context * wctx = nullptr;
    ggml_backend_buffer_t wbuf = nullptr;
    ggml_tensor *tok_embd = nullptr, *output_norm = nullptr, *output = nullptr, *rope_ff = nullptr;
    std::vector<lgh_layer> L;
    std::map<std::string, ggml_tensor *> by_name;
    // the graph of the current (n_tokens, n_kv) bucket, reused token after token (only the cache-view offsets and inputs change)
    ggml_context * gctx = nullptr;
    ggml_gallocr_t galloc = nullptr;   // kept across graph rebuilds: its buffer is reserved for (n_tokens_max, n_ctx)
    int n_tokens_max = 1;
    ggml_cgraph * gf = nullptr;
    int g_tokens = 0;
    int64_t g_nkv = 0;
    ggml_tensor *inp_tokens = nullptr, *inp_pos = nullptr, *kq_mask = nullptr, *logits = nullptr, *l_out = nullptr;
    std::vector<ggml_tensor *> k_views, v_views;
    std::vector<float> mask_host;
    // the KV cells of the one sequence (llama_kv_cell / llama_kv_cache, src/llama.cpp:2860-2960): a cell keeps its slot and carries
    // the position stored in it (-1 = empty) and the RoPE delta accumulated since the last K-shift.  Until the first seq_rm / seq_add
    // after a clear the cells are not consulted (`managed` false): a token at position p goes to cell p, as it always did here.
    struct cell { int32_t pos = -1, delta = 0; };
    std::vector<cell> cells;
    uint32_t head = 0, used = 0;
    bool managed = false, has_shift = false;
    // the K-shift graph of build_k_shift (src/llama.cpp:10665-10719): its own context, built once; inp_K_shift lives in a buffer of
    // the backend (its own allocator, like the scheduler's for this graph), every other node is an in-place view of a K cache
    ggml_context * kctx = nullptr;
    ggml_gallocr_t kgalloc = nullptr;
    ggml_cgraph * kgf = nullptr;
    ggml_tensor * inp_k_shift = nullptr;
    uint64_t n_k_shifts = 0;
    uint64_t n_graph_builds = 0;
    double t_build = 0, t_set = 0, t_enqueue = 0, t_get = 0;   // host seconds spent per phase (diagnostics for bench.py)
};
static double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

static ggml_tensor * new_w(lgh_ctx * c, const char * name, int type, int64_t ne0, int64_t ne1) {
    ggml_tensor * t = ne1 > 0 ? ggml_new_tensor_2d(c->wctx, (ggml_type) type, ne0, ne1) : ggml_new_tensor_1d(c->wctx, (ggml_type) type, ne0);
    ggml_set_name(t, name);
    c->by_name[name] = t;
    return t;
}

// types: ggml_type of every weight matrix, in the order token_embd, output, then per layer wq wk wv wo gate up down (7 * n_layer)
void * lgh_create(const lgh_hparams * hp, const int32_t * types, const char * backend_name, int n_threads) {
    lgh_ctx * c = new lgh_ctx();
    c->hp = *hp;
    ggml_backend_dev_t dev = ggml_backend_dev_by_name(backend_name);
    if (!dev) { fprintf(stderr, "lgh: no backend device named %s\n", backend_name); delete c; return nullptr; }
    c->backend = ggml_backend_dev_init(dev, nullptr);
    if (!c->backend) { delete c; return nullptr; }
    c->is_cpu = ggml_backend_is_cpu(c->backend);
    if (c->is_cpu) ggml_backend_cpu_set_n_threads(c->backend, n_threads);
    const int64_t E = hp->n_embd, QD = (int64_t) hp->n_head * hp->head_dim, EK = (int64_t) hp->n_head_kv * hp->head_dim, F = hp->n_ff;
    ggml_init_params ip = { ggml_tensor_overhead() * (size_t) (16 + 20 * hp->n_layer) + 4096, nullptr, true };
    c->wctx = ggml_init(ip);
    c->tok_embd = new_w(c, "token_embd.weight", types[0], E, hp->n_vocab);
    c->output_norm = new_w(c, "output_norm.weight", GGML_TYPE_F32, E, 0);
    c->output = new_w(c, "output.weight", types[1], E, hp->n_vocab);
    if (hp->has_freq_factors) c->rope_ff = new_w(c, "rope_freqs.weight", GGML_TYPE_F32, hp->head_dim / 2, 0);
    c->L.resize(hp->n_layer);
    char nm[96];
    for (int il = 0; il < hp->n_layer; il++) {
        lgh_layer & l = c->L[il];
        const int32_t * t = types + 2 + 7 * il;
        auto N = [&](const char * s) { snprintf(nm, sizeof nm, "blk.%d.%s", il, s); return nm; };
        l.attn_norm = new_w(c, N("attn_norm.weight"), GGML_TYPE_F32, E, 0);
        l.ffn_norm = new_w(c, N("ffn_norm.weight"), GGML_TYPE_F32, E, 0);
        l.wq = new_w(c, N("attn_q.weight"), t[0], E, QD);
        l.wk = new_w(c, N("attn_k.weight"), t[1], E, EK);
        l.wv = new_w(c, N("attn_v.weight"), t[2], E, EK);
        l.wo = new_w(c, N("attn_output.weight"), t[3], QD, E);
        l.gate = new_w(c, N("ffn_gate.weight"), t[4], E, F);
        l.up = new_w(c, N("ffn_up.weight"), t[5], E, F);
        l.down = new_w(c, N("ffn_down.weight"), t[6], F, E);
        l.bq = l.bk = l.bv = nullptr;
        if (hp->has_bias) {
            l.bq = new_w(c, N("attn_q.bias"), GGML_TYPE_F32, QD, 0);
            l.bk = new_w(c, N("attn_k.bias"), GGML_TYPE_F32, EK, 0);
            l.bv = new_w(c, N("attn_v.bias"), GGML_TYPE_F32, EK, 0);
        }
        // llama_kv_cache_init (src/llama.cpp:3955-3975): 1-D f16 tensors of n_embd_k_gqa * kv_size per layer
        l.k = new_w(c, N("cache_k"), GGML_TYPE_F16, EK * hp->n_ctx, 0);
        l.v = new_w(c, N("cache_v"), GGML_TYPE_F16, EK * hp->n_ctx, 0);
    }
    c->wbuf = ggml_backend_alloc_ctx_tensors(c->wctx, c->backend);
    if (!c->wbuf) { fprintf(stderr, "lgh: weight buffer allocation failed\n"); ggml_free(c->wctx); ggml_backend_free(c->backend); delete c; return nullptr; }
    ggml_backend_buffer_clear(c->wbuf, 0);
    c->cells.resize((size_t) hp->n_ctx);
    return c;
}

void lgh_free(void * p) {
    lgh_ctx * c = (lgh_ctx *) p;
    if (!c) return;
    if (c->kgalloc) ggml_gallocr_free(c->kgalloc);
    if (c->kctx) ggml_free(c->kctx);
    if (c->gctx) ggml_free(c->gctx);
    if (c->galloc) ggml_gallocr_free(c->galloc);
    if (c->wbuf) ggml_backend_buffer_free(c->wbuf);
    if (c->wctx) ggml_free(c->wctx);
    if (c->backend) ggml_backend_free(c->backend);
    delete c;
}

// HOST bytes -> backend tensor (what llm_load_tensors does through ggml_backend_tensor_set)
int lgh_set_tensor(void * p, const char * name, const void * data, size_t nbytes) {
    lgh_ctx * c = (lgh_ctx *) p;
    auto it = c->by_name.find(name);
    if (it == c->by_name.end()) return -1;
    if (nbytes != ggml_nbytes(it->second)) return -2;
    ggml_backend_tensor_set(it->second, data, 0, nbytes);
    return 0;
}
// address and size of a tensor inside its backend buffer (bench.py fills 42 GB of synthetic weights device-to-device)
void * lgh_tensor_data(void * p, const char * name, size_t * nbytes) {
    lgh_ctx * c = (lgh_ctx *) p;
    auto it = c->by_name.find(name);
    if (it == c->by_name.end()) return nullptr;
    if (nbytes) *nbytes = ggml_nbytes(it->second);
    return it->second->data;
}
int lgh_get_tensor(void * p, const char * name, void * data, size_t nbytes) {
    lgh_ctx * c = (lgh_ctx *) p;
    auto it = c->by_name.find(name);
    if (it == c->by_name.end() || nbytes > ggml_nbytes(it->second)) return -1;
    ggml_backend_synchronize(c->backend);
    ggml_backend_tensor_get(it->second, data, 0, nbytes);
    return 0;
}
void lgh_kv_clear(void * p) {
    lgh_ctx * c = (lgh_ctx *) p;
    ggml_backend_synchronize(c->backend);
    for (lgh_layer & l : c->L) {
        std::vector<char> z(ggml_nbytes(l.k), 0);
        ggml_backend_tensor_set(l.k, z.data(), 0, z.size());
        ggml_backend_tensor_set(l.v, z.data(), 0, z.size());
    }
    for (auto & cl : c->cells) cl = lgh_ctx::cell();   // llama_kv_cache_clear (src/llama.cpp:4230-4243)
    c->head = c->used = 0;
    c->managed = c->has_shift = false;
}

// llama_kv_cache_seq_rm of the one sequence (src/llama.cpp:4245-4316, transformer branch): cells with pos in [p0, p1) become empty
int lgh_kv_seq_rm(void * p, int32_t p0, int32_t p1) {
    lgh_ctx * c = (lgh_ctx *) p;
    c->managed = true;   // from here until the next clear, lgh_decode places tokens like llama_decode does
    const uint32_t size = (uint32_t) c->cells.size();
    uint32_t new_head = size;
    if (p0 < 0) p0 = 0;
    if (p1 < 0) p1 = INT32_MAX;
    for (uint32_t i = 0; i < size; i++) {
        lgh_ctx::cell & cl = c->cells[i];
        if (cl.pos >= p0 && cl.pos < p1) {
            cl.pos = -1;
            c->used--;
            if (new_head == size) new_head = i;
        }
    }
    if (new_head != size && new_head < c->head) c->head = new_head;
    return 0;
}
// llama_kv_cache_seq_add (src/llama.cpp:4378-4427): cells with pos in [p0, p1) move by delta in position (not in slot); the K rows
// are re-rotated by the accumulated delta at the next lgh_decode
int lgh_kv_seq_add(void * p, int32_t p0, int32_t p1, int32_t delta) {
    lgh_ctx * c = (lgh_ctx *) p;
    c->managed = true;   // from here until the next clear, lgh_decode places tokens like llama_decode does
    const uint32_t size = (uint32_t) c->cells.size();
    uint32_t new_head = size;
    if (p0 < 0) p0 = 0;
    if (p1 < 0) p1 = INT32_MAX;
    if (p0 == p1) return 0;
    for (uint32_t i = 0; i < size; i++) {
        lgh_ctx::cell & cl = c->cells[i];
        if (cl.pos >= p0 && cl.pos < p1) {
            c->has_shift = true;
            cl.pos += delta;
            cl.delta += delta;
            if (cl.pos < 0) {
                cl.pos = -1;
                c->used--;
                if (new_head == size) new_head = i;
            }
        }
    }
    c->head = new_head != size ? new_head : 0;
    return 0;
}
// position stored in each cell (-1 = empty), n_ctx entries
void lgh_kv_cells(void * p, int32_t * pos_out) {
    lgh_ctx * c = (lgh_ctx *) p;
    for (size_t i = 0; i < c->cells.size(); i++) pos_out[i] = c->cells[i].pos;
}

// build_k_shift: one in-place ROPE per layer on the whole f16 K cache viewed as [head_dim, n_head_kv, n_ctx], positions = the cells'
// deltas (inp_K_shift)
static bool build_k_shift(lgh_ctx * c) {
    if (c->kgf) return true;
    const lgh_hparams & hp = c->hp;
    const int64_t D = hp.head_dim, HK = hp.n_head_kv, n_ctx = hp.n_ctx;
    const size_t max_nodes = (size_t) 16 + 4 * (size_t) hp.n_layer;
    ggml_init_params ip = { ggml_tensor_overhead() * max_nodes + ggml_graph_overhead_custom(max_nodes, false) + (1u << 16), nullptr, true };
    c->kctx = ggml_init(ip);
    c->kgf = ggml_new_graph_custom(c->kctx, max_nodes, false);
    c->inp_k_shift = ggml_new_tensor_1d(c->kctx, GGML_TYPE_I32, n_ctx);
    ggml_set_input(c->inp_k_shift);
    for (lgh_layer & L : c->L) {
        ggml_tensor * k = ggml_view_3d(c->kctx, L.k, D, HK, n_ctx, ggml_row_size(L.k->type, D), ggml_row_size(L.k->type, D * HK), 0);
        ggml_tensor * t = ggml_rope_ext_inplace(c->kctx, k, c->inp_k_shift, c->rope_ff, (int) D, hp.rope_mode, hp.n_ctx_orig, hp.rope_freq_base,
                                                hp.rope_freq_scale, 0.0f, 1.0f, 32.0f, 1.0f);
        ggml_build_forward_expand(c->kgf, t);
    }
    // only inp_K_shift needs memory: every other node is a view of a K cache
    c->kgalloc = ggml_gallocr_new(ggml_backend_get_default_buffer_type(c->backend));
    return ggml_gallocr_alloc_graph(c->kgalloc, c->kgf);
}
// llama_kv_cache_update_internal (src/llama.cpp:19102-19134): run the K-shift graph on the context's backend, then clear the deltas
static bool apply_k_shift(lgh_ctx * c) {
    if (!c->has_shift) return true;
    if (!build_k_shift(c)) return false;
    std::vector<int32_t> d(c->cells.size());
    for (size_t i = 0; i < d.size(); i++) d[i] = c->cells[i].delta;   // llama_set_k_shift (:17262-17273)
    ggml_backend_tensor_set(c->inp_k_shift, d.data(), 0, d.size() * sizeof(int32_t));
    if (ggml_backend_graph_compute(c->backend, c->kgf) != GGML_STATUS_SUCCESS) return false;
    c->has_shift = false;
    for (auto & cl : c->cells) cl.delta = 0;
    c->n_k_shifts++;
    return true;
}
// non-view nodes of the K-shift graph the backend does not support (what ggml_backend_sched checks for a node whose source is a
// pre-allocated tensor in this backend's buffer); -1 if it could not be built
int lgh_kshift_unsupported_nodes(void * p) {
    lgh_ctx * c = (lgh_ctx *) p;
    if (!build_k_shift(c)) return -1;
    int n = 0;
    for (int i = 0; i < ggml_graph_n_nodes(c->kgf); i++) {
        ggml_tensor * t = ggml_graph_node(c->kgf, i);
        if (t->op == GGML_OP_NONE || t->op == GGML_OP_RESHAPE || t->op == GGML_OP_VIEW || t->op == GGML_OP_PERMUTE || t->op == GGML_OP_TRANSPOSE) continue;
        if (!ggml_backend_supports_op(c->backend, t)) n++;
    }
    return n;
}
int lgh_kshift_nodes(void * p) { lgh_ctx * c = (lgh_ctx *) p; return build_k_shift(c) ? ggml_graph_n_nodes(c->kgf) : -1; }
uint64_t lgh_k_shifts(void * p) { return ((lgh_ctx *) p)->n_k_shifts; }

// llama_kv_cache_find_slot, transformer branch (src/llama.cpp:3998-4215): the first run of n_tokens empty cells from head
static int find_slot(lgh_ctx * c, int n_tokens) {
    const uint32_t size = (uint32_t) c->cells.size();
    if ((uint32_t) n_tokens > size) return -1;
    uint32_t n_tested = 0;
    while (true) {
        if (c->head + n_tokens > size) { n_tested += size - c->head; c->head = 0; continue; }
        bool found = true;
        for (int i = 0; i < n_tokens; i++) {
            if (c->cells[c->head + i].pos >= 0) { found = false; c->head += i + 1; n_tested += i + 1; break; }
        }
        if (found) break;
        if (n_tested >= size) return -1;
    }
    return (int) c->head;
}
uint64_t lgh_graph_builds(void * p) { return ((lgh_ctx *) p)->n_graph_builds; }
int lgh_graph_nodes(void * p) { lgh_ctx * c = (lgh_ctx *) p; return c->gf ? ggml_graph_n_nodes(c->gf) : 0; }
// base address of the compute buffer the current graph lives in (NULL before the first lgh_decode)
void * lgh_compute_buffer_base(void * p) {
    lgh_ctx * c = (lgh_ctx *) p;
    return c->gf && c->logits && c->logits->buffer ? ggml_backend_buffer_get_base(c->logits->buffer) : nullptr;
}
// non-view nodes of the current graph the backend does not support; llama.cpp's scheduler would run those on the CPU
int lgh_unsupported_nodes(void * p) {
    lgh_ctx * c = (lgh_ctx *) p;
    if (!c->gf) return -1;
    int n = 0;
    for (int i = 0; i < ggml_graph_n_nodes(c->gf); i++) {
        ggml_tensor * t = ggml_graph_node(c->gf, i);
        if (t->op == GGML_OP_NONE || t->op == GGML_OP_RESHAPE || t->op == GGML_OP_VIEW || t->op == GGML_OP_PERMUTE || t->op == GGML_OP_TRANSPOSE) continue;
        if (!ggml_backend_supports_op(c->backend, t)) n++;
    }
    return n;
}

static void build_graph(lgh_ctx * g, int n_tokens, int64_t n_kv) {
    const lgh_hparams & hp = g->hp;
    const int64_t H = hp.n_head, HK = hp.n_head_kv, D = hp.head_dim;
    const int64_t EK = HK * D;
    const int64_t n_ctx = hp.n_ctx;
    if (g->gctx) { ggml_free(g->gctx); g->gctx = nullptr; g->gf = nullptr; }
    const size_t max_nodes = (size_t) 64 + 40 * (size_t) hp.n_layer;
    ggml_init_params ip = { ggml_tensor_overhead() * max_nodes * 2 + ggml_graph_overhead_custom(max_nodes * 2, false) + (1u << 20), nullptr, true };
    ggml_context * c = g->gctx = ggml_init(ip);
    ggml_cgraph * gf = g->gf = ggml_new_graph_custom(c, max_nodes * 2, false);
    g->k_views.clear(); g->v_views.clear();

    g->inp_tokens = ggml_new_tensor_1d(c, GGML_TYPE_I32, n_tokens);
    ggml_set_input(g->inp_tokens);
    g->inp_pos = ggml_new_tensor_1d(c, GGML_TYPE_I32, n_tokens);
    ggml_set_input(g->inp_pos);
    const int64_t n_tok_pad = GGML_PAD(n_tokens, GGML_KQ_MASK_PAD);
    g->kq_mask = ggml_new_tensor_2d(c, GGML_TYPE_F32, n_kv, n_tok_pad);
    ggml_set_input(g->kq_mask);

    ggml_tensor * inpL = ggml_get_rows(c, g->tok_embd, g->inp_tokens);
    const float kq_scale = 1.0f / sqrtf((float) D);
    ggml_tensor * cur = nullptr;
    for (int il = 0; il < hp.n_layer; il++) {
        lgh_layer & L = g->L[il];
        ggml_tensor * inpSA = inpL;
        cur = ggml_rms_norm(c, inpL, hp.rms_eps);
        cur = ggml_mul(c, cur, L.attn_norm);
        ggml_tensor * Qcur = ggml_mul_mat(c, L.wq, cur);
        if (L.bq) Qcur = ggml_add(c, Qcur, L.bq);
        ggml_tensor * Kcur = ggml_mul_mat(c, L.wk, cur);
        if (L.bk) Kcur = ggml_add(c, Kcur, L.bk);
        ggml_tensor * Vcur = ggml_mul_mat(c, L.wv, cur);
        if (L.bv) Vcur = ggml_add(c, Vcur, L.bv);
        Qcur = ggml_rope_ext(c, ggml_reshape_3d(c, Qcur, D, H, n_tokens), g->inp_pos, g->rope_ff, (int) D, hp.rope_mode, hp.n_ctx_orig,
                             hp.rope_freq_base, hp.rope_freq_scale, 0.0f, 1.0f, 32.0f, 1.0f);
        Kcur = ggml_rope_ext(c, ggml_reshape_3d(c, Kcur, D, HK, n_tokens), g->inp_pos, g->rope_ff, (int) D, hp.rope_mode, hp.n_ctx_orig,
                             hp.rope_freq_base, hp.rope_freq_scale, 0.0f, 1.0f, 32.0f, 1.0f);
        {   // llm_build_kv_store, FA off: V cache transposed.  The views are created at kv_head = 0 and re-pointed before every compute.
            ggml_tensor * k_view = ggml_view_1d(c, L.k, n_tokens * EK, 0);
            ggml_tensor * k_cpy = ggml_cpy(c, Kcur, k_view);
            ggml_build_forward_expand(gf, k_cpy);
            ggml_tensor * v_view = ggml_view_2d(c, L.v, n_tokens, EK, n_ctx * ggml_element_size(L.v), 0);
            ggml_tensor * v_cpy = ggml_cpy(c, ggml_transpose(c, Vcur), v_view);
            ggml_build_forward_expand(gf, v_cpy);
            // the CPY node is itself a view of its destination (ggml_cpy_impl): both carry the offset
            g->k_views.push_back(k_view); g->k_views.push_back(k_cpy);
            g->v_views.push_back(v_view); g->v_views.push_back(v_cpy);
        }
        {   // llm_build_kqv, FA off
            ggml_tensor * q = ggml_permute(c, Qcur, 0, 2, 1, 3);
            ggml_tensor * k = ggml_view_3d(c, L.k, D, n_kv, HK, ggml_row_size(L.k->type, EK), ggml_row_size(L.k->type, D), 0);
            ggml_tensor * kq = ggml_mul_mat(c, k, q);
            if (hp.rope_mode == 2) ggml_mul_mat_set_prec(kq, GGML_PREC_F32);   // LLM_ARCH_QWEN2 (:10100-10104)
            kq = ggml_soft_max_ext(c, kq, g->kq_mask, kq_scale, 0.0f);
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
        {   // llm_build_ffn LLM_FFN_SILU / LLM_FFN_PAR
            ggml_tensor * tmp = ggml_mul_mat(c, L.up, cur);
            cur = ggml_mul_mat(c, L.gate, cur);
            cur = ggml_silu(c, cur);
            cur = ggml_mul(c, cur, tmp);
            cur = ggml_mul_mat(c, L.down, cur);
        }
        cur = ggml_add(c, cur, ffn_inp);
        inpL = cur;
    }
    g->l_out = cur;
    cur = ggml_rms_norm(c, cur, hp.rms_eps);
    cur = ggml_mul(c, cur, g->output_norm);
    cur = ggml_mul_mat(c, g->output, cur);
    ggml_set_output(cur);
    g->logits = cur;
    ggml_build_forward_expand(gf, cur);
    g->g_tokens = n_tokens; g->g_nkv = n_kv;
}

// worst-case reservation (llama_new_context_with_model: ggml_backend_sched_reserve on a graph of n_ubatch tokens over the whole
// cache).  ggml_gallocr_alloc_graph reuses the reserved buffer for every graph that fits it and grows it only for one that does not.
static bool reserve_compute_buffer(lgh_ctx * g) {
    if (!g->galloc) g->galloc = ggml_gallocr_new(ggml_backend_get_default_buffer_type(g->backend));
    build_graph(g, g->n_tokens_max, g->hp.n_ctx);
    const bool ok = ggml_gallocr_reserve(g->galloc, g->gf);
    ggml_free(g->gctx); g->gctx = nullptr; g->gf = nullptr;   // the next lgh_decode builds its own graph
    g->logits = g->l_out = nullptr;
    return ok;
}
// size the compute buffer for prompts of up to n_tokens_max tokens (the context's n_ubatch; 1 unless called)
int lgh_reserve(void * p, int n_tokens_max) {
    lgh_ctx * g = (lgh_ctx *) p;
    if (n_tokens_max < 1 || n_tokens_max > g->hp.n_ctx) return -1;
    g->n_tokens_max = n_tokens_max;
    return reserve_compute_buffer(g) ? 0 : -2;
}

// n_tokens tokens at positions pos0 .. pos0+n_tokens-1, HOST buffers in and out.  The tokens are stored from kv_head = pos0, or, once
// lgh_kv_seq_rm / lgh_kv_seq_add have been called since the last clear, in the first run of empty cells from the search head (a pending
// K-shift runs first).
// logits: [n_tokens][n_vocab] if all_logits, else [n_vocab] of the last token.  Returns 0 on success.
int lgh_decode(void * p, const int32_t * tokens, int n_tokens, int pos0, float * logits, int all_logits) {
    lgh_ctx * g = (lgh_ctx *) p;
    const lgh_hparams & hp = g->hp;
    if (n_tokens <= 0 || pos0 < 0 || pos0 + n_tokens > hp.n_ctx) return -1;
    const int64_t EK = (int64_t) hp.n_head_kv * hp.head_dim;
    if (!apply_k_shift(g)) return -2;   // llama_kv_cache_update before the slot search (src/llama.cpp:18433)
    // the destination cell of the first token: its position until the cells are managed, else the reference's slot search
    int cell0 = pos0;
    if (g->managed) {
        if (g->head > g->used + 2 * (uint32_t) n_tokens) g->head = 0;   // src/llama.cpp:18437-18440
        cell0 = find_slot(g, n_tokens);
        if (cell0 < 0) return -4;
    }
    for (int i = 0; i < n_tokens; i++) {
        lgh_ctx::cell & cl = g->cells[(size_t) (cell0 + i)];
        if (cl.pos < 0) g->used++;
        cl.pos = pos0 + i;
    }
    g->head = (uint32_t) (cell0 + n_tokens) >= g->cells.size() ? 0 : (uint32_t) (cell0 + n_tokens);   // :18578-18586
    // kv_self.n = min(size, max(pad, GGML_PAD(cell_max, pad))), pad = 32 when FA off (src/llama.cpp:4485, 18442-18451)
    int64_t cell_max = pos0 + n_tokens;
    if (g->managed) {
        cell_max = 0;
        for (int64_t i = (int64_t) g->cells.size(); i > 0; i--) if (g->cells[(size_t) (i - 1)].pos >= 0) { cell_max = i; break; }
    }
    int64_t n_kv = ((cell_max + 31) / 32) * 32;
    if (n_kv < 32) n_kv = 32;
    if (n_kv > hp.n_ctx) n_kv = hp.n_ctx;
    double t0 = now_s();
    if (!g->gf || g->g_tokens != n_tokens || g->g_nkv != n_kv) {
        if (!g->galloc && !reserve_compute_buffer(g)) return -3;
        build_graph(g, n_tokens, n_kv);
        if (!ggml_gallocr_alloc_graph(g->galloc, g->gf)) return -3;
        g->n_graph_builds++;
    }
    g->t_build += now_s() - t0; t0 = now_s();
    // re-point the cache store views at kv_head (what a rebuilt graph would carry in view_offs)
    for (size_t iv = 0; iv < g->k_views.size(); iv++) {
        ggml_tensor * kv = g->k_views[iv], * vv = g->v_views[iv];
        kv->view_offs = ggml_row_size(kv->type, EK) * (size_t) cell0;
        kv->data = (char *) kv->view_src->data + kv->view_offs;
        vv->view_offs = (size_t) cell0 * ggml_element_size(vv);
        vv->data = (char *) vv->view_src->data + vv->view_offs;
    }
    std::vector<int32_t> posv(n_tokens);
    for (int i = 0; i < n_tokens; i++) posv[i] = pos0 + i;
    const int64_t n_tok_pad = GGML_PAD(n_tokens, GGML_KQ_MASK_PAD);
    g->mask_host.resize((size_t) (n_kv * n_tok_pad));
    for (int64_t j = 0; j < n_tok_pad; j++)      // llama_set_inputs causal mask (src/llama.cpp:17330-17380): empty cells and later positions hidden
        for (int64_t i = 0; i < n_kv; i++) {
            const int32_t cp = g->managed ? g->cells[(size_t) i].pos : (int32_t) i;
            g->mask_host[(size_t) (j * n_kv + i)] = (j < n_tokens && cp >= 0 && cp <= pos0 + j) ? 0.0f : -INFINITY;
        }
    ggml_backend_tensor_set(g->inp_tokens, tokens, 0, sizeof(int32_t) * (size_t) n_tokens);
    ggml_backend_tensor_set(g->inp_pos, posv.data(), 0, sizeof(int32_t) * (size_t) n_tokens);
    ggml_backend_tensor_set(g->kq_mask, g->mask_host.data(), 0, sizeof(float) * g->mask_host.size());
    g->t_set += now_s() - t0; t0 = now_s();
    const ggml_status st = ggml_backend_graph_compute(g->backend, g->gf);
    if (st != GGML_STATUS_SUCCESS) return -2;
    g->t_enqueue += now_s() - t0; t0 = now_s();
    if (logits) {
        if (all_logits) ggml_backend_tensor_get(g->logits, logits, 0, sizeof(float) * (size_t) hp.n_vocab * (size_t) n_tokens);
        else ggml_backend_tensor_get(g->logits, logits, sizeof(float) * (size_t) hp.n_vocab * (size_t) (n_tokens - 1), sizeof(float) * (size_t) hp.n_vocab);
    } else {
        ggml_backend_synchronize(g->backend);
    }
    g->t_get += now_s() - t0;
    return 0;
}
// host seconds spent so far in {graph (re)build + allocation, input upload, graph_compute call, wait + logits read}; resets the counters
void lgh_phase_seconds(void * p, double * out4) {
    lgh_ctx * g = (lgh_ctx *) p;
    out4[0] = g->t_build; out4[1] = g->t_set; out4[2] = g->t_enqueue; out4[3] = g->t_get;
    g->t_build = g->t_set = g->t_enqueue = g->t_get = 0;
}

// last-layer output of the previous lgh_decode ([n_tokens][n_embd])
int lgh_get_hidden(void * p, float * out) {
    lgh_ctx * g = (lgh_ctx *) p;
    if (!g->l_out) return -1;
    ggml_backend_tensor_get(g->l_out, out, 0, ggml_nbytes(g->l_out));
    return 0;
}

}  // extern "C"
