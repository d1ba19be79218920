// prima.cpp_b200/csrc/engine.cu — the decode engine behind include/prima_b200.h: weights resident in HBM in raw GGUF
// block layout, one fused launch sequence per token (10 kernels per layer instead of the reference's ~30, SURVEY App. A),
// all PDL-chained and replayed as ONE CUDA graph per token; token id and position live in device memory so the graph
// never changes (the reference re-captures / patches cpy nodes, ggml-cuda.cu:2602-2617, 2741-2752).
//
// Graph restated: build_llama / build_qwen2 (src/llama.cpp:11000-11216, 12736-12916), FA off.
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/prima_b200.h"
#include "launch.h"

using namespace pb;

std::atomic<uint64_t> g_launches{0};

#define CK(expr)                                  \
    do {                                          \
        int _e = (int) (expr);                    \
        if (_e != 0) return _e;                   \
    } while (0)

static int dbg_sync(cudaStream_t st, const char * what) {
    static const bool on = getenv("PB200_DEBUG_SYNC") != nullptr;
    if (!on) return 0;
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing(st, &cs);
    if (cs != cudaStreamCaptureStatusNone) return 0;
    fprintf(stderr, "[pb200] launched %s ... ", what);
    fflush(stderr);
    cudaError_t e = cudaStreamSynchronize(st);
    fprintf(stderr, "%s\n", cudaGetErrorString(e));
    return (int) e;
}

namespace {

struct Tensor {
    void * data = nullptr;
    int type = -1;
    int64_t N = 0, K = 0;
    size_t bytes = 0;
};

struct Layer {
    float *attn_norm = nullptr, *ffn_norm = nullptr;
    Tensor wq, wk, wv, wo, gate, up, down;
    float *bq = nullptr, *bk = nullptr, *bv = nullptr;
};

struct ActBuf {
    ActQ q{};
    void * base = nullptr;
};

// Device scratch that only grows.  grow() waits for the stream before it frees the old block, which kernels in flight may still read,
// so it must not run during stream capture; the engine captures only in pb200_model_finalize, which grows nothing.
struct DevBuf {
    void * p = nullptr;
    size_t bytes = 0;
    DevBuf() = default;
    DevBuf(const DevBuf &) = delete;
    DevBuf & operator=(const DevBuf &) = delete;
    ~DevBuf() { if (p) cudaFree(p); }
    int grow(size_t need, cudaStream_t st) {
        if (need <= bytes) return 0;
        if (p) {
            CK(cudaStreamSynchronize(st));
            CK(cudaFree(p));
            p = nullptr;
            bytes = 0;
        }
        CK(cudaMalloc(&p, need));
        bytes = need;
        return 0;
    }
};

struct Penalty {                    // logit bias + penalties of one slot (pb200_penalties_set_seq)
    DevBuf state;                   // penalty_state_bytes(last_n, n_bias) device bytes
    int32_t last_n = 0;             // clamped to >= 0
    bool set = false;
};

// One sequence slot: an independent sequence with its own KV cache, token and position (the pipeline keeps one per stage in flight).
// The device words point into the model's per-slot arrays, whose layouts hosts see: pb200_token_device, pb200_sample_device and
// pb200_kv_device.
struct Slot {
    int32_t * tokpos = nullptr;         // {token, pos}, 16 bytes per slot
    int32_t * sample = nullptr;         // the slot's last sample (pb200_argmax_seq / pb200_sample_seq)
    uint8_t * rng = nullptr;            // mt19937 state of pb200_sample_seq (shards with the head)
    __half *k = nullptr, *v = nullptr;  // the slot's [layer][n_ctx][n_head_kv * head_dim] block of the K and V caches
    size_t layer_elems = 0;             // n_ctx * n_head_kv * head_dim
    pb200_sampling sampling{};          // valid where sampling_set
    bool sampling_set = false;
    Penalty pen;
    cudaGraphExec_t graph = nullptr;    // the captured step (NULL: direct launches)
    __half * kc(int layer) const { return k + layer * layer_elems; }   // layer: index within this shard
    __half * vc(int layer) const { return v + layer * layer_elems; }
};

}  // namespace

struct pb200_model {
    pb200_hparams hp{};
    int device = 0, l0 = 0, l1 = 0;
    bool with_embd = false, with_head = false, finalized = false, use_graph = true;
    cudaStream_t stream = nullptr;
    Tensor tok_embd, output;
    float *output_norm = nullptr, *rope_ff = nullptr;
    std::vector<Layer> layers;   // index il - l0
    __half *kcache = nullptr, *vcache = nullptr;   // [n_seq][layer][n_ctx][n_head_kv * head_dim] each
    size_t kv_bytes = 0;                           // of each
    float *x_in = nullptr, *x_a = nullptr, *x_b = nullptr, *q = nullptr, *k = nullptr, *v = nullptr, *att = nullptr, *g = nullptr, *u = nullptr,
          *xn = nullptr, *x_out = nullptr, *logits = nullptr;
    ActBuf actE, actQD, actF;
    unsigned int * gbar = nullptr;     // grid-barrier state of the distributed GEMV prologues (2 words, self-resetting)
    int32_t * tokpos_host = nullptr;   // pinned
    float * logits_host = nullptr;     // pinned
    RopeParams rp{};
    int n_seq = 1;
    std::vector<Slot> slots;           // [n_seq], from finalize on
    DevBuf pen_logits;                 // [n_vocab] the penalised row the chain reads (one for all slots: they share the stream)
    DevBuf pen_tok;                    // staging of pb200_sampler_accept_seq
    DevBuf head;                       // pb200_prompt_head(_kld): logits [n_rows][n_vocab] | that call's per-row data (head_rows)
    uint64_t launches_per_step = 0;
    int64_t weight_bytes = 0;
    std::vector<void *> allocs;
    bool profiling = false;
    struct Prefill {                   // prompt-processing scratch for up to T tokens: one block, grown on demand
        int T = 0;
        int rows = 0;                  // tokens of the last ubatch, whose hidden states x0 holds (0: no prefill yet)
        DevBuf mem;
        float *x0 = nullptr, *x1 = nullptr, *xn = nullptr, *q = nullptr, *k = nullptr, *v = nullptr, *att = nullptr, *g = nullptr, *u = nullptr;
        void * ws = nullptr;
        int32_t *tok = nullptr, *pos = nullptr;
    } pf;
    std::vector<cudaEvent_t> prof_ev;
    std::vector<int64_t> prof_bytes;
    size_t prof_n = 0;

    int alloc(void ** p, size_t bytes) {
        bytes = (bytes + 255) / 256 * 256;
        cudaError_t e = cudaMalloc(p, bytes);
        if (e != cudaSuccess) return (int) e;
        allocs.push_back(*p);
        return 0;
    }
};

// Argument checks of the entry points.  ready: a NULL or unfinalized model, or a shard without the head where the call needs the logits,
// returns `unready` (PB200_ESTATE; the host copies pb200_get_hidden / pb200_set_hidden / pb200_debug_read answer PB200_EINVAL); ready_seq
// then returns PB200_EINVAL for a seq outside [0, n_seq).  building: the calls that fill an unfinalized model.  Each makes the model's
// device current when its checks pass.
static int ready(pb200_model * m, bool head = false, int unready = PB200_ESTATE) {
    if (!m || !m->finalized || (head && !m->with_head)) return unready;
    cudaSetDevice(m->device);
    return 0;
}
static int ready_seq(pb200_model * m, int seq, bool head = false) {
    CK(ready(m, head));
    return seq < 0 || seq >= m->n_seq ? PB200_EINVAL : 0;
}
static int building(pb200_model * m) {
    if (!m) return PB200_EINVAL;
    if (m->finalized) return PB200_ESTATE;
    cudaSetDevice(m->device);
    return 0;
}
static bool tokpos_ok(const pb200_model * m, int32_t token, int32_t pos) {
    return pos >= 0 && pos < m->hp.n_ctx && token >= 0 && token < m->hp.n_vocab;
}

// ---------------------------------------------------------------------------------------------------------------
// synthetic raw blocks generated on the device (bench without a checkpoint): valid bit patterns, weight std ~ 1/sqrt(K)
__device__ __forceinline__ uint64_t splitmix(uint64_t & s) {
    uint64_t z = (s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
__device__ __forceinline__ float u01(uint64_t & s) { return (float) (splitmix(s) >> 40) * (1.0f / 16777216.0f); }

__global__ void k_synth_blocks(uint8_t * p, int type, int64_t nblocks, int64_t K, uint64_t seed) {
    const int64_t b = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nblocks) return;
    uint64_t s = seed * 0x100000001B3ull + (uint64_t) b * 0x9E3779B97F4A7C15ull;
    const float sc = rsqrtf((float) K);
    const int bytes = (int) row_bytes(type, block_elems(type));
    uint8_t * o = p + b * bytes;
    auto put16 = [&](int off, float v) { __half h = __float2half_rn(v); *reinterpret_cast<uint16_t *>(o + off) = __half_as_ushort(h); };
    auto fill = [&](int off, int n) {
        for (int i = 0; i < n; i += 2) { uint64_t r = splitmix(s); o[off + i] = (uint8_t) r; if (i + 1 < n) o[off + i + 1] = (uint8_t) (r >> 8); }
    };
    if (type == T_Q4_K || type == T_Q5_K) {
        const float qh = type == T_Q4_K ? 7.5f : 15.5f;
        const float d = (0.5f + u01(s)) * sc / (qh * 32.f);
        put16(0, d);
        put16(2, d * qh * (0.9f + 0.2f * u01(s)));
        fill(4, bytes - 4);
    } else if (type == T_Q6_K) {
        fill(0, 208);
        put16(208, (0.5f + u01(s)) * sc / (18.f * 64.f));
    } else if (type == T_Q8_0) {
        put16(0, (0.5f + u01(s)) * sc / 73.f);
        fill(2, 32);
    } else if (type == T_Q4_0 || type == T_Q5_0) {   // d (q - 8) / d (q - 16): symmetric around 0
        put16(0, (0.5f + u01(s)) * sc / (type == T_Q4_0 ? 4.5f : 9.f));
        fill(2, bytes - 2);
    } else if (type == T_Q4_1) {
        const float d = (0.5f + u01(s)) * sc / 4.5f;
        put16(0, d);
        put16(2, -d * 7.5f * (0.9f + 0.2f * u01(s)));
        fill(4, 16);
    } else {
        const float d = (0.5f + u01(s)) * sc / 9.f;
        put16(0, d);
        put16(2, -d * 15.5f * (0.9f + 0.2f * u01(s)));
        fill(4, 20);
    }
}
__global__ void k_set_tokpos(int32_t * tp, int32_t token, int32_t pos) { tp[0] = token; tp[1] = pos; }
__global__ void k_fill_f32(float * p, int64_t n, float base, float jitter, uint64_t seed) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t s = seed + (uint64_t) i * 0x9E3779B97F4A7C15ull;
    p[i] = base + jitter * (u01(s) - 0.5f);
}

// ---------------------------------------------------------------------------------------------------------------
static bool use_more_bits(int i_layer, int n_layers) {   // src/llama.cpp:19278-19280
    return i_layer < n_layers / 8 || i_layer >= 7 * n_layers / 8 || (i_layer - n_layers / 8) % 3 == 2;
}
static int fallback_type(int t, int64_t k) {   // src/llama.cpp:19516-19551
    if (!is_kquant(t) || k % 256 == 0) return t;
    if (t == T_Q4_K) return T_Q5_0;
    if (t == T_Q5_K) return T_Q5_1;
    return T_Q8_0;   // Q6_K
}

// Where a GGUF tensor name goes on this shard.
struct Found {
    enum Kind { UNKNOWN, SKIPPED, QUANT, F32 } kind = UNKNOWN;   // SKIPPED: another stage's tensor, or a per-layer one the engine does not use
    Tensor * t = nullptr;       // QUANT, with its N and K set
    float ** f32 = nullptr;     // F32: where the vector's device address is kept
    int64_t n = 0;              // F32: its length
};
static Found find_tensor(pb200_model * m, const std::string & name) {
    const pb200_hparams & hp = m->hp;
    const int64_t E = hp.n_embd, QD = (int64_t) hp.n_head * hp.head_dim, EK = (int64_t) hp.n_head_kv * hp.head_dim, F = hp.n_ff;
    auto quant = [](Tensor & t, int64_t N, int64_t K) { t.N = N; t.K = K; Found f; f.kind = Found::QUANT; f.t = &t; return f; };
    auto f32 = [](float *& p, int64_t n) { Found f; f.kind = Found::F32; f.f32 = &p; f.n = n; return f; };
    Found skipped;
    skipped.kind = Found::SKIPPED;
    if (name == "token_embd.weight") return m->with_embd ? quant(m->tok_embd, hp.n_vocab, E) : skipped;
    if (name == "output.weight") return m->with_head ? quant(m->output, hp.n_vocab, E) : skipped;
    if (name == "output_norm.weight") return m->with_head ? f32(m->output_norm, E) : skipped;
    if (name == "rope_freqs.weight") return f32(m->rope_ff, hp.head_dim / 2);
    if (name.rfind("blk.", 0) != 0) return Found{};
    int il = -1;
    char what[64] = {0};
    if (sscanf(name.c_str(), "blk.%d.%63s", &il, what) != 2 || il < m->l0 || il >= m->l1) return skipped;
    Layer & L = m->layers[il - m->l0];
    const std::string w(what);
    if (w == "attn_q.weight") return quant(L.wq, QD, E);
    if (w == "attn_k.weight") return quant(L.wk, EK, E);
    if (w == "attn_v.weight") return quant(L.wv, EK, E);
    if (w == "attn_output.weight") return quant(L.wo, E, QD);
    if (w == "ffn_gate.weight") return quant(L.gate, F, E);
    if (w == "ffn_up.weight") return quant(L.up, F, E);
    if (w == "ffn_down.weight") return quant(L.down, E, F);
    if (w == "attn_norm.weight") return f32(L.attn_norm, E);
    if (w == "ffn_norm.weight") return f32(L.ffn_norm, E);
    if (w == "attn_q.bias") return f32(L.bq, QD);
    if (w == "attn_k.bias") return f32(L.bk, EK);
    if (w == "attn_v.bias") return f32(L.bv, EK);
    return skipped;
}

extern "C" {

pb200_model * pb200_model_create(const pb200_hparams * hp, int device, int layer_begin, int layer_end, int with_embd, int with_head) {
    if (!hp || layer_begin < 0 || layer_end > hp->n_layer || layer_begin > layer_end) return nullptr;
    if (hp->n_head_kv <= 0 || hp->n_head <= 0 || hp->n_ff <= 0 || hp->n_vocab <= 0 || hp->n_ctx <= 0 || hp->n_embd <= 0) return nullptr;
    if (hp->head_dim != 128 || hp->n_head % hp->n_head_kv != 0 || hp->n_embd % 256 != 0) return nullptr;
    if (cudaSetDevice(device) != cudaSuccess) return nullptr;
    if (hp->n_ctx > attn_rows_max_kv()) return nullptr;   // the attention fallback keeps a whole score row in shared memory
    pb200_model * m = new pb200_model();
    m->hp = *hp;
    m->device = device;
    m->l0 = layer_begin;
    m->l1 = layer_end;
    m->with_embd = with_embd != 0;
    m->with_head = with_head != 0;
    m->layers.resize(layer_end - layer_begin);
    if (cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking) != cudaSuccess) { delete m; return nullptr; }
    return m;
}

void pb200_model_free(pb200_model * m) {
    if (!m) return;
    cudaSetDevice(m->device);
    cudaStreamSynchronize(m->stream);
    for (Slot & s : m->slots) if (s.graph) cudaGraphExecDestroy(s.graph);
    for (void * p : m->allocs) cudaFree(p);
    for (cudaEvent_t e : m->prof_ev) cudaEventDestroy(e);
    if (m->tokpos_host) cudaFreeHost(m->tokpos_host);
    if (m->logits_host) cudaFreeHost(m->logits_host);
    cudaStreamDestroy(m->stream);
    delete m;   // the grow-only buffers free themselves
}

// Reserves the device memory of one tensor of this shard and returns its address (NULL with rc 0: the tensor lives on another stage).
// The caller fills it (pb200_model_set_tensor: one synchronous copy; gguf.cu: pinned double-buffered stream from the file).
int pb200_model_tensor_alloc(pb200_model * m, const char * name, int type, size_t nbytes, void ** dev_ptr) {
    if (!m || !name || !dev_ptr) return PB200_EINVAL;
    *dev_ptr = nullptr;
    CK(building(m));
    const Found f = find_tensor(m, name);
    if (f.kind == Found::SKIPPED) return 0;
    if (f.kind == Found::UNKNOWN) return PB200_EINVAL;
    if (f.kind == Found::F32) {
        if (type != T_F32 || nbytes != (size_t) f.n * 4) return PB200_EINVAL;
        CK(m->alloc((void **) f.f32, nbytes));
        *dev_ptr = *f.f32;
        return 0;
    }
    Tensor & t = *f.t;
    if (!is_quant_type(type)) return PB200_ENOTSUP;
    if (t.K % block_elems(type) != 0) return PB200_EINVAL;
    const size_t need = (size_t) (row_bytes(type, t.K) * t.N);
    if (nbytes != need) return PB200_EINVAL;
    t.type = type;
    t.bytes = need;
    CK(m->alloc(&t.data, need + 16));
    *dev_ptr = t.data;
    return 0;
}

int pb200_model_set_tensor(pb200_model * m, const char * name, int type, const void * host_data, size_t nbytes) {
    if (!host_data) return PB200_EINVAL;
    void * dev = nullptr;
    const int rc = pb200_model_tensor_alloc(m, name, type, nbytes, &dev);
    if (rc || !dev) return rc;
    return (int) cudaMemcpy(dev, host_data, nbytes, cudaMemcpyHostToDevice);
}

int pb200_model_synth(pb200_model * m, int ftype, uint64_t seed) {
    CK(building(m));
    const pb200_hparams & hp = m->hp;
    const int def = ftype == 0 ? T_Q4_K : ftype == 2 ? T_Q4_0 : T_Q5_K;
    const bool kq = ftype != 2;   // Q4_0 (no imatrix): every matrix and the embedding Q4_0, only the head Q6_K (src/llama.cpp:19296-19460)
    const bool is70b = hp.n_layer == 80;   // MODEL_70B (src/llama.cpp:19385-19390)
    uint64_t sd = seed;
    auto synth = [&](Tensor & t, int type, int64_t N, int64_t K) -> int {
        type = fallback_type(type, K);
        if (type < 0) return PB200_ENOTSUP;
        t.type = type; t.N = N; t.K = K;
        t.bytes = (size_t) (row_bytes(type, K) * N);
        CK(m->alloc(&t.data, t.bytes + 16));
        const int64_t nb = N * K / block_elems(type);
        k_synth_blocks<<<(unsigned) ((nb + 255) / 256), 256, 0, m->stream>>>((uint8_t *) t.data, type, nb, K, ++sd);
        return (int) cudaGetLastError();
    };
    auto fvec = [&](float ** p, int64_t n, float base, float jit) -> int {
        CK(m->alloc((void **) p, (size_t) n * 4));
        k_fill_f32<<<(unsigned) ((n + 255) / 256), 256, 0, m->stream>>>(*p, n, base, jit, ++sd);
        return (int) cudaGetLastError();
    };
    const int64_t E = hp.n_embd, QD = (int64_t) hp.n_head * hp.head_dim, EK = (int64_t) hp.n_head_kv * hp.head_dim, F = hp.n_ff;
    if (m->with_embd) CK(synth(m->tok_embd, def, hp.n_vocab, E));
    if (m->with_head) { CK(synth(m->output, T_Q6_K, hp.n_vocab, E)); CK(fvec(&m->output_norm, E, 1.0f, 0.04f)); }
    for (int il = m->l0; il < m->l1; il++) {
        Layer & L = m->layers[il - m->l0];
        const bool more = use_more_bits(il, hp.n_layer);
        int tv = more && kq ? T_Q6_K : def;
        if (is70b && tv == T_Q4_K) tv = T_Q5_K;
        const int td = more && kq ? T_Q6_K : def;
        CK(fvec(&L.attn_norm, E, 1.0f, 0.04f));
        CK(fvec(&L.ffn_norm, E, 1.0f, 0.04f));
        CK(synth(L.wq, def, QD, E));
        CK(synth(L.wk, def, EK, E));
        CK(synth(L.wv, tv, EK, E));
        CK(synth(L.wo, def, E, QD));
        CK(synth(L.gate, def, F, E));
        CK(synth(L.up, def, F, E));
        CK(synth(L.down, td, E, F));
        if (hp.rope_mode == 2) {   // qwen2 carries q/k/v biases (build_qwen2 :12815-12832)
            CK(fvec(&L.bq, QD, 0.0f, 0.02f));
            CK(fvec(&L.bk, EK, 0.0f, 0.02f));
            CK(fvec(&L.bv, EK, 0.0f, 0.02f));
        }
    }
    return (int) cudaStreamSynchronize(m->stream);
}

// profile pass: CUDA events around every GEMV group (direct launches, no graph) -> per-group durations for the roofline.  The start
// event is handed to launch_gemv, which records it after any producer kernel, right in front of the GEMV kernels.
static int prof_begin(pb200_model * m, int64_t bytes, cudaEvent_t & start) {
    start = nullptr;
    if (!m->profiling) return 0;
    if (m->prof_ev.size() < 2 * (m->prof_n + 1)) {
        cudaEvent_t a, b;
        CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
        m->prof_ev.push_back(a); m->prof_ev.push_back(b);
        m->prof_bytes.push_back(0);
    }
    m->prof_bytes[m->prof_n] = bytes;
    start = m->prof_ev[2 * m->prof_n];
    return 0;
}
static int prof_end(pb200_model * m) {
    if (!m->profiling) return 0;
    int e = (int) cudaEventRecord(m->prof_ev[2 * m->prof_n + 1], m->stream);
    m->prof_n++;
    return e;
}
static int64_t tbytes(const Tensor & t) { return (int64_t) t.bytes; }

// one decode step enqueued on m->stream (captured into the CUDA graph by finalize); every kernel is PDL-chained to the previous one
static int enqueue_step(pb200_model * m, int seq, uint64_t * nlaunch) {
    const pb200_hparams & hp = m->hp;
    const int E = hp.n_embd, H = hp.n_head, HK = hp.n_head_kv, D = hp.head_dim, F = hp.n_ff;
    const int QD = H * D, EK = HK * D;
    cudaStream_t st = m->stream;
    uint64_t n = 0;
    cudaEvent_t ev = nullptr;   // profiling: start event of the next GEMV group
    // one GEMV group between its profiling events
    auto gemv = [&](const GemvDesc * d, int nmat, int K, const ActQ & act, const GemvPrologue & pro, int64_t bytes, bool pdl, const char * what) -> int {
        CK(prof_begin(m, bytes, ev));
        CK(launch_gemv(d, nmat, K, act, pro, st, pdl, n, ev)); CK(dbg_sync(st, what));
        return prof_end(m);
    };
    const Slot & s = m->slots[seq];
    const int32_t * tok_dev = s.tokpos, * pos_dev = s.tokpos + 1;
    float * x = m->x_in;
    if (m->with_embd) {
        CK(launch_get_rows(m->tok_embd.data, m->tok_embd.type, E, tok_dev, 1, m->x_a, st, true)); n++; CK(dbg_sync(st, "get_rows"));
        x = m->x_a;
    }
    const float kq_scale = 1.0f / sqrtf((float) D);
    // three rotating hidden-state buffers so that a residual source is never overwritten by its consumer
    float * bufs[3] = {m->x_a, m->x_b, m->xn};
    for (int il = m->l0; il < m->l1; il++) {
        const int li = il - m->l0;
        Layer & L = m->layers[li];
        float * x1 = nullptr, * x2 = nullptr;
        for (int i = 0; i < 3 && (!x1 || !x2); i++)
            if (bufs[i] != x) { if (!x1) x1 = bufs[i]; else x2 = bufs[i]; }
        if (il + 1 == m->l1) x2 = m->x_out;   // the last layer writes hidden_out in place (a copy node would break the PDL chain)
        // --- attention block ---
        const GemvDesc qkv[3] = {{L.wq.data, m->q, L.bq, nullptr, L.wq.type, QD},
                                 {L.wk.data, m->k, L.bk, nullptr, L.wk.type, EK},
                                 {L.wv.data, m->v, L.bv, nullptr, L.wv.type, EK}};
        CK(gemv(qkv, 3, E, m->actE.q, GemvPrologue{PRO_RMSNORM, x, L.attn_norm, hp.rms_eps, m->gbar, m->g},   // g: scratch
                tbytes(L.wq) + tbytes(L.wk) + tbytes(L.wv), true, "gemv qkv"));
        bool att_quantized = false;   // the attention kernel also wrote wo's activation
        CK(launch_attn_step(m->q, m->k, m->v, s.kc(li), s.vc(li), m->att, m->actQD.q, act_mode_for(L.wo.type), H, HK, D, pos_dev, hp.n_ctx, m->rp,
                            m->rope_ff, kq_scale, st, true, att_quantized)); n++; CK(dbg_sync(st, "attn"));
        const GemvDesc wo = {L.wo.data, x1, nullptr, x, L.wo.type, E};   // ffn_inp = wo.att + inpSA
        CK(gemv(&wo, 1, QD, m->actQD.q, att_quantized ? GemvPrologue{} : GemvPrologue{PRO_QUANTIZE, m->att}, tbytes(L.wo), true, "gemv wo"));
        // --- FFN block ---
        const GemvDesc gu[2] = {{L.gate.data, m->g, nullptr, nullptr, L.gate.type, F}, {L.up.data, m->u, nullptr, nullptr, L.up.type, F}};
        CK(gemv(gu, 2, E, m->actE.q, GemvPrologue{PRO_RMSNORM, x1, L.ffn_norm, hp.rms_eps, m->gbar, m->att},   // att: scratch
                tbytes(L.gate) + tbytes(L.up), true, "gemv gate|up"));
        const GemvDesc down = {L.down.data, x2, nullptr, x1, L.down.type, E};   // l_out = down.act + ffn_inp
        CK(gemv(&down, 1, F, m->actF.q, GemvPrologue{PRO_SILU_MUL, m->g, m->u, 0.f, m->gbar}, tbytes(L.down), true, "gemv down"));
        x = x2;
    }
    // hidden_out has a stable address for the next pipeline stage / tests (a stage without layers forwards its input)
    if (x != m->x_out) { CK(cudaMemcpyAsync(m->x_out, x, (size_t) E * 4, cudaMemcpyDeviceToDevice, st)); }
    if (m->with_head) {
        const GemvDesc head = {m->output.data, m->logits, nullptr, nullptr, m->output.type, hp.n_vocab};
        const bool head_pdl = m->l1 > m->l0;   // a stage without layers starts with a copy node: no programmatic edge
        CK(gemv(&head, 1, E, m->actE.q, GemvPrologue{PRO_RMSNORM, m->x_out, m->output_norm, hp.rms_eps, m->gbar}, tbytes(m->output), head_pdl,
                "gemv head"));
    }
    if (nlaunch) *nlaunch = n;
    return 0;
}

int pb200_model_finalize(pb200_model * m) {
    if (!m) return PB200_EINVAL;
    if (m->finalized) return 0;
    cudaSetDevice(m->device);
    const pb200_hparams & hp = m->hp;
    const int64_t E = hp.n_embd, QD = (int64_t) hp.n_head * hp.head_dim, EK = (int64_t) hp.n_head_kv * hp.head_dim, F = hp.n_ff;
    // completeness + algorithmic bytes
    int64_t wb = 0;
    auto need = [&](const Tensor & t) { if (!t.data) return false; wb += (int64_t) t.bytes; return true; };
    for (Layer & L : m->layers) {
        if (!L.attn_norm || !L.ffn_norm) return PB200_ESTATE;
        if (!need(L.wq) || !need(L.wk) || !need(L.wv) || !need(L.wo) || !need(L.gate) || !need(L.up) || !need(L.down)) return PB200_ESTATE;
        wb += 2 * E * 4;
        if (L.bq) wb += (QD + 2 * EK) * 4;
    }
    if (m->with_embd && !m->tok_embd.data) return PB200_ESTATE;
    if (m->with_head) {
        if (!m->output_norm || !need(m->output)) return PB200_ESTATE;
        wb += E * 4;
    }
    m->weight_bytes = wb;
    const size_t nl = m->layers.size(), layer_elems = (size_t) hp.n_ctx * EK;
    m->kv_bytes = (size_t) m->n_seq * nl * layer_elems * sizeof(__half);
    if (nl) {
        CK(m->alloc((void **) &m->kcache, m->kv_bytes));
        CK(m->alloc((void **) &m->vcache, m->kv_bytes));
        CK(cudaMemset(m->kcache, 0, m->kv_bytes));
        CK(cudaMemset(m->vcache, 0, m->kv_bytes));
    }
    const int64_t big = std::max<int64_t>(std::max<int64_t>(F, QD), E);
    CK(m->alloc((void **) &m->x_in, E * 4));
    CK(m->alloc((void **) &m->x_a, E * 4));
    CK(m->alloc((void **) &m->x_b, E * 4));
    CK(m->alloc((void **) &m->xn, E * 4));
    CK(m->alloc((void **) &m->x_out, E * 4));
    CK(m->alloc((void **) &m->q, QD * 4));
    CK(m->alloc((void **) &m->k, EK * 4));
    CK(m->alloc((void **) &m->v, EK * 4));
    CK(m->alloc((void **) &m->att, big * 4));
    CK(m->alloc((void **) &m->g, big * 4));
    CK(m->alloc((void **) &m->u, big * 4));
    if (m->with_head) CK(m->alloc((void **) &m->logits, (size_t) hp.n_vocab * 4));
    auto mk = [&](ActBuf & a, int64_t K) -> int {
        CK(m->alloc(&a.base, act_ws_bytes(K)));
        CK(cudaMemset(a.base, 0, act_ws_bytes(K)));
        a.q = act_from_ws(a.base, K);
        return 0;
    };
    CK(mk(m->actE, E));
    CK(mk(m->actQD, QD));
    CK(mk(m->actF, F));
    CK(m->alloc((void **) &m->gbar, 16));
    CK(cudaMemset(m->gbar, 0, 16));
    int32_t * tokpos = nullptr, * sample = nullptr;
    uint8_t * rng = nullptr;
    CK(m->alloc((void **) &tokpos, 16 * (size_t) m->n_seq));
    CK(cudaMemset(tokpos, 0, 16 * (size_t) m->n_seq));
    CK(m->alloc((void **) &sample, 4 * (size_t) m->n_seq));
    CK(cudaMemset(sample, 0, 4 * (size_t) m->n_seq));
    if (m->with_head) CK(m->alloc((void **) &rng, sampler_state_bytes() * (size_t) m->n_seq));
    m->slots = std::vector<Slot>((size_t) m->n_seq);
    for (int sq = 0; sq < m->n_seq; sq++) {
        Slot & s = m->slots[sq];
        s.tokpos = tokpos + 4 * sq;
        s.sample = sample + sq;
        s.rng = rng ? rng + sampler_state_bytes() * (size_t) sq : nullptr;
        s.k = m->kcache + (size_t) sq * nl * layer_elems;
        s.v = m->vcache + (size_t) sq * nl * layer_elems;
        s.layer_elems = layer_elems;
    }
    CK(cudaMallocHost((void **) &m->tokpos_host, 16));
    if (m->with_head) CK(cudaMallocHost((void **) &m->logits_host, (size_t) hp.n_vocab * 4));
    rope_params_init(m->rp, hp.head_dim, hp.rope_mode, hp.n_ctx_orig, hp.rope_freq_base, hp.rope_freq_scale, 0.0f, 1.0f, 32.0f, 1.0f);
    CK(cudaDeviceSynchronize());

    // warm-up (sets kernel attributes outside of capture), then capture the whole token as one graph per sequence slot
    CK(enqueue_step(m, 0, &m->launches_per_step));
    CK(cudaStreamSynchronize(m->stream));
    if (nl) { CK(cudaMemset(m->kcache, 0, m->kv_bytes)); CK(cudaMemset(m->vcache, 0, m->kv_bytes)); }
    for (int sq = 0; sq < m->n_seq; sq++) {
        Slot & s = m->slots[sq];
        cudaGraph_t graph = nullptr;
        cudaError_t e = cudaStreamBeginCapture(m->stream, cudaStreamCaptureModeThreadLocal);
        if (e != cudaSuccess) break;
        int rc = enqueue_step(m, sq, nullptr);
        e = cudaStreamEndCapture(m->stream, &graph);
        if (rc == 0 && e == cudaSuccess && graph) {
            e = cudaGraphInstantiate(&s.graph, graph, 0);
            if (e != cudaSuccess) s.graph = nullptr;
        }
        if (graph) cudaGraphDestroy(graph);
    }
    cudaGetLastError();   // a failed capture must not poison later calls: fall back to direct launches
    m->finalized = true;
    return 0;
}

int64_t pb200_model_weight_bytes(const pb200_model * m) { return m ? m->weight_bytes : 0; }

int pb200_model_tensor_device(pb200_model * m, const char * name, const void ** dev_ptr, size_t * nbytes, int * type) {
    if (!m || !name || !dev_ptr || !nbytes) return PB200_EINVAL;
    const Found f = find_tensor(m, name);
    if (f.kind == Found::F32 && *f.f32) {
        *dev_ptr = *f.f32; *nbytes = (size_t) f.n * 4;
        if (type) *type = T_F32;
        return 0;
    }
    if (f.kind == Found::QUANT && f.t->data) {
        *dev_ptr = f.t->data; *nbytes = f.t->bytes;
        if (type) *type = f.t->type;
        return 0;
    }
    return PB200_ESTATE;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------
// Prompt processing: all T tokens through every layer as one batch.  Same graph as enqueue_step (build_llama / build_qwen2,
// src/llama.cpp:11000-11216, 12736-12916) with ne11 = T: the mat-muls run on the tensor cores (mmq.cu), attention is the
// decode kernel over a (head, token) grid reading the K/V rows just written to the cache (causal: token t sees rows <= pos_t).
static int pf_reserve(pb200_model * m, int T) {
    pb200_model::Prefill & P = m->pf;
    if (T <= P.T) return 0;
    const pb200_hparams & hp = m->hp;
    const size_t E = hp.n_embd, QD = (size_t) hp.n_head * hp.head_dim, EK = (size_t) hp.n_head_kv * hp.head_dim, F = hp.n_ff;
    void ** part[] = {(void **) &P.x0, (void **) &P.x1, (void **) &P.xn, (void **) &P.q, (void **) &P.k, (void **) &P.v, (void **) &P.att,
                      (void **) &P.g, (void **) &P.u, &P.ws, (void **) &P.tok, (void **) &P.pos};
    const size_t bytes[] = {T * E * 4, T * E * 4, T * std::max(E, QD) * 4, T * QD * 4, T * EK * 4, T * EK * 4, T * QD * 4, T * F * 4, T * F * 4,
                            mmq_workspace_bytes((int64_t) std::max(std::max(E, QD), F), T) + 256, (size_t) T * 4, (size_t) T * 4};
    auto padded = [](size_t b) { return (b + 255) / 256 * 256; };
    size_t total = 0;
    for (size_t b : bytes) total += padded(b);
    P.T = 0;
    CK(P.mem.grow(total, m->stream));
    char * p = (char *) P.mem.p;
    for (int i = 0; i < 12; i++) { *part[i] = p; p += padded(bytes[i]); }
    P.T = T;
    return 0;
}

// y[t][:] = W . x[t][:] (+ bias): tensor-core path when the type / K allow it, otherwise the decode GEMV row by row
// same_x_as: the matrix of the previous pf_matmul call when it read the same x (q -> k -> v, gate -> up): its tiled fp16 activation image
// in the workspace is reused if both went down the tensor-core path with the same activation format
static bool pf_tc(const Tensor & W, int T) { return mmq_supported(W.type, W.K) && T >= 8; }
static int pf_matmul(pb200_model * m, const Tensor & W, const float * x, int T, float * y, const float * bias, const float * resid, uint64_t & n,
                     const Tensor * same_x_as = nullptr, const MmqPre * pre = nullptr) {
    cudaStream_t st = m->stream;
    if (pf_tc(W, T)) {
        const bool reuse = same_x_as && pf_tc(*same_x_as, T) && same_x_as->K == W.K && is_kquant(same_x_as->type) == is_kquant(W.type);
        n += reuse ? 1 : 2;
        return (int) launch_mmq(W.type, W.data, W.N, W.K, x, W.K, T, y, bias, resid, m->pf.ws, st, reuse, reuse ? nullptr : pre);
    }
    if (pre) return (int) cudaErrorInvalidValue;   // callers fuse a producer only when pf_tc(W, T) && is_kquant(W.type)
    ActQ act = act_from_ws(m->actF.base, W.K);
    for (int t = 0; t < T; t++) {
        GemvDesc d1 = {W.data, y + (size_t) t * W.N, bias, resid ? resid + (size_t) t * W.N : nullptr, W.type, (int) W.N};
        CK(launch_gemv(&d1, 1, (int) W.K, act, GemvPrologue{PRO_QUANTIZE, x + (size_t) t * W.K}, st, false, n));
    }
    return 0;
}

__global__ void k_iota_pos(int32_t * pos, int pos0, int T) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < T) pos[i] = pos0 + i;
}

static int prefill_ubatch(pb200_model * m, int seq, const int32_t * tokens_host, const float * hidden_in_dev, int32_t T, int32_t pos0, float * logits_host,
                          bool sync);
static const int PB200_N_UBATCH = 512;   // the reference's default n_ubatch (common/common.h): longer prompts go through in slices

extern "C" int pb200_prefill_seq(pb200_model * m, int seq, const int32_t * tokens_host, int32_t T, int32_t pos0, float * logits_host) {
    CK(ready_seq(m, seq));
    if (!tokens_host || T <= 0 || pos0 < 0 || pos0 + T > m->hp.n_ctx) return PB200_EINVAL;
    if (!m->with_embd || m->l0 != 0) return PB200_ENOTSUP;   // whole prompts start at the embedding; pipeline shards: pb200_prefill_stage
    for (int32_t done = 0; done < T; done += PB200_N_UBATCH) {
        const int32_t n = std::min<int32_t>(PB200_N_UBATCH, T - done);
        const int rc = prefill_ubatch(m, seq, tokens_host + done, nullptr, n, pos0 + done, done + n == T ? logits_host : nullptr, true);
        if (rc) return rc;
    }
    return 0;
}
extern "C" int pb200_prefill(pb200_model * m, const int32_t * tokens_host, int32_t T, int32_t pos0, float * logits_host) {
    return pb200_prefill_seq(m, 0, tokens_host, T, pos0, logits_host);
}
// One ubatch (<= 512 tokens) through THIS shard's layers: prima's layer windows during prompt processing (src/llama.cpp:17825-18029: every
// rank runs its window of the sub-graph on the ubatch and ships the hidden states on).  The first stage takes token ids, the others the
// previous stage's hidden states [n_tokens][n_embd] f32 in device memory (left untouched); the result stays in pb200_prefill_hidden_device.
extern "C" int pb200_prefill_stage_seq(pb200_model * m, int seq, const int32_t * tokens_host, const float * hidden_in_dev, int32_t T, int32_t pos0,
                                       float * logits_host, int32_t synchronize) {
    CK(ready_seq(m, seq));
    if (T <= 0 || T > PB200_N_UBATCH || pos0 < 0 || pos0 + T > m->hp.n_ctx) return PB200_EINVAL;
    if (m->with_embd ? !tokens_host : !hidden_in_dev) return PB200_EINVAL;
    if (logits_host && !synchronize) return PB200_EINVAL;   // host logits are read back at the synchronisation point
    return prefill_ubatch(m, seq, tokens_host, hidden_in_dev, T, pos0, logits_host, synchronize != 0);
}
extern "C" int pb200_prefill_stage(pb200_model * m, const int32_t * tokens_host, const float * hidden_in_dev, int32_t T, int32_t pos0, float * logits_host,
                                   int32_t synchronize) {
    return pb200_prefill_stage_seq(m, 0, tokens_host, hidden_in_dev, T, pos0, logits_host, synchronize);
}
extern "C" float * pb200_prefill_hidden_device(pb200_model * m) { return (m && m->finalized) ? m->pf.x0 : nullptr; }

// Rows [row0, row0 + n_rows) of the last ubatch: PB200_EINVAL when there is no prefill yet or the range leaves it.
static int head_range(const pb200_model * m, int32_t row0, int32_t n_rows) {
    const int rows = m->pf.rows;
    return rows == 0 || row0 < 0 || n_rows <= 0 || row0 > rows - n_rows ? PB200_EINVAL : 0;
}

static size_t round256(size_t b) { return (b + 255) / 256 * 256; }

// The head over rows [row0, row0 + n_rows) of the last ubatch (the reference's inp_out_ids rows, src/llama.cpp:11120-11125): output_norm
// rides in the tensor-core mat-mul's activation pass like q|k|v's attn_norm, or runs first where pf_matmul takes a fallback.  Reads x0,
// writes only the head buffer and the prefill scratch (xn, ws, actF), which every prefill and decode rewrites before reading.  The head
// buffer grows to the logits [n_rows][n_vocab] (256-byte rounded) and `extra` bytes after them, for the caller's per-row data; lg and ex
// point at both.  Enqueued on the model stream; n counts the launches.  The caller has checked the model and the rows.
static int head_rows(pb200_model * m, int32_t row0, int32_t n_rows, size_t extra, float *& lg, char *& ex, uint64_t & n) {
    pb200_model::Prefill & P = m->pf;
    const pb200_hparams & hp = m->hp;
    const int E = hp.n_embd;
    const size_t lg_bytes = round256((size_t) n_rows * hp.n_vocab * 4);
    CK(m->head.grow(lg_bytes + extra, m->stream));
    lg = (float *) m->head.p;
    ex = (char *) m->head.p + lg_bytes;
    const float * x = P.x0 + (size_t) row0 * E;
    const bool fused = pf_tc(m->output, n_rows) && is_kquant(m->output.type);
    const MmqPre output_norm{PRO_RMSNORM, m->output_norm, 0, hp.rms_eps};
    if (!fused) { CK(launch_rms_norm(x, P.xn, E, n_rows, hp.rms_eps, m->stream, m->output_norm)); n++; }
    return pf_matmul(m, m->output, fused ? x : P.xn, n_rows, lg, nullptr, nullptr, n, nullptr, fused ? &output_norm : nullptr);
}

extern "C" int pb200_prompt_head(pb200_model * m, int32_t row0, int32_t n_rows, const int32_t * targets_host, float * logits_host,
                                 pb200_token_score * scores_host) {
    CK(ready(m, true));
    CK(head_range(m, row0, n_rows));
    if ((!logits_host && !scores_host) || (scores_host && !targets_host)) return PB200_EINVAL;
    const int V = m->hp.n_vocab;
    if (targets_host)
        for (int32_t i = 0; i < n_rows; i++)
            if (targets_host[i] >= V) return PB200_EINVAL;
    cudaStream_t st = m->stream;
    const size_t tg_bytes = round256((size_t) n_rows * 4);
    float * lg;
    char * ex;
    uint64_t n = 0;
    CK(head_rows(m, row0, n_rows, tg_bytes + (size_t) n_rows * sizeof(pb200_token_score), lg, ex, n));
    int32_t * tg = (int32_t *) ex;
    pb200_token_score * sc = (pb200_token_score *) (ex + tg_bytes);
    if (targets_host) {
        // from pageable memory the copy returns once the ids are staged; stream order keeps them until the scores have read them
        CK(cudaMemcpyAsync(tg, targets_host, (size_t) n_rows * 4, cudaMemcpyHostToDevice, st));
        CK(launch_token_scores(lg, n_rows, V, tg, sc, st)); n++;
    }
    g_launches += n;
    if (logits_host) CK(cudaMemcpyAsync(logits_host, lg, (size_t) n_rows * V * 4, cudaMemcpyDeviceToHost, st));
    if (scores_host) CK(cudaMemcpyAsync(scores_host, sc, (size_t) n_rows * sizeof(pb200_token_score), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return check_clear_abort() ? PB200_EABORTED : 0;   // a kernel's wait watchdog gave up: these rows are invalid (flag re-armed)
}

// The same rows' u16 log-probability records (llama-perplexity --kl-divergence-base) and / or their KL-divergence against base records
// (--kl-divergence), from one head computation.  Only the records and the per-row results cross PCIe.
extern "C" int pb200_prompt_head_kld(pb200_model * m, int32_t row0, int32_t n_rows, const int32_t * targets_host, uint16_t * records_host,
                                     float * nll_host, const uint16_t * base_host, pb200_kld_score * kld_host) {
    CK(ready(m, true));
    CK(head_range(m, row0, n_rows));
    if ((!records_host && !kld_host) || (nll_host && !records_host) || (!base_host != !kld_host) || !targets_host) return PB200_EINVAL;
    const int V = m->hp.n_vocab;
    for (int32_t i = 0; i < n_rows; i++)
        if (targets_host[i] < 0 || targets_host[i] >= V) return PB200_EINVAL;
    cudaStream_t st = m->stream;
    const size_t rec_bytes = (size_t) n_rows * pb200_logprob_record_u16s(V) * 2;
    // after the logits: targets | the records written | the base records read | nll | KLD scores, each 256-byte aligned
    const size_t tg_b = round256((size_t) n_rows * 4), rec_b = records_host ? round256(rec_bytes) : 0, base_b = base_host ? round256(rec_bytes) : 0,
                 nll_b = nll_host ? round256((size_t) n_rows * 4) : 0, kld_b = kld_host ? (size_t) n_rows * sizeof(pb200_kld_score) : 0;
    float * lg;
    char * ex;
    uint64_t n = 0;
    CK(head_rows(m, row0, n_rows, tg_b + rec_b + base_b + nll_b + kld_b, lg, ex, n));
    int32_t * tg = (int32_t *) ex;
    uint16_t * rec = (uint16_t *) (ex + tg_b);
    uint16_t * base = (uint16_t *) (ex + tg_b + rec_b);
    float * nll = nll_host ? (float *) (ex + tg_b + rec_b + base_b) : nullptr;
    pb200_kld_score * kld = (pb200_kld_score *) (ex + tg_b + rec_b + base_b + nll_b);
    // from pageable memory the copies return once staged; stream order keeps them until the kernels have read them
    CK(cudaMemcpyAsync(tg, targets_host, (size_t) n_rows * 4, cudaMemcpyHostToDevice, st));
    if (base_host) CK(cudaMemcpyAsync(base, base_host, rec_bytes, cudaMemcpyHostToDevice, st));
    if (records_host) { CK(launch_logprobs_u16(lg, n_rows, V, tg, rec, nll, st)); n++; }
    if (kld_host) { CK(launch_kld_scores(lg, n_rows, V, base, tg, kld, st)); n++; }
    g_launches += n;
    if (records_host) CK(cudaMemcpyAsync(records_host, rec, rec_bytes, cudaMemcpyDeviceToHost, st));
    if (nll_host) CK(cudaMemcpyAsync(nll_host, nll, (size_t) n_rows * 4, cudaMemcpyDeviceToHost, st));
    if (kld_host) CK(cudaMemcpyAsync(kld_host, kld, (size_t) n_rows * sizeof(pb200_kld_score), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return check_clear_abort() ? PB200_EABORTED : 0;
}

// the callers have checked the model, seq, T, pos0 and which input is given; the prompt's K/V rows go to slot seq.  The scratch, x_out and
// the logits are shared by all slots: every call is ordered on the model stream.
static int prefill_ubatch(pb200_model * m, int seq, const int32_t * tokens_host, const float * hidden_in_dev, int32_t T, int32_t pos0, float * logits_host,
                          bool sync) {
    if (m->with_embd)
        for (int t = 0; t < T; t++)
            if (tokens_host[t] < 0 || tokens_host[t] >= m->hp.n_vocab) return PB200_EINVAL;
    CK(pf_reserve(m, T));
    pb200_model::Prefill & P = m->pf;
    const Slot & s = m->slots[seq];
    const pb200_hparams & hp = m->hp;
    const int E = hp.n_embd, H = hp.n_head, HK = hp.n_head_kv, D = hp.head_dim, F = hp.n_ff;
    const int QD = H * D, EK = HK * D;
    cudaStream_t st = m->stream;
    uint64_t n = 0;
    k_iota_pos<<<(T + 255) / 256, 256, 0, st>>>(P.pos, pos0, T); n++;
    CK(cudaGetLastError());
    if (m->with_embd) {
        CK(cudaMemcpyAsync(P.tok, tokens_host, (size_t) T * 4, cudaMemcpyHostToDevice, st));
        CK(launch_get_rows(m->tok_embd.data, m->tok_embd.type, E, P.tok, T, P.x0, st, false)); n++;
    } else {
        CK(cudaMemcpyAsync(P.x0, hidden_in_dev, (size_t) T * E * 4, cudaMemcpyDeviceToDevice, st));   // the layers update the residual stream in place
    }
    const float kq_scale = 1.0f / sqrtf((float) D);
    float * x = P.x0, * y = P.x1;
    for (int il = m->l0; il < m->l1; il++) {
        const int li = il - m->l0;
        Layer & L = m->layers[li];
        __half * kc = s.kc(li), * vc = s.vc(li);
        // Each block's producer (rms_norm * norm weight, silu(g) * u) rides in the activation pass of the block's first mat-mul when the
        // block takes the tensor-core path with k-quants (later mat-muls reuse its image); otherwise a kernel runs it first.
        // --- attention block ---
        const bool qkv_fused = pf_tc(L.wq, T) && pf_tc(L.wk, T) && pf_tc(L.wv, T) && is_kquant(L.wq.type) && is_kquant(L.wk.type) && is_kquant(L.wv.type);
        const MmqPre attn_norm{PRO_RMSNORM, L.attn_norm, 0, hp.rms_eps};
        if (!qkv_fused) { CK(launch_rms_norm(x, P.xn, E, T, hp.rms_eps, st, L.attn_norm)); n++; }
        const float * xa = qkv_fused ? x : P.xn;
        CK(pf_matmul(m, L.wq, xa, T, P.q, L.bq, nullptr, n, nullptr, qkv_fused ? &attn_norm : nullptr));
        CK(pf_matmul(m, L.wk, xa, T, P.k, L.bk, nullptr, n, &L.wq));
        CK(pf_matmul(m, L.wv, xa, T, P.v, L.bv, nullptr, n, &L.wk));
        CK(launch_rope(P.q, P.q, T, H, D, QD, D, P.pos, m->rp, m->rope_ff, st)); n++;
        CK(launch_rope(P.k, P.k, T, HK, D, EK, D, P.pos, m->rp, m->rope_ff, st)); n++;
        CK(launch_cpy_f32_f16(P.k, kc + (size_t) pos0 * EK, (int64_t) T * EK, st)); n++;
        CK(launch_cpy_f32_f16(P.v, vc + (size_t) pos0 * EK, (int64_t) T * EK, st)); n++;
        CK(launch_attn_batch(P.q, kc, vc, P.att, H, HK, D, P.pos, T, pos0 + T, kq_scale, st)); n++;
        CK(pf_matmul(m, L.wo, P.att, T, y, nullptr, x, n));                  // ffn_inp = wo.att + inpSA (residual in the epilogue)
        // --- FFN block ---
        const bool gu_fused = pf_tc(L.gate, T) && pf_tc(L.up, T) && is_kquant(L.gate.type) && is_kquant(L.up.type);
        const MmqPre ffn_norm{PRO_RMSNORM, L.ffn_norm, 0, hp.rms_eps};
        if (!gu_fused) { CK(launch_rms_norm(y, P.xn, E, T, hp.rms_eps, st, L.ffn_norm)); n++; }
        const float * xf = gu_fused ? y : P.xn;
        CK(pf_matmul(m, L.gate, xf, T, P.g, nullptr, nullptr, n, nullptr, gu_fused ? &ffn_norm : nullptr));
        CK(pf_matmul(m, L.up, xf, T, P.u, nullptr, nullptr, n, &L.gate));
        const bool down_fused = pf_tc(L.down, T) && is_kquant(L.down.type);
        const MmqPre silu_mul{PRO_SILU_MUL, P.u, F};
        if (!down_fused) { CK(launch_silu_mul(P.g, P.u, P.g, (int64_t) T * F, st)); n++; }
        CK(pf_matmul(m, L.down, P.g, T, x, nullptr, y, n, nullptr, down_fused ? &silu_mul : nullptr));   // l_out = down.act + ffn_inp (x is free: y holds ffn_inp)
    }
    // hidden state of the last token -> the decode path's output head
    CK(cudaMemcpyAsync(m->x_out, x + (size_t) (T - 1) * E, (size_t) E * 4, cudaMemcpyDeviceToDevice, st));
    if (m->with_head) {
        GemvDesc d1 = {m->output.data, m->logits, nullptr, nullptr, m->output.type, hp.n_vocab};
        CK(launch_gemv(&d1, 1, E, m->actE.q, GemvPrologue{PRO_RMSNORM, m->x_out, m->output_norm, hp.rms_eps}, st, false, n));
    }
    P.rows = T;
    g_launches += n;
    if (!sync) return 0;
    if (m->with_head && logits_host) CK(cudaMemcpyAsync(m->logits_host, m->logits, (size_t) hp.n_vocab * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (check_clear_abort()) return PB200_EABORTED;   // a kernel's wait watchdog gave up: this batch's results are invalid (flag re-armed)
    if (m->with_head && logits_host) memcpy(logits_host, m->logits_host, (size_t) hp.n_vocab * 4);
    return 0;
}

extern "C" {
int pb200_kv_clear(pb200_model * m) {
    CK(ready(m));
    if (m->kv_bytes) { CK(cudaMemsetAsync(m->kcache, 0, m->kv_bytes, m->stream)); CK(cudaMemsetAsync(m->vcache, 0, m->kv_bytes, m->stream)); }
    return (int) cudaStreamSynchronize(m->stream);
}

// prima's context shift on slot seq (llama-cli, examples/main/main.cpp:578-608): one launch on the model stream moves cells [p0, p1) of
// every layer of this shard to c + delta, re-rotating K by delta, and moves the slot's device position with them.  The captured
// per-slot graphs read the position from device memory, so they stay valid.
int pb200_kv_seq_shift(pb200_model * m, int seq, int32_t p0, int32_t p1, int32_t delta) {
    if (delta >= 0 || (int64_t) p0 + delta < 0 || p0 >= p1) return PB200_EINVAL;   // checked before the model: no CUDA call needed
    CK(ready_seq(m, seq));
    if (p1 > m->hp.n_ctx) return PB200_EINVAL;
    const Slot & s = m->slots[seq];
    g_launches++;
    return launch_kv_shift(s.k, s.v, (int) m->layers.size(), m->hp.n_head_kv, m->hp.n_ctx, p0, p1, delta, m->rp, m->rope_ff, s.tokpos, m->stream);
}
// llama_kv_cache_seq_cp (src/llama.cpp:4308-4350): cells [p0, p1) of every layer of this shard from slot src to slot dst.  In the slot layout
// [n_seq][layer][n_ctx][row] the range is one contiguous run per layer at the pitch of one layer's block: one 2-D copy each for K and V on
// the model stream, no kernel, no host synchronisation.
int pb200_kv_seq_cp(pb200_model * m, int seq_src, int seq_dst, int32_t p0, int32_t p1) {
    CK(ready_seq(m, seq_src));
    CK(ready_seq(m, seq_dst));
    const int32_t n_ctx = m->hp.n_ctx;
    if (p0 < 0) p0 = 0;
    if (p1 < 0 || p1 > n_ctx) p1 = n_ctx;
    if (seq_src == seq_dst || p0 >= p1 || m->layers.empty()) return 0;
    const Slot & s = m->slots[seq_src], & d = m->slots[seq_dst];
    const size_t row = (size_t) m->hp.n_head_kv * m->hp.head_dim * sizeof(__half), pitch = s.layer_elems * sizeof(__half);
    const size_t off = (size_t) p0 * row, width = (size_t) (p1 - p0) * row, nl = m->layers.size();
    CK(cudaMemcpy2DAsync((char *) d.k + off, pitch, (const char *) s.k + off, pitch, width, nl, cudaMemcpyDeviceToDevice, m->stream));
    return (int) cudaMemcpy2DAsync((char *) d.v + off, pitch, (const char *) s.v + off, pitch, width, nl, cudaMemcpyDeviceToDevice, m->stream);
}
void * pb200_kv_device(pb200_model * m, int v) { return (m && m->finalized) ? (void *) (v ? m->vcache : m->kcache) : nullptr; }

static int step(pb200_model * m, int seq) {
    const Slot & s = m->slots[seq];
    if (m->use_graph && s.graph) {
        g_launches += m->launches_per_step;
        return (int) cudaGraphLaunch(s.graph, m->stream);
    }
    uint64_t n = 0;
    int rc = enqueue_step(m, seq, &n);
    g_launches += n;
    return rc;
}

// greedy sampling on the device (ggml_cuda_argmax, ggml-cuda/argmax.cu:7; first index of the maximum like ggml_compute_forward_argmax)
__global__ void __launch_bounds__(1024) k_argmax(const float * __restrict__ x, int n, int32_t * __restrict__ out, int32_t * __restrict__ out2) {
    __shared__ float sv[32];
    __shared__ int si[32];
    pdl_trigger();
    pdl_wait();
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = threadIdx.x; i < n; i += 1024) {
        const float v = x[i];
        if (v > best) { best = v; bi = i; }       // ascending i per thread: strict '>' keeps the first occurrence
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    warp_argmax(best, bi);
    if (lane == 0) { sv[warp] = best; si[warp] = bi; }
    __syncthreads();
    if (warp == 0) {
        best = sv[lane]; bi = si[lane];
        warp_argmax(best, bi);
        if (lane == 0) { *out = bi; if (out2) *out2 = bi; }
    }
}
extern "C++" int pb::launch_argmax(const float * x, int n, int32_t * out, int32_t * out2, cudaStream_t stream, bool pdl) {
    LaunchCfg lc(dim3(1), dim3(1024), 0, stream, pdl);
    return (int) cudaLaunchKernelEx(&lc.cfg, k_argmax, x, n, out, out2);
}
__global__ void k_advance_pos(int32_t * tp) { pdl_trigger(); pdl_wait(); tp[1] += 1; }

int pb200_decode(pb200_model * m, int32_t token, int32_t pos, float * logits_host) {
    CK(ready(m));
    if (!tokpos_ok(m, token, pos)) return PB200_EINVAL;
    m->tokpos_host[0] = token;
    m->tokpos_host[1] = pos;
    CK(cudaMemcpyAsync(m->slots[0].tokpos, m->tokpos_host, 8, cudaMemcpyHostToDevice, m->stream));
    CK(step(m, 0));
    if (m->with_head && logits_host) {
        CK(cudaMemcpyAsync(m->logits_host, m->logits, (size_t) m->hp.n_vocab * 4, cudaMemcpyDeviceToHost, m->stream));
        CK(cudaStreamSynchronize(m->stream));
        if (check_clear_abort()) return PB200_EABORTED;   // a wait watchdog fired inside this step: its logits are invalid
        memcpy(logits_host, m->logits_host, (size_t) m->hp.n_vocab * 4);
        return 0;
    }
    CK(cudaStreamSynchronize(m->stream));
    return check_clear_abort() ? PB200_EABORTED : 0;
}

// ---- several sequences in flight (prima's ring keeps every stage busy with a different token, src/llama.cpp:17825-18029, 18299-18387) ----
int pb200_model_set_n_seq(pb200_model * m, int n_seq) {
    if (n_seq < 1 || n_seq > 64) return PB200_EINVAL;
    CK(building(m));
    m->n_seq = n_seq;
    return 0;
}
int pb200_decode_seq_async(pb200_model * m, int seq, int32_t token, int32_t pos) {
    CK(ready_seq(m, seq));
    if (!tokpos_ok(m, token, pos)) return PB200_EINVAL;
    k_set_tokpos<<<1, 1, 0, m->stream>>>(m->slots[seq].tokpos, token, pos);   // by-value kernel args: no host buffer to keep alive
    CK(cudaGetLastError());
    return step(m, seq);
}
int pb200_decode_async(pb200_model * m, int32_t token, int32_t pos) { return pb200_decode_seq_async(m, 0, token, pos); }
// token and position of the slot are ALREADY in device memory (pb200_token_device: written by the previous stage's hand-off or by
// pb200_argmax_seq); nothing crosses the host.  advance_pos: bump the slot's position afterwards for its next step.
int pb200_step_seq_dev(pb200_model * m, int seq, int advance_pos) {
    CK(ready_seq(m, seq));
    CK(step(m, seq));
    if (advance_pos) {
        k_advance_pos<<<1, 1, 0, m->stream>>>(m->slots[seq].tokpos);
        g_launches++;
        CK(cudaGetLastError());
    }
    return 0;
}
int pb200_set_tokpos_seq(pb200_model * m, int seq, int32_t token, int32_t pos) {
    CK(ready_seq(m, seq));
    k_set_tokpos<<<1, 1, 0, m->stream>>>(m->slots[seq].tokpos, token, pos);
    return (int) cudaGetLastError();
}
// greedy token of the slot's logits -> the slot's sample word (and, when this shard also holds the embedding, straight into its token)
int pb200_argmax_seq(pb200_model * m, int seq, int feed_back) {
    CK(ready_seq(m, seq, true));
    const Slot & s = m->slots[seq];
    g_launches++;
    return launch_argmax(m->logits, (int) m->hp.n_vocab, s.sample, feed_back && m->with_embd ? s.tokpos : nullptr, m->stream, true);
}
// seeded sampling of the slot (sample.cu): parameters checked and the slot's generator seeded here, on the model stream
int pb200_sampling_set_seq(pb200_model * m, int seq, const pb200_sampling * p) {
    CK(ready_seq(m, seq, true));
    if (!sampling_params_ok(p)) return PB200_EINVAL;
    Slot & s = m->slots[seq];
    CK(launch_sampler_seed(s.rng, p->seed, m->stream));
    s.sampling = *p;
    s.sampling_set = true;
    return 0;
}
// like pb200_argmax_seq with the slot's sampling parameters (and logit bias + penalties when the slot has them)
int pb200_sample_seq(pb200_model * m, int seq, int feed_back) {
    CK(ready_seq(m, seq, true));
    const Slot & s = m->slots[seq];
    if (!s.sampling_set) return PB200_ESTATE;
    const int n = (int) m->hp.n_vocab;
    const float * row = m->logits;
    if (s.pen.set) {                    // logit bias + penalties on a copy of the row, then the unchanged chain on that copy
        CK(launch_penalize(m->logits, n, s.pen.state.p, (float *) m->pen_logits.p, m->stream, true));
        g_launches++;
        row = (const float *) m->pen_logits.p;
    }
    CK(launch_sample(row, n, s.sampling, s.rng, s.sample, feed_back && m->with_embd ? s.tokpos : nullptr, m->stream, true));
    g_launches++;
    if (s.pen.set && s.pen.last_n > 0) {   // gpt_sampler_accept: the token joins the slot's history
        CK(launch_penalty_accept(s.pen.state.p, s.sample, 1, m->stream, true));
        g_launches++;
    }
    return 0;
}
// logit bias + penalties of the slot: state allocated (or grown) here, configuration uploaded and history cleared on the model stream
int pb200_penalties_set_seq(pb200_model * m, int seq, const pb200_penalties * p) {
    CK(ready_seq(m, seq, true));
    if (p && !penalties_ok(p)) return PB200_EINVAL;
    Penalty & pen = m->slots[seq].pen;
    pen.set = false;                    // until the new configuration is in place
    if (!p) return 0;
    CK(m->pen_logits.grow((size_t) m->hp.n_vocab * 4, m->stream));
    CK(pen.state.grow(penalty_state_bytes(p->last_n, p->n_logit_bias), m->stream));
    uint64_t nl = 0;
    const int rc = launch_penalty_init(pen.state.p, (int) m->hp.n_vocab, *p, m->stream, nl);
    g_launches += nl;
    if (rc) return rc;
    pen.last_n = std::max(p->last_n, 0);
    pen.set = true;
    return 0;
}
// llama-cli accepts the prompt into the sampler (examples/main/main.cpp:720): the last last_n host tokens go to the slot's history
int pb200_sampler_accept_seq(pb200_model * m, int seq, const int32_t * tokens_host, int n) {
    CK(ready_seq(m, seq, true));
    if (n < 0 || (n > 0 && !tokens_host)) return PB200_EINVAL;
    const Penalty & pen = m->slots[seq].pen;
    if (!pen.set) return PB200_ESTATE;
    const int k = std::min(n, pen.last_n);
    if (k == 0) return 0;
    CK(m->pen_tok.grow((size_t) k * 4, m->stream));
    // from pageable memory the copy returns once the tokens are staged, so the caller may reuse its array; stream order keeps the
    // staging buffer until the accept has read it
    CK(cudaMemcpyAsync(m->pen_tok.p, tokens_host + (n - k), (size_t) k * 4, cudaMemcpyHostToDevice, m->stream));
    CK(launch_penalty_accept(pen.state.p, (const int32_t *) m->pen_tok.p, k, m->stream, false));
    g_launches++;
    return 0;
}
int32_t * pb200_token_device(pb200_model * m, int seq) { return (m && seq >= 0 && (size_t) seq < m->slots.size()) ? m->slots[seq].tokpos : nullptr; }
int32_t * pb200_sample_device(pb200_model * m, int seq) { return (m && seq >= 0 && (size_t) seq < m->slots.size()) ? m->slots[seq].sample : nullptr; }

int pb200_synchronize(pb200_model * m) {
    if (!m) return PB200_EINVAL;
    cudaSetDevice(m->device);
    CK(cudaStreamSynchronize(m->stream));
    return check_clear_abort() ? PB200_EABORTED : 0;
}
float * pb200_logits_device(pb200_model * m) { return m ? m->logits : nullptr; }
float * pb200_hidden_in_device(pb200_model * m) { return m ? m->x_in : nullptr; }
float * pb200_hidden_out_device(pb200_model * m) { return m ? m->x_out : nullptr; }
void * pb200_stream(pb200_model * m) { return m ? (void *) m->stream : nullptr; }
int pb200_get_hidden(pb200_model * m, float * hidden_host) {
    if (!hidden_host) return PB200_EINVAL;
    CK(ready(m, false, PB200_EINVAL));
    CK(cudaStreamSynchronize(m->stream));
    return (int) cudaMemcpy(hidden_host, m->x_out, (size_t) m->hp.n_embd * 4, cudaMemcpyDeviceToHost);
}
int pb200_profile_step(pb200_model * m, int32_t token, int32_t pos, double * gemv_ms, int64_t * gemv_bytes, int32_t * gemv_launches, double * step_ms) {
    CK(ready(m));
    if (!tokpos_ok(m, token, pos)) return PB200_EINVAL;
    struct Event {                      // released on every return
        cudaEvent_t e = nullptr;
        ~Event() { if (e) cudaEventDestroy(e); }
    } e0, e1;
    CK(cudaEventCreate(&e0.e)); CK(cudaEventCreate(&e1.e));
    k_set_tokpos<<<1, 1, 0, m->stream>>>(m->slots[0].tokpos, token, pos);
    CK(cudaEventRecord(e0.e, m->stream));
    m->profiling = true;
    m->prof_n = 0;
    uint64_t n = 0;
    int rc = enqueue_step(m, 0, &n);
    m->profiling = false;
    if (rc) return rc;
    g_launches += n;
    CK(cudaEventRecord(e1.e, m->stream));
    CK(cudaStreamSynchronize(m->stream));
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, e0.e, e1.e));
    if (step_ms) *step_ms = ms;
    double tot = 0; int64_t by = 0;
    for (size_t i = 0; i < m->prof_n; i++) {
        float t = 0.f;
        CK(cudaEventElapsedTime(&t, m->prof_ev[2 * i], m->prof_ev[2 * i + 1]));
        tot += t; by += m->prof_bytes[i];
    }
    if (gemv_ms) *gemv_ms = tot;
    if (gemv_bytes) *gemv_bytes = by;
    if (gemv_launches) *gemv_launches = (int32_t) m->prof_n;
    return 0;
}
int pb200_set_hidden(pb200_model * m, const float * hidden_host) {
    if (!hidden_host) return PB200_EINVAL;
    CK(ready(m, false, PB200_EINVAL));
    CK(cudaStreamSynchronize(m->stream));
    return (int) cudaMemcpy(m->x_in, hidden_host, (size_t) m->hp.n_embd * 4, cudaMemcpyHostToDevice);
}
// debugging / white-box tests: copy a named internal activation buffer of the LAST step to the host
int pb200_debug_read(pb200_model * m, const char * name, float * host, int64_t n) {
    if (!name || !host) return PB200_EINVAL;
    CK(ready(m, false, PB200_EINVAL));
    CK(cudaStreamSynchronize(m->stream));
    const std::string s(name);
    const float * p = s == "q" ? m->q : s == "k" ? m->k : s == "v" ? m->v : s == "att" ? m->att : s == "g" ? m->g : s == "u" ? m->u :
                      s == "x_a" ? m->x_a : s == "x_b" ? m->x_b : s == "x_out" ? m->x_out : s == "xn" ? m->xn : s == "x_in" ? m->x_in : s == "logits" ? m->logits : nullptr;
    if (!p) return PB200_EINVAL;
    return (int) cudaMemcpy(host, p, (size_t) n * 4, cudaMemcpyDeviceToHost);
}
int pb200_set_use_graph(pb200_model * m, int on) {
    if (!m) return PB200_EINVAL;
    m->use_graph = on != 0;
    return 0;
}

}  // extern "C"
