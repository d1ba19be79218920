// prima.cpp_b200/csrc/gguf.cu — GGUF file -> device loader (SURVEY §8 row N2).
//
// Replaces, for the tensors of the decode path: gguf_init_from_file (ggml/src/ggml.c, GGUF v2/v3 container: header, KV pairs, tensor
// infos, aligned data section) + llm_load_hparams' key lookups (src/llama.cpp "%s.block_count", "%s.embedding_length", ...) +
// llm_load_tensors' per-tensor ggml_backend_tensor_set, which on the reference CUDA backend is a synchronous cudaMemcpy from pageable
// memory per tensor (ggml-cuda.cu:464-487).
//
// Here: the file is read with pread() into two pinned staging buffers and streamed with cudaMemcpyAsync, so the disk / page-cache read of
// chunk i+1 overlaps the PCIe copy of chunk i; tensors keep their raw GGUF block layout in HBM (no repack: the kernels read the blocks
// byte for byte).  A pipeline shard loads only its layer window (prima's n_layer_window) and skips the rest of the file.
// The parser is host-only and is exercised without a GPU (pb200_gguf_probe).
#include <cuda_runtime.h>
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/prima_b200.h"
#include "common.cuh"

namespace {

using pb::row_bytes;

struct GgufTensor {
    std::string name;
    int type = -1;
    int n_dims = 0;
    int64_t ne[4] = {1, 1, 1, 1};
    uint64_t offset = 0;   // relative to the data section
    uint64_t nbytes = 0;
};
struct GgufFile {
    int fd = -1;
    uint32_t version = 0;
    uint64_t data_start = 0, file_size = 0, alignment = 32;
    std::string arch;
    std::map<std::string, double> num;        // numeric KV pairs (ints and floats widened)
    std::map<std::string, std::string> str;   // string KV pairs
    std::map<std::string, uint64_t> arr_len;  // array KV pairs: length only (tokenizer tables are skipped)
    std::vector<GgufTensor> tensors;
    ~GgufFile() { if (fd >= 0) close(fd); }
};

// buffered sequential reader over the metadata part of the file
struct Reader {
    int fd;
    uint64_t pos = 0, size;
    std::vector<uint8_t> buf;
    uint64_t buf_pos = 0;
    bool ok = true;
    Reader(int f, uint64_t sz) : fd(f), size(sz) {}
    bool fill(uint64_t need) {
        if (pos + need > size) return ok = false;
        if (pos >= buf_pos && pos + need <= buf_pos + buf.size()) return true;
        const uint64_t n = std::min<uint64_t>(std::max<uint64_t>(need, 1u << 20), size - pos);
        buf.resize(n);
        buf_pos = pos;
        uint64_t got = 0;
        while (got < n) {
            const ssize_t r = pread(fd, buf.data() + got, n - got, (off_t) (pos + got));
            if (r <= 0) return ok = false;
            got += (uint64_t) r;
        }
        return true;
    }
    template <typename T> T get() {
        T v{};
        if (!fill(sizeof(T))) return v;
        memcpy(&v, buf.data() + (pos - buf_pos), sizeof(T));
        pos += sizeof(T);
        return v;
    }
    std::string get_str() {
        const uint64_t n = get<uint64_t>();
        if (!ok || n > (1u << 24) || !fill(n)) { ok = false; return std::string(); }
        std::string s((const char *) buf.data() + (pos - buf_pos), n);
        pos += n;
        return s;
    }
    void skip(uint64_t n) { if (pos + n > size) ok = false; else pos += n; }
};

// enum gguf_type (ggml/include/ggml.h:2358-2373)
enum { G_U8 = 0, G_I8, G_U16, G_I16, G_U32, G_I32, G_F32, G_BOOL, G_STR, G_ARR, G_U64, G_I64, G_F64 };
int scalar_size(uint32_t t) {
    switch (t) {
        case G_U8: case G_I8: case G_BOOL: return 1;
        case G_U16: case G_I16: return 2;
        case G_U32: case G_I32: case G_F32: return 4;
        case G_U64: case G_I64: case G_F64: return 8;
    }
    return -1;
}
double read_num(Reader & r, uint32_t t) {
    switch (t) {
        case G_U8: return r.get<uint8_t>();
        case G_I8: return r.get<int8_t>();
        case G_BOOL: return r.get<uint8_t>();
        case G_U16: return r.get<uint16_t>();
        case G_I16: return r.get<int16_t>();
        case G_U32: return r.get<uint32_t>();
        case G_I32: return r.get<int32_t>();
        case G_F32: return r.get<float>();
        case G_U64: return (double) r.get<uint64_t>();
        case G_I64: return (double) r.get<int64_t>();
        case G_F64: return r.get<double>();
    }
    r.ok = false;
    return 0;
}

int64_t type_nbytes(int type, const int64_t ne[4]) {
    if (type != pb::T_F32 && type != pb::T_F16 && !pb::is_quant_type(type)) return -1;
    const int be = pb::block_elems(type);
    if (ne[0] % be != 0) return -1;
    return row_bytes(type, ne[0]) * ne[1] * ne[2] * ne[3];
}

int gguf_parse(const char * path, GgufFile & g) {
    g.fd = open(path, O_RDONLY);
    if (g.fd < 0) return PB200_EINVAL;
    struct stat st;
    if (fstat(g.fd, &st) != 0) return PB200_EINVAL;
    g.file_size = (uint64_t) st.st_size;
    Reader r(g.fd, g.file_size);
    const uint32_t magic = r.get<uint32_t>();
    if (!r.ok || memcmp(&magic, "GGUF", 4) != 0) return PB200_EINVAL;
    g.version = r.get<uint32_t>();
    if (g.version != 2 && g.version != 3) return PB200_ENOTSUP;   // v1 had 32-bit counts (gguf_init_from_file rejects it too)
    const uint64_t n_tensors = r.get<uint64_t>(), n_kv = r.get<uint64_t>();
    if (!r.ok || n_tensors > (1u << 20) || n_kv > (1u << 20)) return PB200_EINVAL;
    for (uint64_t i = 0; i < n_kv && r.ok; i++) {
        const std::string key = r.get_str();
        const uint32_t t = r.get<uint32_t>();
        if (t == G_STR) {
            g.str[key] = r.get_str();
        } else if (t == G_ARR) {
            const uint32_t et = r.get<uint32_t>();
            const uint64_t n = r.get<uint64_t>();
            g.arr_len[key] = n;
            if (et == G_STR) { for (uint64_t j = 0; j < n && r.ok; j++) { const uint64_t l = r.get<uint64_t>(); r.skip(l); } }
            else if (scalar_size(et) > 0) r.skip(n * (uint64_t) scalar_size(et));
            else r.ok = false;
        } else if (scalar_size(t) > 0) {
            g.num[key] = read_num(r, t);
        } else {
            r.ok = false;
        }
    }
    if (!r.ok) return PB200_EINVAL;
    g.tensors.resize(n_tensors);
    for (uint64_t i = 0; i < n_tensors && r.ok; i++) {
        GgufTensor & t = g.tensors[i];
        t.name = r.get_str();
        t.n_dims = (int) r.get<uint32_t>();
        if (t.n_dims < 1 || t.n_dims > 4) { r.ok = false; break; }
        for (int d = 0; d < t.n_dims; d++) t.ne[d] = (int64_t) r.get<uint64_t>();
        t.type = (int) r.get<uint32_t>();
        t.offset = r.get<uint64_t>();
    }
    if (!r.ok) return PB200_EINVAL;
    if (g.num.count("general.alignment")) g.alignment = (uint64_t) g.num["general.alignment"];
    if (g.alignment == 0 || (g.alignment & (g.alignment - 1))) return PB200_EINVAL;
    g.data_start = (r.pos + g.alignment - 1) / g.alignment * g.alignment;
    g.arch = g.str.count("general.architecture") ? g.str["general.architecture"] : std::string();
    for (GgufTensor & t : g.tensors) {
        const int64_t nb = type_nbytes(t.type, t.ne);
        t.nbytes = nb > 0 ? (uint64_t) nb : 0;   // unsupported types are only an error if the decode path needs the tensor
        if (nb > 0 && g.data_start + t.offset + t.nbytes > g.file_size) return PB200_EINVAL;
    }
    return 0;
}

const GgufTensor * find(const GgufFile & g, const std::string & name) {
    for (const GgufTensor & t : g.tensors) if (t.name == name) return &t;
    return nullptr;
}

int gguf_hparams(const GgufFile & g, int n_ctx, pb200_hparams * hp) {
    if (g.arch != "llama" && g.arch != "qwen2") return PB200_ENOTSUP;
    auto key = [&](const char * k) { return g.arch + "." + k; };
    auto geti = [&](const char * k, double def) { auto it = g.num.find(key(k)); return it == g.num.end() ? def : it->second; };
    memset(hp, 0, sizeof *hp);
    hp->n_layer = (int32_t) geti("block_count", 0);
    hp->n_embd = (int32_t) geti("embedding_length", 0);
    hp->n_head = (int32_t) geti("attention.head_count", 0);
    hp->n_head_kv = (int32_t) geti("attention.head_count_kv", hp->n_head);
    hp->n_ff = (int32_t) geti("feed_forward_length", 0);
    if (hp->n_layer <= 0 || hp->n_embd <= 0 || hp->n_head <= 0 || hp->n_head_kv <= 0 || hp->n_ff <= 0) return PB200_EINVAL;
    hp->head_dim = (int32_t) geti("attention.key_length", hp->n_embd / hp->n_head);      // llm_load_hparams: n_embd_head_k
    const int32_t n_rot = (int32_t) geti("rope.dimension_count", hp->head_dim);
    if (n_rot != hp->head_dim) return PB200_ENOTSUP;                                       // partial rotary: not on this path
    hp->n_ctx_orig = (int32_t) geti("rope.scaling.original_context_length", geti("context_length", 0));
    hp->n_ctx = n_ctx > 0 ? n_ctx : (int32_t) std::min<double>(geti("context_length", 4096), 4096);
    hp->rope_freq_base = (float) geti("rope.freq_base", 10000.0);
    const double factor = geti("rope.scaling.factor", 0.0);
    const std::string sc = g.str.count(key("rope.scaling.type")) ? g.str.at(key("rope.scaling.type")) : std::string("none");
    hp->rope_freq_scale = (sc == "linear" && factor > 0.0) ? (float) (1.0 / factor) : 1.0f;   // YaRN etc.: not handled by this loader
    hp->rms_eps = (float) geti("attention.layer_norm_rms_epsilon", 1e-5);
    hp->rope_mode = g.arch == "qwen2" ? 2 : 0;                                             // llama_rope_type (src/llama.cpp): NORM / NEOX
    const GgufTensor * emb = find(g, "token_embd.weight");
    if (!emb || emb->ne[0] != hp->n_embd) return PB200_EINVAL;
    hp->n_vocab = (int32_t) emb->ne[1];
    return 0;
}

}  // namespace

extern "C" {

// host-only: header + hyper-parameters of a GGUF file (no CUDA call).  n_tensors / data_bytes may be NULL.
int pb200_gguf_probe(const char * path, pb200_hparams * hp, int32_t * n_tensors, int64_t * data_bytes, char * arch_out16) {
    if (!path || !hp) return PB200_EINVAL;
    GgufFile g;
    int rc = gguf_parse(path, g);
    if (rc) return rc;
    if (n_tensors) *n_tensors = (int32_t) g.tensors.size();
    if (data_bytes) *data_bytes = (int64_t) (g.file_size - g.data_start);
    if (arch_out16) { memset(arch_out16, 0, 16); strncpy(arch_out16, g.arch.c_str(), 15); }
    return gguf_hparams(g, 0, hp);
}

// Creates the model shard [layer_begin, layer_end) (layer_end < 0: to the last layer) on `device` from a GGUF file and finalizes it.
// with_embd / with_head < 0: decided from the window (first / last stage).  Tied embeddings (no output.weight): token_embd is used.
int pb200_model_load_gguf(const char * path, int device, int layer_begin, int layer_end, int n_ctx, int with_embd, int with_head,
                          pb200_model ** out, double * seconds, int64_t * bytes_loaded) {
    if (!path || !out) return PB200_EINVAL;
    *out = nullptr;
    GgufFile g;
    int rc = gguf_parse(path, g);
    if (rc) return rc;
    pb200_hparams hp;
    rc = gguf_hparams(g, n_ctx, &hp);
    if (rc) return rc;
    if (layer_end < 0) layer_end = hp.n_layer;
    if (layer_begin < 0 || layer_begin > layer_end || layer_end > hp.n_layer) return PB200_EINVAL;
    if (with_embd < 0) with_embd = layer_begin == 0;
    if (with_head < 0) with_head = layer_end == hp.n_layer;
    if (cudaSetDevice(device) != cudaSuccess) return PB200_EINVAL;
    pb200_model * m = pb200_model_create(&hp, device, layer_begin, layer_end, with_embd, with_head);
    if (!m) return PB200_EINVAL;

    constexpr size_t CHUNK = 64u << 20;
    uint8_t * pin[2] = {nullptr, nullptr};
    cudaEvent_t ev[2] = {nullptr, nullptr};
    cudaStream_t st = nullptr;
    auto cleanup = [&](int code) {
        if (st) { cudaStreamSynchronize(st); cudaStreamDestroy(st); }
        for (int i = 0; i < 2; i++) { if (ev[i]) cudaEventDestroy(ev[i]); if (pin[i]) cudaFreeHost(pin[i]); }
        if (code) { pb200_model_free(m); *out = nullptr; }
        return code;
    };
    if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess) return cleanup(PB200_ENOMEM);
    for (int i = 0; i < 2; i++)
        if (cudaHostAlloc((void **) &pin[i], CHUNK, cudaHostAllocDefault) != cudaSuccess || cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming) != cudaSuccess)
            return cleanup(PB200_ENOMEM);
    timespec t0; clock_gettime(CLOCK_MONOTONIC, &t0);
    int64_t total = 0;
    int slot = 0;
    bool used[2] = {false, false};
    bool have_output = find(g, "output.weight") != nullptr;
    for (const GgufTensor & t : g.tensors) {
        std::string name = t.name;
        void * dev = nullptr;
        // Tensors the decode path has no slot for, or whose type / shape it cannot hold, are skipped: pb200_model_finalize below refuses a
        // shard with a missing tensor (PB200_ESTATE), so nothing needed can be dropped silently.
        rc = pb200_model_tensor_alloc(m, name.c_str(), t.type, (size_t) t.nbytes, &dev);
        if (rc == PB200_EINVAL || rc == PB200_ENOTSUP) continue;
        if (rc) return cleanup(rc);
        for (int rep = 0; rep < 2; rep++) {
            if (dev) {
                uint64_t done = 0;
                while (done < t.nbytes) {
                    const size_t n = (size_t) std::min<uint64_t>(CHUNK, t.nbytes - done);
                    if (used[slot] && cudaEventSynchronize(ev[slot]) != cudaSuccess) return cleanup(PB200_ENOMEM);
                    size_t got = 0;
                    while (got < n) {
                        const ssize_t r = pread(g.fd, pin[slot] + got, n - got, (off_t) (g.data_start + t.offset + done + got));
                        if (r <= 0) return cleanup(PB200_EINVAL);
                        got += (size_t) r;
                    }
                    if (cudaMemcpyAsync((uint8_t *) dev + done, pin[slot], n, cudaMemcpyHostToDevice, st) != cudaSuccess) return cleanup(PB200_ENOMEM);
                    if (cudaEventRecord(ev[slot], st) != cudaSuccess) return cleanup(PB200_ENOMEM);
                    used[slot] = true;
                    slot ^= 1;
                    done += n;
                }
                total += (int64_t) t.nbytes;
            }
            // tied embeddings (llm_load_tensors: output = token_embd when output.weight is absent): a second copy for the head
            if (rep == 0 && name == "token_embd.weight" && !have_output && with_head) {
                dev = nullptr;
                rc = pb200_model_tensor_alloc(m, "output.weight", t.type, t.nbytes, &dev);
                if (rc) return cleanup(rc);
            } else break;
        }
    }
    if (cudaStreamSynchronize(st) != cudaSuccess) return cleanup(PB200_ENOMEM);
    rc = pb200_model_finalize(m);
    if (rc) return cleanup(rc);
    timespec t1; clock_gettime(CLOCK_MONOTONIC, &t1);
    if (seconds) *seconds = (double) (t1.tv_sec - t0.tv_sec) + 1e-9 * (double) (t1.tv_nsec - t0.tv_nsec);
    if (bytes_loaded) *bytes_loaded = total;
    *out = m;
    return cleanup(0);
}

}  // extern "C"
