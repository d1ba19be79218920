// prima.cpp_b200/csrc/sample.cu — seeded top-k / top-p / min-p / temperature sampling on the device, the sampler chain the
// reference's gpt_sampler_init builds for temp > 0 and mirostat 0 (common/sampling.cpp:140-224, default order):
//   top-k (src/llama-sampling.cpp:91-165) -> top-p (:557-588) -> min-p (:624-684) -> temp (:913-918) -> softmax (:66-89)
//   -> dist (:18-46, :415-480: std::mt19937 through libstdc++'s std::discrete_distribution).
// Every stage keeps a prefix of the logits in descending order (ties: ascending token id, where the reference's std::sort leaves
// the order unspecified), so each one is a threshold found by a radix select on the 64-bit key {order-preserving logit, id}:
//   top-k        the k-th key by count;
//   top-p        the first key at which the running softmax mass of the top-k set reaches p * total (an exact sum: the reference's
//                float running sum drifts over a whole vocabulary, so with top-k 0 its cut can sit a few tokens away);
//   min-p        a count of the logits >= l0 + logf(min_p) (a prefix of the order, so no select);
//   draw         the first key at which the running mass of exp(l/temp - l0/temp) reaches u * total.
// One launch: a cluster of 16 CTAs, each holding its slice of the logits in shared memory; histograms and reductions are merged
// through distributed shared memory, every CTA ends each pass with the same merged result.  Masses are summed as 64-bit fixed
// point (2^-40 units) so the sums, and hence the picks, do not depend on the order of the atomics.
#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdint>

#include "../../include/prima_b200.h"
#include "launch.h"

namespace cg = cooperative_groups;

namespace pb {
namespace {

constexpr int SCL = 16;               // CTAs per cluster (non-portable size)
constexpr int SNT = 512;              // threads per CTA
constexpr int MT_N = 624, MT_M = 397;
typedef unsigned long long u64;

struct MtState {                      // std::mt19937: 624 words and the index of the next output (624: twist first)
    uint32_t mt[MT_N];
    uint32_t idx;
};

struct SampleArgs {
    int top_k;
    float top_p, min_p, log_min_p, temp;   // log_min_p = logf(min_p), computed on the host like the reference does
    int min_keep;
};

struct Smem {
    uint32_t hc[2][256];              // this CTA's histogram: counts / fixed-point masses, double-buffered across passes
    u64 hw[2][256];
    uint32_t gc[256];                 // merged over the cluster
    u64 gw[256];
    u64 red[2][3];                    // this CTA's reduction slot, double-buffered
    u64 wred[SNT / 32][3];
    u64 gred[3];
    u64 res;                          // key resolved by a select (written by its owner into every CTA)
    u64 sel_w;
    uint32_t sel_c;
    int sel_d;
    uint32_t mt[MT_N];
    uint32_t mt_idx;
};

struct Ctx {
    Smem & S;
    const float * lg;                 // this CTA's slice of the logits (shared memory)
    int lo, cnt;                      // global index of lg[0], slice length
    unsigned pass;                    // parity of the double-buffered histogram / reduction slots
};

__device__ __forceinline__ u64 order_key(float v, uint32_t id) {
    uint32_t u = __float_as_uint(v);
    u ^= (u & 0x80000000u) ? 0xffffffffu : 0x80000000u;   // ascending in v
    return ((u64) ~u << 32) | id;                          // ascending key = descending logit, then ascending id
}
__device__ __forceinline__ float key_logit(u64 k) {
    const uint32_t u = ~(uint32_t) (k >> 32);
    return __uint_as_float((u & 0x80000000u) ? (u ^ 0x80000000u) : ~u);
}
// softmax weight of logit l at temperature T relative to the top logit's l0 / T (= m), in units of 2^-40.  A quotient that is not
// finite (l0 = -inf, or a temperature so small that l / T overflows) gives NaN here: weight 0, never a stray conversion of NaN.
__device__ __forceinline__ u64 mass(float l, float T, float m) {
    const float e = expf(__fdiv_rn(l, T) - m);
    return e > 0.f ? __float2ull_rn(fminf(e, 1.f) * 0x1p40f) : 0ull;
}

// cluster-wide {min, sum, sum} of three per-thread values; every thread of every CTA returns the result.  The peers' slots are read
// after the barrier with no barrier behind them: the kernel ends with a cluster barrier so that no CTA exits while another still
// reads its shared memory.
__device__ void cluster_reduce(Ctx & c, u64 v[3]) {
    Smem & S = c.S;
    cg::cluster_group cl = cg::this_cluster();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, b = c.pass++ & 1;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        v[0] = min(v[0], __shfl_xor_sync(~0u, v[0], o));
        v[1] += __shfl_xor_sync(~0u, v[1], o);
        v[2] += __shfl_xor_sync(~0u, v[2], o);
    }
    if (lane == 0) { S.wred[warp][0] = v[0]; S.wred[warp][1] = v[1]; S.wred[warp][2] = v[2]; }
    __syncthreads();
    if (threadIdx.x == 0) {
        u64 a = ~0ull, s = 0, t = 0;
        for (int w = 0; w < SNT / 32; w++) { a = min(a, S.wred[w][0]); s += S.wred[w][1]; t += S.wred[w][2]; }
        S.red[b][0] = a; S.red[b][1] = s; S.red[b][2] = t;
    }
    cl.sync();
    if (warp == 0) {
        u64 a = ~0ull, s = 0, t = 0;
        if (lane < SCL) {
            const u64 * r = cl.map_shared_rank(&S.red[b][0], lane);
            a = r[0]; s = r[1]; t = r[2];
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            a = min(a, __shfl_xor_sync(~0u, a, o));
            s += __shfl_xor_sync(~0u, s, o);
            t += __shfl_xor_sync(~0u, t, o);
        }
        if (lane == 0) { S.gred[0] = a; S.gred[1] = s; S.gred[2] = t; }
    }
    __syncthreads();
    v[0] = S.gred[0]; v[1] = S.gred[1]; v[2] = S.gred[2];
    __syncthreads();
}

// Radix select over the keys <= bound: the first key x (ascending) at which the running weight reaches tgt (1 <= tgt <= total
// weight): weight 1 per key when !use_mass (x = the tgt-th key), else mass(l, T, m).  *before = how many keys of the set precede x.
__device__ u64 select(Ctx & c, u64 bound, bool use_mass, float T, float m, u64 tgt, uint32_t * before) {
    Smem & S = c.S;
    cg::cluster_group cl = cg::this_cluster();
    u64 prefix = 0, pmask = 0, before_w = 0;
    uint32_t before_c = 0;
    for (int shift = 56;; shift -= 8) {
        const int b = c.pass++ & 1;
        for (int i = threadIdx.x; i < 256; i += SNT) { S.hc[b][i] = 0; S.hw[b][i] = 0; }
        __syncthreads();
        for (int i = threadIdx.x; i < c.cnt; i += SNT) {
            const float l = c.lg[i];
            const u64 k = order_key(l, (uint32_t) (c.lo + i));
            if (k <= bound && (k & pmask) == prefix) {
                const int d = (int) (k >> shift) & 255;
                atomicAdd(&S.hc[b][d], 1u);
                if (use_mass) atomicAdd(&S.hw[b][d], mass(l, T, m));
            }
        }
        cl.sync();
        if (threadIdx.x < 256) {
            uint32_t cc = 0;
            u64 ww = 0;
            for (int r = 0; r < SCL; r++) {
                cc += cl.map_shared_rank(&S.hc[b][0], r)[threadIdx.x];
                if (use_mass) ww += cl.map_shared_rank(&S.hw[b][0], r)[threadIdx.x];
            }
            S.gc[threadIdx.x] = cc;
            S.gw[threadIdx.x] = use_mass ? ww : cc;
        }
        __syncthreads();
        if (threadIdx.x < 32) {              // digit where the running weight reaches tgt: 8 bins per lane, then a warp scan
            const int lane = threadIdx.x;
            u64 w8 = 0;
            uint32_t c8 = 0;
            for (int j = 0; j < 8; j++) { w8 += S.gw[8 * lane + j]; c8 += S.gc[8 * lane + j]; }
            u64 wi = w8;
            uint32_t ci = c8;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const u64 wo = __shfl_up_sync(~0u, wi, o);
                const uint32_t co = __shfl_up_sync(~0u, ci, o);
                if (lane >= o) { wi += wo; ci += co; }
            }
            const unsigned hit = __ballot_sync(~0u, before_w + wi >= tgt);
            const int hl = hit ? __ffs(hit) - 1 : 31;
            if (lane == hl) {
                u64 acc = before_w + wi - w8;
                uint32_t accc = before_c + ci - c8;
                int d = 8 * lane;
                for (; d < 8 * lane + 7 && acc + S.gw[d] < tgt; d++) { acc += S.gw[d]; accc += S.gc[d]; }
                S.sel_d = d; S.sel_w = acc; S.sel_c = accc;
            }
        }
        __syncthreads();
        const int d = S.sel_d;
        before_w = S.sel_w;
        before_c = S.sel_c;
        const uint32_t in_bucket = S.gc[d];
        prefix |= (u64) d << shift;
        pmask |= 255ull << shift;
        __syncthreads();
        if (in_bucket <= 1 || shift == 0) break;
    }
    // the bucket holds one key: its owner writes it into every CTA
    for (int i = threadIdx.x; i < c.cnt; i += SNT) {
        const u64 k = order_key(c.lg[i], (uint32_t) (c.lo + i));
        if (k <= bound && (k & pmask) == prefix)
            for (int r = 0; r < SCL; r++) *cl.map_shared_rank(&S.res, r) = k;
    }
    cl.sync();
    *before = before_c;
    return S.res;
}

// next output of std::mt19937 (every thread of the CTA calls it; the twist is spread over the CTA)
__device__ uint32_t mt_next(Smem & S, bool & twisted) {
    if (S.mt_idx >= MT_N) {
        auto phase = [&](int i0, int i1) {    // in three ranges, each reading only words the sequential twist has (or has not) updated
            const int i = i0 + (int) threadIdx.x;
            uint32_t v = 0;
            if (i < i1) {
                const uint32_t y = (S.mt[i] & 0x80000000u) | (S.mt[(i + 1) % MT_N] & 0x7fffffffu);
                v = S.mt[(i + MT_M) % MT_N] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
            }
            __syncthreads();
            if (i < i1) S.mt[i] = v;
            __syncthreads();
        };
        phase(0, MT_N - MT_M);
        phase(MT_N - MT_M, 2 * (MT_N - MT_M));
        phase(2 * (MT_N - MT_M), MT_N);
        if (threadIdx.x == 0) S.mt_idx = 0;
        twisted = true;
        __syncthreads();
    }
    uint32_t y = S.mt[S.mt_idx];
    __syncthreads();
    if (threadIdx.x == 0) S.mt_idx++;
    __syncthreads();
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= y >> 18;
    return y;
}

__global__ void __launch_bounds__(SNT) k_sample(const float * __restrict__ x, int n, SampleArgs a, MtState * __restrict__ st,
                                               int32_t * __restrict__ out, int32_t * __restrict__ out2) {
    extern __shared__ float s_logit[];
    __shared__ Smem S;
    cg::cluster_group cl = cg::this_cluster();
    const int rank = (int) cl.block_rank();
    const int chunk = (n + SCL - 1) / SCL;
    const int lo = min(n, rank * chunk), cnt = min(n, lo + chunk) - lo;
    pdl_trigger();
    pdl_wait();
    for (int i = threadIdx.x; i < cnt; i += SNT) s_logit[i] = x[lo + i];
    for (int i = threadIdx.x; i < MT_N; i += SNT) S.mt[i] = st->mt[i];   // every CTA reads the state before the first cluster barrier;
    if (threadIdx.x == 0) S.mt_idx = st->idx;                           // only rank 0 writes it back, after later barriers
    __syncthreads();
    Ctx c{S, s_logit, lo, cnt, 0u};

    // the first key of the order: the top logit l0 (lowest id among equals)
    u64 v[3] = {~0ull, 0, 0};
    for (int i = threadIdx.x; i < cnt; i += SNT) v[0] = min(v[0], order_key(s_logit[i], (uint32_t) (lo + i)));
    cluster_reduce(c, v);
    const u64 top = v[0];
    const float l0 = key_logit(top);

    // top-k: k <= 0 keeps the whole vocabulary
    const int K = a.top_k <= 0 ? n : min(a.top_k, n);
    u64 bound = ~0ull;
    uint32_t before = 0;
    if (K < n) bound = select(c, ~0ull, false, 1.f, 0.f, (u64) K, &before);
    int L = K;

    // top-p over the top-k set at temperature 1 (skipped for p >= 1), min-p (skipped for p <= 0); one reduction for both
    const bool do_top_p = a.top_p < 1.f, do_min_p = a.min_p > 0.f;
    if (do_top_p || do_min_p) {
        const float min_logit = l0 + a.log_min_p;
        v[0] = ~0ull; v[1] = 0; v[2] = 0;
        for (int i = threadIdx.x; i < cnt; i += SNT) {
            const float l = s_logit[i];
            if (do_top_p && order_key(l, (uint32_t) (lo + i)) <= bound) v[1] += mass(l, 1.f, l0);
            if (do_min_p && l >= min_logit) v[2] += 1;
        }
        cluster_reduce(c, v);
        if (do_top_p && v[1] > 0) {        // total 0: the top logit is -inf or NaN, no mass to cut by
            const u64 total = v[1];
            u64 tgt = (u64) ceil((double) a.top_p * (double) total);
            tgt = min(max(tgt, 1ull), total);
            select(c, bound, true, 1.f, l0, tgt, &before);
            L = min(K, max((int) before + 1, a.min_keep));     // shortest prefix reaching p, at least min_keep
        }
        if (do_min_p) L = min(L, max(max(1, (int) v[2]), a.min_keep));   // index 0 always stays
    }

    int32_t tok = (int32_t) (uint32_t) top;
    bool twisted = false, drew = false;
    if (L > 1) {                     // one survivor draws nothing and leaves the generator where it was
        if (L < K) bound = select(c, bound, false, 1.f, 0.f, (u64) L, &before);
        const float m = __fdiv_rn(l0, a.temp);
        v[0] = ~0ull; v[1] = 0; v[2] = 0;
        for (int i = threadIdx.x; i < cnt; i += SNT) {
            const float l = s_logit[i];
            if (order_key(l, (uint32_t) (lo + i)) <= bound) v[1] += mass(l, a.temp, m);
        }
        cluster_reduce(c, v);
        const u64 total = v[1];
        // generate_canonical<double, 53> over two 32-bit outputs (libstdc++ bits/random.tcc:3349-3381)
        const uint32_t g1 = mt_next(S, twisted);
        const uint32_t g2 = mt_next(S, twisted);
        double u = __dadd_rn((double) g1, (double) g2 * 4294967296.0) * 0x1p-64;
        if (u >= 1.0) u = nextafter(1.0, 0.0);
        drew = true;
        if (total > 0) {                 // total 0 (l0 / temp not finite): every weight vanished, keep the top key (the greedy limit)
            u64 tgt = (u64) ceil(u * (double) total);
            tgt = min(max(tgt, 1ull), total);
            tok = (int32_t) (uint32_t) select(c, bound, true, a.temp, m, tgt, &before);
        }
    }
    // Distributed shared memory may only be accessed while every CTA of the cluster is resident: on some paths (min-p alone leaving
    // one survivor, n_vocab 1) the last cluster operation is a cluster_reduce whose remote reads no later barrier orders, so no CTA
    // may leave before all of them have finished.
    cg::this_cluster().sync();
    if (rank == 0) {
        if (twisted)
            for (int i = threadIdx.x; i < MT_N; i += SNT) st->mt[i] = S.mt[i];
        if (threadIdx.x == 0) {
            if (drew) st->idx = S.mt_idx;
            *out = tok;
            if (out2) *out2 = tok;
        }
    }
}

__global__ void k_sampler_seed(MtState * st, uint32_t seed) {   // std::mt19937(seed): init_genrand
    uint32_t y = seed;
    st->mt[0] = y;
    for (int i = 1; i < MT_N; i++) {
        y = 1812433253u * (y ^ (y >> 30)) + (uint32_t) i;
        st->mt[i] = y;
    }
    st->idx = MT_N;
}

FuncAttrCache sample_attr;

// ---- logit bias and repeat / frequency / presence penalties (llama_sampler_init_logit_bias, :1568-1645, and
// llama_sampler_init_penalties, :1373-1566): the two samplers gpt_sampler_init puts in front of every chain.  They write a penalised
// copy of the logits row that the chain above (or k_argmax) then reads like any other row.
// Device state: PenHdr, the bias list (n_bias entries), the history ring (last_n int32).
struct PenHdr {
    int32_t last_n;          // ring capacity, >= 0; 0: accept does nothing
    int32_t n_bias;
    int32_t eos;             // -1: no EOS step (ignore_eos off, or no EOS id in [0, n_vocab))
    int32_t nl;              // -1: the newline is penalised like any other token
    int32_t active;          // 0: the early exit (last_n 0, or repeat 1 / freq 0 / present 0): bias and EOS only
    float repeat, freq, present;
    int32_t count, pos;      // tokens in the ring (min(accepted, last_n)) and the next slot to write
    int32_t pad_[6];
};
static_assert(sizeof(PenHdr) == 64, "PenHdr");
constexpr int PEN_CHUNK = 256;        // bias entries per init launch, passed by value
constexpr int PEN_SLICE = 4096;       // vocabulary ids per CTA of k_penalize
constexpr int PEN_NT = 512;
struct BiasChunk { pb200_logit_bias e[PEN_CHUNK]; };

__device__ __forceinline__ const pb200_logit_bias * pen_bias(const PenHdr * h) { return (const pb200_logit_bias *) (h + 1); }
__device__ __forceinline__ int32_t * pen_ring(const PenHdr * h, int n_bias) { return (int32_t *) ((const pb200_logit_bias *) (h + 1) + n_bias); }

// a fresh penalties sampler: header (first chunk only; count = pos = 0 clears the history) and entries [off, off + cnt) of the bias list
__global__ void k_penalty_init(PenHdr * st, PenHdr h, BiasChunk c, int off, int cnt) {
    pb200_logit_bias * b = (pb200_logit_bias *) (st + 1);
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) b[off + i] = c.e[i];
    if (off == 0 && threadIdx.x == 0) *st = h;
}

// out = the penalised copy of x[n].  CTA b owns ids [b * PEN_SLICE, ...): its slice of the row and a count per id in shared memory.
__global__ void __launch_bounds__(PEN_NT) k_penalize(const float * __restrict__ x, int n, const PenHdr * __restrict__ st, float * __restrict__ out) {
    __shared__ float s_row[PEN_SLICE];
    __shared__ int s_cnt[PEN_SLICE];
    __shared__ float s_bv[32];
    pdl_trigger();
    pdl_wait();
    const PenHdr h = *st;
    const int lo = blockIdx.x * PEN_SLICE, cnt = min(n - lo, PEN_SLICE);
    for (int i = threadIdx.x; i < cnt; i += PEN_NT) { s_row[i] = x[lo + i]; s_cnt[i] = 0; }
    __syncthreads();
    // 1. bias, one rounded add per entry in list order: warp 0 takes 32 entries at a time; the lowest lane of each group of equal
    //    ids in this slice adds the group's biases in lane (= list) order.  Ids outside [0, n) fall in no slice.
    if (threadIdx.x < 32) {
        const int lane = threadIdx.x;
        const pb200_logit_bias * b = pen_bias(st);
        for (int j0 = 0; j0 < h.n_bias; j0 += 32) {
            int t = -1;
            float v = 0.f;
            if (j0 + lane < h.n_bias) { t = b[j0 + lane].token; v = b[j0 + lane].bias; }
            const bool mine = t >= lo && t < lo + cnt;
            const unsigned grp = __match_any_sync(~0u, mine ? t : -1);
            s_bv[lane] = v;
            __syncwarp();
            if (mine && __ffs(grp) - 1 == lane) {
                float acc = s_row[t - lo];
                for (unsigned g = grp; g; g &= g - 1) acc = __fadd_rn(acc, s_bv[__ffs(g) - 1]);
                s_row[t - lo] = acc;
            }
            __syncwarp();
        }
    }
    __syncthreads();
    // 2. ignore_eos
    if (threadIdx.x == 0 && h.eos >= lo && h.eos < lo + cnt) s_row[h.eos - lo] = -INFINITY;
    // 3. early exit: bias and EOS only
    if (h.active) {
        // 5. counts of the ids of this slice among the last min(last_n, accepted) tokens (the ring holds exactly those)
        const int32_t * ring = pen_ring(st, h.n_bias);
        for (int i = threadIdx.x; i < h.count; i += PEN_NT) {
            const int t = ring[i];
            if (t >= lo && t < lo + cnt) atomicAdd(&s_cnt[t - lo], 1);
        }
        __syncthreads();
        // 4. + 6. the newline keeps the logit it had before this step: it is simply not penalised
        for (int i = threadIdx.x; i < cnt; i += PEN_NT) {
            const int c = s_cnt[i];
            if (c > 0 && lo + i != h.nl) {
                float l = s_row[i];
                l = l <= 0.f ? __fmul_rn(l, h.repeat) : __fdiv_rn(l, h.repeat);
                s_row[i] = __fsub_rn(l, __fadd_rn(__fmul_rn((float) c, h.freq), __fmul_rn(1.0f, h.present)));
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < cnt; i += PEN_NT) out[lo + i] = s_row[i];
}

// llama_sampler_accept for n tokens: only the last last_n reach the ring
__global__ void k_penalty_accept(PenHdr * st, const int32_t * __restrict__ tok, int n) {
    pdl_trigger();
    pdl_wait();
    const int L = st->last_n;
    if (L <= 0) return;
    int32_t * ring = pen_ring(st, st->n_bias);
    const int m = min(n, L), pos = st->pos, count = st->count;
    for (int i = threadIdx.x; i < m; i += blockDim.x) ring[(pos + i) % L] = tok[n - m + i];
    __syncthreads();
    if (threadIdx.x == 0) { st->pos = (pos + m) % L; st->count = min(count + m, L); }
}

}  // namespace

size_t penalty_state_bytes(int last_n, int n_bias) {
    return (sizeof(PenHdr) + (size_t) std::max(n_bias, 0) * sizeof(pb200_logit_bias) + (size_t) std::max(last_n, 0) * 4 + 255) / 256 * 256;
}

bool penalties_ok(const pb200_penalties * p) {
    if (!p) return false;
    if (!std::isfinite(p->repeat) || !(p->repeat > 0.f) || !std::isfinite(p->freq) || !std::isfinite(p->present)) return false;
    if (p->n_logit_bias < 0 || (p->n_logit_bias > 0 && !p->logit_bias)) return false;
    for (int i = 0; i < p->n_logit_bias; i++)
        if (std::isnan(p->logit_bias[i].bias)) return false;
    return true;
}

int launch_penalty_init(void * state, int n_vocab, const pb200_penalties & p, cudaStream_t stream, uint64_t & nlaunch) {
    PenHdr h{};
    h.last_n = std::max(p.last_n, 0);
    h.n_bias = p.n_logit_bias;
    h.eos = p.ignore_eos && p.eos_token >= 0 && p.eos_token < n_vocab ? p.eos_token : -1;
    h.nl = !p.penalize_nl && p.nl_token >= 0 && p.nl_token < n_vocab ? p.nl_token : -1;
    h.active = h.last_n != 0 && !(p.repeat == 1.f && p.freq == 0.f && p.present == 0.f);
    h.repeat = p.repeat; h.freq = p.freq; h.present = p.present;
    int off = 0;
    do {
        const int cnt = std::min(PEN_CHUNK, p.n_logit_bias - off);
        BiasChunk c;
        for (int i = 0; i < cnt; i++) c.e[i] = p.logit_bias[off + i];
        k_penalty_init<<<1, PEN_CHUNK, 0, stream>>>((PenHdr *) state, h, c, off, cnt);
        nlaunch++;
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return (int) e;
        off += cnt;
    } while (off < p.n_logit_bias);
    return 0;
}

int launch_penalize(const float * x, int n, const void * state, float * out, cudaStream_t stream, bool pdl) {
    LaunchCfg lc(dim3((n + PEN_SLICE - 1) / PEN_SLICE), dim3(PEN_NT), 0, stream, pdl);
    return (int) cudaLaunchKernelEx(&lc.cfg, k_penalize, x, n, (const PenHdr *) state, out);
}

int launch_penalty_accept(void * state, const int32_t * tokens, int n, cudaStream_t stream, bool pdl) {
    LaunchCfg lc(dim3(1), dim3(256), 0, stream, pdl);
    return (int) cudaLaunchKernelEx(&lc.cfg, k_penalty_accept, (PenHdr *) state, tokens, n);
}

size_t sampler_state_bytes() { return (sizeof(MtState) + 255) / 256 * 256; }

bool sampling_params_ok(const pb200_sampling * p) {
    if (!p) return false;
    if (!std::isfinite(p->top_p) || !std::isfinite(p->min_p) || !std::isfinite(p->temp)) return false;
    if (!(p->top_p > 0.f && p->top_p <= 1.f)) return false;
    if (!(p->min_p >= 0.f && p->min_p < 1.f)) return false;
    return p->min_keep >= 0;
}

int launch_sampler_seed(void * state, uint32_t seed, cudaStream_t stream) {
    k_sampler_seed<<<1, 1, 0, stream>>>((MtState *) state, seed);
    return (int) cudaGetLastError();
}

int launch_sample(const float * x, int n, const pb200_sampling & p, void * state, int32_t * out, int32_t * out2, cudaStream_t stream, bool pdl) {
    if (p.temp <= 0.f) return launch_argmax(x, n, out, out2, stream, pdl);   // greedy: first index of the maximum
    const SampleArgs a{p.top_k, p.top_p, p.min_p, p.min_p > 0.f ? logf(p.min_p) : 0.f, p.temp, p.min_keep};
    const size_t smem = (size_t) ((n + SCL - 1) / SCL) * sizeof(float);
    cudaError_t e = ensure_dyn_smem(sample_attr, (const void *) k_sample, smem, true);   // opt in: the static Smem + the slice pass 48 KB at Qwen2.5's vocabulary
    if (e != cudaSuccess) return (int) e;
    static bool cluster_ok[PB_MAX_DEV] = {false};
    const int dev = cur_device();
    if (!cluster_ok[dev]) {
        if ((e = cudaFuncSetAttribute(k_sample, cudaFuncAttributeNonPortableClusterSizeAllowed, 1)) != cudaSuccess) return (int) e;
        cluster_ok[dev] = true;
    }
    LaunchCfg lc(dim3(SCL), dim3(SNT), smem, stream, pdl, SCL);
    return (int) cudaLaunchKernelEx(&lc.cfg, k_sample, x, n, a, (MtState *) state, out, out2);
}

}  // namespace pb
