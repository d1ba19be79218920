// prima.cpp_b200/csrc/gemv.cu — kernels + launchers for the decode GEMV (see gemv.cuh for the design).
#include "gemv.cuh"
#include "launch.h"
#include "quantize.cuh"

#include <algorithm>
#include <cstdlib>

namespace pb {

constexpr int GEMV_ROWQ = 8;   // rows of one warp group whose partials may be pending (> ring depth: see the split-row loop)
struct __align__(16) GemvSmemCtl {
    uint64_t full[GEMV_MAX_STAGE];              // "tile of this stage has landed" (expect_tx)
    uint64_t pbar[GEMV_ROWQ][4];                // split rows: "the partials of the group's row (r mod GEMV_ROWQ) are in shared memory"
    int cnt[GEMV_MAX_STAGE];                    // consumer warps done with the stage; the last one refills it
    float part[GEMV_ROWQ][GEMV_NW];             // cross-warp partial sums, one slot per row in flight of each group
    double red[GEMV_NW];                        // rms_norm partial sums of squares
    volatile int aborted;                       // raised by the wait watchdog (common.cuh)
};
constexpr int GEMV_CTL_BYTES = 768;
static_assert(sizeof(GemvSmemCtl) <= GEMV_CTL_BYTES, "ctl block");

__device__ __forceinline__ float silu_f(float x) { return __fdiv_rn(x, 1.0f + expf(-x)); }   // ggml.c:2560

// TRACE instantiation only: slot k (0..5) of this CTA's 8-entry row = %globaltimer (ns) at stamp k; slots 6 / 7 = clock64 at
// the first / last stamp (the SM clock during the launch follows from the two)
template <bool TRACE>
__device__ __forceinline__ void stamp(const GemvParams & P, int k) {
    if (TRACE) {
        if (threadIdx.x == 0 && P.trace) {
            unsigned long long t;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
            P.trace[blockIdx.x * 8 + k] = t;
            if (k == 0) P.trace[blockIdx.x * 8 + 6] = (unsigned long long) clock64();
            if (k == 5) P.trace[blockIdx.x * 8 + 7] = (unsigned long long) clock64();
        }
    }
}

__device__ __forceinline__ void load8(const float * p, float (&v)[8]) {   // .cg: L2 only (data written by the previous grid)
    const float4 a0 = __ldcg(reinterpret_cast<const float4 *>(p)), a1 = __ldcg(reinterpret_cast<const float4 *>(p + 4));
    v[0] = a0.x; v[1] = a0.y; v[2] = a0.z; v[3] = a0.w; v[4] = a1.x; v[5] = a1.y; v[6] = a1.z; v[7] = a1.w;
}
constexpr int PRO_B = 4;   // super-blocks in flight per warp while summing squares (8 warps x 4 = K 8192 in one batch)

__device__ __forceinline__ void tile_info(const GemvParams & P, int t, int & m, int & r0, int & nrows) {
    m = 0;
#pragma unroll
    for (int i = 1; i < GEMV_MAX_MAT; i++)
        if (i < P.nmat && t >= P.mat[i].tile0) m = i;
    const GemvMat & M = P.mat[m];
    r0 = (t - M.tile0) * M.rows_per_tile;
    nrows = min(M.rows_per_tile, M.N - r0);
}

// one bulk copy (TMA 1-D) of tile t into ring stage s; arms the stage's mbarrier with the byte count first
__device__ __forceinline__ void issue_tile(const GemvParams & P, GemvSmemCtl * ctl, uint8_t * stages, int s, int t, uint64_t pol) {
    int m, r0, nrows;
    tile_info(P, t, m, r0, nrows);
    const GemvMat & M = P.mat[m];
    const int64_t g0 = (int64_t) r0 * M.row_bytes;
    const int64_t g1 = g0 + (int64_t) nrows * M.row_bytes;
    const int64_t a0 = g0 & ~(int64_t) 15;
    int64_t a1 = (g1 + 15) & ~(int64_t) 15;
    const int64_t lim = (M.total_bytes + 15) & ~(int64_t) 15;   // allocations are 16-B granular (include/prima_b200.h: W padding rule)
    if (a1 > lim) a1 = lim;
    const uint32_t bytes = (uint32_t) (a1 - a0);
    mbar_arrive_expect_tx(&ctl->full[s], bytes);
    bulk_g2s(stages + (size_t) s * P.stage_bytes, M.W + a0, bytes, &ctl->full[s], pol);
}
// called by lane 0 of a consumer warp when the warp no longer needs stage s (iteration it): the last of the 8 warps refills it
__device__ __forceinline__ void release_stage(const GemvParams & P, GemvSmemCtl * ctl, uint8_t * stages, int s, int it, uint64_t pol) {
    __threadfence_block();
    if (atomicAdd(&ctl->cnt[s], 1) == P.rel_count - 1) {
        ctl->cnt[s] = 0;
        const int t = blockIdx.x + (it + P.nstage) * gridDim.x;
        if (t < P.ntiles) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy reads of the stage before the async-proxy refill
            issue_tile(P, ctl, stages, s, t, pol);
        }
    }
}

// initial stages that were held back until the activation loads had been issued (P.prefill < P.nstage_init)
__device__ __forceinline__ void fill_rest(const GemvParams & P, GemvSmemCtl * ctl, uint8_t * stages, uint64_t pol) {
    if (threadIdx.x == 0) {
        for (int it = P.prefill; it < P.nstage_init; it++) {
            const int t = blockIdx.x + it * gridDim.x;
            if (t < P.ntiles) issue_tile(P, ctl, stages, it, t, pol);
        }
    }
}

// TYPE = weight type of every matrix of the launch (one dot routine in the hot loop: the three unrolled routines together are
// ~126 KB of SASS, more than the instruction cache holds), or 0 = mixed (q|k|v with a Q5_K / Q6_K v)
template <int TYPE>
__device__ __forceinline__ float dot_block(int type, const uint8_t * bp, const ActRegs & r) {
    if (TYPE == T_Q4_K) return dot_q4K(bp, r);
    if (TYPE == T_Q5_K) return dot_q5K(bp, r);
    if (TYPE == T_Q6_K) return dot_q6K(bp, r);
    if (TYPE == T_Q8_0) return dot_q8_0x8(bp, r);
    if (TYPE == T_Q5_1) return dot_q5_1x8(bp, r);
    if (type == T_Q4_K) return dot_q4K(bp, r);
    if (type == T_Q6_K) return dot_q6K(bp, r);
    return dot_q5K(bp, r);
}

// ---- distributed prologue (PRO_*_DIST): CTA c produces super-blocks c, c + grid, ... of the q8_K activation in P.act ----
__device__ __forceinline__ void dist_prologue(const GemvParams & P, GemvSmemCtl * ctl, int warp, int lane) {
    const int nblk = P.nblk;
    if ((int) blockIdx.x >= nblk) return;                       // nothing to produce: straight to the barrier
    // warp w owns this CTA's w-th block; its operands are requested first so that they travel with the loads of the sum
    const int myblk = (int) blockIdx.x + warp * (int) gridDim.x;
    float bx[8], bw[8];
    if (myblk < nblk) {
        load8(P.in0 + myblk * 256 + lane * 8, bx);
        load8(P.in1 + myblk * 256 + lane * 8, bw);
    }
    float scale = 1.f;
    if (P.prologue == PRO_RMSNORM_DIST) {
        // every producing CTA needs the whole sum of squares (one extra read of the vector per producer: 32 x 32 KB at K = 8192)
        double sum = 0.0;
        if (nblk <= GEMV_NW * PRO_B) {
            float xr[PRO_B][8];
#pragma unroll
            for (int j = 0; j < PRO_B; j++) {
                const int b = warp + j * GEMV_NW;
                if (b < nblk) load8(P.in0 + b * 256 + lane * 8, xr[j]);
            }
#pragma unroll
            for (int j = 0; j < PRO_B; j++) {
                if (warp + j * GEMV_NW < nblk) {
#pragma unroll
                    for (int i = 0; i < 8; i++) sum += (double) __fmul_rn(xr[j][i], xr[j][i]);
                }
            }
        } else {
            for (int i = threadIdx.x; i < P.K; i += GEMV_THREADS) { const float v = __ldcg(P.in0 + i); sum += (double) __fmul_rn(v, v); }
        }
        sum = warp_sum_d(sum);
        if (lane == 0) ctl->red[warp] = sum;
        __syncthreads();
        double t = 0.0;
#pragma unroll
        for (int i = 0; i < GEMV_NW; i++) t += ctl->red[i];
        const float mean = (float) (t / (double) P.K);
        scale = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(mean, P.eps)));
    }
    for (int b = myblk; b < nblk; b += GEMV_NW * (int) gridDim.x) {
        if (b != myblk) { load8(P.in0 + b * 256 + lane * 8, bx); load8(P.in1 + b * 256 + lane * 8, bw); }   // tiny grids only
        if (P.prologue == PRO_RMSNORM_DIST) {
#pragma unroll
            for (int i = 0; i < 8; i++) bx[i] = __fmul_rn(__fmul_rn(bx[i], scale), bw[i]);
        } else {
#pragma unroll
            for (int i = 0; i < 8; i++) bx[i] = __fmul_rn(silu_f(bx[i]), bw[i]);
        }
        quantize_warp_q8K(bx, lane, b, P.act);
    }
}
// All CTAs of the launch meet once.  Safe because the persistent grid is co-resident by construction (launcher: grid <= 2 x SMs,
// gemv_dist_prologue_ok()); bounded like every other wait.  State = {arrivals, departures}; the last CTA to leave re-arms both.
__device__ __forceinline__ void grid_barrier(const GemvParams & P, GemvSmemCtl * ctl) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(P.gbar, 1u);
        const unsigned target = gridDim.x;
        const long long t0 = clock64();
        unsigned v;
        int spins = 0;
        do {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(P.gbar) : "memory");
            if (v < target && (++spins & 63) == 0) {
                if (ctl->aborted) break;
                if (clock64() - t0 > PB_WAIT_TIMEOUT_CYCLES) { wait_gave_up(&ctl->aborted, P.abort_flag); break; }
            }
        } while (v < target);
        if (atomicAdd(P.gbar + 1, 1u) == target - 1) {   // everybody has seen the full count
            P.gbar[1] = 0u;
            __threadfence();
            P.gbar[0] = 0u;
        }
    }
    __syncthreads();
}

// split rows (wpr > 1): the leader warp's row whose partials are still being collected
struct PendingRow { bool active; int q; uint64_t tok; float v, extra; float * y; };
__device__ __forceinline__ void finish_split_row(const GemvParams & P, GemvSmemCtl * ctl, const PendingRow & pr, int group, int wpr, int lane) {
    const uint64_t tok = __shfl_sync(0xffffffffu, pr.tok, 0);
    mbar_wait_token(&ctl->pbar[pr.q][group], tok, &ctl->aborted, P.abort_flag);
    if (lane == 0) {
        float acc = pr.v;
        for (int i = 1; i < wpr; i++) acc += ctl->part[pr.q][group * wpr + i];
        *pr.y = acc + pr.extra;
    }
}

template <int TYPE, bool SPLIT, bool TRACE>
__global__ void __launch_bounds__(GEMV_THREADS, GEMV_CTAS_PER_SM) k_gemv_kquant(const __grid_constant__ GemvParams P) {
    extern __shared__ __align__(128) uint8_t smem[];
    GemvSmemCtl * ctl = reinterpret_cast<GemvSmemCtl *>(smem);
    uint8_t * stages = smem + GEMV_CTL_BYTES;
    // the activation staging area is dead once every lane holds its super-block in registers: it doubles as the last ring stages
    uint8_t * act_smem = stages + (size_t) P.nstage_init * P.stage_bytes;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    stamp<TRACE>(P, 0);
    const uint64_t pol = policy_evict_first();
    if (threadIdx.x == 0) {
        for (int s = 0; s < P.nstage; s++) {
            mbar_init(&ctl->full[s], 1);
            ctl->cnt[s] = 0;
        }
        if (SPLIT) {
#pragma unroll
            for (int q = 0; q < GEMV_ROWQ; q++)
#pragma unroll
                for (int g = 0; g < 4; g++) mbar_init(&ctl->pbar[q][g], P.wpr);
        }
        ctl->aborted = 0;
        mbar_fence_init();
    }
    __syncthreads();
    pdl_trigger();   // the next kernel's CTAs may take this SM's free slots as soon as CTAs of this grid exit
    // Weights never depend on the previous kernel: start streaming BEFORE griddepcontrol.wait.  Under PDL this CTA is resident
    // while the tail of the previous GEMV (or a whole small kernel: attention, silu-quant) still runs on other SMs.
    if (threadIdx.x == 0) {
        for (int it = 0; it < P.prefill; it++) {
            const int t = blockIdx.x + it * gridDim.x;
            if (t < P.ntiles) issue_tile(P, ctl, stages, it, t, pol);
        }
    }
    stamp<TRACE>(P, 1);
    pdl_wait();      // the activation is produced by the previous kernel in the stream
    stamp<TRACE>(P, 2);

    const int wpr = SPLIT ? P.wpr : 1;
    const int ngroups = GEMV_NW / wpr;
    const int group = warp / wpr, wsub = warp % wpr;
    // short rows (nblk <= 16, e.g. K = 4096 of Llama-3-8B): a warp holds 32 / nblk_p2 rows side by side, lane = (row in the slot, super-block)
    const int nbp = SPLIT ? 32 : P.nblk_p2, rpw = 32 / nbp;
    const int rsh = SPLIT ? 0 : 31 - __clz(rpw);   // rpw is a power of two: the per-stage row-slot arithmetic below uses shifts (two integer divisions per stage visit before)
    const int sub = SPLIT ? 0 : lane / nbp;
    const int blk = SPLIT ? wsub * 32 + lane : (lane & (nbp - 1));
    const bool valid = blk < P.nblk;

    ActRegs r;
    ActQ sa;   // the CTA's activation in shared memory: qs[K] | bsums[K/16] i16 | d[K/256] f32   (padded strides, common.cuh)
    sa.qs = reinterpret_cast<int8_t *>(act_smem);
    sa.bsums = reinterpret_cast<int16_t *>(act_smem + P.nblk * ACT_SMEM_QS_STRIDE);
    sa.d = reinterpret_cast<float *>(act_smem + P.nblk * (ACT_SMEM_QS_STRIDE + 2 * ACT_SMEM_BS_STRIDE));
    sa.s = nullptr;
    sa.qs_stride = ACT_SMEM_QS_STRIDE;
    sa.bs_stride = ACT_SMEM_BS_STRIDE;
    const bool dist = P.prologue == PRO_RMSNORM_DIST || P.prologue == PRO_SILU_DIST;
    if (dist) {
        dist_prologue(P, ctl, warp, lane);
        grid_barrier(P, ctl);
    }
    constexpr bool BLK32 = TYPE == T_Q8_0 || TYPE == T_Q5_1;
    if (BLK32) {
        // q8_0 / q8_1 activation (qs[K] | d[K/32] | s[K/32]): columns of 8 blocks, qs with the padded column stride, the scales dense
        // (8 floats per column) behind them
        float * sd = reinterpret_cast<float *>(act_smem + P.nblk * ACT_SMEM_QS_STRIDE);
        float * ss = sd + P.nblk * 8;
        const int nq = P.K / 16, nb32 = P.K / 32;
        for (int i = threadIdx.x; i < nq; i += GEMV_THREADS)
            *reinterpret_cast<int4 *>(sa.qs + (i >> 4) * ACT_SMEM_QS_STRIDE + (i & 15) * 16) = __ldcg(reinterpret_cast<const int4 *>(P.act.qs) + i);
        for (int i = threadIdx.x; i < P.nblk * 8; i += GEMV_THREADS) {
            sd[i] = i < nb32 ? __ldcg(P.act.d + i) : 0.f;
            if (TYPE == T_Q5_1) ss[i] = i < nb32 ? __ldcg(P.act.s + i) : 0.f;
        }
        fill_rest(P, ctl, stages, pol);
        __syncthreads();
        r.nb = valid ? min(8, nb32 - 8 * blk) : 0;
        if (valid) {
            const int4 * q = reinterpret_cast<const int4 *>(sa.qs + blk * ACT_SMEM_QS_STRIDE);
            const int nq4 = r.nb * 2;                                  // the blocks that exist: 2 x 16 bytes each
#pragma unroll
            for (int i = 0; i < 16; i++) {
                int4 v = make_int4(0, 0, 0, 0);
                if (i < nq4) v = q[i];
                r.a[4 * i + 0] = v.x; r.a[4 * i + 1] = v.y; r.a[4 * i + 2] = v.z; r.a[4 * i + 3] = v.w;
            }
#pragma unroll
            for (int j = 0; j < 8; j++) { r.d8[j] = sd[blk * 8 + j]; r.s8[j] = TYPE == T_Q5_1 ? ss[blk * 8 + j] : 0.f; }
        }
    } else {
        // ONE coalesced copy of the quantized activation per CTA (qs | bsums | d), staged with the padded strides
        constexpr int NQ_MAX = (GEMV_ACT_MAX_NBLK * 16 + GEMV_THREADS - 1) / GEMV_THREADS;   // int4 of qs per thread (7)
        const int nq = P.K / 16, nb16 = P.K / 128;
        int4 cq[NQ_MAX], cb;
        float cd = 0.f;
#pragma unroll
        for (int j = 0; j < NQ_MAX; j++) {
            const int i = threadIdx.x + j * GEMV_THREADS;
            if (i < nq) cq[j] = __ldcg(reinterpret_cast<const int4 *>(P.act.qs) + i);
        }
        if ((int) threadIdx.x < nb16) cb = __ldcg(reinterpret_cast<const int4 *>(P.act.bsums) + threadIdx.x);
        if ((int) threadIdx.x < P.nblk) cd = __ldcg(P.act.d + threadIdx.x);
        fill_rest(P, ctl, stages, pol);   // the small activation loads are out: they do not queue behind the rest of the ring fill
#pragma unroll
        for (int j = 0; j < NQ_MAX; j++) {
            const int i = threadIdx.x + j * GEMV_THREADS;
            if (i < nq) *reinterpret_cast<int4 *>(sa.qs + (i >> 4) * ACT_SMEM_QS_STRIDE + (i & 15) * 16) = cq[j];
        }
        if ((int) threadIdx.x < nb16) *reinterpret_cast<int4 *>(reinterpret_cast<char *>(sa.bsums) + (threadIdx.x >> 1) * (2 * ACT_SMEM_BS_STRIDE) + (threadIdx.x & 1) * 16) = cb;
        if ((int) threadIdx.x < P.nblk) sa.d[threadIdx.x] = cd;
        __syncthreads();
        load_act_regs(r, sa, blk, valid);
        finish_act_regs(r);
    }
    if (P.nstage_init < P.nstage) {
        __syncthreads();   // every warp has its registers: hand the staging area to the ring
        if (threadIdx.x == 0) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            for (int it = P.nstage_init; it < P.nstage; it++) {
                const int t = blockIdx.x + it * gridDim.x;
                if (t < P.ntiles) issue_tile(P, ctl, stages, it, t, pol);
            }
        }
    }
    stamp<TRACE>(P, 3);

    // Every warp visits every iteration in order (so a parity wait can never be satisfied by an older phase of the same stage);
    // row `slot` of iteration `it` belongs to warp group (it * rows_per_tile + slot) mod ngroups.
    PendingRow pend;
    pend.active = false;
    int grow = 0;   // rows this warp group has processed (split rows)
    int s = 0;
    uint32_t ph = 0;
    for (int it = 0, t = blockIdx.x; t < P.ntiles; t += gridDim.x, it++, s = (s + 1 == P.nstage ? 0 : s + 1), ph ^= (s == 0 ? 1u : 0u)) {
        int m, r0, nrows;
        tile_info(P, t, m, r0, nrows);
        const GemvMat & M = P.mat[m];
        const int type = TYPE ? TYPE : M.type;
        const int bpb = type == T_Q4_K ? BYTES_Q4_K : type == T_Q5_K ? BYTES_Q5_K : type == T_Q6_K ? BYTES_Q6_K : type == T_Q8_0 ? 8 * BYTES_Q8_0 : 8 * BYTES_Q5_1;
        const uint32_t mis = (uint32_t) (((int64_t) r0 * M.row_bytes) & 15);
        const uint8_t * tile = stages + (size_t) s * P.stage_bytes + mis;
        const int spt = M.rows_per_tile >> rsh;                                                // row slots per tile (a slot = rpw rows, one per sub-warp)
        const int first = (group - it * spt) & (ngroups - 1);                                 // this group's first slot in the stage
        if (P.owner_only && first >= spt) continue;   // not an owner of this stage (stable per stage: see gemv_plan)
        mbar_wait(&ctl->full[s], ph, &ctl->aborted, P.abort_flag);
        if (TRACE && it == 0) stamp<TRACE>(P, 4);
        if (!SPLIT) {
            const int nslots = (nrows + rpw - 1) >> rsh;
            for (int slot = first; slot < nslots; slot += ngroups) {
                const int rit = slot * rpw + sub;                 // row inside the tile
                const int row = r0 + rit;
                const bool has_row = rit < nrows;
                const bool writer = (lane & (nbp - 1)) == 0 && has_row;
                // epilogue operands are requested before the dot so that their L2 latency is off the critical path
                float extra = 0.f;
                if (writer) {
                    if (M.bias) extra = M.bias[row];
                    if (M.resid) extra += __ldcg(M.resid + row);
                }
                float v = 0.f;
                if (valid && has_row) v = dot_block<TYPE>(type, tile + (size_t) rit * M.row_bytes + (size_t) blk * bpb, r);
                if (slot + ngroups >= nslots) {
                    // last row of this stage for this warp: hand the buffer back before reducing
                    __syncwarp();
                    if (lane == 0) release_stage(P, ctl, stages, s, it, pol);
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1)
                    if (o < nbp) v += __shfl_xor_sync(0xffffffffu, v, o);      // reduce inside the sub-warp of the row
                if (writer) M.y[row] = v + extra;
            }
            if (first >= nslots) {   // no row for this warp in the stage: still release it
                __syncwarp();
                if (lane == 0) release_stage(P, ctl, stages, s, it, pol);
            }
        } else {
            // Rows split over wpr warps; rows_per_tile <= ngroups, i.e. at most one row per warp group and stage.  Every warp hands the
            // stage back right after its dot (the ring keeps its full depth); the partial sums travel through part[q] / pbar[q] with
            // q = the group's row count mod GEMV_ROWQ.  Non-leaders publish and move on; the leader finishes row r-1 (which arrived
            // long ago) just before it releases the stage of row r, so a non-leader that has passed the wait of row r+nstage knows that
            // row r-1 has been read: slots are reused GEMV_ROWQ = 8 > nstage rows later at the earliest.
            const int slot = first;
            if (slot >= nrows) {   // this group has no row in the stage
                __syncwarp();
                if (lane == 0) release_stage(P, ctl, stages, s, it, pol);
                continue;
            }
            const int row = r0 + slot;
            const bool lead = wsub == 0;
            const int q = grow & (GEMV_ROWQ - 1);
            grow++;
            float extra = 0.f;
            if (lead && lane == 0) {
                if (M.bias) extra = M.bias[row];
                if (M.resid) extra += __ldcg(M.resid + row);
            }
            float v = 0.f;
            if (valid) v = dot_block<TYPE>(type, tile + (size_t) slot * M.row_bytes + (size_t) blk * bpb, r);
            if (!lead) {
                __syncwarp();
                if (lane == 0) release_stage(P, ctl, stages, s, it, pol);
                v = warp_sum(v);
                if (lane == 0) {
                    ctl->part[q][warp] = v;
                    mbar_arrive(&ctl->pbar[q][group]);   // release semantics: the partial is visible to the waiter
                }
            } else {
                if (pend.active) finish_split_row(P, ctl, pend, group, wpr, lane);
                __syncwarp();
                if (lane == 0) release_stage(P, ctl, stages, s, it, pol);
                v = warp_sum(v);
                uint64_t tok = 0;
                if (lane == 0) tok = mbar_arrive_token(&ctl->pbar[q][group]);
                pend.active = true; pend.q = q; pend.tok = tok; pend.v = v; pend.extra = extra; pend.y = M.y + row;
            }
        }
    }
    if (SPLIT && pend.active) finish_split_row(P, ctl, pend, group, wpr, lane);
    stamp<TRACE>(P, 5);
}

// ---------------------------------------------------------------------------------------------------------------
// Generic fallback: one warp per row, direct global loads, every supported type (incl. the 32-element block types
// Q8_0 / Q5_1 that Qwen2.5-72B's ffn_down falls back to, src/llama.cpp:19516-19551), any K.
// Follows ggml_vec_dot_q8_0_q8_0 (ggml-quants.c:5518) and ggml_vec_dot_q5_1_q8_1 (:5144).
__device__ __forceinline__ uint32_t ld_u16x2(const uint8_t * p) {   // 2-B aligned 32-bit read
    const uint16_t * q = reinterpret_cast<const uint16_t *>(p);
    return (uint32_t) q[0] | ((uint32_t) q[1] << 16);
}

struct GemvGenericParams {
    const uint8_t * W;
    float * y;
    const float * bias;
    const float * resid;
    int64_t row_bytes;
    int type, N, K;
    ActQ act;
};

__global__ void __launch_bounds__(256) k_gemv_generic(const __grid_constant__ GemvGenericParams P) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int row = blockIdx.x * 8 + warp;
    pdl_trigger();   // dependents may launch now; they still wait for this grid's completion in their own pdl_wait()
    pdl_wait();
    if (row >= P.N) return;
    const uint8_t * wrow = P.W + (int64_t) row * P.row_bytes;
    float acc = 0.f;
    if (P.type == T_Q8_0) {
        const int nb = P.K / 32;
        for (int b = lane; b < nb; b += 32) {
            const uint8_t * bp = wrow + (int64_t) b * BYTES_Q8_0;
            const float d = __half2float(__ushort_as_half(*reinterpret_cast<const uint16_t *>(bp)));
            const int4 * a = reinterpret_cast<const int4 *>(P.act.qs + (int64_t) b * 32);
            const int4 a0 = a[0], a1 = a[1];
            const int av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            int sumi = 0;
#pragma unroll
            for (int i = 0; i < 8; i++) sumi = dp4a_ss((int) ld_u16x2(bp + 2 + 4 * i), av[i], sumi);
            acc += (float) sumi * (d * P.act.d[b]);
        }
    } else if (P.type == T_Q5_1) {
        const int nb = P.K / 32;
        for (int b = lane; b < nb; b += 32) {
            const uint8_t * bp = wrow + (int64_t) b * BYTES_Q5_1;   // 24 B: 8-B aligned rows, 4-B aligned fields
            const uint32_t dmw = *reinterpret_cast<const uint32_t *>(bp);
            const float d = __half2float(__ushort_as_half((unsigned short) (dmw & 0xffff)));
            const float mm = __half2float(__ushort_as_half((unsigned short) (dmw >> 16)));
            const uint32_t qh = *reinterpret_cast<const uint32_t *>(bp + 4);
            const int4 * a = reinterpret_cast<const int4 *>(P.act.qs + (int64_t) b * 32);
            const int4 a0 = a[0], a1 = a[1];
            const int av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            int sumi = 0;
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const uint32_t w = *reinterpret_cast<const uint32_t *>(bp + 8 + 4 * i);   // qs bytes 4i..4i+3
                // element j = 4i+k (low nibble) gets bit j of qh; element j+16 (high nibble) gets bit j+16
                uint32_t hb_lo = 0, hb_hi = 0;
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    hb_lo |= ((qh >> (4 * i + k)) & 1u) << (8 * k + 4);
                    hb_hi |= ((qh >> (4 * i + k + 16)) & 1u) << (8 * k + 4);
                }
                sumi = dp4a_us((w & 0x0f0f0f0fu) | hb_lo, av[i], sumi);
                sumi = dp4a_us(((w >> 4) & 0x0f0f0f0fu) | hb_hi, av[4 + i], sumi);
            }
            acc += (d * P.act.d[b]) * (float) sumi + mm * P.act.s[b];
        }
    } else {
        // k-quants without shared-memory staging (used when K > 65 536 or for tiny problems)
        const int nb = P.K / 256;
        for (int b = lane; b < nb; b += 32) {
            ActRegs r;
            load_act_regs(r, P.act, b, true);
            finish_act_regs(r);
            // stage the block through registers -> local array is avoided by reading global memory directly with the
            // same dot routines: they only need byte-addressable memory with the block's natural alignment.
            const int bpb = P.type == T_Q4_K ? BYTES_Q4_K : (P.type == T_Q5_K ? BYTES_Q5_K : BYTES_Q6_K);
            const uint8_t * bp = wrow + (int64_t) b * bpb;
            // dot_q6K uses shared-memory addressing for its alignment probe; use the global-memory variant below
            if (P.type == T_Q4_K && ((uintptr_t) bp & 15) == 0) acc += dot_q4K(bp, r);
            else if (P.type == T_Q5_K && ((uintptr_t) bp & 15) == 0) acc += dot_q5K(bp, r);
            else {
                // byte-wise scalar path (rare): dequantize on the fly against int8 activations
                const int8_t * a8 = P.act.qs + (int64_t) b * 256;
                if (P.type == T_Q6_K) {
                    const float d = __half2float(__ushort_as_half(*reinterpret_cast<const uint16_t *>(bp + 208)));
                    const int8_t * sc = reinterpret_cast<const int8_t *>(bp + 192);
                    int sumi = 0;
                    for (int n = 0; n < 2; n++)
                        for (int l = 0; l < 32; l++) {
                            const uint8_t qa = bp[64 * n + l], qb = bp[64 * n + 32 + l], h = bp[128 + 32 * n + l];
                            const int is = l / 16;
                            const int q1 = (int) ((qa & 0xF) | (((h >> 0) & 3) << 4)) - 32;
                            const int q2 = (int) ((qb & 0xF) | (((h >> 2) & 3) << 4)) - 32;
                            const int q3 = (int) ((qa >> 4) | (((h >> 4) & 3) << 4)) - 32;
                            const int q4 = (int) ((qb >> 4) | (((h >> 6) & 3) << 4)) - 32;
                            sumi += sc[8 * n + is + 0] * q1 * a8[128 * n + l] + sc[8 * n + is + 2] * q2 * a8[128 * n + 32 + l] +
                                    sc[8 * n + is + 4] * q3 * a8[128 * n + 64 + l] + sc[8 * n + is + 6] * q4 * a8[128 * n + 96 + l];
                        }
                    acc += (d * r.d) * (float) sumi;
                } else {
                    const bool q5 = P.type == T_Q5_K;
                    const __half2 dm = *reinterpret_cast<const __half2 *>(bp);
                    const uint8_t * scb = bp + 4;
                    const uint8_t * qhb = bp + 16;
                    const uint8_t * qs = bp + (q5 ? 48 : 16);
                    int sumi = 0, summ = 0;
                    for (int j = 0; j < 8; j++) {
                        int sc, mn;
                        if (j < 4) { sc = scb[j] & 63; mn = scb[j + 4] & 63; }
                        else { sc = (scb[j + 4] & 0xF) | ((scb[j - 4] >> 6) << 4); mn = (scb[j + 4] >> 4) | ((scb[j] >> 6) << 4); }
                        int dsum = 0, asum = 0;
                        for (int l = 0; l < 32; l++) {
                            const uint8_t byte = qs[32 * (j / 2) + l];
                            int q = (j & 1) ? (byte >> 4) : (byte & 0xF);
                            if (q5 && ((qhb[l] >> j) & 1)) q += 16;
                            const int a = a8[32 * j + l];
                            dsum += q * a;
                            asum += a;
                        }
                        sumi += sc * dsum;
                        summ += mn * asum;
                    }
                    acc += (__low2float(dm) * r.d) * (float) sumi - (__high2float(dm) * r.d) * (float) summ;
                }
            }
        }
    }
    acc = warp_sum(acc);
    if (lane == 0) {
        if (P.bias) acc += P.bias[row];
        if (P.resid) acc += P.resid[row];
        P.y[row] = acc;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Streaming GEMV for the 32-element block types (Q8_0 34 B, Q5_1 24 B per block): Qwen2.5-72B's ffn_down (K = 29 568, not a
// multiple of 256) falls back to them (src/llama.cpp:19516-19551) and they are a third of that model's bytes.
// The activation (q8_0 / q8_1) is staged once per CTA in shared memory; every warp streams whole rows through its own 4-deep
// cp.async ring of 32-block chunks (8-byte pieces, all lanes issue, ~100 KB in flight per SM at 3 CTAs/SM); lane l owns block
// l of every chunk, i.e. the same blocks and the same per-lane order as k_gemv_generic => bit-identical results.
constexpr int B32_NST = 4;
struct GemvB32Params {
    const uint8_t * W;
    float * y;
    const float * bias;
    const float * resid;
    int64_t row_bytes;
    int type, N, K, nb, bpb;
    ActQ act;
};
__global__ void __launch_bounds__(256) k_gemv_blk32(const __grid_constant__ GemvB32Params P) {
    extern __shared__ __align__(16) uint8_t b32_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int kp = (P.K + 15) & ~15;
    int8_t * a_qs = reinterpret_cast<int8_t *>(b32_smem);                        // [K]
    float * a_d = reinterpret_cast<float *>(b32_smem + kp);                      // [nb]
    float * a_s = a_d + P.nb;                                                    // [nb]  (Q5_1 only)
    const int cb = 32 * P.bpb;                                                   // chunk bytes: 1088 / 768
    uint8_t * ring = b32_smem + ((kp + 8 * P.nb + 15) & ~15) + (size_t) warp * B32_NST * 1088;
    pdl_trigger();
    pdl_wait();
    for (int i = threadIdx.x; i < P.K / 16; i += 256) reinterpret_cast<int4 *>(a_qs)[i] = reinterpret_cast<const int4 *>(P.act.qs)[i];
    for (int i = threadIdx.x; i < P.nb; i += 256) { a_d[i] = P.act.d[i]; if (P.type == T_Q5_1) a_s[i] = P.act.s[i]; }
    __syncthreads();
    const int nchunk = (P.nb + 31) / 32;
    const int pieces = cb / 8;
    for (int row = blockIdx.x * 8 + warp; row < P.N; row += gridDim.x * 8) {
        const uint8_t * wrow = P.W + (int64_t) row * P.row_bytes;
        auto issue = [&](int c) {
            if (c < nchunk) {
                const int64_t off = (int64_t) c * cb;
                uint8_t * dst = ring + (size_t) (c % B32_NST) * 1088;
                for (int pc = lane; pc < pieces; pc += 32)
                    if (off + pc * 8 + 8 <= P.row_bytes)
                        asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(dst + pc * 8)), "l"(wrow + off + pc * 8) : "memory");
            }
            asm volatile("cp.async.commit_group;" ::: "memory");
        };
        for (int c = 0; c < B32_NST - 1; c++) issue(c);
        float acc = 0.f;
        for (int c = 0; c < nchunk; c++) {
            issue(c + B32_NST - 1);
            asm volatile("cp.async.wait_group %0;" ::"n"(B32_NST - 1) : "memory");
            __syncwarp();
            const int b = c * 32 + lane;
            if (b < P.nb) {
                const uint8_t * bp = ring + (size_t) (c % B32_NST) * 1088 + lane * P.bpb;
                const int4 * a = reinterpret_cast<const int4 *>(a_qs + (int64_t) b * 32);
                const int4 a0 = a[0], a1 = a[1];
                const int av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
                int sumi = 0;
                if (P.type == T_Q8_0) {
                    // 34-byte blocks are only 2-byte aligned: read the 9 aligned words around the block; qs (offset 2) is either
                    // word-aligned already (block at 4k+2) or straddles two words (block at 4k): one PRMT per word, selector per lane
                    const uint32_t * wp = reinterpret_cast<const uint32_t *>(reinterpret_cast<uintptr_t>(bp) & ~(uintptr_t) 3);
                    const bool odd = (reinterpret_cast<uintptr_t>(bp) & 2) != 0;
                    const uint32_t sel = odd ? 0x7654u : 0x5432u;
                    uint32_t w[9];
#pragma unroll
                    for (int i = 0; i < 9; i++) w[i] = wp[i];
                    const float d = __half2float(__ushort_as_half((unsigned short) ((w[0] >> (odd ? 16 : 0)) & 0xffff)));
#pragma unroll
                    for (int i = 0; i < 8; i++) sumi = dp4a_ss((int) __byte_perm(w[i], w[i + 1], sel), av[i], sumi);
                    acc += (float) sumi * (d * a_d[b]);
                } else {
                    const uint32_t dmw = *reinterpret_cast<const uint32_t *>(bp);
                    const float d = __half2float(__ushort_as_half((unsigned short) (dmw & 0xffff)));
                    const float mm = __half2float(__ushort_as_half((unsigned short) (dmw >> 16)));
                    const uint32_t qh = *reinterpret_cast<const uint32_t *>(bp + 4);
#pragma unroll
                    for (int i = 0; i < 4; i++) {
                        const uint32_t w = *reinterpret_cast<const uint32_t *>(bp + 8 + 4 * i);
                        // bit k of a nibble of qh -> bit 4 of byte k: x * 0x00204081 puts bit k at 8k (no carries), then << 4
                        const uint32_t hb_lo = ((((qh >> (4 * i)) & 0xFu) * 0x00204081u) & 0x01010101u) << 4;
                        const uint32_t hb_hi = ((((qh >> (4 * i + 16)) & 0xFu) * 0x00204081u) & 0x01010101u) << 4;
                        sumi = dp4a_us((w & 0x0f0f0f0fu) | hb_lo, av[i], sumi);
                        sumi = dp4a_us(((w >> 4) & 0x0f0f0f0fu) | hb_hi, av[4 + i], sumi);
                    }
                    acc += (d * a_d[b]) * (float) sumi + mm * a_s[b];
                }
            }
            __syncwarp();   // the slot is refilled by the next issue()
        }
        asm volatile("cp.async.wait_all;" ::: "memory");
        acc = warp_sum(acc);
        if (lane == 0) {
            if (P.bias) acc += P.bias[row];
            if (P.resid) acc += P.resid[row];
            P.y[row] = acc;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// host side.  Everything cached here is keyed by device: cudaFuncSetAttribute and the SM count are per-device properties and
// one process may drive several devices through the ggml plugin (ggml_backend_b200_reg registers every CUDA device).
int cur_device() {
    int dev = 0;
    cudaGetDevice(&dev);
    return (dev >= 0 && dev < PB_MAX_DEV) ? dev : 0;
}
int sm_count() {
    static int cache[PB_MAX_DEV] = {0};
    const int dev = cur_device();
    if (!cache[dev]) cudaDeviceGetAttribute(&cache[dev], cudaDevAttrMultiProcessorCount, dev);
    return cache[dev];
}
cudaError_t ensure_dyn_smem(FuncAttrCache & c, const void * fn, size_t bytes, bool max_carveout) {
    const int dev = cur_device();
    if (bytes <= c.bytes[dev]) return cudaSuccess;
    if (bytes > 48 * 1024 || max_carveout) {
        cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) std::max<size_t>(bytes, 48 * 1024));
        if (e != cudaSuccess) return e;
        if (max_carveout) {
            e = cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, (int) cudaSharedmemCarveoutMaxShared);
            if (e != cudaSuccess) return e;
        }
    }
    c.bytes[dev] = bytes;
    return cudaSuccess;
}
// process-wide abort flag of the wait watchdogs: pinned, mapped host memory (UVA: same address on every device)
static int * g_abort_flag = nullptr;
int * abort_flag() {
    static bool tried = false;
    if (!tried) {
        tried = true;
        void * p = nullptr;
        if (cudaHostAlloc(&p, 64, cudaHostAllocMapped | cudaHostAllocPortable) == cudaSuccess) {
            g_abort_flag = (int *) p;
            *g_abort_flag = 0;
        } else {
            cudaGetLastError();
        }
    }
    return g_abort_flag;
}
int check_clear_abort() {
    int * f = abort_flag();
    if (!f || !*(volatile int *) f) return 0;
    *(volatile int *) f = 0;
    return 1;
}

// profiling: device buffer of `slots` rows of u64[GEMV_TRACE_ROW]; launch i writes row i % slots.  TRACE instantiation when set.
constexpr int GEMV_TRACE_ROW = 4096;
static unsigned long long * g_trace_buf = nullptr;
static int g_trace_slots = 0;
static uint64_t g_trace_idx = 0;
int gemv_set_trace(unsigned long long * dev_buf, int slots) {
    g_trace_buf = slots > 0 ? dev_buf : nullptr;
    g_trace_slots = slots;
    g_trace_idx = 0;
    return 0;
}

bool gemv_fused_prologue_ok(int K) { return K > 0 && K % 256 == 0 && K / 256 <= GEMV_ACT_MAX_NBLK; }

// ring geometry of one launch: rows per tile of each matrix, stage size, depth — everything that must fit 2 CTAs on an SM
struct GemvPlan { int wpr, nblk_p2, nstage, nstage_init, stage_bytes, smem, owner_only, rel_count, rows[GEMV_MAX_MAT]; };
// tunables (environment, read once): ring geometry experiments without a rebuild
struct GemvTune { int stage_target, max_stage, prefill; };
static const GemvTune tune = [] {
    GemvTune t{GEMV_STAGE_TARGET, GEMV_MAX_STAGE, GEMV_MAX_STAGE};
    if (const char * e = getenv("PB200_GEMV_STAGE_KB")) t.stage_target = std::max(4, atoi(e)) * 1024;
    if (const char * e = getenv("PB200_GEMV_PREFILL")) t.prefill = std::max(0, atoi(e));
    if (const char * e = getenv("PB200_GEMV_MAX_STAGE")) t.max_stage = std::min(GEMV_MAX_STAGE, std::max(2, atoi(e)));
    return t;
}();
static bool is_blk32(int t) { return t == T_Q8_0 || t == T_Q5_1; }
static bool gemv_plan(const int * types, const int * Ns, int nmat, int K, GemvPlan & pl) {
    // k-quants: K a multiple of 256; 32-element block types (one matrix per launch): K a multiple of 32, columns of 8 blocks
    const bool b32 = nmat == 1 && is_blk32(types[0]);
    if (b32 ? !(K > 0 && K % 32 == 0 && (K + 255) / 256 <= GEMV_ACT_MAX_NBLK) : !gemv_fused_prologue_ok(K)) return false;
    const int nblk = (K + 255) / 256;
    int wpr = 1;
    while (wpr * 32 < nblk) wpr *= 2;
    const int ngroups = GEMV_NW / wpr;
    int nbp = 1;
    while (nbp < nblk && nbp < 32) nbp *= 2;
    const int rpw = wpr > 1 ? 1 : 32 / nbp;          // rows a warp holds side by side (short rows)
    pl.nblk_p2 = nbp;
    int64_t biggest = 0;
    for (int i = 0; i < nmat; i++) {
        if (!(is_kquant(types[i]) || b32) || Ns[i] < 1) return false;
        const int64_t rb = row_bytes(types[i], K);
        if (b32 && rb % 8 != 0) return false;          // the column dots read 64-bit words
        int R = (int) std::max<int64_t>(1, tune.stage_target / rb);
        R = std::max(rpw, R / rpw * rpw);              // whole slots
        if (wpr > 1) {                             // split rows: at most one row per warp group and stage, and a ring of >= 4 stages
            R = std::min(R, ngroups);
            while (R > 1 && (GEMV_SMEM_LIMIT - GEMV_CTL_BYTES) / ((R * rb + 16 + 127) / 128 * 128) < 5) R--;
        }
        if (R > Ns[i]) R = (Ns[i] + rpw - 1) / rpw * rpw;   // (ragged rows of the last slot are masked in the kernel)
        pl.rows[i] = R;
        biggest = std::max<int64_t>(biggest, R * rb);
    }
    pl.wpr = wpr;
    pl.stage_bytes = (int) ((biggest + 16 + 127) / 128 * 128);
    // the activation staging area overlays the last stages of the ring (they are filled once the activation is in registers)
    const int act = gemv_act_smem_bytes(nblk);
    const int act_stages = (act + pl.stage_bytes - 1) / pl.stage_bytes;
    pl.nstage = std::min(tune.max_stage, (GEMV_SMEM_LIMIT - GEMV_CTL_BYTES) / pl.stage_bytes);
    if (pl.nstage >= GEMV_ROWQ) pl.nstage = GEMV_ROWQ - 1;   // split rows reuse their partial-sum slots GEMV_ROWQ rows later (see the kernel)
    // Owner-only visits: row slot j of iteration it belongs to group (it * R + j) mod ngroups; with a common R that pattern has
    // period ngroups / gcd(ngroups, R) in `it`, so if the ring depth is a multiple of it every stage is always consumed by the same
    // warps and the others never touch it (saves their wait + release: 1/4 of the instructions of a split-row launch).
    pl.owner_only = 0;
    pl.rel_count = GEMV_NW;
    {
        bool same = true;
        for (int i = 1; i < nmat; i++) same = same && pl.rows[i] == pl.rows[0];
        const int R = pl.rows[0] / rpw;          // row slots per tile
        if (same && R < ngroups && !getenv("PB200_GEMV_VISIT_ALL")) {
            int g = R, b = ngroups;
            while (b) { const int t = g % b; g = b; b = t; }
            const int period = ngroups / g;
            const int ns = pl.nstage / period * period;
            if (ns >= 3 && ns - act_stages >= 2) {
                pl.nstage = ns;
                pl.owner_only = 1;
                pl.rel_count = R * wpr;
            }
        }
    }
    pl.nstage_init = pl.nstage - act_stages;
    if (pl.nstage_init < (b32 ? 1 : 2)) return false;   // (31-KB Q8_0 rows: a ring of 3, one stage before the activation is in registers)
    pl.smem = GEMV_CTL_BYTES + pl.nstage * pl.stage_bytes;
    return true;
}
bool gemv_dist_prologue_ok() {
    static int cache[PB_MAX_DEV] = {0};   // 0 unknown, 1 yes, 2 no
    const int dev = cur_device();
    if (!cache[dev]) {
        int per_sm = 0;
        static FuncAttrCache tmp;
        bool ok = ensure_dyn_smem(tmp, (const void *) k_gemv_kquant<T_Q4_K, false, false>, GEMV_SMEM_LIMIT, true) == cudaSuccess &&
                  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_gemv_kquant<T_Q4_K, false, false>, GEMV_THREADS, GEMV_SMEM_LIMIT) == cudaSuccess &&
                  per_sm >= GEMV_CTAS_PER_SM;
        if (!ok) cudaGetLastError();
        cache[dev] = ok ? 1 : 2;
    }
    return cache[dev] == 1;
}
int gemv_smem_bytes(int type, int K, int N) {
    GemvPlan pl;
    return gemv_plan(&type, &N, 1, K, pl) ? pl.smem : 0;
}

// Fused launch of up to 3 k-quant matrices sharing one q8_K activation.  Returns cudaError_t as int.
int launch_gemv_kquant(const GemvDesc * d, int nmat, int K, const ActQ & act, cudaStream_t stream, bool pdl) {
    GemvFused none{};
    return launch_gemv_kquant_fused(d, nmat, K, act, none, stream, pdl);
}

int launch_gemv_kquant_fused(const GemvDesc * d, int nmat, int K, const ActQ & act, const GemvFused & pro, cudaStream_t stream, bool pdl) {
    const bool b32 = nmat == 1 && is_blk32(d[0].type);   // Q8_0 / Q5_1 (act: q8_0 / q8_1): same ring, columns of 8 blocks, no fused prologue
    if (nmat < 1 || nmat > GEMV_MAX_MAT || K <= 0 || (b32 ? K % 32 != 0 : K % 256 != 0)) return (int) cudaErrorInvalidValue;
    if (b32 && pro.kind != PRO_NONE) return (int) cudaErrorInvalidValue;
    int types[GEMV_MAX_MAT], Ns[GEMV_MAX_MAT];
    bool fast = true;
    for (int i = 0; i < nmat; i++) {
        types[i] = d[i].type; Ns[i] = d[i].N;
        if (!is_kquant(d[i].type) && !b32) return (int) cudaErrorInvalidValue;
        if ((uintptr_t) d[i].W & 15) fast = false;      // bulk copies need 16-byte aligned sources
    }
    GemvPlan pl;
    fast = fast && gemv_plan(types, Ns, nmat, K, pl);
    if (!fast) {
        if (pro.kind != PRO_NONE) return (int) cudaErrorInvalidValue;   // callers must check gemv_fused_prologue_ok / alignment
        if (b32) return (int) cudaErrorNotSupported;                     // launch_gemv_generic falls back to its own kernels
        for (int i = 0; i < nmat; i++) {
            int e = launch_gemv_generic(d[i], K, act, stream, pdl);
            if (e) return e;
        }
        return 0;
    }
    GemvParams P{};
    P.wpr = pl.wpr;
    P.nblk_p2 = pl.nblk_p2;
    P.nblk = (K + 255) / 256;
    P.K = K;
    P.nmat = nmat;
    P.nstage = pl.nstage;
    P.nstage_init = pl.nstage_init;
    P.owner_only = pl.owner_only;
    P.rel_count = pl.rel_count;
    P.prefill = std::min(pl.nstage_init, tune.prefill);
    P.stage_bytes = pl.stage_bytes;
    P.act = act;
    P.prologue = pro.kind;
    P.in0 = pro.in0;
    P.in1 = pro.in1;
    P.eps = pro.eps;
    P.abort_flag = abort_flag();
    P.trace = g_trace_buf ? g_trace_buf + (size_t) (g_trace_idx++ % (uint64_t) g_trace_slots) * GEMV_TRACE_ROW : nullptr;
    int tiles = 0;
    for (int i = 0; i < nmat; i++) {
        GemvMat & M = P.mat[i];
        M.W = (const uint8_t *) d[i].W;
        M.y = d[i].y;
        M.bias = d[i].bias;
        M.resid = d[i].resid;
        M.type = d[i].type;
        M.N = d[i].N;
        M.row_bytes = row_bytes(d[i].type, K);
        M.total_bytes = M.row_bytes * d[i].N;
        M.rows_per_tile = pl.rows[i];
        M.tile0 = tiles;
        tiles += (d[i].N + M.rows_per_tile - 1) / M.rows_per_tile;
    }
    P.ntiles = tiles;
    P.gbar = pro.gbar;
    if ((pro.kind == PRO_RMSNORM_DIST || pro.kind == PRO_SILU_DIST) && (!pro.gbar || !gemv_dist_prologue_ok())) return (int) cudaErrorInvalidValue;
    // instantiation: weight type (0 = mixed) x split rows x instrumented
    int ty = types[0];
    for (int i = 1; i < nmat; i++) if (types[i] != ty) ty = 0;
    const int ti = ty == T_Q4_K ? 1 : ty == T_Q5_K ? 2 : ty == T_Q6_K ? 3 : ty == T_Q8_0 ? 4 : ty == T_Q5_1 ? 5 : 0;
    const bool tr = g_trace_buf != nullptr;
    typedef void (*kern_t)(const GemvParams);
    static const kern_t table[6][2][2] = {
        {{k_gemv_kquant<0, false, false>, k_gemv_kquant<0, false, true>}, {k_gemv_kquant<0, true, false>, k_gemv_kquant<0, true, true>}},
        {{k_gemv_kquant<T_Q4_K, false, false>, k_gemv_kquant<T_Q4_K, false, true>}, {k_gemv_kquant<T_Q4_K, true, false>, k_gemv_kquant<T_Q4_K, true, true>}},
        {{k_gemv_kquant<T_Q5_K, false, false>, k_gemv_kquant<T_Q5_K, false, true>}, {k_gemv_kquant<T_Q5_K, true, false>, k_gemv_kquant<T_Q5_K, true, true>}},
        {{k_gemv_kquant<T_Q6_K, false, false>, k_gemv_kquant<T_Q6_K, false, true>}, {k_gemv_kquant<T_Q6_K, true, false>, k_gemv_kquant<T_Q6_K, true, true>}},
        {{k_gemv_kquant<T_Q8_0, false, false>, k_gemv_kquant<T_Q8_0, false, true>}, {k_gemv_kquant<T_Q8_0, true, false>, k_gemv_kquant<T_Q8_0, true, true>}},
        {{k_gemv_kquant<T_Q5_1, false, false>, k_gemv_kquant<T_Q5_1, false, true>}, {k_gemv_kquant<T_Q5_1, true, false>, k_gemv_kquant<T_Q5_1, true, true>}}};
    static FuncAttrCache attr_cache[6][2][2];
    const int si = pl.wpr > 1 ? 1 : 0;
    const kern_t fn = table[ti][si][tr ? 1 : 0];
    cudaError_t e = ensure_dyn_smem(attr_cache[ti][si][tr ? 1 : 0], (const void *) fn, GEMV_SMEM_LIMIT, true);
    if (e != cudaSuccess) return (int) e;
    int grid = sm_count() * GEMV_CTAS_PER_SM;
    if (grid > P.ntiles) grid = P.ntiles;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(GEMV_THREADS);
    cfg.dynamicSmemBytes = pl.smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return (int) cudaLaunchKernelEx(&cfg, fn, P);
}

static int launch_gemv_blk32(const GemvDesc & d, int K, const ActQ & act, cudaStream_t stream, bool pdl) {
    GemvB32Params P{};
    P.W = (const uint8_t *) d.W;
    P.y = d.y;
    P.bias = d.bias;
    P.resid = d.resid;
    P.type = d.type;
    P.N = d.N;
    P.K = K;
    P.nb = K / 32;
    P.bpb = d.type == T_Q8_0 ? BYTES_Q8_0 : BYTES_Q5_1;
    P.row_bytes = row_bytes(d.type, K);
    P.act = act;
    const int kp = (K + 15) & ~15;
    const size_t smem = (size_t) ((kp + 8 * P.nb + 15) & ~15) + (size_t) 8 * B32_NST * 1088;
    static FuncAttrCache attr_cache;
    {
        cudaError_t e = ensure_dyn_smem(attr_cache, (const void *) k_gemv_blk32, smem, false);
        if (e != cudaSuccess) return (int) e;
    }
    const int per_sm = (int) std::max<size_t>(1, std::min<size_t>(4, (224 * 1024) / (smem + 1024)));
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(std::min((d.N + 7) / 8, sm_count() * per_sm));
    cfg.blockDim = dim3(256);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return (int) cudaLaunchKernelEx(&cfg, k_gemv_blk32, P);
}

int launch_gemv_generic(const GemvDesc & d, int K, const ActQ & act, cudaStream_t stream, bool pdl) {
    // 32-element block types: the bulk-copy ring of the k-quant kernel (columns of 8 blocks) when the shape fits it ...
    static const bool no_ring32 = getenv("PB200_NO_BLK32_RING") != nullptr;
    if (!no_ring32 && (d.type == T_Q8_0 || d.type == T_Q5_1)) {
        GemvFused none{};
        const int rc = launch_gemv_kquant_fused(&d, 1, K, act, none, stream, pdl);
        if (rc != (int) cudaErrorNotSupported && rc != (int) cudaErrorInvalidValue) return rc;
    }
    // ... else, with 8-byte aligned rows and an activation that fits in shared memory, the per-warp cp.async streaming kernel
    static const bool no_b32 = getenv("PB200_NO_BLK32") != nullptr;
    if (!no_b32 && (d.type == T_Q8_0 || d.type == T_Q5_1) && K % 32 == 0 && row_bytes(d.type, K) % 8 == 0 && K % 16 == 0 && K <= 131072 &&
        ((uintptr_t) d.W & 7) == 0)
        return launch_gemv_blk32(d, K, act, stream, pdl);
    GemvGenericParams P{};
    P.W = (const uint8_t *) d.W;
    P.y = d.y;
    P.bias = d.bias;
    P.resid = d.resid;
    P.type = d.type;
    P.N = d.N;
    P.K = K;
    P.row_bytes = row_bytes(d.type, K);
    P.act = act;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((d.N + 7) / 8);
    cfg.blockDim = dim3(256);
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return (int) cudaLaunchKernelEx(&cfg, k_gemv_generic, P);
}

}  // namespace pb
