// rollout_closedw.cuh -- the closed-loop cluster rollout's code (see rollout_closedw.cu for the design and the barrier argument):
// the shared-memory layout, the body every CTA of a cluster runs and the launch configuration.
#pragma once
#include <math.h>
#include "common.cuh"
#include "mt19937.cuh"

namespace {

constexpr int CW_THREADS = 512;
constexpr int CW_WARPS = CW_THREADS / 32;
constexpr int CW_MAX_LAYERS = 5;           // 2 to 4 hidden layers
constexpr int CW_MAX_WIDTH = 256;
constexpr int CW_MAX_OBS = 384;
constexpr int CW_MAX_ACT = 64;
constexpr int CW_HALO = 16;                // band <= 16
constexpr int CW_SMEM_MAX = 227 * 1024 - 1024;    // dynamic shared memory per CTA: 227 KiB less 1 KiB for the static cw_layers

struct CwParams {
    EsRollout r;
    EsClosedEnv env;                        // ep_rows: [clusters][T] per-step episode sums (n_episodes > 1)
    EsTerm term;                            // term.steps == NULL: the episodes run T steps whatever the position
    unsigned* next;                         // the evaluation counter of dynamic scheduling, zero before the launch
};

// The stream walk of es_rollout_closedloop_terminal_streams (rollout_closedw_walk.cu states the design): every stream's
// tempered MT19937 words from its block 0 on, and what the walk reads and writes of the streams
struct CwWalk {
    const uint32_t* words;      // [n_streams][stride] (mj_launch_fill)
    size_t stride;
    uint32_t limit;             // a cursor past it has left the generated words (the buffer is padded past it by >= 4096 words)
    uint32_t rng, mask;         // the randint bound (mt19937_randint_bound)
    int n_per_stream, coins;
    double ac_std;
    uint32_t* mt_key;           // [n_streams][624], position, has_gauss, gauss: in and out
    int32_t* mt_pos;
    int32_t* has_gauss;
    double* gauss;
    int64_t* idx_out;           // [n_streams * n_per_stream]
    uint32_t* coin_out;         // [n_streams * n_per_stream][4 coins] or NULL
    float* trace;               // [n_streams * n_per_stream][2][E T act] the noise each executed step added, or NULL
};
struct CwWalkParams : CwParams { CwWalk w; };

// the walk's shared memory after the layout's end (floats): the noise of the step being run and of the next one, the staged
// words of the next step's attempts, the pair's index and the evaluation's save_obs decision
constexpr int CW_WALK_NZ = CW_MAX_ACT, CW_WALK_STAGE = 256;
constexpr int CW_WALK_FLOATS = 2 * CW_WALK_NZ + CW_WALK_STAGE + 4;

__host__ __device__ inline int cw_pad32(int n) { return (n + 31) & ~31; }
__host__ __device__ inline int cw_pad4(int n) { return (n + 3) & ~3; }

struct CwLayout {                          // offsets in floats into dynamic shared memory (all multiples of 4)
    int norm, racc, x, prod, abin, stat, o2, o2_stride, env_a, env_b, total;
    int act[CW_MAX_LAYERS], w[CW_MAX_LAYERS], bias[CW_MAX_LAYERS], rows[CW_MAX_LAYERS], stride[CW_MAX_LAYERS];
};
// act: the actions the env sees (dims[n_layers], or adim for a binned head, whose actions get their own buffer `abin`)
__host__ __device__ inline CwLayout cw_layout(int n_layers, const int* dims, int C, int band, int act, bool binned) {
    CwLayout L;
    const int obs = dims[0];
    int at = 0;
    L.norm = at; at += 4 * obs;                            // double mean[obs], double std[obs]  (first: 8-byte aligned)
    L.racc = at; at += 8;                                  // double fitness, float position[3]
    L.x = at; at += cw_pad32(obs);                         // the normalised observation, zero padded
    for (int l = 0; l < n_layers; ++l) { L.act[l] = at; at += cw_pad32(dims[l + 1]); }    // a_l, zero padded
    for (int l = 0; l < n_layers; ++l) {
        L.rows[l] = (dims[l + 1] + C - 1) / C;
        L.stride[l] = cw_pad32(dims[l]);
        L.w[l] = at; at += cw_pad4(L.rows[l]) * L.stride[l];
        L.bias[l] = at; at += cw_pad4(L.rows[l]);
    }
    L.prod = at; at += cw_pad4(act);
    L.abin = at; if (binned) at += cw_pad4(act);
    L.stat = at; at += 2 * obs;                            // float2 (sum, sumsq) of the post-step observations
    L.o2_stride = cw_pad4(obs + CW_HALO);
    L.o2 = at; at += 2 * L.o2_stride;                      // [2 buffers] raw observations with halo
    L.env_a = at; at += cw_pad4(band * obs);
    L.env_b = at; at += cw_pad4(act * obs);
    L.total = at;
    return L;
}
__host__ __device__ inline CwLayout cw_layout(int n_layers, const int* dims, int C, int band) {
    return cw_layout(n_layers, dims, C, band, dims[n_layers], false);
}

__device__ __forceinline__ float cw_normalise(float o, double mean, double std, double clip) {
    double x = ((double)o - mean) / std;
    x = isnan(x) ? x : fmin(fmax(x, -clip), clip);    // torch.clamp passes a NaN (fmax(NaN, -clip) is -clip)
    return (float)x;
}
// the warp-wide sums of v[0..3] in 7 shuffles (transposing butterfly, the xor-16, 8, 4, 2, 1 tree for every row): lane L
// returns the sum over the lanes of v[L / 8]
__device__ __forceinline__ float cw_warp_sum4(const float (&v)[4], int lane) {
    const bool h16 = lane & 16, h8 = lane & 8;
    float a[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) a[i] = (h16 ? v[i + 2] : v[i]) + __shfl_xor_sync(0xffffffffu, h16 ? v[i] : v[i + 2], 16);
    float c = (h8 ? a[1] : a[0]) + __shfl_xor_sync(0xffffffffu, h8 ? a[0] : a[1], 8);
    c += __shfl_xor_sync(0xffffffffu, c, 4);
    c += __shfl_xor_sync(0xffffffffu, c, 2);
    c += __shfl_xor_sync(0xffffffffu, c, 1);
    return c;
}
// all threads of all CTAs of the cluster; orders every earlier shared-memory access (local and remote) before every later one
__device__ __forceinline__ void cw_cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ unsigned cw_cluster_rank() {
    unsigned r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ unsigned cw_cluster_nctas() {
    unsigned r;
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
    return r;
}
// v into the same shared-memory word of CTA `rank` of the cluster
__device__ __forceinline__ void cw_store_remote(float* local, unsigned rank, float v) {
    const unsigned a = (unsigned)__cvta_generic_to_shared(local);
    unsigned r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(rank));
    asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(r), "f"(v) : "memory");
}

// one layer of this CTA in the step loop (read from shared memory: a per-layer index into registers would go to local memory)
struct CwLayer { int in, nr, S, r0, w, bias, xin, out, woff, boff; };

// One stream's walk, run by one warp (every lane holds the same state): the committed state after the draws of every executed
// step (cur, hg, gv: word cursor, has_gauss, cached gaussian) and the state after the draws formed ahead for a step that may not
// run (fcur, fhg, fgv).  Draws act on the formed state; commit() keeps them, discard() drops them.  numpy's order per pair:
// randint, then per evaluation the coin words and randn(act) per executed step (legacy_gauss: the cached value first, then
// polar attempts of 4 words, f x2 returned and f x1 cached).
struct CwWalker {
    const uint32_t* gw;
    uint32_t cur, fcur;
    int hg, fhg;
    double gv, fgv;
    bool bad;

    __device__ void load(const CwWalk& w, int sid) {
        gw = w.words + (size_t)sid * w.stride;
        cur = fcur = (uint32_t)w.mt_pos[sid];
        hg = fhg = w.has_gauss[sid] ? 1 : 0;
        gv = fgv = w.gauss[sid];
        bad = false;
    }
    __device__ void commit() { cur = fcur; hg = fhg; gv = fgv; }
    __device__ void discard() { fcur = cur; fhg = hg; fgv = gv; }
    // n more words from the formed cursor must lie in the generated words; otherwise the ctx's error word is set and the walk
    // stops consuming (its remaining draws are garbage, es_check_async raises)
    __device__ bool room(const CwWalk& w, uint32_t n, int* err) {
        if (!bad && fcur + n > w.limit) {
            bad = true;
            if (err) *(volatile int*)err = ES_ASYNC_WALK_OVERFLOW;
        }
        return !bad;
    }
    // rs.randint(0, upper_bound): masked rejection, 32 candidates at a time
    __device__ uint32_t randint(const CwWalk& w, int lane, int* err) {
        while (room(w, 32, err)) {
            const uint32_t v = __ldg(gw + fcur + lane) & w.mask;
            const unsigned ok = __ballot_sync(0xffffffffu, v <= w.rng);
            if (ok) {
                const int f = __ffs((int)ok) - 1;
                fcur += (uint32_t)f + 1u;
                return __shfl_sync(0xffffffffu, v, f);
            }
            fcur += 32u;
        }
        return 0u;
    }
    // the next two words (one rs.random() coin)
    __device__ uint2 coin(const CwWalk& w, int* err) {
        if (!room(w, 2, err)) return make_uint2(0u, 0u);
        const uint2 c = make_uint2(__ldg(gw + fcur), __ldg(gw + fcur + 1));
        fcur += 2u;
        return c;
    }
    // start copying the CW_WALK_STAGE words from the formed cursor into `stage` (cp.async: no registers held across the layers)
    __device__ void prefetch(uint32_t* stage, int lane) const {
#pragma unroll
        for (int j = 0; j < CW_WALK_STAGE / 32; ++j) {
            const int i = lane + 32 * j;
            const unsigned s = (unsigned)__cvta_generic_to_shared(stage + i);
            asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(s), "l"(gw + fcur + i) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    // randn(act) * ac_std rounded to float32 into out[0 .. act), from the formed state; `stage`: the words prefetch() copied
    // from the same cursor, or NULL
    __device__ void form(const CwWalk& w, int act, float* out, const uint32_t* stage, int lane, int* err) {
        if (stage) {
            asm volatile("cp.async.wait_all;" ::: "memory");
            __syncwarp();
        }
        const uint32_t s0 = fcur;
        int k = 0;
        if (fhg) {
            if (lane == 0) out[0] = (float)__dmul_rn(fgv, w.ac_std);
            k = 1; fhg = 0; fgv = 0.0;
        }
        while (k < act && room(w, 128, err)) {
            const int need = (act - k + 1) >> 1;                  // accepted attempts still to find
            uint32_t wd[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const uint32_t rel = fcur - s0 + 4u * (uint32_t)lane + (uint32_t)q;
                wd[q] = (stage && rel < (uint32_t)CW_WALK_STAGE) ? stage[rel] : __ldg(gw + fcur + 4u * (uint32_t)lane + q);
            }
            const bool acc = mt19937_polar_accept(wd[0], wd[1], wd[2], wd[3]);
            const unsigned bal = __ballot_sync(0xffffffffu, acc);
            const int rank = __popc(bal & ((1u << lane) - 1u));
            double cache = 0.0;
            if (acc && rank < need) {
                const double2 g = mt19937_polar_pair(wd[0], wd[1], wd[2], wd[3]);
                const int v = k + 2 * rank;
                out[v] = (float)__dmul_rn(g.x, w.ac_std);
                if (v + 1 < act) out[v + 1] = (float)__dmul_rn(g.y, w.ac_std);
                else cache = g.y;
            }
            const int n_acc = __popc(bal);
            if (n_acc >= need) {                                 // the need-th accepted attempt (lane L) ends the draw
                const int L = __ffs((int)__ballot_sync(0xffffffffu, acc && rank == need - 1)) - 1;
                const double c = __shfl_sync(0xffffffffu, cache, L);
                fhg = (act - k) & 1;
                fgv = fhg ? c : 0.0;
                fcur += 4u * (uint32_t)(L + 1);
                k = act;
            } else {
                fcur += 128u;
                k += 2 * n_acc;
            }
        }
        __syncwarp();
    }
    // the committed state into the stream's state, in DeviceGeneration.mt_state's layout: the raw words behind the tempered
    // words of the cursor's block (position 624: the block is exhausted), the position and the gaussian cache
    __device__ void store(const CwWalk& w, int sid, int lane) const {
        const uint32_t blk = cur / MT_NW, off = cur % MT_NW;
        const bool at_end = off == 0 && blk > 0;
        const uint32_t b_last = at_end ? blk - 1 : blk;
        for (int i = lane; i < MT_NW; i += 32) w.mt_key[(size_t)sid * MT_NW + i] = mt19937_untemper(__ldg(gw + (size_t)b_last * MT_NW + i));
        if (lane == 0) {
            w.mt_pos[sid] = at_end ? MT_NW : (int32_t)off;
            w.has_gauss[sid] = hg;
            w.gauss[sid] = gv;
        }
    }
};

// ACT: every layer of the policy applies the call's activation (p.r.activation, es_act) instead of tanh; the env's own
// tanh(A obs + B a) stays tanh.  p.term.steps set: the env ends an episode when its position falls (rollout_closedw.cu states
// the changes and why the barrier argument holds); unset, no episode ends before T, whatever the position (a NaN included).
// WALK (NOISY, with p a CwWalkParams and p.term.steps set): clusters take streams, not evaluations, and one warp per CTA walks
// the stream's words into the indices, coins and action noise (rollout_closedw_walk.cu)
template <int NL, bool BINNED, bool NOISY, bool ACT, bool WALK = false, class Params = CwParams>
__device__ __forceinline__ void cw_rollout(const Params& p) {
    static_assert(!WALK || (NOISY && !BINNED), "the stream walk draws action noise");
    extern __shared__ __align__(16) float cw_smem[];
    __shared__ CwLayer cw_layers[NL];
    const unsigned C = cw_cluster_nctas(), rank = cw_cluster_rank();
    const int n_clusters = gridDim.x / C, cluster = blockIdx.x / C;
    const int obs = p.r.dims[0], act = p.r.act, T = p.r.T, band = p.env.band;
    const CwLayout L = BINNED ? cw_layout(NL, p.r.dims, (int)C, band, act, true) : cw_layout(NL, p.r.dims, (int)C, band);
    double* __restrict__ nmean = reinterpret_cast<double*>(cw_smem + L.norm);
    double* __restrict__ nstd = nmean + obs;
    double* __restrict__ rfit = reinterpret_cast<double*>(cw_smem + L.racc);
    float* __restrict__ rpos = cw_smem + L.racc + 2;
    float* __restrict__ x = cw_smem + L.x;
    float* __restrict__ prod = cw_smem + L.prod;
    float2* __restrict__ stat = reinterpret_cast<float2*>(cw_smem + L.stat);
    float* __restrict__ o2 = cw_smem + L.o2;
    const float* __restrict__ envA = cw_smem + L.env_a;
    const float* __restrict__ envB = cw_smem + L.env_b;
    const float* __restrict__ action = cw_smem + (BINNED ? L.abin : L.act[NL - 1]);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const bool rew_warp = rank == 0 && warp == CW_WARPS - 1;
    const bool term = p.term.steps != nullptr;

    for (int i = tid; i < band * obs; i += CW_THREADS) cw_smem[L.env_a + i] = p.env.env_a[i];
    for (int i = tid; i < act * obs; i += CW_THREADS) cw_smem[L.env_b + i] = p.env.env_b[i];
    for (int i = tid; i < obs; i += CW_THREADS) { nmean[i] = p.env.ob_mean[i]; nstd[i] = p.env.ob_std[i]; }
    for (int i = tid; i < L.w[0] - L.x; i += CW_THREADS) cw_smem[L.x + i] = 0.f;     // x and every a_l, padding included
    if (tid == 0) {
#pragma unroll
        for (int l = 0; l < NL; ++l) {                      // this CTA owns rows [r0, r0 + nr) of layer l (nr may be <= 0)
            const int r0 = (int)rank * L.rows[l];
            cw_layers[l] = {p.r.dims[l], min(L.rows[l], p.r.dims[l + 1] - r0), L.stride[l], r0, L.w[l], L.bias[l],
                            l ? L.act[l - 1] : L.x, L.act[l], p.r.w_off[l], p.r.b_off[l]};
        }
    }
    cw_cluster_sync();                                      // START: every CTA of the cluster runs and has zeroed its buffers

    // the fell flag of the step (every CTA's own) and the cluster's next evaluation (rank 0 stores it into every CTA) in the
    // two free words after the position
    int* __restrict__ tflag = reinterpret_cast<int*>(cw_smem + L.racc + 5);
    int* __restrict__ tnext = reinterpret_cast<int*>(cw_smem + L.racc + 6);
    // the stream walk: its warp (idle in the env step, obs <= 384), the step noise [2][CW_WALK_NZ] (by step parity), the staged
    // words, and the pair's index and the save_obs decision it publishes
    [[maybe_unused]] const bool walker = WALK && warp == CW_WARPS - 2;
    [[maybe_unused]] float* __restrict__ wnz = cw_smem + L.total;
    [[maybe_unused]] uint32_t* __restrict__ wstage = reinterpret_cast<uint32_t*>(cw_smem + L.total + 2 * CW_WALK_NZ);
    [[maybe_unused]] uint32_t* __restrict__ wmisc = wstage + CW_WALK_STAGE;
    [[maybe_unused]] CwWalker wk;
    [[maybe_unused]] int n_ev = 0;                          // a stream's evaluations (WALK)
    int ev0 = cluster;
    if constexpr (WALK) {
        n_ev = 2 * p.w.n_per_stream;
        ev0 = cluster * n_ev;                               // (>= 2 n_pairs when the cluster has no stream)
    }
    for (int ev = ev0; ev < 2 * p.r.n_pairs; ev = *tnext) {
        const int pair = ev >> 1, neg = ev & 1;
        [[maybe_unused]] const int e_loc = WALK ? ev % n_ev : 0;
        if constexpr (WALK) {
            // the pair's index (before +), the evaluation's coin and its first step's noise, published by the barrier below
            // (every read of this CTA's previous evaluation preceded REUSE)
            if (walker) {
                const CwWalk& w = p.w;
                if (e_loc == 0) wk.load(w, ev / n_ev);
                if (!neg) {
                    const uint32_t ix = wk.randint(w, lane, p.r.err);
                    if (lane == 0) {
                        wmisc[0] = ix;
                        if (rank == 0) w.idx_out[pair] = (int64_t)ix;
                    }
                }
                if (w.coins) {
                    const uint2 c = wk.coin(w, p.r.err);
                    if (lane == 0) {
                        wmisc[1] = mt19937_random_sample(c.x, c.y) < p.env.save_obs_chance;
                        if (rank == 0 && w.coin_out) { w.coin_out[(size_t)pair * 4 + 2 * neg] = c.x; w.coin_out[(size_t)pair * 4 + 2 * neg + 1] = c.y; }
                    }
                } else if (lane == 0) {
                    wmisc[1] = 0u;
                }
                wk.form(w, act, wnz, nullptr, lane, p.r.err);
                wk.commit();
            }
            __syncthreads();
        }
        const long long base = es_checked_slice(WALK ? (long long)wmisc[0] : p.r.idx[pair], p.r.P, p.r.table_len, p.r.err);
        const float* __restrict__ eps = p.r.table + base;
        const float* __restrict__ th = p.r.theta;
        const float sg = p.r.sigma;
        auto w_at = [&](int at) {                           // theta + sigma eps or theta - sigma eps
            float wp, wm;
            es_pheno_pm(sg, eps[at], th[at], wp, wm);
            return neg ? wm : wp;
        };
#pragma unroll 1
        for (int l = 0; l < NL; ++l) {                      // this CTA's rows of every layer, zero padded to a multiple of 4
            const CwLayer ly = cw_layers[l];
            const int R4 = cw_pad4(max(ly.nr, 0)), in = ly.in, S = ly.S;
            float* __restrict__ W = cw_smem + ly.w;
            for (int r = warp; r < R4; r += CW_WARPS)
                for (int k = lane; k < S; k += 32)
                    W[r * S + k] = (r < ly.nr && k < in) ? w_at(ly.woff + (ly.r0 + r) * in + k) : 0.f;
            for (int r = tid; r < R4; r += CW_THREADS) cw_smem[ly.bias + r] = r < ly.nr ? w_at(ly.boff + ly.r0 + r) : 0.f;
        }
        auto start_episode = [&]() {                        // a fresh env: obs_0, position 0
            for (int i = tid; i < obs; i += CW_THREADS) {
                const float v = p.env.obs0[i];
                es_put_obs(o2, i, v, obs, band);
                x[i] = cw_normalise(v, nmean[i], nstd[i], p.env.ob_clip);
                stat[i] = make_float2(0.f, 0.f);
            }
        };
        start_episode();
        if (tid == 0) { rfit[0] = 0.0; rpos[0] = 0.f; rpos[1] = 0.f; rpos[2] = 0.f; }
        bool save = false;                                  // the evaluation's save_obs coin (legacy random_sample < chance)
        if constexpr (WALK) {
            save = wmisc[1] != 0u;
        } else if (p.env.coins) {
            const uint32_t* c = p.env.coins + (size_t)pair * 4 + 2 * neg;
            save = mt19937_random_sample(c[0], c[1]) < p.env.save_obs_chance;
        }
        const bool keep_stat = rank == 0 && p.env.ob_sum && save;
        __syncthreads();

        const int n_eps = NOISY ? p.r.n_episodes : 1;
        // the step the episode ended at (the same in every thread of the cluster), the noise values consumed so far, and the
        // steps the earlier episodes' per-step sums reach (the longest of them)
        int t_end = T - 1, reach = 0;
        long long used = 0;
        for (int ep = 0; ep < n_eps; ++ep) {
            const bool last_ep = ep == n_eps - 1;
            const bool add_stat = keep_stat && last_ep;     // behaviour and ObStat: the last episode's
            if (NOISY && ep > 0) {
                start_episode();
                if (tid == 0) { rpos[0] = 0.f; rpos[1] = 0.f; rpos[2] = 0.f; }
                if constexpr (WALK) {                       // the episode's first step draws where the last one stopped
                    if (walker) { wk.form(p.w, act, wnz, nullptr, lane, p.r.err); wk.commit(); }
                }
                __syncthreads();
            }

            // this cluster's episode sums, and the noise of the output row this lane owns (row 4 warp + lane / 8 of the last
            // layer's pass, lanes 8 i)
            double* __restrict__ erow = NOISY ? p.env.ep_rows + (size_t)cluster * T : nullptr;
            const float* __restrict__ nzp = nullptr;
            [[maybe_unused]] float* __restrict__ trp = nullptr;    // (WALK) the row's noise trace
            if (NOISY && (lane & 7) == 0) {
                const CwLayer& lo = cw_layers[NL - 1];
                const int r = 4 * warp + (lane >> 3);
                if (r < lo.nr) {
                    if constexpr (WALK) {
                        nzp = wnz + lo.r0 + r;
                        if (p.w.trace) trp = p.w.trace + ((size_t)pair * 2 + neg) * n_eps * T * act + used + lo.r0 + r;
                    } else {
                        nzp = p.r.act_noise + ((size_t)pair * 2 + neg) * n_eps * T * act + used + lo.r0 + r;
                    }
                }
            }

            t_end = T - 1;
            for (int t = 0; t < T; ++t) {
                const int cur = t & 1;
                float crow0 = 0.f, crow1 = 0.f;
                double esum = 0.0;                              // the earlier episodes' rewards of this step
                if (rew_warp) {                                 // this step's reward coefficients: in flight under the layers
                    const float* __restrict__ c = p.r.rew_vec + (size_t)t * act;
                    if (lane < act) crow0 = __ldg(c + lane);
                    if (lane + 32 < act) crow1 = __ldg(c + lane + 32);
                    if (NOISY && lane == 0 && ep > 0 && t < reach) esum = erow[t];
                }
                float nz = 0.f;                                 // this lane's action noise: in flight under the layers
                if constexpr (WALK) {
                    if (nzp) {
                        nz = nzp[(t & 1) * CW_WALK_NZ];
                        if (trp) trp[(size_t)t * act] = nz;
                    }
                    if (walker && t + 1 < T) wk.prefetch(wstage, lane);     // the next step's words, under the layers
                } else {
                    if (NOISY && nzp) nz = __ldg(nzp + (size_t)t * act);
                }
                // ---- the layers: 4 rows per warp and pass, each row's tanh stored into every CTA's a_l, then B_l ----
#pragma unroll 1
                for (int l = 0; l < NL; ++l) {
                    const CwLayer ly = cw_layers[l];
                    const int S = ly.S, r0 = ly.r0, nr = ly.nr, nj = S >> 5;
                    const float* __restrict__ xin = cw_smem + ly.xin + lane;
                    const float* __restrict__ W = cw_smem + ly.w + lane;
                    const float* __restrict__ bias = cw_smem + ly.bias;
                    float* __restrict__ out = cw_smem + ly.out;
                    for (int g = 4 * warp; g < nr; g += 4 * CW_WARPS) {
                        float z[4] = {0.f, 0.f, 0.f, 0.f};
                        const float* __restrict__ wr = W + g * S;
#pragma unroll 4
                        for (int j = 0; j < nj; ++j) {
                            const float xv = xin[32 * j];
#pragma unroll
                            for (int r = 0; r < 4; ++r) z[r] = fmaf(wr[r * S + 32 * j], xv, z[r]);
                        }
                        const float s = cw_warp_sum4(z, lane);
                        const int r = g + (lane >> 3);
                        if ((lane & 7) == 0 && r < nr) {
                            const float h = ACT ? es_act(p.r.activation, p.r.act_param, s + bias[r]) : es_tanh_exp(s + bias[r]);
                            const float y = (NOISY && l == NL - 1) ? __fadd_rn(h, nz) : h;
                            for (unsigned q = 0; q < C; ++q) cw_store_remote(out + r0 + r, q, y);
                        }
                    }
                    cw_cluster_sync();                          // B_l
                }
                if (BINNED) {                                   // the actions from this CTA's copy of the last layer's outputs
                    if (tid < act) {
                        const float* __restrict__ o = cw_smem + L.act[NL - 1] + tid * p.r.bins;
                        cw_smem[L.abin + tid] = es_binned_action(p.r.bins, p.r.head_scale, p.r.head_low, p.r.head_range, tid,
                                                                 [&](int b) { return o[b]; });
                    }
                    __syncthreads();
                }
                // ---- env step, redundantly in every CTA: thread i owns observation i ----
                if (tid < obs) {
                    const float* __restrict__ oc = o2 + cur * L.o2_stride;
                    const int i = tid;
                    float acc = 0.f;
                    for (int d = 0; d < band; ++d) acc = __fadd_rn(acc, __fmul_rn(envA[d * obs + i], oc[i + d]));
                    for (int j = 0; j < act; ++j) acc = __fadd_rn(acc, __fmul_rn(envB[j * obs + i], action[j]));
                    const float nv = es_tanh_exp(acc);
                    es_put_obs(o2 + (cur ^ 1) * L.o2_stride, i, nv, obs, band);
                    x[i] = cw_normalise(nv, nmean[i], nstd[i], p.env.ob_clip);
                    if (add_stat) {                             // float32 column sums in step order (numpy's axis-0 reduction)
                        float2 st = stat[i];
                        st.x = __fadd_rn(st.x, nv); st.y = __fadd_rn(st.y, __fmul_rn(nv, nv));
                        stat[i] = st;
                    }
                }
                // ---- reward (float32 dot in index order, summed in float64) and position: rank 0's last warp ----
                if (rew_warp) {
                    if (lane < act) prod[lane] = __fmul_rn(action[lane], crow0);
                    if (lane + 32 < act) prod[lane + 32] = __fmul_rn(action[lane + 32], crow1);
                    __syncwarp();
                    if (lane == 0) {
                        float acc = 0.f;
                        for (int j = 0; j < act; ++j) acc = __fadd_rn(acc, prod[j]);
                        if (!NOISY) {
                            rfit[0] += (double)acc;
                        } else if (!last_ep) {                  // the float64 per-step sum over the episodes, in their order
                            erow[t] = esum + (double)acc;
                        } else {                                // ... and its mean (obj.py:57-61)
                            rfit[0] += (esum + (double)acc) / n_eps;
                        }
                        const float ps = p.r.pos_scale;
                        rpos[0] = __fadd_rn(rpos[0], __fmul_rn(ps, action[0]));
                        rpos[1] = __fadd_rn(rpos[1], __fmul_rn(ps, action[1 % act]));
                        rpos[2] = __fadd_rn(rpos[2], __fmul_rn(ps, action[2 % act]));
                    }
                    __syncwarp();
                }
                if (warp == CW_WARPS - 1 && lane == 0) {
                    // every CTA forms the position as rank 0's reward lane does (same action, same operations), so every CTA
                    // decides the fall alike.  The flag is stored and read at every step, also without an early end: a read
                    // gated on `term` made the step loop measurably slower
                    if (term && rank != 0) {
                        const float ps = p.r.pos_scale;
                        rpos[0] = __fadd_rn(rpos[0], __fmul_rn(ps, action[0]));
                        rpos[1] = __fadd_rn(rpos[1], __fmul_rn(ps, action[1 % act]));
                        rpos[2] = __fadd_rn(rpos[2], __fmul_rn(ps, action[2 % act]));
                    }
                    *tflag = term && !(fabsf(rpos[2]) <= p.term.fall_height);
                }
                if constexpr (WALK) {                           // the next step's noise, kept if the step runs
                    if (walker && t + 1 < T) wk.form(p.w, act, wnz + ((t + 1) & 1) * CW_WALK_NZ, wstage, lane, p.r.err);
                }
                __syncthreads();                                // x and the raw observation before the next step's layer 0
                if constexpr (WALK) {
                    if (walker) { if (*tflag) wk.discard(); else wk.commit(); }
                }
                if (*tflag) { t_end = t; break; }
            }
            used += (long long)(t_end + 1) * act;
            if (NOISY && rew_warp && lane == 0 && last_ep)      // the steps only earlier episodes reached (obj.py:58-61)
                for (int t = t_end + 1; t < reach; ++t) rfit[0] += erow[t] / n_eps;
            reach = max(reach, t_end + 1);
        }
        if (rew_warp && lane == 0) {
            (neg ? p.r.fit_neg : p.r.fit_pos)[(size_t)pair * p.r.fit_stride] = rfit[0];
            float* bv = neg ? p.r.behv_neg : p.r.behv_pos;
            if (bv) { bv[(size_t)pair * 3 + 0] = rpos[0]; bv[(size_t)pair * 3 + 1] = rpos[1]; bv[(size_t)pair * 3 + 2] = rpos[2]; }
            if (term) {
                p.term.steps[(size_t)neg * p.r.n_pairs + pair] = t_end;
                if (p.term.noise_used) p.term.noise_used[(size_t)neg * p.r.n_pairs + pair] = used;
            }
        }
        if (keep_stat) {
            // ObStat.inc of a saved rollout: float32 column sums added in float64 (the order over rollouts is the atomics')
            for (int i = tid; i < obs; i += CW_THREADS) {
                const float2 st = stat[i];
                atomicAdd(p.env.ob_sum + i, (double)st.x);
                atomicAdd(p.env.ob_sumsq + i, (double)st.y);
            }
            if (tid == 0) { atomicAdd(p.env.ob_count, (double)(t_end + 1)); atomicAdd(p.env.ob_count + 1, 1.0); }
        }
        if constexpr (WALK) {                               // the stream's state after its last evaluation
            if (walker && rank == 0 && e_loc == n_ev - 1) wk.store(p.w, ev / n_ev, lane);
        }
        if (rank == 0 && tid == 0) {                        // the cluster's next evaluation, into every CTA before REUSE
            int nx;
            if constexpr (WALK) {                           // the stream's next one, or the first of the next stream
                if (e_loc + 1 < n_ev) {
                    nx = ev + 1;
                } else {
                    const long long s = n_clusters + (long long)atomicAdd(p.next, 1u);
                    nx = s * n_ev < 2ll * p.r.n_pairs ? (int)(s * n_ev) : 2 * p.r.n_pairs;
                }
            } else {
                nx = n_clusters + (int)atomicAdd(p.next, 1u);
            }
            for (unsigned q = 0; q < C; ++q) cw_store_remote(reinterpret_cast<float*>(tnext), q, __int_as_float(nx));
        }
        cw_cluster_sync();                                  // REUSE (the last one: EXIT)
    }
}

typedef void (*CwKernel)(const CwParams);

// a launch of `clusters` clusters of C CTAs (attr: the cluster-dimension attribute the config points to)
static cudaLaunchConfig_t cw_config(int C, size_t smem, int clusters, cudaStream_t stream, cudaLaunchAttribute* attr) {
    attr->id = cudaLaunchAttributeClusterDimension;
    attr->val.clusterDim.x = C; attr->val.clusterDim.y = 1; attr->val.clusterDim.z = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(clusters * C); cfg.blockDim = dim3(CW_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cfg.attrs = attr; cfg.numAttrs = 1;
    return cfg;
}

// the number of clusters of the shape that can be resident at once (the persistent grid), 0 when none fits
template <class Kernel>
static int cw_max_clusters(Kernel k, int C, size_t smem, int* clusters) {
    ES_CHECK_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaLaunchAttribute attr;
    const cudaLaunchConfig_t cfg = cw_config(C, smem, 1, nullptr, &attr);
    ES_CHECK_CUDA(cudaOccupancyMaxActiveClusters(clusters, k, &cfg));
    return ES_OK;
}
}  // namespace
