// rollout_tcw.cuh -- the wide tensor-core rollout's code (see rollout_tcw.cu for the design): the weight-image builder, the
// consumer / producer body, the finish kernel and the host driver.  rollout_tcw.cu instantiates it for tanh policies and binned
// heads, rollout_tcw_act.cu for the other activations.
#pragma once
#include <cuda_fp16.h>
#include <type_traits>
#include "common.cuh"
#include "pipeline.cuh"
#include "wgmma.cuh"

namespace {

constexpr int TW_THREADS = 384;
constexpr int TW_CONS_WARP0 = 4, TW_CONS_WARPS = 8;
constexpr int TW_MT = 128;                   // time steps per tile
constexpr int TW_BLOCK = 64 * 128;           // 8 KB: 64 rows x 64 float16, K-major, 128-byte swizzle
constexpr int TW_ACT_KC = 4;                 // K chunks of the activation buffer (widths <= 256)
constexpr int TW_MAX_HID = 4;
constexpr int TW_MAX_LAYERS = TW_MAX_HID + 1;
// ES_ROLLOUT_TC (single float16 products) is refused for shorter episodes.  Largest per-evaluation error against the float64
// truth, relative to the reward mass, over 64 evaluations each of 15-256-256-3, 28-256x3-8 and 28-128-256-256-128-8 on an
// H100: T = 1: 2.5e-3, 2: 1.6e-3, 3: 1.9e-3 (above the mode's 1e-3 bound); T = 4 .. 128: at most 5.2e-4, falling with T
// (a long episode averages the per-step errors).  ES_ROLLOUT_TC3 measured at most 4.0e-6 at T = 1.
constexpr int TW_TC_MIN_T = 4;
// registers per thread after the split: 128 x 24 + 256 x 240 = 64 512 <= 384 x 168 allocated at launch
constexpr int TW_REGS_DATA = 24, TW_REGS_MATH = 240;

template <bool SPLIT> struct TwCfg {
    static constexpr int NP = SPLIT ? 2 : 1;                                  // pieces per operand
    static constexpr int NSTAGE = SPLIT ? 6 : 12;                             // weight ring stages
    static constexpr uint32_t PIECE = 2 * TW_BLOCK;                           // one K chunk piece of the 128-row tile
    static constexpr uint32_t ACT = TW_ACT_KC * NP * PIECE;                   // [kc][piece][128 rows x 128 B]
    static constexpr uint32_t STAGE = NP * TW_BLOCK;                          // [piece][64 rows x 128 B]
    static constexpr uint32_t BARS = ACT + NSTAGE * STAGE;
    static constexpr uint32_t SMEM = BARS + 2 * NSTAGE * 8 + 1024;            // + alignment slack
};
static_assert(TwCfg<true>::SMEM <= 227 * 1024 && TwCfg<false>::SMEM <= 227 * 1024, "shared memory layout too large");

// the layers of one launch: sizes, their 64-blocks, where they sit in the flat parameters and in the image
struct TwLayers {
    int n_layers;
    int in[TW_MAX_LAYERS], out[TW_MAX_LAYERS];
    int kc[TW_MAX_LAYERS], nb[TW_MAX_LAYERS];         // K chunks / 64-wide N blocks (zero-padded)
    int pw[TW_MAX_LAYERS], pb[TW_MAX_LAYERS];         // offsets of W_l [out][in] and b_l in the flat parameters
    uint32_t w_off[TW_MAX_LAYERS], b_off[TW_MAX_LAYERS];   // byte offsets of the weight blocks / float32 biases in an image
    uint32_t img_bytes;                               // one evaluation's image
};

struct TwParams {
    TwLayers L;
    const uint8_t* images;        // [n_evals][img_bytes], evaluation 2 j + s = pair j of the chunk, sign s
    const float* obsn;            // [T][obs]
    const float* rew_vec;         // [T][act]
    const float* act_noise;       // [n_evals][n_eps][T][act] or NULL
    double* part;                 // [n_evals][n_mtiles][8 consumer warps][4]: reward, position sums 0..2
    int n_evals, n_mtiles, obs, act, T, n_eps;
    int bins; float scale; const float* low; const float* range;    // binned head (act = adim), rollout_tcw_binned_kernel only
};

template <bool SPLIT>
__global__ void __launch_bounds__(256) rollout_tcw_build_kernel(const float* __restrict__ table, const int64_t* __restrict__ idx,
                                                                const float* __restrict__ theta, float sigma, long long table_len,
                                                                int P, int* err, const __grid_constant__ TwLayers L,
                                                                uint8_t* __restrict__ images) {
    constexpr int NP = SPLIT ? 2 : 1;
    const float* __restrict__ eps = table + es_checked_slice(idx[blockIdx.x], P, table_len, err);
    uint8_t* ip = images + (size_t)(2 * blockIdx.x) * L.img_bytes;
    uint8_t* in_ = ip + L.img_bytes;
    for (int l = 0; l < L.n_layers; ++l) {
        const int in = L.in[l], out = L.out[l], Kp = L.kc[l] * 64, NB = L.nb[l];
        const int pw = L.pw[l];
        for (int e = threadIdx.x; e < NB * 64 * Kp / 2; e += blockDim.x) {
            const int n = (2 * e) / Kp, k = 2 * e - n * Kp;
            float p0 = 0.f, p1 = 0.f, m0 = 0.f, m1 = 0.f;
            if (n < out) {
                if (k < in) es_pheno_pm(sigma, __ldg(eps + pw + n * in + k), __ldg(theta + pw + n * in + k), p0, m0);
                if (k + 1 < in) es_pheno_pm(sigma, __ldg(eps + pw + n * in + k + 1), __ldg(theta + pw + n * in + k + 1), p1, m1);
            }
            const uint32_t off = L.w_off[l] + (uint32_t)(((k >> 6) * NB + (n >> 6)) * NP) * TW_BLOCK + sw128_off(n & 63, k & 63);
            if (SPLIT) {
                __half h0, l0, h1, l1;
                split_h1(p0, h0, l0); split_h1(p1, h1, l1);
                *(uint32_t*)(ip + off) = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
                *(uint32_t*)(ip + off + TW_BLOCK) = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
                split_h1(m0, h0, l0); split_h1(m1, h1, l1);
                *(uint32_t*)(in_ + off) = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
                *(uint32_t*)(in_ + off + TW_BLOCK) = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
            } else {
                *(uint32_t*)(ip + off) = pack_h2(p0, p1);
                *(uint32_t*)(in_ + off) = pack_h2(m0, m1);
            }
        }
        for (int n = threadIdx.x; n < NB * 64; n += blockDim.x) {
            float vp = 0.f, vn = 0.f;
            if (n < out) es_pheno_pm(sigma, __ldg(eps + L.pb[l] + n), __ldg(theta + L.pb[l] + n), vp, vn);
            ((float*)(ip + L.b_off[l]))[n] = vp;
            ((float*)(in_ + L.b_off[l]))[n] = vn;
        }
    }
}

__device__ __forceinline__ void st_shared_u32(void* p, uint32_t v) {
    asm volatile("st.shared.u32 [%0], %1;" ::"r"(smem_u32(p)), "r"(v) : "memory");
}
__device__ __forceinline__ void wg_bar(int half) { asm volatile("bar.sync %0, 128;" ::"r"(1 + half) : "memory"); }

// ACT: the activation of every layer (ES_ACT_*, es_act with act_param; SPLIT only for kinds other than tanh).  A hidden value
// the float16 hi part cannot hold (|y| > 65504: ReLU, leaky ReLU and ELU are unbounded) on a row of the episode (t < T) flags
// ES_ASYNC_F16_RANGE in *err
template <bool SPLIT, bool NOISE, bool BINNED, int ACT = ES_ACT_TANH>
__device__ __forceinline__ void tw_rollout(const TwParams& p, float act_param = 0.f, int* err = nullptr) {
    static_assert(ACT == ES_ACT_TANH || (SPLIT && !BINNED), "other activations: ES_ROLLOUT_TC3, tanh-free heads only");
    using C = TwCfg<SPLIT>;
    constexpr int NP = C::NP, NSTAGE = C::NSTAGE;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint8_t* ring = smem + C::ACT;
    uint64_t* full = (uint64_t*)(smem + C::BARS);
    uint64_t* empty = full + NSTAGE;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int n_items = p.n_evals * p.n_mtiles;
    const int n_layers = p.L.n_layers;

    if (tid == 0) {
        for (int s = 0; s < NSTAGE; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], TW_CONS_WARPS); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < TW_CONS_WARP0) {
        reg_dealloc<TW_REGS_DATA>();
        if (warp == 0 && lane == 0) {
            // ===================== producer: the weight blocks of every item, layer, K chunk and N block, in order =====================
            uint32_t s = 0, ph = 0;
            for (int it = blockIdx.x; it < n_items; it += gridDim.x) {
                const uint8_t* img = p.images + (size_t)(it / p.n_mtiles) * p.L.img_bytes;
                for (int l = 0; l < n_layers; ++l) {
                    const int nblk = p.L.kc[l] * p.L.nb[l];
                    for (int b = 0; b < nblk; ++b) {
                        mbar_wait(&empty[s], ph ^ 1);
                        mbar_expect_tx(&full[s], C::STAGE);
                        bulk_g2s(ring + s * C::STAGE, img + p.L.w_off[l] + (size_t)b * C::STAGE, C::STAGE, &full[s]);
                        if (++s == NSTAGE) { s = 0; ph ^= 1; }
                    }
                }
            }
        }
        return;
    }

    reg_alloc<TW_REGS_MATH>();
    // ===================== consumer warpgroups: rows 64*half .. 64*half + 63 of every tile =====================
    const int cw = warp - TW_CONS_WARP0, half = cw >> 2, q = lane & 3;
    const int wt = tid - TW_CONS_WARP0 * 32 - half * 128;       // thread of the warpgroup, 0..127
    const int rw = (cw & 3) * 16 + (lane >> 2);                  // this thread's rows of the warpgroup: rw, rw + 8
    uint8_t* act_wg = smem + half * TW_BLOCK;                    // the warpgroup's 64 rows in K chunk 0, piece 0
    const uint64_t a_desc0 = wg_desc_sw128(smem_u32(act_wg));
    const uint64_t ring_d = wg_desc_sw128(smem_u32(ring));
    constexpr uint64_t PIECE_D = C::PIECE >> 4, STAGE_D = C::STAGE >> 4, BLOCK_D = TW_BLOCK >> 4;
    uint32_t s = 0, ph = 0;

    for (int it = blockIdx.x; it < n_items; it += gridDim.x) {
        const int ev = it / p.n_mtiles, m = it - ev * p.n_mtiles;
        const int t0 = m * TW_MT + half * 64;
        const uint8_t* img = p.images + (size_t)ev * p.L.img_bytes;

        // ---- observation rows -> activation buffer (float16 hi[, lo]), zero beyond obs and T ----
        wg_bar(half);                                            // the previous item's last MMAs of every warp have retired
        {
            const int kp2 = p.L.kc[0] * 32;                      // column pairs per row
            for (int e = wt; e < 64 * kp2; e += 128) {
                const int row = e / kp2, k = 2 * (e - row * kp2), t = t0 + row;
                float x0 = 0.f, x1 = 0.f;
                if (t < p.T) {
                    const float* xr = p.obsn + (size_t)t * p.obs;
                    if (k < p.obs) x0 = __ldg(xr + k);
                    if (k + 1 < p.obs) x1 = __ldg(xr + k + 1);
                }
                uint8_t* dst = act_wg + (size_t)((k >> 6) * NP) * C::PIECE + sw128_off(row, k & 63);
                if (SPLIT) {
                    uint32_t hi, lo;
                    split_h2(x0, x1, hi, lo);
                    *(uint32_t*)dst = hi;
                    *(uint32_t*)(dst + C::PIECE) = lo;
                } else {
                    *(uint32_t*)dst = pack_h2(x0, x1);
                }
            }
        }
        fence_async_smem();
        wg_bar(half);

        double fitd = 0.0;
        float q0s = 0.f, q1s = 0.f, q2s = 0.f;
        for (int l = 0; l < n_layers; ++l) {
            const int KC = p.L.kc[l];
            const float* __restrict__ bias = (const float*)(img + p.L.b_off[l]);
            const bool last = l == n_layers - 1;
            auto layer = [&](auto nb_c) {
                constexpr int NB = decltype(nb_c)::value;
                float acc[NB][32];
                // bias -> accumulators: this thread's columns 64 nb + 8 c + 2 q (+1), rows rw and rw + 8
#pragma unroll
                for (int nb = 0; nb < NB; ++nb)
#pragma unroll
                    for (int c = 0; c < 8; ++c) {
                        const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + 64 * nb + 8 * c + 2 * q));
                        acc[nb][4 * c + 0] = bb.x; acc[nb][4 * c + 1] = bb.y; acc[nb][4 * c + 2] = bb.x; acc[nb][4 * c + 3] = bb.y;
                    }
                wg_fence();
                uint32_t prev = 0;
                for (int kc = 0; kc < KC; ++kc) {
                    const uint64_t ah = a_desc0 + (uint64_t)(kc * NP) * PIECE_D, al = ah + PIECE_D;
#pragma unroll
                    for (int nb = 0; nb < NB; ++nb) {
                        mbar_wait_warp(&full[s], ph);
                        const uint64_t bh = ring_d + s * STAGE_D, bl = bh + BLOCK_D;
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            wgmma64_ss(acc[nb], ah + 2 * k, bh + 2 * k, 1);
                            if (SPLIT) {
                                wgmma64_ss(acc[nb], ah + 2 * k, bl + 2 * k, 1);
                                wgmma64_ss(acc[nb], al + 2 * k, bh + 2 * k, 1);
                            }
                        }
                        wg_commit();
                        if (kc > 0 || nb > 0) {                  // the previous block has retired: its stage goes back
                            wg_wait<1>();
                            if (lane == 0) mbar_arrive(&empty[prev]);
                        }
                        prev = s;
                        if (++s == NSTAGE) { s = 0; ph ^= 1; }
                    }
                }
                wg_wait<0>();
#pragma unroll
                for (int nb = 0; nb < NB; ++nb) reg_fence(acc[nb]);
                if (lane == 0) mbar_arrive(&empty[prev]);
                if (!last) {
                    // ---- hidden layer: tanh -> the warpgroup's rows of the activation buffer, N block nb = next K chunk ----
                    wg_bar(half);                                // every warp's MMAs of this layer have read the buffer
#pragma unroll
                    for (int nb = 0; nb < NB; ++nb) {
                        uint8_t* dst = act_wg + (size_t)(nb * NP) * C::PIECE;
#pragma unroll
                        for (int c = 0; c < 8; ++c) {
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                const float z0 = acc[nb][4 * c + 2 * h], z1 = acc[nb][4 * c + 2 * h + 1];
                                const uint32_t o = sw128_off(rw + 8 * h, 8 * c + 2 * q);
                                if constexpr (ACT != ES_ACT_TANH) {
                                    const float y0 = es_act<ACT>(z0, act_param), y1 = es_act<ACT>(z1, act_param);
                                    // rows at t >= T (the zero observations of a partial tile) are no part of the episode:
                                    // whatever they reach is never read
                                    if (ACT != ES_ACT_SIGMOID && err && t0 + rw + 8 * h < p.T &&
                                        (fabsf(y0) > 65504.f || fabsf(y1) > 65504.f))
                                        *(volatile int*)err = ES_ASYNC_F16_RANGE;
                                    uint32_t hi, lo;
                                    split_h2(y0, y1, hi, lo);
                                    st_shared_u32(dst + o, hi);
                                    st_shared_u32(dst + o + C::PIECE, lo);
                                } else if (SPLIT) {
                                    uint32_t hi, lo;
                                    split_h2(tanh_acc(z0), tanh_acc(z1), hi, lo);
                                    st_shared_u32(dst + o, hi);
                                    st_shared_u32(dst + o + C::PIECE, lo);
                                } else {
                                    st_shared_u32(dst + o, pack_h2(tanh_fast(z0), tanh_fast(z1)));
                                }
                            }
                        }
                        // the next blocks' accumulators stay untouched until this block is stored: computed all at once, the
                        // tanh and hi / lo values of a 256-wide layer do not fit beside the accumulators (TC3 spilled)
#pragma unroll
                        for (int j = nb + 1; j < NB; ++j) reg_fence(acc[j]);
                    }
                    fence_async_smem();
                    wg_bar(half);
                    return;
                }
                if (BINNED) {
                    // ---- binned head: float32 tanh outputs -> the warpgroup's rows of the free activation buffer; then one
                    //      thread per row: the arg-max bin of every dimension, the action, the float32 reward in index order ----
                    wg_bar(half);                                // every warp's MMAs of this layer have read the buffer
#pragma unroll
                    for (int nb = 0; nb < NB; ++nb)
#pragma unroll
                        for (int c = 0; c < 8; ++c)
#pragma unroll
                            for (int e = 0; e < 4; ++e) {
                                const int col = 64 * nb + 8 * c + 2 * q + (e & 1), row = rw + 8 * (e >> 1);
                                *(float*)(act_wg + (size_t)(col >> 5) * C::PIECE + row * 128 + (((col ^ row) & 31) << 2)) =
                                    tanh_acc(acc[nb][4 * c + e]);
                            }
                    wg_bar(half);
                    const int t = t0 + wt;
                    if (wt < 64 && t < p.T) {
                        const uint8_t* rowp = act_wg + wt * 128;
                        float r = 0.f, a0 = 0.f, a1 = 0.f, a2 = 0.f;
                        for (int j = 0; j < p.act; ++j) {
                            int best = 0;
                            float bv = 0.f;
                            for (int b = 0; b < p.bins; ++b) {
                                const int col = j * p.bins + b;
                                const float v = *(const float*)(rowp + (size_t)(col >> 5) * C::PIECE + (((col ^ wt) & 31) << 2));
                                if (b == 0 || (bv == bv && (v > bv || v != v))) { bv = v; best = b; }    // a NaN is the maximum
                            }
                            const float a = __fadd_rn(__fmul_rn(__fmul_rn(p.scale, (float)best), __ldg(p.range + j)), __ldg(p.low + j));
                            r = __fadd_rn(r, __fmul_rn(a, __ldg(p.rew_vec + (size_t)t * p.act + j)));
                            if (j == 0) a0 = a;
                            if (j == 1) a1 = a;
                            if (j == 2) a2 = a;
                        }
                        fitd = (double)r; q0s = a0; q1s = a1; q2s = a2;
                    }
                    return;
                }
                // ---- last layer: a = tanh(z) [+ action noise of each episode]; r_t = <a_t, c_t>; positions (act <= 32: N block 0,
                //      columns 8 c + 2 q (+1) for c < 4) ----
                const int ta = t0 + rw, tb = ta + 8;
                const float* __restrict__ nz0 = (NOISE && p.act_noise) ? p.act_noise + (size_t)ev * p.n_eps * p.T * p.act : nullptr;
                const int n_ep = nz0 ? p.n_eps : 1;
                double sa = 0.0, sb = 0.0;
                for (int ep = 0; ep < n_ep; ++ep) {
                    const float* __restrict__ nz = nz0 ? nz0 + (size_t)ep * p.T * p.act : nullptr;
                    float ra = 0.f, rb = 0.f, a0 = 0.f, a1 = 0.f, a2 = 0.f;
    #pragma unroll
                    for (int c = 0; c < 4; ++c) {
    #pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const int col = 8 * c + 2 * q + (e & 1);
                            const int t = (e & 2) ? tb : ta;
                            float a = ACT != ES_ACT_TANH ? es_act<ACT>(acc[0][4 * c + e], act_param)
                                      : SPLIT ? tanh_acc(acc[0][4 * c + e]) : tanh_fast(acc[0][4 * c + e]);
                            if (col < p.act && t < p.T) {
                                if (NOISE && nz) a += __ldg(nz + (size_t)t * p.act + col);   // src/nn/nn.py:47-48
                                const float r = a * __ldg(p.rew_vec + (size_t)t * p.act + col);
                                if (e & 2) rb += r; else ra += r;
                                a0 += (col == 0) ? a : 0.f; a1 += (col == 1) ? a : 0.f; a2 += (col == 2) ? a : 0.f;
                            }
                        }
                    }
                    ra += __shfl_xor_sync(0xffffffffu, ra, 1); ra += __shfl_xor_sync(0xffffffffu, ra, 2);
                    rb += __shfl_xor_sync(0xffffffffu, rb, 1); rb += __shfl_xor_sync(0xffffffffu, rb, 2);
                    sa += (double)ra; sb += (double)rb;
                    q0s = a0; q1s = a1; q2s = a2;                    // the last episode's actions
                }
                fitd = (q == 0) ? sa / n_ep + sb / n_ep : 0.0;      // rows beyond T contribute 0
            };
            switch (p.L.nb[l]) {
                case 1: layer(std::integral_constant<int, 1>{}); break;
                case 2: layer(std::integral_constant<int, 2>{}); break;
                case 3: layer(std::integral_constant<int, 3>{}); break;
                default: layer(std::integral_constant<int, 4>{}); break;
            }
        }
        // ---- this warp's sums of the tile -> its partial slot ----
        const double f = es_warp_sum(fitd);
        const double g0 = es_warp_sum((double)q0s), g1 = es_warp_sum((double)q1s), g2 = es_warp_sum((double)q2s);
        if (lane == 0) {
            double* o = p.part + (((size_t)ev * p.n_mtiles + m) * TW_CONS_WARPS + cw) * 4;
            o[0] = f; o[1] = g0; o[2] = g1; o[3] = g2;
        }
    }
}

// the partial sums of every evaluation, tile by tile and warp by warp -> fitness and behaviour
__global__ void rollout_tcw_finish_kernel(const double* __restrict__ part, int n_evals, int n_mtiles, int act, float pos_scale,
                                          double* fit_pos, double* fit_neg, int fit_stride, float* behv_pos, float* behv_neg) {
    const int ev = blockIdx.x * blockDim.x + threadIdx.x;
    if (ev >= n_evals) return;
    double t[4] = {0.0, 0.0, 0.0, 0.0};
    const double* src = part + (size_t)ev * n_mtiles * TW_CONS_WARPS * 4;
    for (int i = 0; i < n_mtiles * TW_CONS_WARPS; ++i)
#pragma unroll
        for (int k = 0; k < 4; ++k) t[k] += src[4 * i + k];
    const int pair = ev >> 1, sgn = ev & 1;
    (sgn ? fit_neg : fit_pos)[(size_t)pair * fit_stride] = t[0];
    if (behv_pos) {
        // components 1 and 2 of an action narrower than 3 repeat component 0 (index % act)
        float* o = (sgn ? behv_neg : behv_pos) + (size_t)pair * 3;
        o[0] = pos_scale * (float)t[1];
        o[1] = pos_scale * (float)(act > 1 ? t[2] : t[1]);
        o[2] = pos_scale * (float)(act > 2 ? t[3] : t[1]);
    }
}

// the rollout of r: per chunk of pairs the weight images, `launch(ctx, p, grid, stream)` (the main kernel over the chunk's
// items, returning ES_OK or an error) and the finish kernel
template <bool SPLIT, typename Launch>
int tw_run(es_ctx* ctx, const EsRollout& r, cudaStream_t stream, Launch launch) {
    constexpr int NP = SPLIT ? 2 : 1;
    TwParams p;
    memset(&p, 0, sizeof(p));
    TwLayers& L = p.L;
    L.n_layers = r.n_layers;
    uint32_t o = 0;
    for (int l = 0; l < r.n_layers; ++l) {
        L.in[l] = r.dims[l];
        L.out[l] = r.dims[l + 1];
        L.kc[l] = es_div_up(L.in[l], 64);
        L.nb[l] = es_div_up(L.out[l], 64);
        L.pw[l] = r.w_off[l];
        L.pb[l] = r.b_off[l];
        L.w_off[l] = o; o += (uint32_t)(L.kc[l] * L.nb[l] * NP) * TW_BLOCK;
    }
    for (int l = 0; l < r.n_layers; ++l) { L.b_off[l] = o; o += (uint32_t)L.nb[l] * 64 * sizeof(float); }
    L.img_bytes = (o + 1023) & ~1023u;
    const int T = r.T, n_mtiles = es_div_up(T, TW_MT);
    // pairs per launch: <= 256 MiB of images
    int chunk = (int)((256u << 20) / (2 * (size_t)L.img_bytes));
    if (chunk < 1) chunk = 1;
    if (chunk > r.n_pairs) chunk = r.n_pairs;
    const size_t img_total = (size_t)2 * chunk * L.img_bytes;
    const size_t part_total = (size_t)2 * chunk * n_mtiles * TW_CONS_WARPS * 4 * sizeof(double);
    void* scratch = nullptr;
    int rc = es_ctx_scratch(ctx, img_total + part_total, &scratch);
    if (rc) return rc;
    uint8_t* images = (uint8_t*)scratch;
    double* part = (double*)((uint8_t*)scratch + img_total);
    if (r.bins) { p.bins = r.bins; p.scale = r.head_scale; p.low = r.head_low; p.range = r.head_range; }
    for (int p0 = 0; p0 < r.n_pairs; p0 += chunk) {
        const int np = (r.n_pairs - p0 < chunk) ? r.n_pairs - p0 : chunk;
        const EsRollout c = es_rollout_rows(r, p0, np);
        rollout_tcw_build_kernel<SPLIT><<<np, 256, 0, stream>>>(c.table, c.idx, c.theta, c.sigma, c.table_len, c.P, c.err, L, images);
        ES_LAUNCHED(ctx);
        p.images = images;
        p.obsn = r.obsn; p.rew_vec = r.rew_vec;
        p.act_noise = c.act_noise;
        p.part = part;
        p.n_evals = 2 * np; p.n_mtiles = n_mtiles; p.obs = L.in[0]; p.act = r.act; p.T = T; p.n_eps = r.n_episodes;
        const int n_items = p.n_evals * n_mtiles;
        const int grid = n_items < ctx->sm_count ? n_items : ctx->sm_count;
        rc = launch(ctx, p, grid, stream);
        if (rc) return rc;
        rollout_tcw_finish_kernel<<<es_div_up(2 * np, 128), 128, 0, stream>>>(part, 2 * np, n_mtiles, c.act, c.pos_scale, c.fit_pos,
                                                                            c.fit_neg, c.fit_stride, c.behv_pos, c.behv_neg);
        ES_LAUNCHED(ctx);
    }
    return ES_OK;
}

}  // namespace
