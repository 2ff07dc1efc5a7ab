// rollout_tc2.cu -- fused perturb + MLP rollout + fitness on the Hopper tensor cores (wgmma), float16 operands, two precisions:
//
//   SPLIT = false (ES_ROLLOUT_TC):   one wgmma per product, tanh.approx                 -> float16-grade fitness
//   SPLIT = true  (ES_ROLLOUT_TC3):  every operand is a float16 hi + lo pair (x = hi + lo to ~2^-22) and every product is
//                                    THREE MMAs  hi*hi + hi*lo + lo*hi  accumulated in float32, the tanh is evaluated to
//                                    float32 accuracy (1 - 2 / (1 + e^2x)) and rewards are summed in float64
//                                    -> float32-equivalent fitness (the reference's arithmetic is float32:
//                                    src/nn/nn.py:42-50, src/core/policy.py:61-64)
//
// Same contract as rollout_f32.cu (reference: src/core/policy.py:61-64, src/nn/nn.py:35-46, src/gym/gym_runner.py:50-54,
// src/gym/training_result.py:28) for obs -> 64 -> 64 -> act (act <= 32) tanh MLPs.
//
// One CTA = one antithetic pair at a time (persistent over pairs), episode time on the MMA M dimension.  A tile is 128 time
// steps; each of the two consumer warpgroups owns 64 of them (wgmma M = 64) and keeps its accumulators in registers:
//   L1   V (64 x 64 f32) = Xn_tile . eps1^T      eps1 UNSCALED, straight from a float16 shadow of the noise table (both
//        operands in shared memory); z1+- = U +- sigma*V with U = Xn . theta1^T + b1 computed once per generation in float64
//        -> float32 (ubase kernel), so one MMA chain serves both signs and the unperturbed term carries no tensor-core rounding
//   epi1 h1+- = tanh(z1+-) -> float16 (hi[, lo]) packed in registers: the accumulator fragment of an m64n64 wgmma is, pair by
//        pair, the A-operand fragment of the next layer's m64nNk16 wgmma, so the activations never touch shared memory
//   L2   D2+- = h1+- . (theta2 +- sigma*eps2)^T,  epi2: h2+- = tanh(D2+- + b2+-) -> registers
//   L3   D3+- = h2+- . (theta3 +- sigma*eps3)^T (N = 32),  epi3: a = tanh(D3 + b3), r_t = <a_t, c_t>, fitness += r_t
//
// Operand staging:
//   * Xn: pre-tiled once per generation into the exact shared-memory image of every (tile, K chunk[, piece]) stage
//     (rollout_tc2_prep_kernel).  The ring holds 8 KB slots, one warpgroup's 64 rows of a stage each (one cp.async.bulk per
//     slot), filled as one FIFO in the order (pair, tile, warpgroup, K chunk, piece); each slot is released by the 4 warps of
//     the warpgroup that reads it.  SPLIT: 8 slots = 4 K chunks of lookahead, otherwise 16 slots = 16 chunks;
//   * eps1 (82 % of a perturbation): the library keeps float16 shadows of the table (hi, and lo for SPLIT) in 8 copies shifted
//     by 0..7 elements; in copy idx % 8 every row of eps1 is 16-byte aligned, and ONE 3-D TMA tensor copy per K chunk
//     (dims {64 elements, origin in 16-byte units, 64 rows of stride obs*2 bytes}: overlapping strides, 128-byte swizzle)
//     lands the 64 x 64 block in the K-major swizzled layout the wgmma descriptor expects.  No thread touches eps1.
//     (Shapes without 16-byte aligned rows, or no memory for the shadows: builder warps convert the float32 slice.)
//   * theta2/3 +- sigma*eps2/3 and the biases: builder warps compute them one pair ahead into an L2-resident image, a copier
//     warp moves the image into shared memory with two bulk copies when the previous pair's MMAs have retired.
//   * with the shadows, the copier also prefetches the next pair's eps1 into L2 (TMA prefetch, same maps and coordinates)
//     one pair ahead, so the eps1 copy at the pair boundary reads L2 and not HBM.
//   * U and the reward weights c (the same for every pair): each consumer thread loads its 32 values of U for a tile into
//     registers before the tile's L1 chain, which hides the load, and its 16 values of c once per tile; both signs use the
//     registers.  Loaded once per sign inside the epilogues, their latency sat between the wgmma chains (pointing them at
//     rows already in L1 recovered only a small part of what this saves).  The NOISE instantiations still load c element by
//     element in the epilogue: holding it in registers there spills at 208.
//
// 12 warps (3 warpgroups):
//   warpgroup 0: warp 0 producer (Xn ring) | warp 1 copier | warps 2-3 builders      -> setmaxnreg 72 registers
//   warpgroup 1: consumers, rows 0-63 of every tile | warpgroup 2: rows 64-127     -> setmaxnreg 208 registers
//
// Consumer schedule per tile: the L1 chain (one commit group per K chunk, the chunk before retired and its ring slots
// released while the next one runs), then the two signs staggered by one phase so that each short L2 / L3 chain runs on
// the tensor pipe under the other sign's tanh:
//   epi1+ | L2+ . epi1- | L2- . epi2+ | L3+ . epi2- | L3- . epi3+ | epi3-      ("X . e": X in flight while e runs)
// The FIFO order of the ring staggers the two warpgroups by one L1 chain: warpgroup 1's chain of tile m is fed after
// warpgroup 0's, so it runs while warpgroup 0 is in its epilogues, and warpgroup 0's chain of tile m + 1 runs under warpgroup
// 1's epilogues.  No other synchronisation orders the warpgroups (an explicit turn token on top of the FIFO order measured no
// faster at float32-equivalent precision and slower with single float16 products).
// The waits inside the chains are warp-uniform (mbar_wait_warp, pipeline.cuh).
#include <cuda_fp16.h>
#include <stdlib.h>
#include "common.cuh"
#include "pipeline.cuh"
#include "wgmma.cuh"

namespace {

constexpr int T2_THREADS = 384;
constexpr int T2_W_PROD = 0, T2_W_COPY = 1, T2_BLD_WARP0 = 2, T2_BLD_WARPS = 2, T2_CONS_WARP0 = 4, T2_CONS_WARPS = 8;
constexpr int T2_H = 64, T2_MT = 128, T2_KC = 64, T2_ACT_PAD = 32;
constexpr int T2_STAGE = T2_MT * 128;          // 16 KB: 128 rows x 64 f16 (one tile's K chunk piece in the xnt image)
constexpr int T2_SLOT = T2_STAGE / 2;          // 8 KB: the 64 rows of one consumer warpgroup (one observation ring slot)
constexpr int T2_WG_WARPS = T2_CONS_WARPS / 2; // warps per consumer warpgroup
constexpr int T2_B1_CHUNK = T2_H * 128;        // 8 KB: 64 rows x 64 f16
constexpr int T2_W3_BLOCK = T2_ACT_PAD * 128;  // 4 KB
// registers per thread after the split: 128 x 72 + 256 x 208 = 62 464 <= 384 x 168 = 64 512 allocated at launch
constexpr int T2_REGS_DATA = 72, T2_REGS_MATH = 208;

// first 16-byte unit of a slice's eps1 in the shifted shadow copy where its rows are 16-byte aligned
__device__ __forceinline__ int t2_shadow_unit(long long at, size_t shadow_stride) {
    return (int)(((long long)(at & 7) * (long long)shadow_stride + (at - (at & 7))) >> 3);
}

struct T2Maps {
    CUtensorMap hi, lo;           // 3-D maps over the float16 shadows: dims {64 elements, origin (16-byte units), 64 rows}
};

struct T2Params {
    EsRollout r;
    const uint8_t* xnt;           // [n_mtiles][nkc][pieces][16 KB stage image]
    const float* ubase;           // [n_mtiles * 128][64] row-major
    uint8_t* images;              // [gridDim.x][2][image bytes]
    size_t shadow_stride;         // elements per shifted copy
    int use_tma;                  // eps1 by TMA from the shadows; 0: the builders convert the float32 slice
    int nkc, n_mtiles;
};

template <bool SPLIT> struct T2Cfg {
    static constexpr int NP = SPLIT ? 2 : 1;              // pieces per operand
    static constexpr int NSLOT = SPLIT ? 8 : 16;          // 8 KB slots in the observation ring (a power of 2)
};

struct T2Smem { uint32_t b1, xst, w2, w3, bias, red, bars, total; };
template <bool SPLIT> __host__ __device__ inline T2Smem t2_layout(int nkc) {
    using C = T2Cfg<SPLIT>;
    T2Smem L;
    uint32_t o = 0;
    L.b1 = o;   o += (uint32_t)C::NP * nkc * T2_B1_CHUNK;         // [kc][piece][64 rows x 128 B]
    L.xst = o;  o += (uint32_t)C::NSLOT * T2_SLOT;
    L.w2 = o;   o += 2u * C::NP * T2_B1_CHUNK;                    // [sign][piece][64 rows x 128 B]
    L.w3 = o;   o += 2u * C::NP * T2_W3_BLOCK;                    // [sign][piece][32 rows x 128 B]
    L.bias = o; o += 2 * 1024;                                    // double-buffered by pair parity
    L.red = o;  o += 2 * T2_CONS_WARPS * 64 + 64;                 // per-pair sums of the consumer warps [parity][warp][8 doubles] + counters
    L.bars = o; o += 1024;
    L.total = o;
    return L;
}
// operand image in global scratch: [W2 | W3 | bias 1 KB | (B1 when the builders make it)]
struct T2Image { uint32_t w2, w3, bias, b1, total; };
template <bool SPLIT> __host__ __device__ inline T2Image t2_image(int nkc, int with_b1) {
    using C = T2Cfg<SPLIT>;
    T2Image I;
    uint32_t o = 0;
    I.w2 = o;   o += 2u * C::NP * T2_B1_CHUNK;
    I.w3 = o;   o += 2u * C::NP * T2_W3_BLOCK;
    I.bias = o; o += 1024;
    I.b1 = o;   o += with_b1 ? (uint32_t)C::NP * nkc * T2_B1_CHUNK : 0u;
    I.total = o;
    return I;
}

enum { B2_FULL = 0, B2_EMPTY = 16, B2_EPS_TX = 32, B2_EPS_READY, B2_EPS_FREE, B2_W_READY, B2_W_FREE, B2_IMG_READY,
       B2_IMG_FREE = B2_IMG_READY + 2, B2_COUNT = B2_IMG_FREE + 2 };
static_assert(T2Cfg<true>::NSLOT <= B2_EMPTY && T2Cfg<false>::NSLOT <= B2_EMPTY, "barrier enum too small for the ring");
static_assert(B2_COUNT * 8 + 16 <= 1024, "barrier block too small");

// tanh of an accumulator fragment (+ bias / + U +- sigma V) packed into the A fragments of the next layer: the m64nN
// accumulator of a thread holds, for column block i, (row r, cols 8i + 2q, +1) in d[4i], d[4i+1] and (row r + 8, same cols)
// in d[4i+2], d[4i+3]; the k16 A fragment j of the next layer wants exactly the pairs d[8j .. 8j+7] in that order.
template <bool SPLIT> __device__ __forceinline__ void act_pack(const float (&z)[32], uint32_t (&hi)[16], uint32_t (&lo)[16]) {
#pragma unroll
    for (int k = 0; k < 16; ++k) {
        if (SPLIT) split_h2(tanh_acc(z[2 * k]), tanh_acc(z[2 * k + 1]), hi[k], lo[k]);
        else hi[k] = pack_h2(tanh_fast(z[2 * k]), tanh_fast(z[2 * k + 1]));
    }
}

// NOISE: the action-noise variant (loads of the noise array and the episode loop in the layer-3 epilogue); a separate
// instantiation so that the registers it needs do not cost the noise-free kernel anything
template <bool SPLIT, bool NOISE>
__global__ void __launch_bounds__(T2_THREADS, 1) rollout_tc2_kernel(const __grid_constant__ T2Params p,
                                                                     const __grid_constant__ T2Maps maps) {
    using C = T2Cfg<SPLIT>;
    constexpr int NP = C::NP, NSLOT = C::NSLOT;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    const T2Smem L = t2_layout<SPLIT>(p.nkc);
    uint64_t* bars = (uint64_t*)(smem + L.bars);
    float* bias_all = (float*)(smem + L.bias);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int NMT = p.n_mtiles, NKC = p.nkc;
    const int my_pairs = (p.r.n_pairs - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;

    // ---- one-time setup -----------------------------------------------------------------------------------------------
    if (tid == 0) {
        ((unsigned*)(smem + L.red + 2 * T2_CONS_WARPS * 64))[0] = 0;
        ((unsigned*)(smem + L.red + 2 * T2_CONS_WARPS * 64))[1] = 0;
        for (int s = 0; s < NSLOT; ++s) { mbar_init(&bars[B2_FULL + s], 1); mbar_init(&bars[B2_EMPTY + s], T2_WG_WARPS); }
        mbar_init(&bars[B2_EPS_TX], 1); mbar_init(&bars[B2_EPS_READY], 1); mbar_init(&bars[B2_EPS_FREE], T2_CONS_WARPS);
        mbar_init(&bars[B2_W_READY], 1); mbar_init(&bars[B2_W_FREE], T2_CONS_WARPS);
        for (int b = 0; b < 2; ++b) { mbar_init(&bars[B2_IMG_READY + b], T2_BLD_WARPS); mbar_init(&bars[B2_IMG_FREE + b], 1); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < T2_CONS_WARP0) {
        // warpgroup 0 (producer, copier, builders) only moves data: its registers go to the two consumer warpgroups
        reg_dealloc<T2_REGS_DATA>();
        if (warp == T2_W_PROD) {
            // ===================== producer: observation ring =====================
            // One FIFO of 8 KB slots in the order (pair, tile, warpgroup half, K chunk, piece): a slot is one warpgroup's 64
            // rows of a 16 KB stage image, so warpgroup 1's chain of a tile is fed after warpgroup 0's, and warpgroup 0's chain
            // of the next tile after that.
            if (lane == 0) {
                uint32_t slot = 0, phase = 0;
                const int per_tile = NKC * NP;
                for (int i = 0; i < my_pairs; ++i)
                    for (int m = 0; m < NMT; ++m)
                        for (int h = 0; h < 2; ++h)
                            for (int s = 0; s < per_tile; ++s) {
                                mbar_wait(&bars[B2_EMPTY + slot], phase ^ 1);
                                mbar_expect_tx(&bars[B2_FULL + slot], T2_SLOT);
                                bulk_g2s(smem + L.xst + slot * T2_SLOT, p.xnt + ((size_t)m * per_tile + s) * T2_STAGE + h * T2_SLOT,
                                         T2_SLOT, &bars[B2_FULL + slot]);
                                if (++slot == NSLOT) { slot = 0; phase ^= 1; }
                            }
            }
        } else if (warp == T2_W_COPY) {
            // ===================== copier: eps1 by TMA from the shadows (or from the image), W2/W3/bias from the image =====================
            const T2Image I = t2_image<SPLIT>(NKC, !p.use_tma);
            const uint8_t* my_images = p.images + (size_t)blockIdx.x * 2 * I.total;
            const uint32_t w_bytes = 2u * NP * (T2_B1_CHUNK + T2_W3_BLOCK);
            for (int i = 0; i < my_pairs; ++i) {
                const uint32_t b = i & 1, u = i >> 1;
                const uint8_t* img = my_images + (size_t)b * I.total;
                const int pair = blockIdx.x + i * gridDim.x;
                const long long slice = es_checked_slice(p.r.idx[pair], p.r.P, p.r.table_len, p.r.err);
                mbar_wait(&bars[B2_IMG_READY + b], u & 1);                             // builders have finished image i
                if (i > 0) mbar_wait(&bars[B2_EPS_FREE], (i - 1) & 1);                 // previous pair's last L1 has retired
                if (lane == 0) {
                    mbar_expect_tx(&bars[B2_EPS_TX], (uint32_t)(NP * NKC * T2_B1_CHUNK));
                    if (p.use_tma) {
                        const int unit0 = t2_shadow_unit(slice + p.r.w_off[0], p.shadow_stride);
#pragma unroll
                        for (int pc = 0; pc < NP; ++pc)
                            for (int kc = 0; kc < NKC; ++kc)
                                tma_load_3d(smem + L.b1 + (size_t)(kc * NP + pc) * T2_B1_CHUNK, pc ? &maps.lo : &maps.hi, 0, unit0 + 8 * kc, 0,
                                            &bars[B2_EPS_TX]);
                    } else {
                        for (int c = 0; c < NP * NKC; ++c)
                            bulk_g2s(smem + L.b1 + (size_t)c * T2_B1_CHUNK, img + I.b1 + (size_t)c * T2_B1_CHUNK, T2_B1_CHUNK, &bars[B2_EPS_TX]);
                    }
                }
                mbar_wait(&bars[B2_EPS_TX], i & 1);
                if (p.use_tma) {
                    // the unit holding column `obs` received the first elements of the next row: it carries the bias element
                    // eps_b1[n] (the observation tile has a constant 1 there) and zeros (obs % 8 == 0 on this path)
                    const int kcb = p.r.dims[0] >> 6, ub = (p.r.dims[0] & 63) >> 3;
#pragma unroll
                    for (int rr = 0; rr < 2; ++rr) {
                        const int n = 2 * lane + rr;
                        const float eb = ldg_stream(p.r.table + slice + p.r.b_off[0] + n);
                        __half hi, lo;
                        split_h1(eb, hi, lo);
                        const uint32_t off = (uint32_t)(kcb * NP) * T2_B1_CHUNK + n * 128 + ((ub ^ (n & 7)) << 4);      // [kc][piece] blocks
                        *(uint4*)(smem + L.b1 + off) = make_uint4((uint32_t)__half_as_ushort(hi), 0, 0, 0);
                        if (SPLIT) *(uint4*)(smem + L.b1 + T2_B1_CHUNK + off) = make_uint4((uint32_t)__half_as_ushort(lo), 0, 0, 0);
                    }
                    fence_async_smem();
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&bars[B2_EPS_READY]);
                if (p.use_tma && lane == 0 && i + 1 < my_pairs) {
                    // the next pair's eps1 rows into L2 now, so that its TMA at the pair boundary does not wait on HBM
                    const long long nslice = es_checked_slice(p.r.idx[pair + gridDim.x], p.r.P, p.r.table_len, nullptr);
                    const int nunit0 = t2_shadow_unit(nslice + p.r.w_off[0], p.shadow_stride);
#pragma unroll
                    for (int pc = 0; pc < NP; ++pc)
                        for (int kc = 0; kc < NKC; ++kc) tma_prefetch_3d(pc ? &maps.lo : &maps.hi, 0, nunit0 + 8 * kc, 0);
                }
                if (i > 0) mbar_wait(&bars[B2_W_FREE], (i - 1) & 1);                   // previous pair's last L3 has retired
                if (lane == 0) {
                    mbar_expect_tx(&bars[B2_W_READY], w_bytes + 1024);
                    bulk_g2s(smem + L.w2, img + I.w2, w_bytes, &bars[B2_W_READY]);     // W2 [sign][piece], W3 [sign][piece]: contiguous in both
                    bulk_g2s((uint8_t*)bias_all + (i & 1) * 1024, img + I.bias, 1024, &bars[B2_W_READY]);
                }
                mbar_wait(&bars[B2_W_READY], i & 1);                                   // landed: the image slot may be rewritten
                __syncwarp();
                if (lane == 0) mbar_arrive(&bars[B2_IMG_FREE + b]);
            }
        } else {
            // ===================== builder warps: W2+-, W3+-, biases (and eps1 without the shadows) one pair ahead =====================
            const int btid = tid - T2_BLD_WARP0 * 32;
            constexpr int BT = T2_BLD_WARPS * 32;
            const T2Image I = t2_image<SPLIT>(NKC, !p.use_tma);
            uint8_t* my_images = p.images + (size_t)blockIdx.x * 2 * I.total;
            const float sg = p.r.sigma;
            for (int j = 0; j < my_pairs; ++j) {
                const int pair = blockIdx.x + j * gridDim.x;
                mbar_wait(&bars[B2_IMG_FREE + (j & 1)], (((uint32_t)j >> 1) & 1) ^ 1);
                const long long slice = es_checked_slice(p.r.idx[pair], p.r.P, p.r.table_len, nullptr);
                const float* __restrict__ eps = p.r.table + slice;
                uint8_t* img = my_images + (size_t)(j & 1) * I.total;
                // W2+- / W3+-: element pairs (n, k), (n, k+1)
                const int n2 = T2_H * T2_H / 2, n3 = T2_ACT_PAD * T2_H / 2;
                for (int e2 = btid; e2 < n2 + n3; e2 += BT) {
                    const bool l3 = e2 >= n2;
                    const int k2 = 2 * (l3 ? e2 - n2 : e2);
                    const int n = k2 >> 6, kk = k2 & 63;
                    const int at = (l3 ? p.r.w_off[2] : p.r.w_off[1]) + k2;
                    const bool live = !l3 || n < p.r.act;
                    float wp0 = 0.f, wp1 = 0.f, wn0 = 0.f, wn1 = 0.f;
                    if (live) {
                        es_pheno_pm(sg, ldg_stream(eps + at), __ldg(p.r.theta + at), wp0, wn0);
                        es_pheno_pm(sg, ldg_stream(eps + at + 1), __ldg(p.r.theta + at + 1), wp1, wn1);
                    }
                    const uint32_t blk = l3 ? T2_W3_BLOCK : T2_B1_CHUNK;
                    uint8_t* base = img + (l3 ? I.w3 : I.w2) + sw128_off(n, kk);
                    if (SPLIT) {
                        __half h0, l0, h1, l1;
                        split_h1(wp0, h0, l0); split_h1(wp1, h1, l1);
                        *(uint32_t*)(base + 0 * blk) = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
                        *(uint32_t*)(base + 1 * blk) = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
                        split_h1(wn0, h0, l0); split_h1(wn1, h1, l1);
                        *(uint32_t*)(base + 2 * blk) = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
                        *(uint32_t*)(base + 3 * blk) = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
                    } else {
                        *(uint32_t*)(base + 0 * blk) = pack_h2(wp0, wp1);
                        *(uint32_t*)(base + 1 * blk) = pack_h2(wn0, wn1);
                    }
                }
                {
                    float* bias = (float*)(img + I.bias);
                    for (int e = btid; e < T2_H + T2_ACT_PAD; e += BT) {
                        if (e < T2_H) {
                            es_pheno_pm(sg, ldg_stream(eps + p.r.b_off[1] + e), __ldg(p.r.theta + p.r.b_off[1] + e), bias[e], bias[T2_H + e]);
                        } else {
                            const int j2 = e - T2_H;
                            float vp = 0.f, vn = 0.f;
                            if (j2 < p.r.act) es_pheno_pm(sg, ldg_stream(eps + p.r.b_off[2] + j2), __ldg(p.r.theta + p.r.b_off[2] + j2), vp, vn);
                            bias[2 * T2_H + j2] = vp; bias[2 * T2_H + T2_ACT_PAD + j2] = vn;
                        }
                    }
                }
                if (!p.use_tma) {
                    // eps1 (unscaled) converted from the float32 slice: rows of 64, K padded to nkc*64, column `obs` = eps_b1
                    const int Kp = NKC * T2_KC;
                    for (int e2 = btid; e2 < T2_H * Kp / 2; e2 += BT) {
                        const int n = (2 * e2) / Kp, k = (2 * e2) - n * Kp;
                        float x0 = 0.f, x1 = 0.f;
                        if (k < p.r.dims[0]) x0 = ldg_stream(eps + p.r.w_off[0] + (size_t)n * p.r.dims[0] + k); else if (k == p.r.dims[0]) x0 = ldg_stream(eps + p.r.b_off[0] + n);
                        if (k + 1 < p.r.dims[0]) x1 = ldg_stream(eps + p.r.w_off[0] + (size_t)n * p.r.dims[0] + k + 1); else if (k + 1 == p.r.dims[0]) x1 = ldg_stream(eps + p.r.b_off[0] + n);
                        uint8_t* dst = img + I.b1 + (size_t)((k >> 6) * NP) * T2_B1_CHUNK + sw128_off(n, k & 63);     // [kc][piece] blocks
                        if (SPLIT) {
                            __half h0, l0, h1, l1;
                            split_h1(x0, h0, l0); split_h1(x1, h1, l1);
                            *(uint32_t*)dst = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
                            *(uint32_t*)(dst + T2_B1_CHUNK) = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
                        } else {
                            *(uint32_t*)dst = pack_h2(x0, x1);
                        }
                    }
                }
                __threadfence();                                             // image visible device-wide (L2)
                asm volatile("fence.proxy.async;" ::: "memory");             // ... and to the async proxy that will copy it
                __syncwarp();
                if (lane == 0) mbar_arrive(&bars[B2_IMG_READY + (j & 1)]);
                if (j + 1 < my_pairs) {                                      // L2 prefetch of the next pair's operands
                    const long long nidx = es_checked_slice(p.r.idx[blockIdx.x + (j + 1) * gridDim.x], p.r.P, p.r.table_len, nullptr);
                    const char* nxt = (const char*)(p.r.table + nidx);
                    const int lines = (p.r.b_off[2] + p.r.act) * 4 / 128 + 2;
                    const int skip = p.use_tma ? p.r.b_off[0] * 4 / 128 : 0;         // with the shadows eps1 comes by TMA
                    for (int l = skip + btid; l < lines; l += BT) prefetch_l2(nxt + (size_t)l * 128);
                }
            }
    }
    } else {
        reg_alloc<T2_REGS_MATH>();
        // ===================== consumer warpgroups: MMAs and epilogues of 64 rows of every tile =====================
        const int cw = warp - T2_CONS_WARP0;                  // 0..7
        const int half = cw >> 2;                             // rows 64*half .. 64*half + 63 of the tile
        const int q = lane & 3;
        const int r0 = half * 64 + (cw & 3) * 16 + (lane >> 2);   // this thread's rows: r0 and r0 + 8
        const float sg = p.r.sigma;
        const bool want_pos = p.r.behv_pos != nullptr;
        const uint64_t a_desc0 = wg_desc_sw128(smem_u32(smem + L.xst));
        const uint64_t b1_desc0 = wg_desc_sw128(smem_u32(smem + L.b1));
        const uint64_t w2d = wg_desc_sw128(smem_u32(smem + L.w2)), w3d = wg_desc_sw128(smem_u32(smem + L.w3));
        constexpr uint64_t SLOT_D = T2_SLOT >> 4, B1_D = T2_B1_CHUNK >> 4, W3_D = T2_W3_BLOCK >> 4;
        double* red = (double*)(smem + L.red);                // [pair parity][8 warps][8]: per-pair sums of every consumer warp
        unsigned* red_cnt = (unsigned*)(smem + L.red + 2 * T2_CONS_WARPS * 64);
        // The ring holds the chains of both warpgroups in turn: warpgroup 0's slots of tile m, then warpgroup 1's, then
        // warpgroup 0's of tile m + 1, ...  `fifo` is the ring position of this warpgroup's next slot.
        uint32_t fifo = (uint32_t)(half * NKC * NP);
        for (int i = 0; i < my_pairs; ++i) {
            const int pair = blockIdx.x + i * gridDim.x;
            const float* bias = bias_all + (i & 1) * 256;
            double fit_p = 0.0, fit_n = 0.0;
            float pp0 = 0.f, pp1 = 0.f, pp2 = 0.f, pn0 = 0.f, pn1 = 0.f, pn2 = 0.f;     // position sums of this thread's rows
            mbar_wait_warp(&bars[B2_EPS_READY], i & 1);
            for (int m = 0; m < NMT; ++m) {
                const int ta = m * T2_MT + r0, tb = ta + 8;                        // time steps of this thread's two rows
                // U of this thread's two rows, loaded once for both signs (issued before the L1 chain, which hides the latency)
                float u[32];
                {
                    const float* __restrict__ urow = p.ubase + (size_t)ta * T2_H + 2 * q;
#pragma unroll
                    for (int c = 0; c < 8; ++c) {
                        const float2 u0 = __ldg(reinterpret_cast<const float2*>(urow + 8 * c));
                        const float2 u1 = __ldg(reinterpret_cast<const float2*>(urow + 8 * T2_H + 8 * c));
                        u[4 * c + 0] = u0.x; u[4 * c + 1] = u0.y; u[4 * c + 2] = u1.x; u[4 * c + 3] = u1.y;
                    }
                }
                // ---- L1: V = Xn . eps1^T (SPLIT: x_hi.eps_hi + x_hi.eps_lo + x_lo.eps_hi), chunk by chunk through the ring ----
                float v[32];
                reg_fence(v);
                wg_fence();
                uint32_t prev = 0;
                for (int kc = 0; kc < NKC; ++kc) {
                    const uint32_t st = fifo & (NSLOT - 1), phase = (fifo / NSLOT) & 1;
                    mbar_wait_warp(&bars[B2_FULL + st], phase);
                    if (SPLIT) mbar_wait_warp(&bars[B2_FULL + st + 1], phase);
                    const uint64_t ah = a_desc0 + st * SLOT_D, al = ah + SLOT_D;
                    const uint64_t bh = b1_desc0 + (uint64_t)kc * NP * B1_D, bl = bh + B1_D;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        wgmma64_ss(v, ah + 2 * k, bh + 2 * k, (kc | k) != 0);
                        if (SPLIT) {
                            wgmma64_ss(v, ah + 2 * k, bl + 2 * k, 1);
                            wgmma64_ss(v, al + 2 * k, bh + 2 * k, 1);
                        }
                    }
                    wg_commit();
                    if (kc > 0) {                                  // chunk kc - 1 has retired: its slots go back to the producer
                        wg_wait<1>();
                        if (lane == 0) { mbar_arrive(&bars[B2_EMPTY + prev]); if (SPLIT) mbar_arrive(&bars[B2_EMPTY + prev + 1]); }
                    }
                    prev = st;
                    fifo += NP;
                }
                fifo += (uint32_t)(NKC * NP);                      // the other warpgroup's chain of this tile
                wg_wait<0>();
                reg_fence(v);
                if (lane == 0) {
                    mbar_arrive(&bars[B2_EMPTY + prev]);
                    if (SPLIT) mbar_arrive(&bars[B2_EMPTY + prev + 1]);
                    if (m == NMT - 1) mbar_arrive(&bars[B2_EPS_FREE]);            // the pair's last L1 has retired
                }
                if (m == 0) mbar_wait_warp(&bars[B2_W_READY], i & 1);                  // W2, W3 and the biases of the pair in place?

                // ---- epi1: h1 = tanh(U +- sigma V) ----
                auto epi1 = [&](float s, uint32_t (&hh)[16], uint32_t (&hl)[16]) {
                    float z[32];
#pragma unroll
                    for (int k = 0; k < 32; ++k) z[k] = __fmaf_rn(v[k], s, u[k]);
                    act_pack<SPLIT>(z, hh, hl);
                };
                // ---- L2: D2 = h1 . W2^T (SPLIT: h_hi.w_hi + h_hi.w_lo + h_lo.w_hi), one commit group ----
                auto mma2 = [&](int sgn, const uint32_t (&hh)[16], const uint32_t (&hl)[16], float (&d2)[32]) {
                    const uint64_t w2h = w2d + (uint64_t)(sgn * NP) * B1_D, w2l = w2h + B1_D;
                    reg_fence(d2);
                    wg_fence();
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        const uint32_t ah[4] = {hh[4 * k], hh[4 * k + 1], hh[4 * k + 2], hh[4 * k + 3]};
                        wgmma64_rs(d2, ah, w2h + 2 * k, k != 0);
                        if (SPLIT) {
                            const uint32_t al[4] = {hl[4 * k], hl[4 * k + 1], hl[4 * k + 2], hl[4 * k + 3]};
                            wgmma64_rs(d2, ah, w2l + 2 * k, 1);
                            wgmma64_rs(d2, al, w2h + 2 * k, 1);
                        }
                    }
                    wg_commit();
                };
                // ---- epi2: h2 = tanh(D2 + b2) ----
                auto epi2 = [&](int sgn, float (&d2)[32], uint32_t (&hh)[16], uint32_t (&hl)[16]) {
                    const float* b2 = bias + sgn * T2_H + 2 * q;
#pragma unroll
                    for (int c = 0; c < 8; ++c) {
                        const float2 bb = *reinterpret_cast<const float2*>(b2 + 8 * c);
                        d2[4 * c + 0] = __fadd_rn(d2[4 * c + 0], bb.x); d2[4 * c + 1] = __fadd_rn(d2[4 * c + 1], bb.y);
                        d2[4 * c + 2] = __fadd_rn(d2[4 * c + 2], bb.x); d2[4 * c + 3] = __fadd_rn(d2[4 * c + 3], bb.y);
                    }
                    act_pack<SPLIT>(d2, hh, hl);
                };
                // ---- L3: D3 = h2 . W3^T (N = 32), one commit group ----
                auto mma3 = [&](int sgn, const uint32_t (&hh)[16], const uint32_t (&hl)[16], float (&d3)[16]) {
                    const uint64_t w3h = w3d + (uint64_t)(sgn * NP) * W3_D, w3l = w3h + W3_D;
                    reg_fence(d3);
                    wg_fence();
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        const uint32_t ah[4] = {hh[4 * k], hh[4 * k + 1], hh[4 * k + 2], hh[4 * k + 3]};
                        wgmma32_rs(d3, ah, w3h + 2 * k, k != 0);
                        if (SPLIT) {
                            const uint32_t al[4] = {hl[4 * k], hl[4 * k + 1], hl[4 * k + 2], hl[4 * k + 3]};
                            wgmma32_rs(d3, ah, w3l + 2 * k, 1);
                            wgmma32_rs(d3, al, w3h + 2 * k, 1);
                        }
                    }
                    wg_commit();
                };
                // ---- epi3: a = tanh(D3 + b3) [+ action noise]; r_t = <a_t, c_t>; positions ----
                // With action noise, episode ep of n_eps sees a + its own noise; the two rows' float32 rewards are summed over
                // the episodes in float64, in order, and divided by n_eps (obj.py:54-63); the positions are the last episode's.
                // The first episode is straight-line code as in the single-episode kernel; the others loop and recompute the
                // tanh (keeping the 16 actions live across the loop would cost registers).  (epi3_episode serves the NOISE
                // instantiations only.)
                float rw[16];                                                      // c_t of this thread's D3 elements (!NOISE)
                auto epi3_episode = [&](int sgn, const float (&d3)[16], const float* __restrict__ nz, float& ra, float& rb,
                                        float& q0, float& q1, float& q2) {
                    const float* b3 = bias + 2 * T2_H + sgn * T2_ACT_PAD;
                    ra = 0.f; rb = 0.f; q0 = 0.f; q1 = 0.f; q2 = 0.f;
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const int col = 8 * c + 2 * q + (e & 1);
                            const int t = (e & 2) ? tb : ta;
                            const float z = __fadd_rn(d3[4 * c + e], b3[col]);
                            float a = SPLIT ? tanh_acc(z) : tanh_fast(z);
                            if (col < p.r.act && t < p.r.T) {
                                if (NOISE && nz)                // a += rs.randn(act) * ac_std (src/nn/nn.py:47-48), drawn by mt_gauss.cu
                                    a += __ldg(nz + (size_t)t * p.r.act + col);
                                const float r = a * __ldg(p.r.rew_vec + (size_t)t * p.r.act + col);
                                if (e & 2) rb += r; else ra += r;
                                // position integrator: action components 0, 1, 2
                                q0 += (col == 0) ? a : 0.f; q1 += (col == 1) ? a : 0.f; q2 += (col == 2) ? a : 0.f;
                            }
                        }
                    }
                    ra += __shfl_xor_sync(0xffffffffu, ra, 1); ra += __shfl_xor_sync(0xffffffffu, ra, 2);
                    rb += __shfl_xor_sync(0xffffffffu, rb, 1); rb += __shfl_xor_sync(0xffffffffu, rb, 2);
                };
                auto epi3 = [&](int sgn, const float (&d3)[16]) {
                    if (!NOISE) {          // the noise-free kernels: one episode, c from registers
                        const float* b3 = bias + 2 * T2_H + sgn * T2_ACT_PAD;
                        float ra = 0.f, rb = 0.f, q0 = 0.f, q1 = 0.f, q2 = 0.f;
#pragma unroll
                        for (int c = 0; c < 4; ++c) {
#pragma unroll
                            for (int e = 0; e < 4; ++e) {
                                const int col = 8 * c + 2 * q + (e & 1);
                                const int t = (e & 2) ? tb : ta;
                                const float z = __fadd_rn(d3[4 * c + e], b3[col]);
                                const float a = SPLIT ? tanh_acc(z) : tanh_fast(z);
                                if (col < p.r.act && t < p.r.T) {
                                    const float r = a * rw[4 * c + e];
                                    if (e & 2) rb += r; else ra += r;
                                    q0 += (col == 0) ? a : 0.f; q1 += (col == 1) ? a : 0.f; q2 += (col == 2) ? a : 0.f;
                                }
                            }
                        }
                        ra += __shfl_xor_sync(0xffffffffu, ra, 1); ra += __shfl_xor_sync(0xffffffffu, ra, 2);
                        rb += __shfl_xor_sync(0xffffffffu, rb, 1); rb += __shfl_xor_sync(0xffffffffu, rb, 2);
                        const double r2 = (q == 0) ? (double)ra + (double)rb : 0.0;   // rows beyond T contribute 0
                        if (sgn) { fit_n += r2; pn0 += q0; pn1 += q1; pn2 += q2; }
                        else     { fit_p += r2; pp0 += q0; pp1 += q1; pp2 += q2; }
                        return;
                    }
                    const int n_ep = p.r.n_episodes;
                    const float* __restrict__ nz = p.r.act_noise ? p.r.act_noise + ((size_t)pair * 2 + sgn) * n_ep * p.r.T * p.r.act : nullptr;
                    float ra, rb, q0, q1, q2;
                    epi3_episode(sgn, d3, nz, ra, rb, q0, q1, q2);
                    double r2 = (q == 0) ? (double)ra + (double)rb : 0.0;   // rows beyond T contribute 0
                    if (n_ep > 1) {
                        double sa = (double)ra, sb = (double)rb;
#pragma unroll 1
                        for (int ep = 1; ep < n_ep; ++ep) {
                            epi3_episode(sgn, d3, nz + (size_t)ep * p.r.T * p.r.act, ra, rb, q0, q1, q2);
                            sa += (double)ra; sb += (double)rb;
                        }
                        if (q == 0) r2 = sa / n_ep + sb / n_ep;
                    }
                    if (sgn) { fit_n += r2; pn0 += q0; pn1 += q1; pn2 += q2; }
                    else     { fit_p += r2; pp0 += q0; pp1 += q1; pp2 += q2; }
                };
                // The + sign runs one phase ahead of the - sign, so every L2 / L3 chain is in flight on the tensor pipe while the
                // tanh of the other sign runs: L2+ under epi1-, L2- under epi2+, L3+ under epi2-, L3- under epi3+.  Each wait
                // leaves the most recent group in flight; the reg_fences after it keep the retired chain's A fragments alive
                // until then, and its accumulators from being read before.
                uint32_t hp[16], lp[16], hn[16], ln[16];
                float d2p[32], d2n[32], d3p[16], d3n[16];
                epi1(sg, hp, lp);
                mma2(0, hp, lp, d2p);
                epi1(-sg, hn, ln);
                mma2(1, hn, ln, d2n);
                wg_wait<1>();
                reg_fence(d2p); reg_fence(hp); if (SPLIT) reg_fence(lp);
                epi2(0, d2p, hp, lp);
                mma3(0, hp, lp, d3p);
                wg_wait<1>();
                reg_fence(d2n); reg_fence(hn); if (SPLIT) reg_fence(ln);
                epi2(1, d2n, hn, ln);
                mma3(1, hn, ln, d3n);
                // c_t of this thread's 16 elements of D3, loaded once for both signs (NOISE: element by element in epi3_episode)
                if (!NOISE) {
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const int col = 8 * c + 2 * q + (e & 1);
                            const int t = (e & 2) ? tb : ta;
                            rw[4 * c + e] = (col < p.r.act && t < p.r.T) ? __ldg(p.r.rew_vec + (size_t)t * p.r.act + col) : 0.f;
                        }
                    }
                }
                wg_wait<1>();
                reg_fence(d3p); reg_fence(hp); if (SPLIT) reg_fence(lp);
                epi3(0, d3p);
                wg_wait<0>();
                reg_fence(d3n); reg_fence(hn); if (SPLIT) reg_fence(ln);
                if (m == NMT - 1 && lane == 0) mbar_arrive(&bars[B2_W_FREE]);   // the pair's last L3 has retired
                epi3(1, d3n);
            }
            // ---- this warp's sums of the pair -> shared memory; the last of the 8 warps adds them in warp order and writes the
            //      pair's results (no global scratch, no device-wide fence: a CTA-scope release/acquire on a shared counter) ----
            double* mine = red + ((size_t)(i & 1) * T2_CONS_WARPS + cw) * 8;
            const double fitp = es_warp_sum(fit_p), fitn = es_warp_sum(fit_n);
            const double ps[6] = {es_warp_sum<double>(pp0), es_warp_sum<double>(pp1), es_warp_sum<double>(pp2),
                                  es_warp_sum<double>(pn0), es_warp_sum<double>(pn1), es_warp_sum<double>(pn2)};
            if (lane == 0) {
                mine[0] = fitp; mine[1] = fitn;
#pragma unroll
                for (int k = 0; k < 6; ++k) mine[2 + k] = ps[k];
                __threadfence_block();
                // monotonic arrival counter per parity slot (pairs i, i+2, ... share one: no warp can be a whole pair ahead)
                if (atomicAdd(red_cnt + (i & 1), 1u) == (unsigned)(T2_CONS_WARPS * ((i >> 1) + 1) - 1)) {
                    __threadfence_block();
                    double tot[8] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
                    const volatile double* all = red + (size_t)(i & 1) * T2_CONS_WARPS * 8;
                    for (int w = 0; w < T2_CONS_WARPS; ++w)
#pragma unroll
                        for (int k = 0; k < 8; ++k) tot[k] += all[w * 8 + k];
                    p.r.fit_pos[(size_t)pair * p.r.fit_stride] = tot[0];
                    p.r.fit_neg[(size_t)pair * p.r.fit_stride] = tot[1];
                    if (want_pos) {
                        // components 1 and 2 of an action narrower than 3 repeat component 0 (index % act)
                        for (int s2 = 0; s2 < 2; ++s2) {
                            const double* ts = tot + 2 + 3 * s2;
                            float* out = (s2 ? p.r.behv_neg : p.r.behv_pos) + pair * 3;
                            out[0] = p.r.pos_scale * (float)ts[0];
                            out[1] = p.r.pos_scale * (float)(p.r.act > 1 ? ts[1] : ts[0]);
                            out[2] = p.r.pos_scale * (float)(p.r.act > 2 ? ts[2] : ts[0]);
                        }
                    }
                }
            }
            __syncwarp();
        }
    }
}

// observation stream -> float16 (hi[, lo]), tiled into the shared-memory image of each (M tile, K chunk, piece) stage
template <bool SPLIT>
__global__ void rollout_tc2_prep_kernel(const float* __restrict__ obsn, int T, int obs, int nkc, int n_mtiles, uint8_t* __restrict__ xnt) {
    constexpr int NP = SPLIT ? 2 : 1;
    const size_t total = (size_t)n_mtiles * nkc * T2_MT * T2_KC;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int k = (int)(i % T2_KC);
        const int row = (int)((i / T2_KC) % T2_MT);
        const int kc = (int)((i / (T2_KC * T2_MT)) % nkc);
        const int m = (int)(i / ((size_t)T2_KC * T2_MT * nkc));
        const int t = m * T2_MT + row, kk = kc * T2_KC + k;
        const float v = (kk < obs) ? ((t < T) ? obsn[(size_t)t * obs + kk] : 0.f) : ((kk == obs) ? 1.0f : 0.f);   // col `obs` = 1: bias
        uint8_t* stage = xnt + ((size_t)(m * nkc + kc) * NP) * T2_STAGE;
        __half hi, lo;
        split_h1(v, hi, lo);
        *(__half*)(stage + sw128_off(row, k)) = hi;
        if (SPLIT) *(__half*)(stage + T2_STAGE + sw128_off(row, k)) = lo;
    }
}

// U[t][n] = b1[n] + sum_k Xn[t][k] * theta1[n][k], the unperturbed part of layer 1 that the pair kernels (this file and
// rollout_f32x.cu) share between the two signs of a pair: accumulated in float64 (k ascending) and rounded once to float32, so
// that splitting z1+- = U +- sigma V adds no rounding of its own to the theta term.  Output: row-major [n_tiles * 128][64]
// (0 beyond T).
constexpr int T2_UB_ROWS = 8, T2_UB_KT = 64, T2_UB_RPT = T2_UB_ROWS / 4;
__global__ void __launch_bounds__(256) rollout_ubase_kernel(const float* __restrict__ obsn, const float* __restrict__ theta,
                                                             int w1, int b1, int T, int obs, float* __restrict__ ubase) {
    __shared__ float s_w[T2_UB_KT][T2_H + 1];
    __shared__ float s_x[T2_UB_ROWS][T2_UB_KT];
    const int n = threadIdx.x & 63, rg = threadIdx.x >> 6;
    const int t0 = blockIdx.x * T2_UB_ROWS;
    double acc[T2_UB_RPT];
#pragma unroll
    for (int r = 0; r < T2_UB_RPT; ++r) acc[r] = (double)__ldg(theta + b1 + n);
    for (int k0 = 0; k0 < obs; k0 += T2_UB_KT) {
        const int kn = min(T2_UB_KT, obs - k0);
        for (int i = threadIdx.x; i < T2_H * T2_UB_KT; i += 256) {
            const int nn = i / T2_UB_KT, kk = i - nn * T2_UB_KT;
            s_w[kk][nn] = (kk < kn) ? __ldg(theta + w1 + (size_t)nn * obs + k0 + kk) : 0.f;
        }
        for (int i = threadIdx.x; i < T2_UB_ROWS * T2_UB_KT; i += 256) {
            const int r = i / T2_UB_KT, kk = i - r * T2_UB_KT;
            const int t = t0 + r;
            s_x[r][kk] = (kk < kn && t < T) ? obsn[(size_t)t * obs + k0 + kk] : 0.f;
        }
        __syncthreads();
        for (int kk = 0; kk < kn; ++kk) {
            const double w = (double)s_w[kk][n];
#pragma unroll
            for (int r = 0; r < T2_UB_RPT; ++r) acc[r] = fma((double)s_x[rg * T2_UB_RPT + r][kk], w, acc[r]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int r = 0; r < T2_UB_RPT; ++r) {
        const int t = t0 + rg * T2_UB_RPT + r;
        ubase[(size_t)t * T2_H + n] = (t < T) ? (float)acc[r] : 0.f;
    }
}

// float16 shadows of the table: copy s, element j = f16(table[j + s]) (hi) / f16(table[j+s] - hi) (lo); zero beyond the end
__global__ void rollout_tc2_shadow_kernel(const float* __restrict__ table, int64_t len, size_t stride, __half* __restrict__ hi,
                                          __half* __restrict__ lo) {
    const size_t total = stride / 2;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int s = blockIdx.y;
        const int64_t j = (int64_t)(2 * i) + s;
        const float a = (j < len) ? __ldg(table + j) : 0.f, b = (j + 1 < len) ? __ldg(table + j + 1) : 0.f;
        __half ah, al, bh, bl;
        split_h1(a, ah, al); split_h1(b, bh, bl);
        *(__half2*)(hi + (size_t)s * stride + 2 * i) = __halves2half2(ah, bh);
        if (lo) *(__half2*)(lo + (size_t)s * stride + 2 * i) = __halves2half2(al, bl);
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// 3-D map over a shadow allocation of 8 x stride float16: {64 elements, origin in 16-byte units (stride 16 B), 64 rows (stride
// obs*2 B)}; box {64, 1, 64} with the 128-byte swizzle = one K chunk of eps1 in the K-major operand layout
int t2_encode_map(CUtensorMap* map, void* base, size_t stride, int obs) {
    static EncodeTiledFn encode = nullptr;
    if (!encode) {
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", (void**)&encode, cudaEnableDefault, &qres) != cudaSuccess || !encode) {
            (void)cudaGetLastError();
            encode = nullptr;
            return -1;
        }
    }
    const cuuint64_t gdim[3] = {64, (cuuint64_t)stride /* = 8*stride/8 units */, 64};
    const cuuint64_t gstr[2] = {16, (cuuint64_t)obs * 2};
    const cuuint32_t box[3] = {64, 1, 64}, estr[3] = {1, 1, 1};
    return encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, base, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS ? 0 : -1;
}

template <bool SPLIT>
int t2_launch(es_ctx* ctx, T2Params& p, const T2Maps& maps, cudaStream_t stream) {
    const T2Smem L = t2_layout<SPLIT>(p.nkc);
    const size_t smem = (size_t)L.total + 1024;       // + alignment slack
    if (smem > 227 * 1024) {
        es_set_error("es_rollout_openloop(TC%s): obs_dim %d needs %zu bytes of shared memory (> 227 KB)", SPLIT ? "3" : "", p.r.dims[0], smem);
        return ES_ERR_UNSUPPORTED;
    }
    constexpr int NP = SPLIT ? 2 : 1;
    const size_t xnt_bytes = (size_t)p.n_mtiles * p.nkc * NP * T2_STAGE;
    const size_t ub_bytes = (size_t)p.n_mtiles * T2_MT * T2_H * sizeof(float);
    const int grid = p.r.n_pairs < ctx->sm_count ? p.r.n_pairs : ctx->sm_count;
    const size_t img_bytes = (((size_t)grid * 2 * t2_image<SPLIT>(p.nkc, !p.use_tma).total) + 255) & ~(size_t)255;
    void* scratch = nullptr;
    int rc = es_ctx_scratch(ctx, xnt_bytes + ub_bytes + img_bytes, &scratch);
    if (rc) return rc;
    char* at = (char*)scratch;
    uint8_t* xnt = (uint8_t*)at; at += xnt_bytes;
    float* ubase = (float*)at; at += ub_bytes;
    p.images = (uint8_t*)at;
    p.xnt = xnt; p.ubase = ubase;
    {
        const size_t total = (size_t)p.n_mtiles * p.nkc * T2_MT * T2_KC;
        int blocks = es_div_up((int64_t)total, 256);
        if (blocks > ctx->sm_count * 8) blocks = ctx->sm_count * 8;
        rollout_tc2_prep_kernel<SPLIT><<<blocks, 256, 0, stream>>>(p.r.obsn, p.r.T, p.r.dims[0], p.nkc, p.n_mtiles, xnt);
        ES_LAUNCHED(ctx);
        rc = es_launch_ubase(ctx, p.r, p.n_mtiles, ubase, stream);
        if (rc) return rc;
    }
    if (p.r.act_noise) {
        ES_CHECK_CUDA(cudaFuncSetAttribute(rollout_tc2_kernel<SPLIT, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        rollout_tc2_kernel<SPLIT, true><<<grid, T2_THREADS, smem, stream>>>(p, maps);
    } else {
        ES_CHECK_CUDA(cudaFuncSetAttribute(rollout_tc2_kernel<SPLIT, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        rollout_tc2_kernel<SPLIT, false><<<grid, T2_THREADS, smem, stream>>>(p, maps);
    }
    ES_LAUNCHED(ctx);
    return ES_OK;
}

}  // namespace

int es_launch_ubase(es_ctx* ctx, const EsRollout& r, int n_tiles, float* ubase, cudaStream_t stream) {
    rollout_ubase_kernel<<<n_tiles * T2_MT / T2_UB_ROWS, 256, 0, stream>>>(r.obsn, r.theta, r.w_off[0], r.b_off[0], r.T, r.dims[0], ubase);
    ES_LAUNCHED(ctx);
    return ES_OK;
}

void es_tc2_free_shadows(es_ctx* ctx) {
    if (ctx->sh16_hi) cudaFree(ctx->sh16_hi);
    if (ctx->sh16_lo) cudaFree(ctx->sh16_lo);
    if (ctx->sh16_maps) free(ctx->sh16_maps);
    ctx->sh16_hi = ctx->sh16_lo = nullptr;
    ctx->sh16_maps = nullptr;
    ctx->sh16_src = nullptr;
}

// the largest obs_dim whose layout fits in shared memory: 511 (TC, 8 K chunks) / 383 (TC3, 6 K chunks)
template <bool SPLIT> static int t2_max_obs() {
    int nkc = 1;
    while ((size_t)t2_layout<SPLIT>(nkc + 1).total + 1024 <= 227 * 1024) ++nkc;
    return nkc * T2_KC - 1;                              // nkc = ceil((obs + 1) / 64)
}

int es_impl_rollout_tc2(es_ctx* ctx, const EsRollout& r, int split, cudaStream_t stream) {
    const int* ls = r.dims;
    const int max_obs = split ? t2_max_obs<true>() : t2_max_obs<false>();
    if (r.n_layers != 3 || ls[1] != T2_H || ls[2] != T2_H || ls[3] > T2_ACT_PAD) {
        es_set_error("es_rollout_openloop(TC%s): the tensor-core path covers obs(<=%d)-64-64-act(<=32) tanh MLPs; "
                     "use ES_ROLLOUT_F32 for other shapes (the wide tensor-core path covers obs(<=256) with 2 to 4 hidden layers "
                     "of widths in {64, 128, 192, 256} and act(<=32))", split ? "3" : "", max_obs);
        return ES_ERR_UNSUPPORTED;
    }
    if (ls[0] > max_obs) {                               // refused before any float16 shadow of the table is built
        es_set_error("es_rollout_openloop(TC%s): obs_dim %d needs more than 227 KB of shared memory (this mode covers "
                     "obs_dim <= %d)", split ? "3" : "", ls[0], max_obs);
        return ES_ERR_UNSUPPORTED;
    }
    const int obs = ls[0];
    T2Params p;
    memset(&p, 0, sizeof(p));
    p.r = r;
    p.nkc = es_div_up(obs + 1, T2_KC);                   // + the constant-1 column that carries the L1 bias
    p.n_mtiles = es_div_up(r.T, T2_MT);

    // float16 shadows of the table (hi always, lo when a split rollout asks for it): 8 shifted copies each, built once per
    // (table pointer, length) and addressed through two TMA tensor maps.  Needs 16-byte aligned rows in every slice (obs % 8
    // == 0).  Without them (other shapes, no memory, no driver entry point) the builder warps convert the float32 slice.
    T2Maps maps;
    memset(&maps, 0, sizeof(maps));
    p.use_tma = 0;
    if (obs % 8 == 0 && !ctx->sh16_failed) {
        const size_t stride = ((size_t)r.table_len + 64 * (size_t)obs + 79) & ~(size_t)7;       // room for the last slice's rows
        const bool fresh = ctx->sh16_src != r.table || ctx->sh16_len != r.table_len || ctx->sh16_stride != stride || ctx->sh16_obs != obs;
        if (fresh) es_tc2_free_shadows(ctx);
        bool ok = true;
        if (!ctx->sh16_hi) {
            ok = cudaMalloc(&ctx->sh16_hi, 8 * stride * sizeof(__half)) == cudaSuccess;
            if (ok) {
                rollout_tc2_shadow_kernel<<<dim3(ctx->sm_count * 8, 8), 256, 0, stream>>>(r.table, r.table_len, stride, (__half*)ctx->sh16_hi, nullptr);
                ES_LAUNCHED(ctx);
            }
        }
        if (ok && split && !ctx->sh16_lo) {
            ok = cudaMalloc(&ctx->sh16_lo, 8 * stride * sizeof(__half)) == cudaSuccess;
            if (ok) {
                // (recomputes hi: simpler than a second kernel, runs once per table)
                rollout_tc2_shadow_kernel<<<dim3(ctx->sm_count * 8, 8), 256, 0, stream>>>(r.table, r.table_len, stride, (__half*)ctx->sh16_hi,
                                                                                        (__half*)ctx->sh16_lo);
                ES_LAUNCHED(ctx);
            }
        }
        if (ok && !ctx->sh16_maps) {
            void* m = nullptr;
            ok = posix_memalign(&m, 64, sizeof(T2Maps)) == 0;
            if (ok) { memset(m, 0, sizeof(T2Maps)); ctx->sh16_maps = m; ctx->sh16_maps_lo = 0; }
            if (ok) ok = t2_encode_map(&((T2Maps*)ctx->sh16_maps)->hi, ctx->sh16_hi, stride, obs) == 0;
        }
        if (ok && split && !ctx->sh16_maps_lo) {
            ok = t2_encode_map(&((T2Maps*)ctx->sh16_maps)->lo, ctx->sh16_lo, stride, obs) == 0;
            if (ok) ctx->sh16_maps_lo = 1;
        }
        if (!ok) {
            (void)cudaGetLastError();
            es_tc2_free_shadows(ctx);
            ctx->sh16_failed = 1;
        } else {
            ctx->sh16_src = r.table; ctx->sh16_len = r.table_len; ctx->sh16_stride = stride; ctx->sh16_obs = obs;
            maps = *(T2Maps*)ctx->sh16_maps;
            p.use_tma = 1;
            p.shadow_stride = stride;
        }
    }
    return split ? t2_launch<true>(ctx, p, maps, stream) : t2_launch<false>(ctx, p, maps, stream);
}
