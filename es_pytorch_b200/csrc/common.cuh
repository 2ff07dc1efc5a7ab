// common.cuh -- shared host/device helpers for libes_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include "../../include/es_b200.h"

#ifndef __CUDA_ARCH_LIST__
#endif

struct es_ctx {
    int device;
    int sm_count;
    int64_t launches;
    // scratch owned by the ctx (grown on demand, never shrunk)
    void* scratch;          // generic scratch (reconstruct partials, rank keys, ...)
    size_t scratch_bytes;
    unsigned* counters;     // small zero-initialised counter array (last-block detection)
    size_t n_counters;
    // float16 shadows for rollout_tc2.cu: hi = f16(table), lo = f16(table - hi) (split rollout only), 8 shifted copies each,
    // plus the two TMA tensor maps over them (host copy, 64-byte aligned)
    const float* sh16_src;
    int64_t sh16_len;
    void* sh16_hi;
    void* sh16_lo;
    void* sh16_maps;
    int sh16_maps_lo;
    size_t sh16_stride;
    int sh16_obs;
    int sh16_failed;
    // asynchronous kernel-side argument errors: a mapped, page-locked host word the kernels set when a noise index is
    // out of range (the reference asserts `len > i + size`, src/core/noisetable.py:34); surfaced by es_check_async and
    // by the next entry point
    volatile int* err_host;
    int* err_dev;
    int mj_lists_ready;     // mt_gauss.cu: the set-bit lists of the jump polynomials have been built on this device
};

#define ES_ASYNC_BAD_INDEX 1
#define ES_ASYNC_RNG_OVERFLOW 2      // es_draw_noisy (jump-ahead path): the stream consumed more words than were generated ahead
#define ES_ASYNC_RANDN_OVERFLOW 3    // es_randn: the n values needed more words than its windows generated
#define ES_ASYNC_F16_RANGE 4         // es_rollout_openloop_activation (TC3): a hidden activation beyond float16 range
#define ES_ASYNC_WALK_OVERFLOW 5     // es_rollout_closedloop_terminal_streams: a stream walked past the words generated ahead

void es_set_error(const char* fmt, ...);

#define ES_CHECK_CUDA(expr)                                                              \
    do {                                                                                 \
        cudaError_t _e = (expr);                                                         \
        if (_e != cudaSuccess) {                                                         \
            es_set_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #expr,              \
                         cudaGetErrorString(_e));                                        \
            return ES_ERR_CUDA;                                                          \
        }                                                                                \
    } while (0)

#define ES_REQUIRE(cond, ...)                                                            \
    do {                                                                                 \
        if (!(cond)) {                                                                   \
            es_set_error(__VA_ARGS__);                                                   \
            return ES_ERR_INVALID;                                                       \
        }                                                                                \
    } while (0)

// after a kernel launch: count it and surface launch-configuration errors
#define ES_LAUNCHED(ctx)                                                                 \
    do {                                                                                 \
        (ctx)->launches++;                                                               \
        ES_CHECK_CUDA(cudaGetLastError());                                               \
    } while (0)

int es_ctx_scratch(es_ctx* ctx, size_t bytes, void** out);
int es_ctx_counters(es_ctx* ctx, size_t n, unsigned** out);

static inline int es_div_up(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

// flat offsets of the parameters of an obs-h1-h2-act MLP in state-dict order (src/core/policy.py:33-35):
// W1 [h1][obs], b1, W2 [h2][h1], b2, W3 [act][h2], b3
struct EsMlpOffsets { int w1, b1, w2, b2, w3, b3; };
__host__ __device__ inline EsMlpOffsets es_mlp_offsets(int obs, int h1, int h2, int act) {
    EsMlpOffsets o;
    o.w1 = 0; o.b1 = h1 * obs; o.w2 = o.b1 + h1; o.b2 = o.w2 + h2 * h1; o.w3 = o.b2 + h2; o.b3 = o.w3 + act * h2;
    return o;
}

// one rollout call of the antithetic pairs idx[0 .. n_pairs), validated and completed by api.cu; the kernels take it by value
struct EsRollout {
    const float* table;
    int64_t table_len;
    const int64_t* idx;
    int n_pairs;
    const float* theta;
    int P;
    float sigma;
    int n_layers;
    // the policy's activation after every layer (ES_ACT_*; 0 = tanh) and its float32 parameter (leaky ReLU's slope, ELU's
    // alpha).  Both sit in alignment holes of the struct, so its size and every other member's offset are those of a call
    // without them, and the kernels that take the struct by value are unchanged
    int activation;
    const float* obsn;          // open loop: normalised observations [T][obs]
    const float* rew_vec;       // [T][act]
    int T;
    float pos_scale;
    double* fit_pos;
    double* fit_neg;
    int fit_stride;
    float* behv_pos;            // [n_pairs][3] or NULL
    float* behv_neg;
    const float* act_noise;     // scaled action noise [n_pairs][2][n_episodes][T][act] (mt_gauss.cu) or NULL
    int* err;                   // the ctx's error word (es_checked_slice)
    int n_episodes;             // episodes per evaluation, averaged per step (>= 1; 1 when act_noise is NULL)
    // the policy head: bins == 0, the tanh outputs are the actions; bins >= 2, a binned-action policy (FFBinned): the last
    // layer's adim * bins outputs become adim actions, low[j] + range[j] * (arg-max bin) / (bins - 1)
    int bins;
    const float* head_low;      // dev float [adim]
    const float* head_range;    // dev float [adim]
    // filled by api.cu from the caller's layer sizes once they are checked
    int dims[ES_MAX_LAYERS + 1];                        // obs, hidden..., the last layer's outputs
    int w_off[ES_MAX_LAYERS], b_off[ES_MAX_LAYERS];     // flat offsets of W_l [dims[l+1]][dims[l]] and b_l, state-dict order
    int act;                    // the env's action dimension: dims[n_layers], or adim = dims[n_layers] / bins
    float head_scale;           // a binned head's float32(1 / (bins - 1))
    float act_param;
};
static_assert(sizeof(void*) != 8 || sizeof(EsRollout) == 272, "EsRollout's members must keep their offsets");

// the call restricted to the pairs [p0, p0 + np)
static inline EsRollout es_rollout_rows(const EsRollout& r, int p0, int np) {
    EsRollout c = r;
    c.idx += p0;
    c.n_pairs = np;
    c.fit_pos += (size_t)p0 * r.fit_stride;
    c.fit_neg += (size_t)p0 * r.fit_stride;
    if (r.behv_pos) { c.behv_pos += (size_t)p0 * 3; c.behv_neg += (size_t)p0 * 3; }
    if (r.act_noise) c.act_noise += (size_t)p0 * 2 * r.n_episodes * r.T * r.act;
    return c;
}

// the closed-loop env, the observation normalisation and the ObStat increments of es_rollout_closedloop
struct EsClosedEnv {
    const double* ob_mean;
    const double* ob_std;
    double ob_clip;
    const float* obs0;
    const float* env_a;         // [band][obs]
    int band;
    const float* env_b;         // [act][obs]
    const uint32_t* coins;      // [n_pairs][4] save_obs coin words or NULL
    double save_obs_chance;
    double* ob_sum;             // [obs], or NULL with ob_sumsq and ob_count
    double* ob_sumsq;
    double* ob_count;           // [2]
    // with action noise and n_episodes > 1: the per-step float64 episode sums, [2 sm_count][T] (a [2][T] pair per CTA of
    // rollout_closed.cu, a [T] row per cluster of rollout_closedw.cu; either grid has at most sm_count CTAs / clusters)
    double* ep_rows;
};

// an env whose episodes end early (es_rollout_closedloop_terminal), uniform over the launch.  Every other closed-loop call
// passes steps == NULL: its episodes run T steps whatever the position (a NaN included; fall_height = inf would not do that,
// since !(|NaN| <= inf))
struct EsTerm {
    float fall_height;          // h > 0: an episode ends after the step whose position leaves |z| <= h (or at T - 1)
    int32_t* steps;             // [2][n_pairs] (+ then -): the last episode's t_d
    int64_t* noise_used;        // [2][n_pairs] action-noise values the evaluation consumed (sum_e (t_{d,e} + 1) act), or NULL
};

// ---- entry points implemented one per .cu file (called from api.cu) -------------------------
int es_impl_draw_indices(es_ctx*, uint32_t*, int32_t*, int, int, uint64_t, int, int64_t*, uint32_t*, cudaStream_t);
int es_impl_mt_skip(es_ctx*, uint32_t*, int32_t*, int, int, cudaStream_t);
int es_impl_perturb(es_ctx*, const float*, const float*, int64_t, const int64_t*, int, int, float, float*, float*,
                    cudaStream_t);
int es_impl_normalise_obs(es_ctx*, const float*, const double*, const double*, double, int, int, float*, cudaStream_t);
int es_impl_obs_colsum(es_ctx*, const float*, int, int, float*, float*, cudaStream_t);
int es_impl_obstat_accumulate(es_ctx*, double*, double*, const float*, const float*, int, int, cudaStream_t);
int es_impl_obstat_accumulate_coins(es_ctx*, double*, double*, double*, const float*, const float*, int, int,
                                    const uint32_t*, int, double, cudaStream_t);
int es_impl_draw_noisy(es_ctx*, uint32_t*, int32_t*, int32_t*, double*, int, int, uint64_t, int, int, double, int64_t*, uint32_t*,
                       float*, cudaStream_t);
int es_impl_randn(es_ctx*, uint32_t*, int32_t*, int32_t*, double*, int64_t, float*, cudaStream_t);
int es_impl_randn_plan(const es_ctx*, int64_t, size_t*, int*);
int es_impl_rollout_f32(es_ctx*, const EsRollout&, cudaStream_t);
int es_impl_rollout_f32x(es_ctx*, const EsRollout&, cudaStream_t);
int es_impl_rollout_tc2(es_ctx*, const EsRollout&, int split, cudaStream_t);
void es_tc2_free_shadows(es_ctx* ctx);
// tanh MLPs with 2 to 4 hidden layers of widths in {64, 128, 192, 256}, obs <= 256, act <= 32, other than obs-64-64-act
bool es_tcw_covers(const EsRollout&);
int es_impl_rollout_tcw(es_ctx*, const EsRollout&, int split, cudaStream_t);
// binned heads on ES_ROLLOUT_TC3: 2 to 4 hidden layers of widths in {64, 128, 192, 256} (obs-64-64-X included), obs <= 256,
// adim * bins <= 256
bool es_tcw_covers_binned(const EsRollout&);
int es_impl_rollout_closed(es_ctx*, const EsRollout&, const EsClosedEnv&, cudaStream_t);
// the closed loop for MLPs with 2 to 4 hidden layers of <= 256 units, obs <= 384, act <= 64, an even band <= 16, on a
// thread-block cluster per evaluation (rollout_closedw.cu): tanh, binned heads (EsRollout::bins >= 2: every shape
// es_closedw_plan covers with act = adim) and the other activations, with or without action noise and an early end.  The
// cluster size and shared memory per CTA of a shape (or ES_ERR_UNSUPPORTED with the limit in es_last_error()), the clusters
// resident at once (bins: 0, or the binned head's; act: an activation other than tanh), and the rollout (`next`: a device
// word the launch zeroes)
int es_closedw_plan(const int* layer_sizes, int n_layers, int band, int* cluster_size, size_t* smem_bytes);
int es_closedw_binned_plan(const int* layer_sizes, int n_layers, int band, int bins, int* cluster_size, size_t* smem_bytes);
int es_closedw_max_clusters(int n_layers, int bins, bool act, int cluster_size, size_t smem_bytes, int* clusters);
int es_impl_rollout_closedw(es_ctx*, const EsRollout&, const EsClosedEnv&, const EsTerm&, unsigned* next, cudaStream_t);
// The words of es_rollout_closedloop_terminal_streams (mt_gauss.cu): every stream's tempered MT19937 words from its block 0 on,
// as far as n_pairs pairs of evaluations of N gaussians and `coins` coins each reach at es_draw_noisy's mean + 12 sigma, by
// the jump-ahead fill.  plan: no device work; ES_ERR_UNSUPPORTED beyond the jump-ahead range
struct EsStreamWords {
    int lb_log2, n_seg;
    size_t stride_words;        // per stream (a chunk of padding past the generated words included)
    uint32_t limit;             // the last word index a walk may reach
    size_t words_bytes, order_bytes;    // the scratch of the fill (256-byte multiples)
};
int es_impl_stream_words_plan(const es_ctx*, const char* fn, int n_streams, int n_pairs, int coins, int N, EsStreamWords*);
int es_impl_stream_words_fill(es_ctx*, const uint32_t* mt_key, int n_streams, const EsStreamWords&, uint32_t* words,
                              uint16_t* order, cudaStream_t);
// the stream walk (rollout_closedw_walk.cu): the arguments of es_rollout_closedloop_terminal_streams beyond the rollout's
struct EsStreamWalk {
    uint32_t* mt_key; int32_t* mt_pos; int32_t* has_gauss; double* gauss;
    int n_streams, n_per_stream;
    uint64_t upper_bound;
    int coins;
    double ac_std;
    int64_t* idx_out; uint32_t* coin_out; float* noise_trace;
};
int es_impl_rollout_closedw_walk(es_ctx*, const EsRollout&, const EsClosedEnv&, const EsTerm&, const EsStreamWalk&, cudaStream_t);
// policies with an activation other than tanh (EsRollout::activation != ES_ACT_TANH) on ES_ROLLOUT_TC3: the shapes of
// es_tcw_covers_act, rollout_tcw.cu's code (rollout_tcw_act.cu)
bool es_tcw_covers_act(const EsRollout&);
int es_impl_rollout_tcw_act(es_ctx*, const EsRollout&, cudaStream_t);
// U = Xn . theta1^T + b1 of an obs-64-... MLP for the pair kernels (rollout_tc2.cu): row-major [n_tiles * 128][64], 0 beyond T
int es_launch_ubase(es_ctx*, const EsRollout&, int n_tiles, float* ubase, cudaStream_t);
int es_impl_novelty(es_ctx*, const float*, int, const double*, int, int, double*, int, cudaStream_t);
int es_impl_fitness_objective(es_ctx*, int, double*, int, const float*, int, int, cudaStream_t);
int es_impl_mean_reward_steps(es_ctx*, double*, int, const int*, int, cudaStream_t);
int es_impl_rank_transform(es_ctx*, const double*, const double*, int, int, int, double, double, int, int, int,
                           const int64_t*, float*, double*, int32_t*, double*, int32_t*, int64_t*, cudaStream_t);
int es_impl_grad_reconstruct(es_ctx*, const float*, int64_t, const int64_t*, const float*, int, int, float*,
                             cudaStream_t);
int es_impl_adam(es_ctx*, float*, float*, float*, const float*, float, float, float, float, float, float, float, float,
                 int, cudaStream_t);
int es_impl_sgd(es_ctx*, float*, float*, const float*, float, float, float, float, float, int, cudaStream_t);
int es_impl_simple(es_ctx*, float*, const float*, float, float, float, int, cudaStream_t);

#ifdef __CUDACC__
// start of the noise slice of one perturbation, checked like NoiseTable.get (src/core/noisetable.py:34:
// `assert len(self) > i + size`).  An out-of-range index is reported through the ctx's mapped error word and replaced
// by 0 (a valid address): the launch's results are garbage and the caller is told so by the next entry point /
// es_check_async.
__device__ __forceinline__ long long es_checked_slice(long long i, int P, long long table_len, int* err) {
    if (i < 0 || i + (long long)P >= table_len) {
        if (err) *(volatile int*)err = ES_ASYNC_BAD_INDEX;
        return 0;
    }
    return i;
}
// Policy.pheno (src/core/policy.py:61-64): `params = self.flat_params + self.std * noise` for noise and -noise, the product
// and the sum rounded separately
__device__ __forceinline__ void es_pheno_pm(float sigma, float e, float t, float& w_plus, float& w_minus) {
    const float d = __fmul_rn(sigma, e);
    w_plus = __fadd_rn(t, d);
    w_minus = __fadd_rn(t, -d);
}
template <typename T> __device__ __forceinline__ T es_warp_sum(T v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// the warp-wide sums of v[0..7] in 9 shuffles (transposing butterfly): lane L returns the sum over the lanes of v[L / 4]
__device__ __forceinline__ float es_warp_sum8(const float (&v)[8], int lane) {
    const bool h16 = lane & 16, h8 = lane & 8, h4 = lane & 4;
    float a[4], b[2], c;
#pragma unroll
    for (int i = 0; i < 4; ++i) a[i] = (h16 ? v[i + 4] : v[i]) + __shfl_xor_sync(0xffffffffu, h16 ? v[i] : v[i + 4], 16);
#pragma unroll
    for (int i = 0; i < 2; ++i) b[i] = (h8 ? a[i + 2] : a[i]) + __shfl_xor_sync(0xffffffffu, h8 ? a[i] : a[i + 2], 8);
    c = (h4 ? b[1] : b[0]) + __shfl_xor_sync(0xffffffffu, h4 ? b[0] : b[1], 4);
    c += __shfl_xor_sync(0xffffffffu, c, 2);
    c += __shfl_xor_sync(0xffffffffu, c, 1);
    return c;
}
// a float32 pair held in one 64-bit register (element 0 in the low half), updated by two independent, identically rounded
// FMAs (sm_90 has no packed f32x2 FMA)
typedef unsigned long long es_f32x2;
__device__ __forceinline__ es_f32x2 es_pack2(float lo, float hi) {
    es_f32x2 v;
    asm("mov.b64 %0, {%1, %2};" : "=l"(v) : "f"(lo), "f"(hi));
    return v;
}
__device__ __forceinline__ void es_unpack2(es_f32x2 v, float& lo, float& hi) { asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v)); }
__device__ __forceinline__ es_f32x2 es_fma2(es_f32x2 a, es_f32x2 b, es_f32x2 c) {
    float a0, a1, b0, b1, c0, c1;
    es_unpack2(a, a0, a1); es_unpack2(b, b0, b1); es_unpack2(c, c0, c1);
    return es_pack2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ float es_hsum2(es_f32x2 v) {
    float a, b;
    es_unpack2(v, a, b);
    return a + b;
}
// the action of dimension j of a binned-action policy (FFBinned, src/nn/nn.py:99-117) from its bins outputs out(0 .. bins - 1):
// the first maximal bin, as torch.argmax (a NaN counts as the maximum), mapped to (scale * idx) * range[j] + low[j] with every
// operation rounded to float32 as the reference's torch expression does
template <typename Out>
__device__ __forceinline__ float es_binned_action(int bins, float scale, const float* low, const float* range, int j, Out out) {
    int best = 0;
    float bv = out(0);
    for (int b = 1; b < bins && bv == bv; ++b) {
        const float v = out(b);
        if (v > bv || v != v) { bv = v; best = b; }
    }
    return __fadd_rn(__fmul_rn(__fmul_rn(scale, (float)best), __ldg(range + j)), __ldg(low + j));
}
// a policy activation (ES_ACT_*, include/es_b200.h) other than tanh, in float32 as torch's CPU kernels evaluate it: ReLU is
// clamp_min(x, 0) (a NaN passes), leaky ReLU and ELU round their float32 parameter's product once, ELU takes expm1 (exp(x) - 1
// loses every digit near 0), sigmoid is 1 / (1 + e^-x) with the fast exponential and division (absolute error ~1e-7: e^-x
// carries (2 + 1.2 |x|) ulp, scaled by sigmoid(x) (1 - sigmoid(x)) <= 0.25, which falls as e^-|x|; the division 2 ulp; the IEEE
// forms made the wide tensor-core kernel with action noise spill)
template <int ACT>
__device__ __forceinline__ float es_act(float x, float param) {
    if constexpr (ACT == ES_ACT_RELU) return x < 0.f ? 0.f : x;
    else if constexpr (ACT == ES_ACT_LEAKY_RELU) return x > 0.f ? x : __fmul_rn(x, param);
    else if constexpr (ACT == ES_ACT_ELU) return x > 0.f ? x : __fmul_rn(param, expm1f(x));
    else return __fdividef(1.f, 1.f + __expf(-x));
}
// the same for a kind known at run time (uniform over the launch)
__device__ __forceinline__ float es_act(int kind, float param, float x) {
    switch (kind) {
        case ES_ACT_RELU: return es_act<ES_ACT_RELU>(x, param);
        case ES_ACT_LEAKY_RELU: return es_act<ES_ACT_LEAKY_RELU>(x, param);
        case ES_ACT_ELU: return es_act<ES_ACT_ELU>(x, param);
        default: return es_act<ES_ACT_SIGMOID>(x, param);
    }
}
// tanh(x) = 1 - 2 / (1 + e^2x) with the fast exponential and division: absolute error ~1e-7 (tanhf is ~40 dependent
// instructions per call); the closed-loop kernels end every phase of a step in one
__device__ __forceinline__ float es_tanh_exp(float x) {
    const float e = __expf(2.f * x);
    return 1.f - __fdividef(2.f, 1.f + e);
}
// raw observation i of the closed-loop env into a buffer with a wrap-around halo of the band (band <= obs): slot q = k + band / 2
// holds observation k mod obs for k in [-band / 2, obs + band - band / 2), so the band around any i is a linear read
template <typename V>
__device__ __forceinline__ void es_put_obs(V* __restrict__ buf, int i, V v, int obs, int band) {
    const int half = band >> 1;
    buf[i + half] = v;
    if (i >= obs - half) buf[i - obs + half] = v;
    if (i < band - half) buf[i + obs + half] = v;
}
#endif
