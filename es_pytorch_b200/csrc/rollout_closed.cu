// rollout_closed.cu -- antithetic pairs on the CLOSED-LOOP synthetic env (SURVEY.md section 8d's optional variant, reported
// separately from the open-loop headline): obs_{t+1} = tanh(A obs_t + B a_t), so the observation a policy sees depends on what
// it did and an episode cannot be batched over time like rollout_tc2.cu / rollout_f32x.cu do.  What replaces the reference here
// is the same loop as in the open-loop kernels -- Policy.pheno (src/core/policy.py:61-64), FeedForward.forward
// (src/nn/nn.py:42-50: clip((ob - mean) / std), Linear + Tanh x3), run_model's reward / position / saved observations
// (src/gym/gym_runner.py:33-67) -- with the env step inside it.
//
// Every step is a batch-1 matrix-vector product per policy, with weights that are unique per pair: the shape that is bound by
// where the WEIGHTS live.  Re-reading a pair's 117 KB slice from HBM at each of 1 000 steps is 1.2 PB per generation; so one
// CTA keeps one pair's perturbed weights on chip for the whole episode and the grid is persistent over the pairs:
//   * the three layers share one thread map: warp w owns rows 4 w .. 4 w + 3 of a layer, lane s the elements k = 32 j + s of
//     each of them.  Layer 1 (82 % of the weights): BOTH signs' weights of a thread's 4 x 12 elements live in registers (96)
//     as (+, -) pairs, so one pair of FMAs with the (x+, x-) pair of an input updates both evaluations; a warp reads every
//     input exactly once per step (one 8-byte load per lane and j);
//     the eight row sums of a warp meet in a transposing butterfly (9 shuffles).  Layers 2 / 3: the same with the weights in
//     shared memory, [row][j][lane] pairs;
//   * the env step: thread i owns observation i of both signs (A's diagonals and B transposed in shared memory; the raw
//     observations carry a wrap-around halo so the band is a linear read), normalises the new observation with its mean / std
//     (float64 like the reference: a float32 tensor minus a float64 ndarray) and keeps the float32 column sums of the
//     post-step observations for the ObStat of a rollout whose save_obs coin fell;
//   * reward (float32 dot in index order, summed in float64 like python's sum) and position by the last warp.
// Four barriers per step.
//
// Action noise and episodes (rollout_closed_noisy_kernel, es_rollout_closedloop_mlp_episodes): FeedForward.forward adds
// rs.randn(act) * ac_std to the action (src/nn/nn.py:47-48) and obj.py:54-63 averages E episodes per evaluation.  The lane
// that writes a row of layer 3 adds its (+ or -) noise value, loaded at the top of the step like the reward coefficients, so
// the env step, the reward and the position all see the noisy action.  Each episode restarts the env from obs_0 with the
// weights left in place; the per-step float64 sums of episodes 0 .. E - 2 go to a [2][T] row per CTA in global memory, and the
// last episode adds (row[t] + r) / E to the fitness and keeps the behaviour and the ObStat sums.
#include <math.h>
#include "common.cuh"
#include "mt19937.cuh"

namespace {

constexpr int CL_THREADS = 512;
constexpr int CL_WARPS = CL_THREADS / 32;
constexpr int CL_H = 64;                   // rows per layer at most (4 per warp)
constexpr int CL_A = 64;                   // action units at most
constexpr int CL_J23 = CL_H / 32;          // elements per lane and row in layers 2 / 3
constexpr int CL_HALO = 16;                // the raw observations carry a wrap-around halo of band entries (band <= 16)

struct ClParams {
    const float* table; long long table_len; const int64_t* idx; int n_pairs;
    const float* theta; float sigma;
    int obs, h1, h2, act, T, n_params;
    const double* ob_mean; const double* ob_std; double ob_clip;
    const float* obs0; const float* env_a; const float* env_b; int band;
    const float* crew; float pos_scale;
    const uint32_t* coins; double chance;
    double* fit_pos; double* fit_neg; int fit_stride;
    float* behv_pos; float* behv_neg;
    double* ob_sum; double* ob_sumsq; double* ob_count;
    int* err;
    const float* act_noise; int n_eps;      // [n_pairs][2][n_eps][T][act] (rollout_closed_noisy_kernel only)
    double* ep_row;                         // [gridDim.x][2][T] per-step episode sums (n_eps > 1)
};

struct ClLayout {                          // offsets in floats into dynamic shared memory
    int norm, w2, w3, bias, env_a, env_b, x2, o2, h1, h2, a2, prod, stat, racc, total, o2_stride, act_pad;
};
__host__ __device__ inline ClLayout cl_layout(int JL, int obs, int act, int band) {
    ClLayout L;
    int at = 0;
    L.act_pad = (act + 3) & ~3;
    L.o2_stride = obs + CL_HALO;
    L.norm = at; at += 4 * obs;             // double mean[obs], double 1/std[obs]  (first: 8-byte aligned)
    L.racc = at; at += 16;                  // fitness (double x 2) and position (float x 6) of the pair, last warp
    L.x2 = at; at += 2 * 32 * JL;           // float2 (x+, x-) normalised observations, zero padded to 32 JL
    L.w2 = at; at += 2 * CL_H * CL_J23 * 32;        // float2 (w+, w-) at [row][j][lane]
    L.w3 = at; at += 2 * CL_H * CL_J23 * 32;
    L.h1 = at; at += 2 * CL_H;              // float2 (h+, h-)
    L.h2 = at; at += 2 * CL_H;
    L.a2 = at; at += 2 * CL_A;
    L.prod = at; at += 2 * CL_A;
    L.stat = at; at += 4 * obs;             // float4 (sum+, sumsq+, sum-, sumsq-) of the post-step observations
    L.bias = at; at += 6 * CL_H;            // b1+ b1- b2+ b2- b3+ b3-
    L.o2 = at; at += 2 * 2 * L.o2_stride;   // [2 buffers] float2 raw observations with halo
    L.env_a = at; at += band * obs;
    L.env_b = at; at += L.act_pad * obs;
    L.total = at;
    return L;
}

// clip((ob - mean) / std) in float64 like the reference (a float32 tensor minus a float64 ndarray), the quotient as a product
// with the rounded reciprocal: the float64 result can differ in its last bit, which survives the rounding to float32 once in
// ~2^28 values (and then by one float32 ulp) -- far inside the tolerance this variant is held to
__device__ __forceinline__ float cl_normalise(float o, double mean, double rstd, double clip) {
    double x = ((double)o - mean) * rstd;
    x = isnan(x) ? x : fmin(fmax(x, -clip), clip);    // torch.clamp passes a NaN (fmax(NaN, -clip) is -clip)
    return (float)x;
}
// the float32 pairs (es_f32x2) of this kernel hold (+, -) of a weight times (x+, x-) of an input
// the four rows of a warp: z[r] (+, -) -> tanh(z + bias) of row 4 w + r, written by the lane that ends up with that sum
// (lanes 4 q: row 4 w + q / 2, sign q & 1); NZ: plus that lane's action noise nz
template <bool NZ = false>
__device__ __forceinline__ void cl_finish_rows(const es_f32x2 (&z)[4], int warp, int lane, int rows, const float* __restrict__ bias_p,
                                               const float* __restrict__ bias_m, float* __restrict__ out2, float nz = 0.f) {
    float v[8];
#pragma unroll
    for (int r = 0; r < 4; ++r) es_unpack2(z[r], v[2 * r], v[2 * r + 1]);
    const float c = es_warp_sum8(v, lane);
    if ((lane & 3) == 0) {
        const int q = lane >> 2, o = 4 * warp + (q >> 1), sg = q & 1;
        out2[2 * o + sg] = (o < rows) ? (NZ ? __fadd_rn(es_tanh_exp(c + (sg ? bias_m : bias_p)[o]), nz)
                                            : es_tanh_exp(c + (sg ? bias_m : bias_p)[o])) : 0.f;
    }
}

template <int JL, bool NOISY>
__device__ __forceinline__ void cl_rollout(const ClParams& p) {
    extern __shared__ __align__(16) float cl_smem[];
    const ClLayout L = cl_layout(JL, p.obs, p.act, p.band);
    double* __restrict__ nmean = reinterpret_cast<double*>(cl_smem + L.norm);
    double* __restrict__ nrstd = nmean + p.obs;
    double* __restrict__ rfit = reinterpret_cast<double*>(cl_smem + L.racc);        // [2]
    float* __restrict__ rpos = cl_smem + L.racc + 4;                                  // [2][3]
    es_f32x2* __restrict__ W2 = reinterpret_cast<es_f32x2*>(cl_smem + L.w2);
    es_f32x2* __restrict__ W3 = reinterpret_cast<es_f32x2*>(cl_smem + L.w3);
    float* __restrict__ bias = cl_smem + L.bias;
    float* __restrict__ envA = cl_smem + L.env_a;
    float* __restrict__ envB = cl_smem + L.env_b;
    float2* __restrict__ x2 = reinterpret_cast<float2*>(cl_smem + L.x2);
    float2* __restrict__ o2 = reinterpret_cast<float2*>(cl_smem + L.o2);
    float2* __restrict__ h1v = reinterpret_cast<float2*>(cl_smem + L.h1);
    float2* __restrict__ h2v = reinterpret_cast<float2*>(cl_smem + L.h2);
    float2* __restrict__ a2 = reinterpret_cast<float2*>(cl_smem + L.a2);
    float2* __restrict__ prod = reinterpret_cast<float2*>(cl_smem + L.prod);
    float4* __restrict__ stat = reinterpret_cast<float4*>(cl_smem + L.stat);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int obs = p.obs, h1 = p.h1, h2 = p.h2, act = p.act, T = p.T, band = p.band;
    const int act_pad = L.act_pad, o2s = L.o2_stride;
    const EsMlpOffsets off = es_mlp_offsets(obs, h1, h2, act);
    const bool l3_warp = 4 * warp < act;                        // warps that hold rows of layer 3
    const bool rew_warp = warp == CL_WARPS - 1;

    for (int i = tid; i < band * obs; i += CL_THREADS) envA[i] = p.env_a[i];
    for (int i = tid; i < act_pad * obs; i += CL_THREADS) envB[i] = i < act * obs ? p.env_b[i] : 0.f;
    for (int i = tid; i < 32 * JL; i += CL_THREADS) x2[i] = make_float2(0.f, 0.f);
    for (int i = tid; i < CL_H; i += CL_THREADS) { h1v[i] = make_float2(0.f, 0.f); h2v[i] = make_float2(0.f, 0.f); }
    for (int i = tid; i < CL_A; i += CL_THREADS) a2[i] = make_float2(0.f, 0.f);
    for (int i = tid; i < obs; i += CL_THREADS) { nmean[i] = p.ob_mean[i]; nrstd[i] = 1.0 / p.ob_std[i]; }
    __syncthreads();

    for (int pair = blockIdx.x; pair < p.n_pairs; pair += gridDim.x) {
        const long long base = es_checked_slice(p.idx[pair], p.n_params, p.table_len, p.err);
        const float* __restrict__ eps = p.table + base;
        const float* __restrict__ th = p.theta;
        const float sg = p.sigma;
        auto wpm = [&](int at) {                                   // (theta + sigma eps, theta - sigma eps)
            const float t = th[at];
            float wp, wm;
            es_pheno_pm(sg, eps[at], t, wp, wm);
            return es_pack2(wp, wm);
        };
        es_f32x2 w1[4][JL];                                        // (w+, w-) of rows 4 warp + r, elements 32 j + lane
#pragma unroll
        for (int r = 0; r < 4; ++r) {
#pragma unroll
            for (int j = 0; j < JL; ++j) {
                const int o = 4 * warp + r, k = 32 * j + lane;
                w1[r][j] = (o < h1 && k < obs) ? wpm(o * obs + k) : 0ull;
            }
        }
#pragma unroll
        for (int r = 0; r < 4; ++r) {
#pragma unroll
            for (int j = 0; j < CL_J23; ++j) {
                const int o = 4 * warp + r, k = 32 * j + lane;
                W2[(o * CL_J23 + j) * 32 + lane] = (o < h2 && k < h1) ? wpm(off.w2 + o * h1 + k) : 0ull;
                W3[(o * CL_J23 + j) * 32 + lane] = (o < act && k < h2) ? wpm(off.w3 + o * h2 + k) : 0ull;
            }
        }
        if (tid < CL_H) {
            float a, b;
            es_unpack2(tid < h1 ? wpm(off.b1 + tid) : 0ull, a, b);
            bias[tid] = a; bias[CL_H + tid] = b;
            es_unpack2(tid < h2 ? wpm(off.b2 + tid) : 0ull, a, b);
            bias[2 * CL_H + tid] = a; bias[3 * CL_H + tid] = b;
            es_unpack2(tid < act ? wpm(off.b3 + tid) : 0ull, a, b);
            bias[4 * CL_H + tid] = a; bias[5 * CL_H + tid] = b;
        }
        auto start_episode = [&]() {                                // a fresh env: obs_0, position 0
            for (int i = tid; i < obs; i += CL_THREADS) {
                const float v = p.obs0[i];
                es_put_obs(o2, i, make_float2(v, v), obs, band);
                const float xn = cl_normalise(v, nmean[i], nrstd[i], p.ob_clip);
                x2[i] = make_float2(xn, xn);
                stat[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
        };
        start_episode();
        if (tid < 2) rfit[tid] = 0.0;
        if (tid < 6) rpos[tid] = 0.f;
        // the save_obs coins of the pair's two evaluations (legacy random_sample < chance)
        bool save_p = false, save_m = false;
        if (p.coins) {
            const uint32_t* c = p.coins + (size_t)pair * 4;
            save_p = mt19937_random_sample(c[0], c[1]) < p.chance;
            save_m = mt19937_random_sample(c[2], c[3]) < p.chance;
        }
        const bool keep_stat = p.ob_sum && (save_p || save_m);
        __syncthreads();

        const int n_eps = NOISY ? p.n_eps : 1;
        for (int ep = 0; ep < n_eps; ++ep) {
            const bool last_ep = ep == n_eps - 1;
            const bool add_stat = keep_stat && last_ep;                 // behaviour and ObStat: the last episode's
            if (NOISY && ep > 0) {
                start_episode();
                if (tid < 6) rpos[tid] = 0.f;
                __syncthreads();
            }

            // this CTA's episode sums of the + / - evaluation, and the noise of the episode (row o of sign sg at lanes 4 q of the
            // warps that hold layer 3's rows, as cl_finish_rows writes them)
            double* __restrict__ erow = NOISY ? p.ep_row + (size_t)blockIdx.x * 2 * T : nullptr;
            const float* __restrict__ nzp = nullptr;
            if (NOISY && l3_warp && (lane & 3) == 0) {
                const int q = lane >> 2, o = 4 * warp + (q >> 1), sg = q & 1;
                if (o < act) nzp = p.act_noise + (((size_t)pair * 2 + sg) * n_eps + ep) * T * act + o;
            }

            for (int t = 0; t < T; ++t) {
                const int cur = t & 1;
                float crow0 = 0.f, crow1 = 0.f;
                double esum = 0.0;                                      // the earlier episodes' rewards of this step
                if (rew_warp) {                                         // this step's reward coefficients: in flight under the layers
                    const float* __restrict__ c = p.crew + (size_t)t * act;
                    if (lane < act) crow0 = __ldg(c + lane);
                    if (lane + 32 < act) crow1 = __ldg(c + lane + 32);
                    if (NOISY && lane < 2 && ep > 0) esum = erow[(size_t)lane * T + t];
                }
                float nz = 0.f;                                         // this lane's action noise: in flight under layers 1 / 2
                if (NOISY && nzp) nz = __ldg(nzp + (size_t)t * act);
                // ---- layer 1: 4 rows x JL elements per lane, weights in registers, every input read once per warp ----
                {
                    es_f32x2 z[4] = {0ull, 0ull, 0ull, 0ull};
                    const es_f32x2* __restrict__ xv = reinterpret_cast<const es_f32x2*>(x2) + lane;
    #pragma unroll
                    for (int j = 0; j < JL; ++j) {
                        const es_f32x2 x = xv[32 * j];
    #pragma unroll
                        for (int r = 0; r < 4; ++r) z[r] = es_fma2(w1[r][j], x, z[r]);
                    }
                    cl_finish_rows(z, warp, lane, h1, bias, bias + CL_H, reinterpret_cast<float*>(h1v));
                }
                __syncthreads();
                // ---- layer 2 ----
                {
                    es_f32x2 z[4] = {0ull, 0ull, 0ull, 0ull};
                    const es_f32x2* __restrict__ hv = reinterpret_cast<const es_f32x2*>(h1v) + lane;
                    const es_f32x2* __restrict__ wr = W2 + (size_t)(4 * warp) * CL_J23 * 32 + lane;
    #pragma unroll
                    for (int j = 0; j < CL_J23; ++j) {
                        const es_f32x2 x = hv[32 * j];
    #pragma unroll
                        for (int r = 0; r < 4; ++r) z[r] = es_fma2(wr[(r * CL_J23 + j) * 32], x, z[r]);
                    }
                    cl_finish_rows(z, warp, lane, h2, bias + 2 * CL_H, bias + 3 * CL_H, reinterpret_cast<float*>(h2v));
                }
                __syncthreads();
                // ---- layer 3 (only the warps that hold its rows) ----
                if (l3_warp) {
                    es_f32x2 z[4] = {0ull, 0ull, 0ull, 0ull};
                    const es_f32x2* __restrict__ hv = reinterpret_cast<const es_f32x2*>(h2v) + lane;
                    const es_f32x2* __restrict__ wr = W3 + (size_t)(4 * warp) * CL_J23 * 32 + lane;
    #pragma unroll
                    for (int j = 0; j < CL_J23; ++j) {
                        const es_f32x2 x = hv[32 * j];
    #pragma unroll
                        for (int r = 0; r < 4; ++r) z[r] = es_fma2(wr[(r * CL_J23 + j) * 32], x, z[r]);
                    }
                    cl_finish_rows<NOISY>(z, warp, lane, act, bias + 4 * CL_H, bias + 5 * CL_H, reinterpret_cast<float*>(a2), nz);
                }
                __syncthreads();
                // ---- env step: thread i owns observation i; the raw observations carry a wrap-around halo, so the band is a
                //      linear read ----
                if (tid < obs) {
                    const float2* __restrict__ oc = o2 + cur * o2s;
                    const int i = tid;
                    float ap = 0.f, am = 0.f, ap1 = 0.f, am1 = 0.f;
    #pragma unroll 4
                    for (int d = 0; d < band; d += 2) {                 // (band is even, checked on the host)
                        const float w0 = envA[d * obs + i], w1_ = envA[(d + 1) * obs + i];
                        const float2 u0 = oc[i + d], u1 = oc[i + d + 1];
                        ap = fmaf(w0, u0.x, ap); am = fmaf(w0, u0.y, am);
                        ap1 = fmaf(w1_, u1.x, ap1); am1 = fmaf(w1_, u1.y, am1);
                    }
    #pragma unroll 2
                    for (int j = 0; j < act_pad; j += 2) {
                        const float w0 = envB[j * obs + i], w1_ = envB[(j + 1) * obs + i];
                        const float4 av = *reinterpret_cast<const float4*>(a2 + j);
                        ap = fmaf(w0, av.x, ap); am = fmaf(w0, av.y, am);
                        ap1 = fmaf(w1_, av.z, ap1); am1 = fmaf(w1_, av.w, am1);
                    }
                    const float np_ = es_tanh_exp(ap + ap1), nm = es_tanh_exp(am + am1);
                    es_put_obs(o2 + (cur ^ 1) * o2s, i, make_float2(np_, nm), obs, band);
                    const double mu = nmean[i], rs_ = nrstd[i];
                    x2[i] = make_float2(cl_normalise(np_, mu, rs_, p.ob_clip), cl_normalise(nm, mu, rs_, p.ob_clip));
                    if (add_stat) {                                     // float32 column sums in step order (numpy's axis-0 reduction)
                        float4 st = stat[i];
                        st.x = __fadd_rn(st.x, np_); st.y = __fadd_rn(st.y, __fmul_rn(np_, np_));
                        st.z = __fadd_rn(st.z, nm);  st.w = __fadd_rn(st.w, __fmul_rn(nm, nm));
                        stat[i] = st;
                    }
                }
                // ---- reward and position: the last warp's lanes form the products, lanes 0 / 1 add them in index order (the env's
                //      float32 dot) for the + / - evaluation ----
                if (rew_warp) {
                    if (lane < act) { const float2 av = a2[lane]; prod[lane] = make_float2(__fmul_rn(av.x, crow0), __fmul_rn(av.y, crow0)); }
                    if (lane + 32 < act) { const float2 av = a2[lane + 32]; prod[lane + 32] = make_float2(__fmul_rn(av.x, crow1), __fmul_rn(av.y, crow1)); }
                    __syncwarp();
                    if (lane < 2) {
                        float acc = 0.f;
    #pragma unroll 8
                        for (int j = 0; j < act; ++j) {
                            const float2 pv = prod[j];
                            acc = __fadd_rn(acc, lane ? pv.y : pv.x);
                        }
                        if (!NOISY) {
                            rfit[lane] += (double)acc;
                        } else if (!last_ep) {                          // the float64 per-step sum over the episodes, in their order
                            erow[(size_t)lane * T + t] = esum + (double)acc;
                        } else {                                        // ... and its mean (obj.py:57-61)
                            rfit[lane] += (esum + (double)acc) / n_eps;
                        }
                        const float ps = p.pos_scale;
                        const float2 q0 = a2[0], q1 = a2[1 % act], q2 = a2[2 % act];
                        rpos[lane * 3 + 0] = __fadd_rn(rpos[lane * 3 + 0], __fmul_rn(ps, lane ? q0.y : q0.x));
                        rpos[lane * 3 + 1] = __fadd_rn(rpos[lane * 3 + 1], __fmul_rn(ps, lane ? q1.y : q1.x));
                        rpos[lane * 3 + 2] = __fadd_rn(rpos[lane * 3 + 2], __fmul_rn(ps, lane ? q2.y : q2.x));
                    }
                    __syncwarp();
                }
                __syncthreads();
            }
        }
        if (rew_warp && lane < 2) {
            (lane ? p.fit_neg : p.fit_pos)[(size_t)pair * p.fit_stride] = rfit[lane];
            float* bv = lane ? p.behv_neg : p.behv_pos;
            if (bv) { bv[(size_t)pair * 3 + 0] = rpos[lane * 3 + 0]; bv[(size_t)pair * 3 + 1] = rpos[lane * 3 + 1]; bv[(size_t)pair * 3 + 2] = rpos[lane * 3 + 2]; }
        }
        if (keep_stat) {
            // ObStat.inc of the saved rollouts (src/core/es.py:73-74, src/gym/training_result.py:17-21): float32 column sums
            // added in float64 (the order over rollouts is the atomics' -- float64 sums of a handful of terms)
            for (int i = tid; i < obs; i += CL_THREADS) {
                const float4 st = stat[i];
                if (save_p) { atomicAdd(p.ob_sum + i, (double)st.x); atomicAdd(p.ob_sumsq + i, (double)st.y); }
                if (save_m) { atomicAdd(p.ob_sum + i, (double)st.z); atomicAdd(p.ob_sumsq + i, (double)st.w); }
            }
            if (tid == 0) {
                const int n = (save_p ? 1 : 0) + (save_m ? 1 : 0);
                atomicAdd(p.ob_count, (double)(n * T));
                atomicAdd(p.ob_count + 1, (double)n);
            }
        }
        __syncthreads();                                            // the next pair overwrites the shared weights
    }
}

template <int JL>
__global__ void __launch_bounds__(CL_THREADS, 1) rollout_closed_kernel(const ClParams p) { cl_rollout<JL, false>(p); }
template <int JL>
__global__ void __launch_bounds__(CL_THREADS, 1) rollout_closed_noisy_kernel(const ClParams p) { cl_rollout<JL, true>(p); }

template <int JL>
int cl_launch(es_ctx* ctx, const ClParams& p, cudaStream_t stream) {
    const ClLayout L = cl_layout(JL, p.obs, p.act, p.band);
    const size_t smem = (size_t)L.total * sizeof(float);
    if (smem > 227 * 1024) {
        es_set_error("es_rollout_closedloop: %zu bytes of shared memory needed (obs %d, act %d, band %d), 227 KB available", smem, p.obs,
                     p.act, p.band);
        return ES_ERR_UNSUPPORTED;
    }
    const int grid = p.n_pairs < ctx->sm_count ? p.n_pairs : ctx->sm_count;
    if (p.act_noise) {
        ES_CHECK_CUDA(cudaFuncSetAttribute(rollout_closed_noisy_kernel<JL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        rollout_closed_noisy_kernel<JL><<<grid, CL_THREADS, smem, stream>>>(p);
    } else {
        ES_CHECK_CUDA(cudaFuncSetAttribute(rollout_closed_kernel<JL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        rollout_closed_kernel<JL><<<grid, CL_THREADS, smem, stream>>>(p);
    }
    ES_LAUNCHED(ctx);
    return ES_OK;
}

}  // namespace

int es_impl_rollout_closed(es_ctx* ctx, const EsRollout& r, const EsClosedEnv& env, cudaStream_t stream) {
    const int* dims = r.dims;
    ClParams p;
    p.table = r.table; p.table_len = r.table_len; p.idx = r.idx; p.n_pairs = r.n_pairs; p.theta = r.theta; p.sigma = r.sigma;
    p.obs = dims[0]; p.h1 = dims[1]; p.h2 = dims[2]; p.act = dims[3]; p.T = r.T; p.n_params = r.P;
    p.ob_mean = env.ob_mean; p.ob_std = env.ob_std; p.ob_clip = env.ob_clip;
    p.obs0 = env.obs0; p.env_a = env.env_a; p.env_b = env.env_b; p.band = env.band; p.crew = r.rew_vec; p.pos_scale = r.pos_scale;
    p.coins = env.coins; p.chance = env.save_obs_chance;
    p.fit_pos = r.fit_pos; p.fit_neg = r.fit_neg; p.fit_stride = r.fit_stride; p.behv_pos = r.behv_pos; p.behv_neg = r.behv_neg;
    p.ob_sum = env.ob_sum; p.ob_sumsq = env.ob_sumsq; p.ob_count = env.ob_count;
    p.err = r.err;
    p.act_noise = r.act_noise; p.n_eps = r.n_episodes; p.ep_row = env.ep_rows;
    if (p.h1 > CL_H || p.h2 > CL_H || p.act > CL_A || p.obs > 384 || p.band > CL_HALO || p.obs < p.band || (p.band & 1)) {
        es_set_error("es_rollout_closedloop: supports even band <= obs <= 384, hidden <= %d, act <= %d, band <= %d (got %d-%d-%d-%d, band %d)",
                     CL_H, CL_A, CL_HALO, p.obs, p.h1, p.h2, p.act, p.band);
        return ES_ERR_UNSUPPORTED;
    }
    if (p.obs <= 32) return cl_launch<1>(ctx, p, stream);
    if (p.obs <= 128) return cl_launch<4>(ctx, p, stream);
    return cl_launch<12>(ctx, p, stream);
}
