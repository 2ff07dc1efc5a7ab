// elementwise.cu -- the small kernels around the hot path: perturbation materialise,
// observation normalisation / column sums, novelty, and the optimizer steps.
// All float32 arithmetic mirrors the reference one IEEE operation at a time
// (__fmul_rn / __fadd_rn / ... so ptxas cannot contract a*b+c into an FMA).
#include "common.cuh"
#include "mt19937.cuh"

// ---- a3: theta +- sigma*eps  (src/core/policy.py:61-64) ----------------------------------------
__global__ void perturb_kernel(const float* __restrict__ theta, const float* __restrict__ table,
                               const int64_t* __restrict__ idx, int P, long long table_len, int* __restrict__ err,
                               float sigma, float* __restrict__ out_pos, float* __restrict__ out_neg) {
    const int k = blockIdx.y;
    const float* __restrict__ eps = table + es_checked_slice(idx[k], P, table_len, err);   // noisetable.py:34
    float* op = out_pos + (size_t)k * P;
    float* on = out_neg ? out_neg + (size_t)k * P : nullptr;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < P; p += gridDim.x * blockDim.x) {
        float wp, wm;
        es_pheno_pm(sigma, __ldg(eps + p), theta[p], wp, wm);
        op[p] = wp;
        if (on) on[p] = wm;
    }
}

int es_impl_perturb(es_ctx* ctx, const float* theta, const float* table, int64_t table_len, const int64_t* idx,
                    int n_idx, int P, float sigma, float* out_pos, float* out_neg, cudaStream_t stream) {
    ES_REQUIRE(n_idx <= 65535, "es_perturb: at most 65535 slices per call");
    dim3 grid(es_div_up(P, 256) < 64 ? es_div_up(P, 256) : 64, n_idx);
    perturb_kernel<<<grid, 256, 0, stream>>>(theta, table, idx, P, (long long)table_len, ctx->err_dev, sigma, out_pos, out_neg);
    ES_LAUNCHED(ctx);
    return ES_OK;
}

// ---- a4: clamp((o - mean)/std, +-clip) in float64, cast float32 (src/nn/nn.py:45) ----------------
__global__ void normalise_kernel(const float* __restrict__ obs, const double* __restrict__ mean,
                                 const double* __restrict__ std, double clip, int64_t n, int obs_dim,
                                 float* __restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int d = (int)(i % obs_dim);
        double x = __ddiv_rn(__dsub_rn((double)obs[i], mean[d]), std[d]);
        x = isnan(x) ? x : fmin(fmax(x, -clip), clip);              // torch.clamp passes a NaN (fmax(NaN, -clip) is -clip)
        out[i] = (float)x;
    }
}

int es_impl_normalise_obs(es_ctx* ctx, const float* obs, const double* mean, const double* std, double clip, int rows,
                          int obs_dim, float* out, cudaStream_t stream) {
    const int64_t n = (int64_t)rows * obs_dim;
    int blocks = es_div_up(n, 256);
    if (blocks > ctx->sm_count * 8) blocks = ctx->sm_count * 8;
    normalise_kernel<<<blocks, 256, 0, stream>>>(obs, mean, std, clip, n, obs_dim, out);
    ES_LAUNCHED(ctx);
    return ES_OK;
}

// ---- a14: float32 column sums in row order (src/gym/training_result.py:17-21) --------------------
// block = 64 columns x 4 row-lanes; tiles of 64 rows are staged in shared memory with coalesced loads (the next tile is
// prefetched into registers while the current one is summed); the sums themselves stay float32 in row order.
constexpr int CS_COLS = 64, CS_ROWS = 64;
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ obs, int rows, int obs_dim,
                                                     float* __restrict__ sum_out, float* __restrict__ sumsq_out) {
    __shared__ float tile[CS_ROWS][CS_COLS + 1];
    const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;          // column, row lane (0..3)
    const int d = blockIdx.x * CS_COLS + tx;
    const bool col_ok = d < obs_dim;
    float s = 0.f, q = 0.f;
    float pre[CS_ROWS / 4];
    auto load = [&](int r0) {
#pragma unroll
        for (int u = 0; u < CS_ROWS / 4; ++u) {
            const int r = r0 + ty + 4 * u;
            pre[u] = (col_ok && r < rows) ? __ldg(obs + (size_t)r * obs_dim + d) : 0.f;
        }
    };
    load(0);
    for (int r0 = 0; r0 < rows; r0 += CS_ROWS) {
#pragma unroll
        for (int u = 0; u < CS_ROWS / 4; ++u) tile[ty + 4 * u][tx] = pre[u];
        __syncthreads();
        if (r0 + CS_ROWS < rows) load(r0 + CS_ROWS);
        if (ty == 0) {
            const int n = min(CS_ROWS, rows - r0);
            for (int r = 0; r < n; ++r) {
                const float x = tile[r][tx];
                s = __fadd_rn(s, x);
                q = __fadd_rn(q, __fmul_rn(x, x));
            }
        }
        __syncthreads();
    }
    if (ty == 0 && col_ok) { sum_out[d] = s; sumsq_out[d] = q; }
}

int es_impl_obs_colsum(es_ctx* ctx, const float* obs, int rows, int obs_dim, float* sum_out, float* sumsq_out,
                       cudaStream_t stream) {
    colsum_kernel<<<es_div_up(obs_dim, CS_COLS), 256, 0, stream>>>(obs, rows, obs_dim, sum_out, sumsq_out);
    ES_LAUNCHED(ctx);
    return ES_OK;
}

__global__ void obstat_acc_kernel(double* __restrict__ sum, double* __restrict__ sumsq, const float* __restrict__ s,
                                  const float* __restrict__ ssq, int obs_dim, int n) {
    const int d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= obs_dim) return;
    double a = sum[d], b = sumsq[d];
    const double sa = (double)s[d], sb = (double)ssq[d];
    for (int i = 0; i < n; ++i) { a = __dadd_rn(a, sa); b = __dadd_rn(b, sb); }   // obstat.py:20-21
    sum[d] = a;
    sumsq[d] = b;
}

int es_impl_obstat_accumulate(es_ctx* ctx, double* sum, double* sumsq, const float* s, const float* ssq, int obs_dim,
                              int n, cudaStream_t stream) {
    obstat_acc_kernel<<<es_div_up(obs_dim, 64), 64, 0, stream>>>(sum, sumsq, s, ssq, obs_dim, n);
    ES_LAUNCHED(ctx);
    return ES_OK;
}

__global__ void coin_count_kernel(const uint32_t* __restrict__ coins, int n_coins, double chance, int* __restrict__ count) {
    int c = 0;
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n_coins; e += gridDim.x * blockDim.x) {
        const uint2 w = *reinterpret_cast<const uint2*>(coins + 2 * (size_t)e);
        c += (mt19937_random_sample(w.x, w.y) < chance) ? 1 : 0;
    }
    c = es_warp_sum(c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(count, c);
}

__global__ void obstat_coins_kernel(double* __restrict__ sum, double* __restrict__ sumsq, double* __restrict__ count_io,
                                    const float* __restrict__ s, const float* __restrict__ ssq, int obs_dim,
                                    int rows_per_rollout, const int* __restrict__ n_saved) {
    const int n = *n_saved;
    const int d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d < obs_dim) {
        double a = sum[d], b = sumsq[d];
        const double sa = (double)s[d], sb = (double)ssq[d];
        for (int i = 0; i < n; ++i) { a = __dadd_rn(a, sa); b = __dadd_rn(b, sb); }      // obstat.py:20-21, n times in order
        sum[d] = a;
        sumsq[d] = b;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        double cnt = count_io[0];
        for (int i = 0; i < n; ++i) cnt = __dadd_rn(cnt, (double)rows_per_rollout);
        count_io[0] = cnt;
        count_io[1] = (double)n;
    }
}

int es_impl_obstat_accumulate_coins(es_ctx* ctx, double* sum, double* sumsq, double* count_io, const float* s,
                                    const float* ssq, int obs_dim, int rows, const uint32_t* coins, int n_coins,
                                    double chance, cudaStream_t stream) {
    unsigned* cnt = nullptr;
    int rc = es_ctx_counters(ctx, 4096, &cnt);                    // slot 4095: coin counter (tickets use the low slots)
    if (rc) return rc;
    int* n_saved = (int*)(cnt + 4095);
    ES_CHECK_CUDA(cudaMemsetAsync(n_saved, 0, sizeof(int), stream));
    if (n_coins > 0) {
        int blocks = es_div_up(n_coins, 256);
        if (blocks > ctx->sm_count) blocks = ctx->sm_count;
        coin_count_kernel<<<blocks, 256, 0, stream>>>(coins, n_coins, chance, n_saved);
        ES_LAUNCHED(ctx);
    }
    obstat_coins_kernel<<<es_div_up(obs_dim, 64), 64, 0, stream>>>(sum, sumsq, count_io, s, ssq, obs_dim, rows, n_saved);
    ES_LAUNCHED(ctx);
    return ES_OK;
}

// ---- a13: novelty = mean of the k smallest distances (src/utils/novelty.py:16-18) ---------------
constexpr int NV_MAXK = 64;
__global__ void novelty_kernel(const float* __restrict__ behv, int n, const double* __restrict__ archive, int A, int k,
                               double* __restrict__ out, int out_stride) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const double bx = (double)behv[(size_t)e * 3 + 0], by = (double)behv[(size_t)e * 3 + 1];
    const int kk = k < A ? k : A;               // heapq.nsmallest clips to the archive size
    double best[NV_MAXK];                       // ascending
    int m = 0;
    for (int a = 0; a < A; ++a) {
        const double dx = __dsub_rn(archive[2 * a + 0], bx), dy = __dsub_rn(archive[2 * a + 1], by);
        const double d = sqrt(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
        if (m < kk) {
            int p = m++;
            while (p > 0 && best[p - 1] > d) { best[p] = best[p - 1]; --p; }
            best[p] = d;
        } else if (d < best[kk - 1]) {
            int p = kk - 1;
            while (p > 0 && best[p - 1] > d) { best[p] = best[p - 1]; --p; }
            best[p] = d;
        }
    }
    // np.mean's sum (numpy's pairwise_sum for n <= 128): sequential below 8 terms, else 8 strided accumulators combined
    // as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the n % 8 leftover terms in order
    double s = 0.0;
    if (kk < 8) {
        for (int i = 0; i < kk; ++i) s = __dadd_rn(s, best[i]);
    } else {
        double r[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = best[j];
        int i = 8;
        for (; i < kk - kk % 8; i += 8)
#pragma unroll
            for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], best[i + j]);
        s = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                      __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
        for (; i < kk; ++i) s = __dadd_rn(s, best[i]);
    }
    out[(size_t)e * out_stride] = __ddiv_rn(s, (double)kk);
}

int es_impl_novelty(es_ctx* ctx, const float* behv, int n, const double* archive, int A, int k, double* out,
                    int out_stride, cudaStream_t stream) {
    novelty_kernel<<<es_div_up(n, 128), 128, 0, stream>>>(behv, n, archive, A, k, out, out_stride);
    ES_LAUNCHED(ctx);
    return ES_OK;
}

// ---- a11/a12: g = l2*theta - gsum/n ; optimizer ; theta += step ------------------------------------
__device__ __forceinline__ float es_total_grad(float theta, float gsum, float n_ranked, float l2coeff) {
    const float grad = __fdiv_rn(gsum, n_ranked);                  // scale_noise(...) / n_fits_ranked  (es.py:100)
    return __fsub_rn(__fmul_rn(l2coeff, theta), grad);             // l2coeff * params - grad          (es.py:101)
}

__global__ void adam_kernel(float* __restrict__ theta, float* __restrict__ m, float* __restrict__ v,
                            const float* __restrict__ gsum, float n_ranked, float l2coeff, float neg_a, float b1,
                            float omb1, float b2, float omb2, float eps, int P) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const float t = theta[p];
    const float g = es_total_grad(t, gsum[p], n_ranked, l2coeff);
    const float mm = __fadd_rn(__fmul_rn(b1, m[p]), __fmul_rn(omb1, g));                 // optimizers.py:57
    const float vv = __fadd_rn(__fmul_rn(b2, v[p]), __fmul_rn(omb2, __fmul_rn(g, g)));   // optimizers.py:58
    const float step = __fdiv_rn(__fmul_rn(neg_a, mm), __fadd_rn(__fsqrt_rn(vv), eps)); // optimizers.py:59
    m[p] = mm;
    v[p] = vv;
    theta[p] = __fadd_rn(t, step);                                                       // policy.py:74
}

__global__ void sgd_kernel(float* __restrict__ theta, float* __restrict__ v, const float* __restrict__ gsum,
                           float n_ranked, float l2coeff, float neg_lr, float mu, float ommu, int P) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const float t = theta[p];
    const float g = es_total_grad(t, gsum[p], n_ranked, l2coeff);
    const float vv = __fadd_rn(__fmul_rn(mu, v[p]), __fmul_rn(ommu, g));   // optimizers.py:43
    v[p] = vv;
    theta[p] = __fadd_rn(t, __fmul_rn(neg_lr, vv));                        // optimizers.py:44
}

__global__ void simple_kernel(float* __restrict__ theta, const float* __restrict__ gsum, float n_ranked, float l2coeff,
                              float lr, int P) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const float t = theta[p];
    theta[p] = __fadd_rn(t, __fmul_rn(lr, es_total_grad(t, gsum[p], n_ranked, l2coeff)));   // optimizers.py:33
}

int es_impl_adam(es_ctx* ctx, float* theta, float* m, float* v, const float* gsum, float n_ranked, float l2coeff,
                 float neg_a, float b1, float omb1, float b2, float omb2, float eps, int P, cudaStream_t stream) {
    adam_kernel<<<es_div_up(P, 256), 256, 0, stream>>>(theta, m, v, gsum, n_ranked, l2coeff, neg_a, b1, omb1, b2, omb2,
                                                       eps, P);
    ES_LAUNCHED(ctx);
    return ES_OK;
}

int es_impl_sgd(es_ctx* ctx, float* theta, float* v, const float* gsum, float n_ranked, float l2coeff, float neg_lr,
                float mu, float ommu, int P, cudaStream_t stream) {
    sgd_kernel<<<es_div_up(P, 256), 256, 0, stream>>>(theta, v, gsum, n_ranked, l2coeff, neg_lr, mu, ommu, P);
    ES_LAUNCHED(ctx);
    return ES_OK;
}

int es_impl_simple(es_ctx* ctx, float* theta, const float* gsum, float n_ranked, float l2coeff, float lr, int P,
                   cudaStream_t stream) {
    simple_kernel<<<es_div_up(P, 256), 256, 0, stream>>>(theta, gsum, n_ranked, l2coeff, lr, P);
    ES_LAUNCHED(ctx);
    return ES_OK;
}
