// rank.cu -- centered-rank transform of the 2K antithetic fitnesses -> K weights
// (reference: rank / Ranker / CenteredRanker / MultiObjectiveRanker,
//  src/utils/rankers.py:9-17,37-58,106-120).
//
// rank(x_i) = #{j : x_j < x_i} + #{j < i : x_j == x_i}  over x = concat(pos, neg)
// which equals ``ranks[argsort(x, kind='stable')] = arange`` -- integer-exact.
// The float64 fitnesses are mapped to order-preserving uint64 keys (-0.0 == +0.0, NaNs last, like numpy's sort) and
// ranked exactly in O(n) expected work with a monotone value bucketing (any non-decreasing bucket function is
// correct; balance only affects speed):
//   1. rank_keys_kernel     keys[n_obj][2K] + min/max of the finite values
//   2. rank_hist_kernel     bucket histogram (RK_BUCKETS linear buckets over [min, max]; -inf first, +inf/NaN last)
//   3. rank_scan_kernel     exclusive scan of the histogram (one block per objective)
//   4. rank_scatter_kernel  (key, index) pairs grouped by bucket
//   5. rank_finalize_kernel rank = bucket start + #{(key_j, j) < (key_i, i) inside the bucket}, only for the
//                           elements of this GPU's shard [k_begin, k_begin+k_count) -- ranks are global;
//                           y = shape(rank) (centered: float32(rank)/(2K-1) - 0.5; also the double-positive, semi-centered
//                           and max-normalised shapings of rankers.py:61-83), blend, weight = y+ - y- (or the elite
//                           selection of rankers.py:86-103)
// The float32 ops are the reference's, one IEEE operation each (no contraction).  Steps 1-4 are replicated on every
// GPU (O(2K)), step 5 is O(shard * bucket occupancy): the cost no longer grows with the number of GPUs.
#include "common.cuh"

constexpr int RK_THREADS = 256;
constexpr int RK_BUCKETS = 8192;        // linear value buckets (+2 edge buckets)
constexpr int RK_NB = RK_BUCKETS + 2;

__device__ __forceinline__ unsigned long long rk_key(double x) {
    if (x != x) return 0xFFFFFFFFFFFFFFFFull;     // NaN sorts last
    unsigned long long b = (unsigned long long)__double_as_longlong(x);
    if ((b << 1) == 0ull) b = 0ull;               // -0.0 -> +0.0 (they compare equal)
    return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ double rk_unkey(unsigned long long k) {
    const unsigned long long b = (k & 0x8000000000000000ull) ? (k & 0x7FFFFFFFFFFFFFFFull) : ~k;
    return __longlong_as_double((long long)b);
}

// keys of the smallest / largest finite value (per objective) and of the smallest / largest value of all (np.min / np.max,
// which return NaN if there is one: its key is the largest); the minima are stored inverted so that all-zero bytes mean
// "no value yet" (one memset initialises the histogram and the statistics)
struct RkStats { unsigned long long kmin_inv, kmax, kall_min_inv, kall_max; };
__device__ __forceinline__ unsigned long long rk_kmin(const RkStats& st) { return ~st.kmin_inv; }

__device__ __forceinline__ double rk_value(const double* __restrict__ fpos, const double* __restrict__ fneg, int K,
                                           int n_obj, int c, int e) {
    return (e < K) ? fpos[(size_t)e * n_obj + c] : fneg[(size_t)(e - K) * n_obj + c];
}

__global__ void rank_keys_kernel(const double* __restrict__ fpos, const double* __restrict__ fneg, int K, int n_obj,
                                 unsigned long long* __restrict__ keys, RkStats* __restrict__ stats) {
    const int n = 2 * K;
    const int c = blockIdx.y;
    unsigned long long lo = 0xFFFFFFFFFFFFFFFFull, hi = 0ull, alo = 0xFFFFFFFFFFFFFFFFull, ahi = 0ull;
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
        const double x = rk_value(fpos, fneg, K, n_obj, c, e);
        const unsigned long long k = rk_key(x);
        keys[(size_t)c * n + e] = k;
        if (isfinite(x)) { lo = min(lo, k); hi = max(hi, k); }
        alo = min(alo, k); ahi = max(ahi, k);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
        hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
        alo = min(alo, __shfl_xor_sync(0xffffffffu, alo, o));
        ahi = max(ahi, __shfl_xor_sync(0xffffffffu, ahi, o));
    }
    if ((threadIdx.x & 31) == 0) {
        if (lo != 0xFFFFFFFFFFFFFFFFull) atomicMax(&stats[c].kmin_inv, ~lo);
        if (hi != 0ull) atomicMax(&stats[c].kmax, hi);
        if (alo != 0xFFFFFFFFFFFFFFFFull) atomicMax(&stats[c].kall_min_inv, ~alo);
        if (ahi != 0ull) atomicMax(&stats[c].kall_max, ahi);
    }
}

// monotone (non-decreasing in x) bucket index in [0, RK_NB)
__device__ __forceinline__ int rk_bucket(unsigned long long key, double mn, double scale) {
    if (key == 0xFFFFFFFFFFFFFFFFull) return RK_NB - 1;              // NaN
    const double x = rk_unkey(key);
    if (x == -INFINITY) return 0;
    if (x == INFINITY) return RK_NB - 1;
    int b = (int)((x - mn) * scale);
    b = b < 0 ? 0 : (b > RK_BUCKETS - 1 ? RK_BUCKETS - 1 : b);
    return 1 + b;
}
__device__ __forceinline__ void rk_range(const RkStats& st, double& mn, double& scale) {
    if (rk_kmin(st) > st.kmax) { mn = 0.0; scale = 0.0; return; }      // no finite value
    mn = rk_unkey(rk_kmin(st));
    const double mx = rk_unkey(st.kmax), span = mx - mn;
    scale = (span > 0.0 && isfinite(span)) ? (double)RK_BUCKETS / span : 0.0;
    if (!isfinite(scale)) scale = 0.0;
}

__global__ void rank_hist_kernel(const unsigned long long* __restrict__ keys, int n, const RkStats* __restrict__ stats,
                                 unsigned* __restrict__ hist) {
    const int c = blockIdx.y;
    double mn, scale;
    rk_range(stats[c], mn, scale);
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x)
        atomicAdd(&hist[(size_t)c * RK_NB + rk_bucket(keys[(size_t)c * n + e], mn, scale)], 1u);
}

// one block per objective: start[b] = sum_{b' < b} hist[b'];  cursor[b] = 0
__global__ void __launch_bounds__(1024) rank_scan_kernel(const unsigned* __restrict__ hist, unsigned* __restrict__ start,
                                                         unsigned* __restrict__ cursor) {
    __shared__ unsigned s_warp[32];
    const int c = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    constexpr int PER = (RK_NB + 1023) / 1024;
    unsigned loc[PER], sum = 0;
#pragma unroll
    for (int i = 0; i < PER; ++i) {
        const int b = t * PER + i;
        loc[i] = (b < RK_NB) ? hist[(size_t)c * RK_NB + b] : 0u;
        sum += loc[i];
    }
    // inclusive scan of the per-thread sums: shuffles inside a warp, then the 32 warp totals
    unsigned inc = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned v = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += v;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        unsigned w = s_warp[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned v = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += v;
        }
        s_warp[lane] = w;                                                // inclusive totals of warps 0..lane
    }
    __syncthreads();
    unsigned run = inc - sum + (warp > 0 ? s_warp[warp - 1] : 0u);      // exclusive prefix of this thread's buckets
#pragma unroll
    for (int i = 0; i < PER; ++i) {
        const int b = t * PER + i;
        if (b < RK_NB) { start[(size_t)c * RK_NB + b] = run; cursor[(size_t)c * RK_NB + b] = 0u; }
        run += loc[i];
    }
}

__global__ void rank_scatter_kernel(const unsigned long long* __restrict__ keys, int n, const RkStats* __restrict__ stats,
                                    const unsigned* __restrict__ start, unsigned* __restrict__ cursor,
                                    unsigned long long* __restrict__ skeys, int* __restrict__ sidx) {
    const int c = blockIdx.y;
    double mn, scale;
    rk_range(stats[c], mn, scale);
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
        const unsigned long long k = keys[(size_t)c * n + e];
        const int b = rk_bucket(k, mn, scale);
        const unsigned at = start[(size_t)c * RK_NB + b] + atomicAdd(&cursor[(size_t)c * RK_NB + b], 1u);
        skeys[(size_t)c * n + at] = k;
        sidx[(size_t)c * n + at] = e;
    }
}

// rank of global element gi of objective c: bucket start + #{(key_j, j) < (key_i, i) inside the bucket}.
// *rev = its rank by descending key with equal keys still by ascending index: the q-th of a tie group of g whose ascending
// ranks start at s goes to n - s - g + q (equal keys share a bucket)
struct RkTables {
    const unsigned long long* keys;      // [n_obj][2K]
    const RkStats* stats;
    const unsigned* hist;
    const unsigned* start;
    const unsigned long long* skeys;     // keys grouped by bucket
    const int* sidx;                     // their element indices
};
__device__ __forceinline__ int rk_rank_of(const RkTables& tb, int n, int c, int gi, int* rev) {
    double mn, scale;
    rk_range(tb.stats[c], mn, scale);
    const unsigned long long k = tb.keys[(size_t)c * n + gi];
    const int b = rk_bucket(k, mn, scale);
    const unsigned s0 = tb.start[(size_t)c * RK_NB + b], cnt = tb.hist[(size_t)c * RK_NB + b];
    int lt = 0, q = 0, g = 0;
    for (unsigned j = 0; j < cnt; ++j) {
        const unsigned long long kj = tb.skeys[(size_t)c * n + s0 + j];
        const int ij = tb.sidx[(size_t)c * n + s0 + j];
        lt += kj < k;
        q += kj == k && ij < gi;
        g += kj == k;
    }
    *rev = n - (int)s0 - lt - g + q;
    return (int)s0 + lt + q;
}

// ---- rank -> fitness-shaping value (the _rank of each Ranker subclass, src/utils/rankers.py:53-83) -----------------
struct RkXform {
    int kind;            // ES_RANK_*
    int n;               // 2K
    float denom;         // float32(2K - 1)                        rankers.py:56
    float semi_c1;       // float32(0.29 * s)                      rankers.py:82 (python float -> float32 operand)
    float semi_inv_s;    // float32(1 / s)
    float semi_s;        // float32(s)
    double w0, w1;       // MultiObjectiveRanker blend             rankers.py:120
    int elite_n;         // > 0: EliteRanker keeps the elite_n largest values (rankers.py:93-97)
};

// float32 kinds: every reference operation is one IEEE float32 operation; the result is returned widened (exact)
__device__ __forceinline__ double rk_shape(const RkXform& xf, int r, double x, double shift, double ymax) {
    switch (xf.kind) {
    case ES_RANK_CENTERED:
        return (double)__fsub_rn(__fdiv_rn((float)r, xf.denom), 0.5f);                       // rankers.py:55-57
    case ES_RANK_DOUBLE_POSITIVE: {
        float y = __fsub_rn(__fdiv_rn((float)r, xf.denom), 0.5f);
        if (y > 0.0f) y = __fmul_rn(y, 2.0f);                                                // rankers.py:64
        return (double)y;
    }
    case ES_RANK_SEMI_CENTERED: {
        const float t = __fadd_rn((float)r, xf.semi_c1);                                     // y + 0.29*s
        const float u = __fmul_rn(xf.semi_inv_s, __fmul_rn(t, t));                           // (1/s) * square(.)
        return (double)__fsub_rn(__fdiv_rn(u, xf.semi_s), 0.5f);                             // / s - 0.5
    }
    default: {                                                                                // ES_RANK_MAX_NORMALIZED
        const double y = __ddiv_rn(__dadd_rn(x, shift), ymax);                                // rankers.py:71-72
        return __dsub_rn(__dmul_rn(2.0, y), 1.0);                                             // rankers.py:73
    }
    }
}

__device__ __forceinline__ double rk_blend(const RkXform& xf, double y0, double y1) {
    if (xf.kind == ES_RANK_MAX_NORMALIZED)                                                    // float64 values
        return __dadd_rn(__dmul_rn(y0, xf.w0), __dmul_rn(y1, xf.w1));
    return (double)__fadd_rn(__fmul_rn((float)y0, (float)xf.w0), __fmul_rn((float)y1, (float)xf.w1));
}

__global__ void rank_finalize_kernel(const RkTables tb, const double* __restrict__ fpos,
                                     const double* __restrict__ fneg, const RkStats* __restrict__ stats, int K,
                                     int n_obj, RkXform xf, int k_begin, int k_count,
                                     const int64_t* __restrict__ noise_idx, float* __restrict__ weights_out,
                                     double* __restrict__ weights64_out, int32_t* __restrict__ ranks_out,
                                     double* __restrict__ elite_vals, int32_t* __restrict__ elite_fit,
                                     int64_t* __restrict__ elite_idx) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= k_count) return;
    const int n_local = 2 * k_count;
    double yp = 0.0, yn = 0.0;
    int rp0 = 0, rn0 = 0, vp0 = 0, vn0 = 0;
    bool reversed = false, all_nan = false;
    for (int c = 0; c < n_obj; ++c) {
        int vp, vn;
        const int rp = rk_rank_of(tb, 2 * K, c, k_begin + k, &vp), rn = rk_rank_of(tb, 2 * K, c, K + k_begin + k, &vn);
        if (c == 0) { rp0 = rp; rn0 = rn; vp0 = vp; vn0 = vn; }
        if (ranks_out) { ranks_out[(size_t)c * n_local + k] = rp; ranks_out[(size_t)c * n_local + k_count + k] = rn; }
        double shift = 0.0, ymax = 1.0, xp = 0.0, xn = 0.0;
        if (xf.kind == ES_RANK_MAX_NORMALIZED) {
            // np.min / np.max: NaN if there is one (its key is the largest), else the infinities count
            const double mx = rk_unkey(stats[c].kall_max);
            const double mn = (mx != mx) ? mx : rk_unkey(~stats[c].kall_min_inv);
            shift = (mn > 0.0) ? -mn : mn;                      // x + (-mn if mn > 0 else mn), rankers.py:71
            ymax = __dadd_rn(mx, shift);                        // np.max(y): the add is monotone (and propagates NaN)
            if (c == 0) {
                reversed = ymax < 0.0;                          // dividing by a negative maximum reverses the order
                // every y <= ymax is -inf or NaN: every shaped value is NaN, and a stable sort keeps them in index order
                all_nan = !(ymax > -INFINITY);
            }
            xp = fpos[(size_t)(k_begin + k) * n_obj + c];
            xn = fneg[(size_t)(k_begin + k) * n_obj + c];
        }
        const double sp = rk_shape(xf, rp, xp, shift, ymax), sn = rk_shape(xf, rn, xn, shift, ymax);
        if (n_obj == 1) { yp = sp; yn = sn; }
        else if (c == 0) { yp = sp; yn = sn; }
        else { yp = rk_blend(xf, yp, sp); yn = rk_blend(xf, yn, sn); }
    }
    double w;
    if (xf.elite_n > 0) {
        // EliteRanker (rankers.py:86-103): the elite_n largest shaped values are kept with their own sign-less weight and
        // the noise index of their pair; nothing is subtracted.  Slot = distance from the elite threshold (rank order).
        const int thr = xf.n - xf.elite_n;
        if (all_nan) { rp0 = k_begin + k; rn0 = K + k_begin + k; }
        else if (reversed) { rp0 = vp0; rn0 = vn0; }           // equal shaped values stay in index order (stable sort)
        const bool ep = rp0 >= thr, en = rn0 >= thr;
        if (ep) {
            if (elite_vals) elite_vals[rp0 - thr] = yp;
            if (elite_fit) elite_fit[rp0 - thr] = k_begin + k;
            if (elite_idx) elite_idx[rp0 - thr] = noise_idx[k_begin + k];
        }
        if (en) {
            if (elite_vals) elite_vals[rn0 - thr] = yn;
            if (elite_fit) elite_fit[rn0 - thr] = K + k_begin + k;
            if (elite_idx) elite_idx[rn0 - thr] = noise_idx[k_begin + k];
        }
        const double a = ep ? yp : 0.0, b = en ? yn : 0.0;
        w = (xf.kind == ES_RANK_MAX_NORMALIZED) ? __dadd_rn(a, b) : (double)__fadd_rn((float)a, (float)b);
    } else {
        w = (xf.kind == ES_RANK_MAX_NORMALIZED) ? __dsub_rn(yp, yn)                 // Ranker._post_rank, rankers.py:44
                                                : (double)__fsub_rn((float)yp, (float)yn);
    }
    weights_out[k] = (float)w;
    if (weights64_out) weights64_out[k] = w;
}

int es_impl_rank_transform(es_ctx* ctx, const double* fpos, const double* fneg, int K, int n_obj, int kind, double w0,
                           double w1, int elite_n, int k_begin, int k_count, const int64_t* noise_idx,
                           float* weights_out, double* weights64_out, int32_t* ranks_out, double* elite_vals,
                           int32_t* elite_fit, int64_t* elite_idx, cudaStream_t stream) {
    const size_t n = 2 * (size_t)K;
    auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
    const size_t key_b = al(n * n_obj * 8), skey_b = key_b, sidx_b = al(n * n_obj * 4);
    const size_t tab_b = al((size_t)RK_NB * n_obj * 4), stat_b = al(sizeof(RkStats) * n_obj);
    void* scratch = nullptr;
    int rc = es_ctx_scratch(ctx, key_b + skey_b + sidx_b + 3 * tab_b + stat_b, &scratch);
    if (rc) return rc;
    char* base = (char*)scratch;
    unsigned long long* keys = (unsigned long long*)base;   base += key_b;
    unsigned long long* skeys = (unsigned long long*)base;  base += skey_b;
    int* sidx = (int*)base;                                 base += sidx_b;
    unsigned* hist = (unsigned*)base;                       base += tab_b;
    RkStats* stats = (RkStats*)base;                        base += stat_b;      // right behind the histogram: one memset
    unsigned* start = (unsigned*)base;                      base += tab_b;
    unsigned* cursor = (unsigned*)base;

    // histogram = 0, statistics = "no finite value yet"
    ES_CHECK_CUDA(cudaMemsetAsync(hist, 0, tab_b + stat_b, stream));
    int blocks = es_div_up((int64_t)n, RK_THREADS);
    if (blocks > ctx->sm_count * 4) blocks = ctx->sm_count * 4;
    dim3 grid(blocks, n_obj);
    rank_keys_kernel<<<grid, RK_THREADS, 0, stream>>>(fpos, fneg, K, n_obj, keys, stats);
    ES_LAUNCHED(ctx);
    rank_hist_kernel<<<grid, RK_THREADS, 0, stream>>>(keys, (int)n, stats, hist);
    ES_LAUNCHED(ctx);
    rank_scan_kernel<<<n_obj, 1024, 0, stream>>>(hist, start, cursor);
    ES_LAUNCHED(ctx);
    rank_scatter_kernel<<<grid, RK_THREADS, 0, stream>>>(keys, (int)n, stats, start, cursor, skeys, sidx);
    ES_LAUNCHED(ctx);
    RkXform xf;
    xf.kind = kind;
    xf.n = (int)n;
    xf.denom = (float)(n - 1);
    xf.semi_c1 = (float)(0.29 * (double)n);
    xf.semi_inv_s = (float)(1.0 / (double)n);
    xf.semi_s = (float)n;
    xf.w0 = w0;
    xf.w1 = w1;
    xf.elite_n = elite_n;
    const RkTables tb = {keys, stats, hist, start, skeys, sidx};
    rank_finalize_kernel<<<es_div_up(k_count, 128), 128, 0, stream>>>(
        tb, fpos, fneg, stats, K, n_obj, xf, k_begin, k_count, noise_idx, weights_out, weights64_out, ranks_out,
        elite_vals, elite_fit, elite_idx);
    ES_LAUNCHED(ctx);
    return ES_OK;
}
