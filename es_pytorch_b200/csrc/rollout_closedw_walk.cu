// rollout_closedw_walk.cu -- es_rollout_closedloop_terminal_streams: the closed-loop cluster rollout (rollout_closedw.cu) on an
// env whose episodes end early, WITH action noise, drawing every stream's indices, coins and gaussians inside the rollout.
//
// Why inside: per reference rank the stream order is nt.sample (randint), then for each sign the save_obs coin, then randn(act)
// for each EXECUTED step (src/core/es.py:66-74, src/nn/nn.py:47-48, src/gym/gym_runner.py:50-67).  Where the next pair's index
// lies in the stream depends on where the previous evaluation fell, so nothing after the first fall can be drawn ahead.  Within
// one stream the evaluations are sequential, as on one MPI rank of the reference; across streams they are independent.
//
// Design:
//   * words: before the launch every stream's tempered MT19937 words are generated from its block 0 on by the jump-ahead fill
//     (mj_launch_fill, mt_gauss.cu), up to what the stream consumes when nothing falls (n pairs x (randint + 2 (coins +
//     E T act gaussians)) at es_draw_noisy's mean + 12 sigma).  Turning words into an index, a coin and polar-method gaussians
//     is cheap sequential bookkeeping, done here;
//   * scheduling: the unit of dynamic scheduling is a STREAM.  A cluster takes the next stream from the device counter and runs
//     its 2n evaluations in the reference's order (pair-major, + before -); the E episodes of an evaluation continue the walk
//     where the previous one stopped.  One stream per cluster at a time: with fewer streams than resident clusters part of the
//     GPU is idle;
//   * the walk: one warp of EVERY CTA of the cluster (warp CW_WARPS - 2, idle in the env step since obs <= 384) walks the
//     stream redundantly (CwWalker in rollout_closedw.cuh), as the env step is computed redundantly: each CTA then holds the
//     noise of its own output rows with no exchange.  Every CTA reads the same words with the same operations, so every CTA
//     forms the same values and the same cursor.  Per step: at the top of step t the warp starts copying the next step's first
//     256 words into shared memory (cp.async), the layers run, and in the env-step phase it forms step t + 1's act gaussians
//     (polar attempts tested 32 at a time, ranked by a ballot) into the other half of a [2][64] noise buffer.  After the step's
//     closing __syncthreads it keeps them if step t + 1 runs (the episode did not end) and otherwise drops them and leaves the
//     cursor where step t's draws ended: only executed steps consume words.  The first step of an evaluation or episode is
//     formed before the barrier that starts it, after the pair's randint (before +) and the evaluation's coin words;
//   * barrier argument: the walk adds no cluster barrier and touches only its CTA's shared memory.  Step t + 1's noise half is
//     written in step t's env-step phase (after B_{L-1}(t)) and read at the top of step t + 1 (after step t's __syncthreads);
//     the previous reads of that half, at the top of step t - 1, precede step t - 1's __syncthreads.  The staging words are
//     written and read by the walk warp alone (cp.async.wait_all, then __syncwarp).  The index and coin decision are written
//     before a __syncthreads at the evaluation's start, after REUSE, which every read of the previous evaluation preceded;
//   * the stream's state (key untempered from the 624 words of the cursor's block, position, has_gauss, cached gaussian) is
//     written back by rank 0's walk warp after the stream's last evaluation, in DeviceGeneration.mt_state's layout;
//   * a cursor past the generated words (a > 12 sigma event) sets the ctx's error word (ES_ASYNC_WALK_OVERFLOW): es_check_async
//     raises and the call's results are not used.
// The float32 noise is (float)(g * ac_std), the float64 product rounded once, as the reference's (randn * ac_std) reaches the
// float32 env; g uses CUDA's log (<= 1 ulp of float64), so a value can differ from numpy's where it lies next to a float32
// rounding midpoint.  Everything else -- the step, the fall, the fitness, ObStat and steps -- is rollout_closedw.cu's.
#include "rollout_closedw.cuh"

namespace {

template <int NL, bool ACT>
__global__ void __launch_bounds__(CW_THREADS, 1) rollout_closedw_walk_kernel(const CwWalkParams p) {
    cw_rollout<NL, false, true, ACT, true>(p);
}

typedef void (*CwwKernel)(const CwWalkParams);

template <bool ACT>
CwwKernel cww_depth(int n_layers) {
    return n_layers == 3 ? rollout_closedw_walk_kernel<3, ACT>
         : n_layers == 4 ? rollout_closedw_walk_kernel<4, ACT> : rollout_closedw_walk_kernel<5, ACT>;
}

size_t cww_pad(size_t b) { return (b + 255) & ~(size_t)255; }

}  // namespace

// the cluster rollout's plan with the walk's shared memory: the smallest cluster size that holds both
static int cww_plan(const EsRollout& r, int band, int* cluster_size, size_t* smem_bytes) {
    int C = 0;
    size_t smem = 0;
    const int rc = es_closedw_plan(r.dims, r.n_layers, band, &C, &smem);
    if (rc) return rc;
    for (; C <= 8; C *= 2) {
        const size_t bytes = ((size_t)cw_layout(r.n_layers, r.dims, C, band).total + CW_WALK_FLOATS) * sizeof(float);
        if (bytes <= (size_t)CW_SMEM_MAX) {
            *cluster_size = C;
            *smem_bytes = bytes;
            return ES_OK;
        }
    }
    es_set_error("es_rollout_closedloop_terminal_streams: the weights, env matrices and the stream walk do not fit the shared "
                 "memory of a cluster of 8 CTAs");
    return ES_ERR_UNSUPPORTED;
}

int es_impl_rollout_closedw_walk(es_ctx* ctx, const EsRollout& r, const EsClosedEnv& env_in, const EsTerm& term,
                                 const EsStreamWalk& s, cudaStream_t stream) {
    const char* fn = "es_rollout_closedloop_terminal_streams";
    int C = 0, max_clusters = 0;
    size_t smem = 0;
    int rc = cww_plan(r, env_in.band, &C, &smem);
    if (rc) return rc;
    const long long N = (long long)r.n_episodes * r.T * r.act;
    if (N > 0x7FFFFFFFLL) {
        es_set_error("%s: %d episodes x %d steps x %d actions = %lld gaussians per evaluation, more than 2^31 - 1", fn, r.n_episodes,
                     r.T, r.act, N);
        return ES_ERR_UNSUPPORTED;
    }
    EsStreamWords wp;
    rc = es_impl_stream_words_plan(ctx, fn, s.n_streams, s.n_per_stream, s.coins, (int)N, &wp);
    if (rc) return rc;
    const CwwKernel kernel = r.activation != ES_ACT_TANH ? cww_depth<true>(r.n_layers) : cww_depth<false>(r.n_layers);
    rc = cw_max_clusters(kernel, C, smem, &max_clusters);
    if (rc) return rc;
    if (max_clusters < 1) {
        es_set_error("%s: no cluster of %d CTAs with %zu bytes of shared memory each fits on this device", fn, C, smem);
        return ES_ERR_UNSUPPORTED;
    }
    // scratch: the stream counter | the per-step episode rows of E > 1 episodes ([T] per cluster) | the words | segment order
    const size_t rows_bytes = r.n_episodes > 1 ? cww_pad((size_t)max_clusters * r.T * sizeof(double)) : 0;
    void* scratch = nullptr;
    rc = es_ctx_scratch(ctx, 256 + rows_bytes + wp.words_bytes + wp.order_bytes, &scratch);
    if (rc) return rc;
    char* at = (char*)scratch;
    unsigned* next = (unsigned*)at; at += 256;
    EsClosedEnv env = env_in;
    env.coins = nullptr;                                       // (the walk draws them)
    env.ep_rows = r.n_episodes > 1 ? (double*)at : nullptr; at += rows_bytes;
    uint32_t* words = (uint32_t*)at; at += wp.words_bytes;
    uint16_t* order = (uint16_t*)at;
    rc = es_impl_stream_words_fill(ctx, s.mt_key, s.n_streams, wp, words, order, stream);
    if (rc) return rc;

    const Mt19937Bound bd = mt19937_randint_bound(s.upper_bound);
    CwWalkParams p;
    p.r = r;
    p.env = env;
    p.term = term;
    p.next = next;
    p.w = CwWalk{words, wp.stride_words, wp.limit, bd.rng, bd.mask, s.n_per_stream, s.coins, s.ac_std, s.mt_key, s.mt_pos,
                 s.has_gauss, s.gauss, s.idx_out, s.coin_out, s.noise_trace};
    const int clusters = s.n_streams < max_clusters ? s.n_streams : max_clusters;
    ES_CHECK_CUDA(cudaMemsetAsync(next, 0, sizeof(unsigned), stream));
    cudaLaunchAttribute attr;
    const cudaLaunchConfig_t cfg = cw_config(C, smem, clusters, stream, &attr);
    ES_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kernel, p));
    ES_LAUNCHED(ctx);
    return ES_OK;
}
