// rollout_closedt.cu -- the closed-loop cluster rollout (rollout_closedw.cuh, design and barrier argument in rollout_closedw.cu)
// on an env whose episodes end early (ClosedLoopEnv(fall_height=h), es_rollout_closedloop_terminal): the reference's run_model
// leaves its step loop when env.step returns done (src/gym/gym_runner.py:50-67), and the pybullet Hopper and Ant envs the
// shipped configs name return it when the robot falls.  Here step t returns done when t = T - 1 or !(|z_t| <= h), z_t the third
// position component after step t's update (a NaN falls).  Every shape es_closedw_plan covers runs here, tanh, binned heads and
// the other activations, with or without action noise and episodes, a cluster of one CTA included: one cluster steps one
// evaluation, so stopping at a data-dependent step costs nothing; rollout_closed.cu and the tensor-core kernels stay as they are.
//
// The template flag TERM of cw_rollout changes, and the instantiations without it (rollout_closedw.cu, rollout_closedw_act.cu)
// compile to the same code as before:
//   * uniform exit: the last warp's lane 0 of EVERY CTA forms the position (rank 0's is the reward lane, which already does;
//     every CTA holds the same action after B_{L-1}, or forms the same binned action from the same outputs), with rank 0's
//     operations in rank 0's order, and writes its CTA's fell flag before the step's closing __syncthreads; every thread reads
//     it after that barrier and leaves the step loop at the same t_d in every CTA, without another cluster barrier;
//   * barrier argument: a step that ends the episode has run all its barriers B_0 .. B_{L-1} and its __syncthreads, as any
//     step.  The next cluster barrier is REUSE (or B_0 of the next episode's first step) instead of B_0(t_d + 1): every read
//     of a_{L-1} (env step, reward, position) precedes the reader's arrival there, and the next write of any a_l comes from
//     a later step's layer, after its writer waited at that barrier -- the write-after-read order of rollout_closedw.cu with
//     B_0(t + 1) replaced by the next barrier the cluster meets.  The fell flag is local: written after the reader's last read
//     of it (the previous step's __syncthreads, then the step's cluster barriers) and read after the step's __syncthreads;
//   * the accumulators stop at t_d: the fitness (float64, step order) and position, the ObStat column sums over the t_d + 1
//     post-step rows, and the ObStat count, which adds t_d + 1 per saved evaluation instead of T;
//   * steps [2][n_pairs]: the last episode's t_d (T - 1 if nothing fell), what run_model returns;
//   * dynamic scheduling: a cluster takes its next evaluation from a device counter (rank 0's thread 0 adds to it after the
//     step loop and stores the result into every CTA's shared memory, which the REUSE barrier publishes; every CTA read the
//     previous value before the evaluation's first cluster barrier, which that thread has passed), so a cluster whose
//     evaluations fall early takes more of them.  An evaluation's arithmetic does not depend on the cluster that runs it;
//   * episodes (obj.py:54-63): each episode ends on its own; rank 0's reward lane keeps the per-step float64 sums of the
//     earlier episodes in the cluster's [T] row as far as the longest of them reached (`reach`; a step beyond it adds to 0),
//     and after the last episode folds row[t] / E into the fitness for t_d < t < reach, so the fitness is
//     sum_t (sum_e r_{e,t}) / E in step order to the longest episode's end.  Behaviour, ObStat and steps are the last
//     episode's.  Without action noise the call runs one episode (the E are identical);
//   * action noise: the reference draws randn(act) for executed steps only, so episode e reads its gaussians from where
//     episode e - 1 stopped, at offset sum_{e' < e} (t_{d,e'} + 1) act of the evaluation's E T act values; noise_used
//     reports the total.
#include "rollout_closedw.cuh"

namespace {

template <int NL, bool BINNED, bool NOISY, bool ACT>
__global__ void __launch_bounds__(CW_THREADS, 1) rollout_closedt_kernel(const CwParams p, const CwTerm tm) {
    cw_rollout<NL, BINNED, NOISY, ACT, true>(p, tm);
}

typedef void (*CtKernel)(const CwParams, const CwTerm);

template <bool BINNED, bool NOISY, bool ACT>
CtKernel ct_depth(int n_layers) {
    return n_layers == 3 ? rollout_closedt_kernel<3, BINNED, NOISY, ACT>
         : n_layers == 4 ? rollout_closedt_kernel<4, BINNED, NOISY, ACT> : rollout_closedt_kernel<5, BINNED, NOISY, ACT>;
}

// binned heads draw no noise (FFBinned.forward ignores rs)
CtKernel ct_kernel(int n_layers, bool binned, bool noisy, bool act) {
    if (binned) return ct_depth<true, false, false>(n_layers);
    if (act) return noisy ? ct_depth<false, true, true>(n_layers) : ct_depth<false, false, true>(n_layers);
    return noisy ? ct_depth<false, true, false>(n_layers) : ct_depth<false, false, false>(n_layers);
}

}  // namespace

int es_impl_rollout_closedt(es_ctx* ctx, const EsRollout& r, const EsClosedEnv& env, float fall_height, int* steps,
                            long long* noise_used, unsigned* next, cudaStream_t stream) {
    const char* fn = "es_rollout_closedloop_terminal";
    int C = 0;
    size_t smem = 0;
    const bool binned = r.bins != 0, noisy = r.act_noise != nullptr, act = r.activation != ES_ACT_TANH;
    int rc = binned ? es_closedw_binned_plan(r.dims, r.n_layers, env.band, r.bins, &C, &smem)
                    : es_closedw_plan(r.dims, r.n_layers, env.band, &C, &smem);
    if (rc) return rc;
    const CtKernel kernel = ct_kernel(r.n_layers, binned, noisy, act);
    ES_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaLaunchAttribute attr;
    int max_clusters = 0;
    {
        const cudaLaunchConfig_t q = cw_config(C, smem, 1, nullptr, &attr);
        ES_CHECK_CUDA(cudaOccupancyMaxActiveClusters(&max_clusters, kernel, &q));
    }
    if (max_clusters < 1) {
        es_set_error("%s: no cluster of %d CTAs with %zu bytes of shared memory each fits on this device", fn, C, smem);
        return ES_ERR_UNSUPPORTED;
    }
    const CwParams p = {r, env};
    const CwTerm tm = {fall_height, steps, noise_used, next};
    const long long evals = 2ll * r.n_pairs;
    const int clusters = evals < max_clusters ? (int)evals : max_clusters;
    ES_CHECK_CUDA(cudaMemsetAsync(next, 0, sizeof(unsigned), stream));
    const cudaLaunchConfig_t cfg = cw_config(C, smem, clusters, stream, &attr);
    ES_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kernel, p, tm));
    ES_LAUNCHED(ctx);
    return ES_OK;
}

