// rollout_closedw.cu -- the CLOSED-LOOP synthetic env (obs_{t+1} = tanh(A obs_t + B a_t)) for policies too wide for
// rollout_closed.cu's one pair per CTA: MLPs with 2 to 4 hidden layers of 1 .. 256 units, obs <= 384, act <= 64 -- every
// shipped config's policy (15-256-256-3, 17/26/28-256-256-256-6/8, 28-128-256-256-128-8) and a Humanoid-shaped 376-256-256-17 --
// with tanh, a binned head or another activation, with or without action noise and episodes, on an env whose episodes run T
// steps or end when the position falls.  One kernel family, cw_rollout<depth, binned, noisy, activation> in
// rollout_closedw.cuh: 15 instantiations, each serving every call of its variant.
//
// Semantics are rollout_closed.cu's: theta +- sigma eps through es_pheno_pm (slices checked by es_checked_slice and the ctx's
// error word), clip((o - mean) / std) in float64 (here an exact float64 division, as the reference), Linear + tanh after every
// layer including the output (the same fast tanh as rollout_closed.cu, es_tanh_exp: absolute error ~1e-7), the reward as a
// float32 dot in index order summed in float64 in step order, the position integrator, behaviour outputs with fit_stride, and
// the ObStat increments (float32 column sums in step order, added in float64) of evaluations whose save_obs coin fell.  The env
// step is the oracle's arithmetic exactly: one float32 accumulator, A's diagonals then B's columns in index order, every product
// and sum rounded separately (rollout_closed.cu interleaves two FMA accumulators instead).
//
// Why a cluster: one evaluation's float32 weights are 276 KiB (15-256-256-3) to 651 KiB (376-256-256-17), more than one SM's
// 227 KiB of shared memory, and re-reading them from L2 at every step would move ~1.3 PB per simple_conf generation.  So:
//   * one thread-block cluster of C CTAs (C in {1, 2, 4, 8}, the smallest that holds the weights; a function of the shape
//     only, es_closedw_plan) runs one evaluation (one sign of a pair) at a time, and clusters loop over the 2 n_pairs
//     evaluations (persistent grid: cudaOccupancyMaxActiveClusters clusters -- a cluster lives inside one GPC and H100's GPCs
//     do not all have the same SM count, so sm_count / C would overestimate);
//   * row split: CTA q of the cluster owns the contiguous output rows [q R_l, (q + 1) R_l) of every layer l
//     (R_l = ceil(d_{l+1} / C)) and keeps their weights and biases in its shared memory, rows [R_l][pad32(d_l)] zero padded;
//   * one warp computes 4 rows at a time: lane s accumulates the elements k = 32 j + s of each row in j order (fmaf), and a
//     transposing butterfly (7 shuffles) adds the 32 lane sums in the fixed xor-16, 8, 4, 2, 1 tree.  A row's value therefore
//     depends on neither C, nor the warp that computes it, nor the grid, nor the order of the pairs;
//   * activation exchange: the lane that holds a row's tanh stores it into the layer's activation buffer of EVERY CTA of the
//     cluster (mapa + st.shared::cluster, its own included; for the output layer with action noise, the tanh plus the row's
//     noise, so every CTA receives the noisy action), then the cluster meets at barrier.cluster.arrive.release /
//     wait.acquire.  Every layer has its own buffer (the input x, a_0 .. a_{L-1}, the last being the action), so that one
//     barrier per layer (B_0 .. B_{L-1} of a step) orders all remote writes:
//       - write-after-read: a_l is read by layer l + 1 of step t before the reader arrives at B_{l+1}(t) (for the action
//         a_{L-1}: by the env step and the reward of step t, before the reader arrives at B_0(t + 1)); the next write of a_l
//         comes from layer l of step t + 1, after the writer waited at B_{L-1}(t) >= B_{l+1}(t) (for the action: after it
//         waited at B_0(t + 1), which precedes layer L - 1 because L >= 3).  With a single buffer the write of layer l + 1
//         would race with the peers' reads of layer l, and a second barrier per layer would be needed;
//       - read-after-write: the release / acquire pair of B_l orders every store of layer l before every read of layer l + 1;
//   * env step: every CTA computes the whole step redundantly (thread i < obs owns observation i; A's diagonals and B in its
//     own shared memory, the raw observation double buffered with a wrap-around halo), so the next input x needs no exchange,
//     only a __syncthreads.  Rank 0's last warp (idle in the env step: obs <= 384 < 480) forms the reward and the position,
//     and rank 0 keeps the ObStat column sums and writes the results;
//   * other cluster barriers: START after the buffers are zeroed and before the first remote store (a peer's shared memory
//     may only be written once that CTA runs), and REUSE at the end of every evaluation, before the cluster reloads its
//     weights and restarts its buffers for the next one; the last REUSE is the EXIT barrier, so no CTA exits while a peer
//     might still store into its shared memory;
//   * arithmetic on float32 CUDA cores: each weight matrix meets one activation column per step, so a wgmma (N >= 8) would
//     run at most 1/8 full.
// Binned-action policies (FFBinned, src/nn/nn.py:99-117; BINNED): the last layer has adim * bins outputs
// and every CTA holds all of them after B_{L-1}, so each CTA forms the adim actions locally (threads j < adim: the first
// maximal bin, as torch.argmax, mapped to low[j] + range[j] * idx / (bins - 1) in the reference's float32 operation order) into
// a local action buffer, then a __syncthreads, before the env step.  The env's B, the reward and the position use adim.  That
// buffer is written after B_{L-1}(t) and read within step t only, so the barrier argument above is unchanged.  Binned shapes
// always run here (C = 1 included): rollout_closed.cu has no head.
// Action noise and episodes (NOISY, es_rollout_closedloop_mlp_episodes; no binned head): the lane that
// owns an output row adds its noise value (loaded at the top of the step: a CTA owns <= 64 output rows, so one pass of its 16
// warps covers them) before the remote stores above, which is the only change inside a step, so the barrier argument holds as
// it is.  The E episodes of an evaluation run in sequence in its cluster, the weights left in place: each restarts x, the raw
// observation and the position locally (a step boundary as far as the barriers are concerned); rank 0's reward lane keeps the
// float64 per-step sums of episodes 0 .. E - 2 in a [T] row per cluster in global memory, and the last episode adds
// (row[t] + r) / E to the fitness and keeps the behaviour and the ObStat sums.  Spreading the episodes over clusters would
// only help with fewer evaluations than resident clusters, and would make the result depend on the grid.
// Other activations (ACT; es_rollout_closedloop_mlp_activation): the lane that owns a row applies ReLU, leaky ReLU, ELU or
// sigmoid (es_act, in float32) where the tanh variants apply es_tanh_exp; the env's tanh(A obs + B a) is the env's and stays.
// The kind is uniform over the launch and the branch sits in the per-row epilogue, outside the dot products, so one kernel per
// depth and noise variant serves every kind.
// Episodes that end early (EsTerm, es_rollout_closedloop_terminal: ClosedLoopEnv(fall_height=h)): the reference's run_model
// leaves its step loop when env.step returns done (src/gym/gym_runner.py:50-67), and the pybullet Hopper and Ant envs the
// shipped configs name return it when the robot falls.  Here step t returns done when t = T - 1 or !(|z_t| <= h), z_t the third
// position component after step t's update (a NaN falls).  One cluster steps one evaluation, so stopping at a data-dependent
// step costs nothing.  The flag is uniform over the launch; it gates only the position the other ranks form, the fall and the
// break, and the steps / noise_used stores.  Everything else below takes its general form in every call, and with nothing
// falling that form is the fixed-length one: t_d = T - 1, the noise offset is e T act, `reach` is T after the first episode,
// and the fold after the last episode is empty.  A call without the flag never ends an episode early, a NaN position included:
//   * uniform exit: the last warp's lane 0 of EVERY CTA forms the position (rank 0's is the reward lane, which already does;
//     every CTA holds the same action after B_{L-1}, or forms the same binned action from the same outputs), with rank 0's
//     operations in rank 0's order, and writes its CTA's fell flag before the step's closing __syncthreads; every thread reads
//     it after that barrier and leaves the step loop at the same t_d in every CTA, without another cluster barrier;
//   * barrier argument: a step that ends the episode has run all its barriers B_0 .. B_{L-1} and its __syncthreads, as any
//     step.  The next cluster barrier is REUSE (or B_0 of the next episode's first step) instead of B_0(t_d + 1): every read
//     of a_{L-1} (env step, reward, position) precedes the reader's arrival there, and the next write of any a_l comes from
//     a later step's layer, after its writer waited at that barrier -- the write-after-read order above with B_0(t + 1)
//     replaced by the next barrier the cluster meets.  The fell flag is local: written after the reader's last read of it
//     (the previous step's __syncthreads, then the step's cluster barriers) and read after the step's __syncthreads;
//   * the accumulators stop at t_d: the fitness (float64, step order) and position, the ObStat column sums over the t_d + 1
//     post-step rows, and the ObStat count, which adds t_d + 1 per saved evaluation;
//   * steps [2][n_pairs]: the last episode's t_d (T - 1 if nothing fell), what run_model returns;
//   * episodes (obj.py:54-63): each episode ends on its own; rank 0's reward lane keeps the per-step float64 sums of the
//     earlier episodes in the cluster's [T] row as far as the longest of them reached (`reach`; a step beyond it adds to 0),
//     and after the last episode folds row[t] / E into the fitness for t_d < t < reach, so the fitness is
//     sum_t (sum_e r_{e,t}) / E in step order to the longest episode's end.  Behaviour, ObStat and steps are the last
//     episode's.  Without action noise the call runs one episode (the E are identical);
//   * action noise: the reference draws randn(act) for executed steps only, so episode e reads its gaussians from where
//     episode e - 1 stopped, at offset sum_{e' < e} (t_{d,e'} + 1) act of the evaluation's E T act values; noise_used
//     reports the total.
// Dynamic scheduling (every call): a cluster takes its next evaluation from a device counter (rank 0's thread 0 adds to it
// after the step loop and stores the result into every CTA's shared memory, which the REUSE barrier publishes; every CTA read
// the previous value before the evaluation's first cluster barrier, which that thread has passed), so a cluster whose
// evaluations fall early takes more of them.  An evaluation's arithmetic does not depend on the cluster that runs it.
// Alternatives not built (so not measured): weights partly in registers (rollout_closed.cu's layer 1), and a pair (both signs)
// per cluster, which doubles the footprint to save only the load-time reads of eps.
#include "rollout_closedw.cuh"

namespace {

template <int NL, bool BINNED, bool NOISY, bool ACT>
__global__ void __launch_bounds__(CW_THREADS, 1) rollout_closedw_kernel(const CwParams p) { cw_rollout<NL, BINNED, NOISY, ACT>(p); }

template <bool BINNED, bool NOISY, bool ACT>
CwKernel cw_depth(int n_layers) {
    return n_layers == 3 ? rollout_closedw_kernel<3, BINNED, NOISY, ACT>
         : n_layers == 4 ? rollout_closedw_kernel<4, BINNED, NOISY, ACT> : rollout_closedw_kernel<5, BINNED, NOISY, ACT>;
}

// binned heads are tanh stacks that draw no noise (FFBinned.forward ignores rs)
CwKernel cw_kernel(int n_layers, bool binned, bool noisy, bool act) {
    if (binned) return cw_depth<true, false, false>(n_layers);
    if (act) return noisy ? cw_depth<false, true, true>(n_layers) : cw_depth<false, false, true>(n_layers);
    return noisy ? cw_depth<false, true, false>(n_layers) : cw_depth<false, false, false>(n_layers);
}

}  // namespace

// the smallest cluster size that holds the shape (act: the env's actions; binned: a binned head), its shared memory per CTA, or
// an error message naming `fn`; no device work
static int cw_plan(const char* fn, const int* dims, int n_layers, int band, int act, bool binned, int* cluster_size,
                   size_t* smem_bytes) {
    const int obs = dims[0];
    if (n_layers < 3 || n_layers > CW_MAX_LAYERS) {
        es_set_error("%s: 2 to 4 hidden layers (n_layers 3 to %d) supported, got n_layers %d", fn, CW_MAX_LAYERS, n_layers);
        return ES_ERR_UNSUPPORTED;
    }
    for (int l = 1; l < n_layers; ++l)
        if (dims[l] > CW_MAX_WIDTH) {
            es_set_error("%s: hidden widths up to %d supported, hidden layer %d has %d", fn, CW_MAX_WIDTH, l, dims[l]);
            return ES_ERR_UNSUPPORTED;
        }
    if (obs > CW_MAX_OBS || act > CW_MAX_ACT) {
        es_set_error("%s: obs <= %d and act <= %d supported, got obs %d, act %d", fn, CW_MAX_OBS, CW_MAX_ACT, obs, act);
        return ES_ERR_UNSUPPORTED;
    }
    if ((band & 1) || band > CW_HALO || band > obs) {
        es_set_error("%s: the band must be even, <= %d and <= obs (got band %d, obs %d)", fn, CW_HALO, band, obs);
        return ES_ERR_UNSUPPORTED;
    }
    size_t bytes = 0;
    for (int C = 1; C <= 8; C *= 2) {
        bytes = (size_t)cw_layout(n_layers, dims, C, band, act, binned).total * sizeof(float);
        if (bytes <= (size_t)CW_SMEM_MAX) {
            *cluster_size = C;
            *smem_bytes = bytes;
            return ES_OK;
        }
    }
    es_set_error("%s: the weights and env matrices need %zu bytes of shared memory per CTA in a cluster of 8 CTAs, %d available",
                 fn, bytes, CW_SMEM_MAX);
    return ES_ERR_UNSUPPORTED;
}

int es_closedw_plan(const int* dims, int n_layers, int band, int* cluster_size, size_t* smem_bytes) {
    return cw_plan("es_rollout_closedloop_mlp", dims, n_layers, band, dims[n_layers], false, cluster_size, smem_bytes);
}
// binned heads: the last layer is adim * bins <= 256 wide (checked as a hidden width), the env sees adim <= 64 actions
int es_closedw_binned_plan(const int* dims, int n_layers, int band, int bins, int* cluster_size, size_t* smem_bytes) {
    const char* fn = "es_rollout_closedloop_mlp_binned";
    const int out = dims[n_layers];
    if (bins < 2 || out % bins || out > CW_MAX_WIDTH) {
        es_set_error("%s: the last layer must have adim * bins <= %d outputs with bins >= 2, got %d outputs, bins %d", fn,
                     CW_MAX_WIDTH, out, bins);
        return ES_ERR_UNSUPPORTED;
    }
    return cw_plan(fn, dims, n_layers, band, out / bins, true, cluster_size, smem_bytes);
}

// the plan entry points' resident clusters (the noise-free variant's: every variant runs one CTA per SM)
int es_closedw_max_clusters(int n_layers, int bins, bool act, int C, size_t smem, int* clusters) {
    return cw_max_clusters(cw_kernel(n_layers, bins != 0, false, act), C, smem, clusters);
}

int es_impl_rollout_closedw(es_ctx* ctx, const EsRollout& r, const EsClosedEnv& env, const EsTerm& term, unsigned* next,
                            cudaStream_t stream) {
    int C = 0, max_clusters = 0;
    size_t smem = 0;
    const bool binned = r.bins != 0;
    int rc = binned ? es_closedw_binned_plan(r.dims, r.n_layers, env.band, r.bins, &C, &smem)
                    : es_closedw_plan(r.dims, r.n_layers, env.band, &C, &smem);
    if (rc) return rc;
    const CwKernel kernel = cw_kernel(r.n_layers, binned, r.act_noise != nullptr, r.activation != ES_ACT_TANH);
    rc = cw_max_clusters(kernel, C, smem, &max_clusters);
    if (rc) return rc;
    if (max_clusters < 1) {
        es_set_error("the closed-loop cluster rollout: no cluster of %d CTAs with %zu bytes of shared memory each fits on this "
                     "device", C, smem);
        return ES_ERR_UNSUPPORTED;
    }
    const CwParams p = {r, env, term, next};
    const long long evals = 2ll * r.n_pairs;
    const int clusters = evals < max_clusters ? (int)evals : max_clusters;
    ES_CHECK_CUDA(cudaMemsetAsync(next, 0, sizeof(unsigned), stream));
    cudaLaunchAttribute attr;
    const cudaLaunchConfig_t cfg = cw_config(C, smem, clusters, stream, &attr);
    ES_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kernel, p));
    ES_LAUNCHED(ctx);
    return ES_OK;
}
