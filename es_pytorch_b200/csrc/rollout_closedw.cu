// rollout_closedw.cu -- the CLOSED-LOOP synthetic env (obs_{t+1} = tanh(A obs_t + B a_t)) for policies too wide for
// rollout_closed.cu's one pair per CTA: tanh MLPs with 2 to 4 hidden layers of 1 .. 256 units, obs <= 384, act <= 64 -- every
// shipped config's policy (15-256-256-3, 17/26/28-256-256-256-6/8, 28-128-256-256-128-8) and a Humanoid-shaped 376-256-256-17.
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
// Binned-action policies (FFBinned, src/nn/nn.py:99-117; rollout_closedw_binned_kernel): the last layer has adim * bins outputs
// and every CTA holds all of them after B_{L-1}, so each CTA forms the adim actions locally (threads j < adim: the first
// maximal bin, as torch.argmax, mapped to low[j] + range[j] * idx / (bins - 1) in the reference's float32 operation order) into
// a local action buffer, then a __syncthreads, before the env step.  The env's B, the reward and the position use adim.  That
// buffer is written after B_{L-1}(t) and read within step t only, so the barrier argument above is unchanged.  Binned shapes
// always run here (C = 1 included): rollout_closed.cu has no head.
// Action noise and episodes (rollout_closedw_noisy_kernel, es_rollout_closedloop_mlp_episodes; tanh heads only): the lane that
// owns an output row adds its noise value (loaded at the top of the step: a CTA owns <= 64 output rows, so one pass of its 16
// warps covers them) before the remote stores above, which is the only change inside a step, so the barrier argument holds as
// it is.  The E episodes of an evaluation run in sequence in its cluster, the weights left in place: each restarts x, the raw
// observation and the position locally (a step boundary as far as the barriers are concerned); rank 0's reward lane keeps the
// float64 per-step sums of episodes 0 .. E - 2 in a [T] row per cluster in global memory, and the last episode adds
// (row[t] + r) / E to the fitness and keeps the behaviour and the ObStat sums.  Spreading the episodes over clusters would
// only help with fewer evaluations than resident clusters, and would make the result depend on the grid.
// Alternatives not built (so not measured): weights partly in registers (rollout_closed.cu's layer 1), and a pair (both signs)
// per cluster, which doubles the footprint to save only the load-time reads of eps.
#include "rollout_closedw.cuh"

namespace {

template <int NL>
__global__ void __launch_bounds__(CW_THREADS, 1) rollout_closedw_kernel(const CwParams p) { cw_rollout<NL, false, false>(p); }
template <int NL>
__global__ void __launch_bounds__(CW_THREADS, 1) rollout_closedw_binned_kernel(const CwParams p) { cw_rollout<NL, true, false>(p); }
template <int NL>
__global__ void __launch_bounds__(CW_THREADS, 1) rollout_closedw_noisy_kernel(const CwParams p) { cw_rollout<NL, false, true>(p); }

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

static CwKernel cw_kernel(int n_layers, bool binned = false, bool noisy = false) {
    if (noisy)
        return n_layers == 3 ? rollout_closedw_noisy_kernel<3> : n_layers == 4 ? rollout_closedw_noisy_kernel<4>
                                                                                : rollout_closedw_noisy_kernel<5>;
    if (binned)
        return n_layers == 3 ? rollout_closedw_binned_kernel<3> : n_layers == 4 ? rollout_closedw_binned_kernel<4>
                                                                                 : rollout_closedw_binned_kernel<5>;
    return n_layers == 3 ? rollout_closedw_kernel<3> : n_layers == 4 ? rollout_closedw_kernel<4> : rollout_closedw_kernel<5>;
}
int es_closedw_max_clusters(int n_layers, int bins, int C, size_t smem, int* clusters) {
    return cw_max_clusters(cw_kernel(n_layers, bins != 0), C, smem, clusters);
}

int es_impl_rollout_closedw(es_ctx* ctx, const EsRollout& r, const EsClosedEnv& env, cudaStream_t stream) {
    int C = 0, max_clusters = 0;
    size_t smem = 0;
    const bool binned = r.bins != 0, noisy = r.act_noise != nullptr;       // (never both: the binned entry passes no noise)
    int rc = binned ? es_closedw_binned_plan(r.dims, r.n_layers, env.band, r.bins, &C, &smem)
                    : es_closedw_plan(r.dims, r.n_layers, env.band, &C, &smem);
    if (rc) return rc;
    const CwKernel kernel = cw_kernel(r.n_layers, binned, noisy);
    rc = cw_max_clusters(kernel, C, smem, &max_clusters);
    if (rc) return rc;
    if (max_clusters < 1) {
        es_set_error("es_rollout_closedloop_mlp: no cluster of %d CTAs with %zu bytes of shared memory each fits on this device", C, smem);
        return ES_ERR_UNSUPPORTED;
    }
    const CwParams p = {r, env};
    const long long evals = 2ll * r.n_pairs;
    const int clusters = evals < max_clusters ? (int)evals : max_clusters;
    cudaLaunchAttribute attr;
    const cudaLaunchConfig_t cfg = cw_config(C, smem, clusters, stream, &attr);
    ES_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kernel, p));
    ES_LAUNCHED(ctx);
    return ES_OK;
}
