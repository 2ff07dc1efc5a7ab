// rollout_closedw_act.cu -- the closed-loop cluster rollout (rollout_closedw.cuh, design in rollout_closedw.cu) for policies
// whose activation is ReLU, leaky ReLU, ELU or sigmoid (es_rollout_closedloop_mlp_activation): every shape es_closedw_plan
// covers, with or without action noise and episodes, a cluster of one CTA included (rollout_closed.cu stays tanh-only).
//
// The lane that owns a row applies the activation (es_act, in float32) where the tanh kernels apply es_tanh_exp; the env's
// tanh(A obs + B a) is the env's and stays.  The kind is uniform over the launch and the branch sits in the per-row epilogue,
// outside the dot products, so one kernel per depth and noise variant serves every kind.  The plan (cluster size, shared
// memory) is es_closedw_plan's; the resident clusters are queried for these kernels.
#include "rollout_closedw.cuh"

namespace {

template <int NL, bool NOISY>
__global__ void __launch_bounds__(CW_THREADS, 1) rollout_closeda_kernel(const CwParams p) { cw_rollout<NL, false, NOISY, true>(p); }

CwKernel cwa_kernel(int n_layers, bool noisy) {
    if (noisy)
        return n_layers == 3 ? rollout_closeda_kernel<3, true> : n_layers == 4 ? rollout_closeda_kernel<4, true>
                                                                                : rollout_closeda_kernel<5, true>;
    return n_layers == 3 ? rollout_closeda_kernel<3, false> : n_layers == 4 ? rollout_closeda_kernel<4, false>
                                                                             : rollout_closeda_kernel<5, false>;
}

}  // namespace

int es_closedw_act_max_clusters(int n_layers, int C, size_t smem, int* clusters) {
    return cw_max_clusters(cwa_kernel(n_layers, false), C, smem, clusters);
}

int es_impl_rollout_closedw_act(es_ctx* ctx, const EsRollout& r, const EsClosedEnv& env, cudaStream_t stream) {
    int C = 0, max_clusters = 0;
    size_t smem = 0;
    int rc = es_closedw_plan(r.dims, r.n_layers, env.band, &C, &smem);
    if (rc) return rc;
    const CwKernel kernel = cwa_kernel(r.n_layers, r.act_noise != nullptr);
    rc = cw_max_clusters(kernel, C, smem, &max_clusters);
    if (rc) return rc;
    if (max_clusters < 1) {
        es_set_error("es_rollout_closedloop_mlp_activation: no cluster of %d CTAs with %zu bytes of shared memory each fits on this "
                     "device", C, smem);
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
