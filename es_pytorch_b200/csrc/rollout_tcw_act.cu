// rollout_tcw_act.cu -- the wide tensor-core rollout (rollout_tcw.cuh, design in rollout_tcw.cu) for policies whose activation
// is ReLU, leaky ReLU, ELU or sigmoid (es_rollout_openloop_activation, ES_ROLLOUT_TC3 only): 2 to 4 hidden layers of widths in
// {64, 128, 192, 256}, obs-64-64-act included (rollout_tc2.cu stays tanh-only), obs <= 256, act <= 32.
//
// Every layer's epilogue applies the activation in float32 (es_act) where the tanh kernels apply tanh; nothing else changes, so
// the results keep the tanh kernels' contract (fixed summation order, independent of the grid, the chunking and the order of
// the pairs).  The hidden activations enter the next layer split into float16 hi + lo parts: tanh's [-1, 1] always fits, but
// ReLU, leaky ReLU and ELU are unbounded above (ELU below too, by alpha), and a value beyond 65504 in magnitude has no finite
// float16 hi part.  The epilogue flags such a value as ES_ASYNC_F16_RANGE through the ctx's error word: the call's results are
// invalid and the caller learns it from es_check_async or the next entry point (the float32 kernel, ES_ROLLOUT_F32, has no
// such limit).  Sigmoid's (0, 1) needs no check.
//
// One kernel per kind and action-noise variant (8), under a name of their own.
#include "rollout_tcw.cuh"

namespace {

template <int ACT, bool NOISE>
__global__ void __launch_bounds__(TW_THREADS, 1) rollout_tcwa_kernel(const __grid_constant__ TwParams p, float act_param, int* err) {
    tw_rollout<true, NOISE, false, ACT>(p, act_param, err);
}

template <int ACT, bool NOISE>
int twa_launch(es_ctx* ctx, const TwParams& p, int grid, float act_param, int* err, cudaStream_t stream) {
    constexpr size_t smem = TwCfg<true>::SMEM;
    ES_CHECK_CUDA(cudaFuncSetAttribute(rollout_tcwa_kernel<ACT, NOISE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    rollout_tcwa_kernel<ACT, NOISE><<<grid, TW_THREADS, smem, stream>>>(p, act_param, err);
    ES_LAUNCHED(ctx);
    return ES_OK;
}

template <int ACT>
int twa_launch_kind(es_ctx* ctx, const TwParams& p, int grid, float act_param, int* err, cudaStream_t stream) {
    return p.act_noise ? twa_launch<ACT, true>(ctx, p, grid, act_param, err, stream)
                       : twa_launch<ACT, false>(ctx, p, grid, act_param, err, stream);
}

}  // namespace

// 2 to 4 hidden layers of multiples of 64 in [64, 256] (obs-64-64-act included), obs <= 256, act <= 32 (N block 0 of the last
// layer's epilogue)
bool es_tcw_covers_act(const EsRollout& r) {
    const int* ls = r.dims;
    if (r.n_layers < 3 || r.n_layers > TW_MAX_LAYERS) return false;
    if (ls[0] < 1 || ls[0] > 256 || ls[r.n_layers] < 1 || ls[r.n_layers] > 32) return false;
    for (int l = 1; l < r.n_layers; ++l)
        if (ls[l] % 64 != 0 || ls[l] < 64 || ls[l] > 256) return false;
    return true;
}

int es_impl_rollout_tcw_act(es_ctx* ctx, const EsRollout& r, cudaStream_t stream) {
    const int kind = r.activation;
    const float prm = r.act_param;
    int* err = r.err;
    return tw_run<true>(ctx, r, stream, [kind, prm, err](es_ctx* c, const TwParams& p, int grid, cudaStream_t s) {
        switch (kind) {
            case ES_ACT_RELU: return twa_launch_kind<ES_ACT_RELU>(c, p, grid, prm, err, s);
            case ES_ACT_LEAKY_RELU: return twa_launch_kind<ES_ACT_LEAKY_RELU>(c, p, grid, prm, err, s);
            case ES_ACT_ELU: return twa_launch_kind<ES_ACT_ELU>(c, p, grid, prm, err, s);
            default: return twa_launch_kind<ES_ACT_SIGMOID>(c, p, grid, prm, err, s);
        }
    });
}
