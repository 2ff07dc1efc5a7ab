// rollout_tcw.cu -- fused rollout + fitness on the Hopper tensor cores (wgmma) for WIDE tanh MLPs: 2 to 4 hidden layers, every
// hidden width a multiple of 64 in [64, 256], obs <= 256, act <= 32 (the shipped configs' policies: 15-256-256-3,
// 17/26/28-256-256-256-6/8, 28-128-256-256-128-8).  Same two precisions as rollout_tc2.cu:
//
//   SPLIT = false (ES_ROLLOUT_TC):   one float16 wgmma per product, tanh.approx
//   SPLIT = true  (ES_ROLLOUT_TC3):  operands split into float16 hi + lo, three MMAs per product (hi.hi + hi.lo + lo.hi)
//                                    accumulated in float32, tanh to float32 accuracy (1 - 2 / (1 + e^2x))
// Rewards are summed in float64 in both.
//
// and the contract of rollout_f32.cu: action noise [n_pairs][2][E][T][act] with the per-step mean over the E episodes in
// float64, behaviour of the last episode, fit_stride, out-of-table indices through es_checked_slice.
//
// Per launch chunk of pairs (<= 256 MiB of weight images):
//   1. rollout_tcw_build_kernel (one CTA per pair) writes theta +- sigma*eps of both evaluations as float16 hi (+ lo) images
//      in the K-major, 128-byte-swizzled layout the wgmma B descriptor reads: per layer [K chunk][64-wide N block][piece] blocks
//      of 64 rows x 128 B, zero-padded to multiples of 64 in K and N, then the float32 biases.  The table is read as float32
//      directly (no float16 shadows: these shapes would pay 16-32 B of HBM per table element for them).  Layer 1 is <= 5 % of
//      these shapes' MACs, so rollout_tc2.cu's U +- sigma V split of layer 1 is not carried over.
//   2. rollout_tcw_kernel: persistent CTAs take work items (evaluation, 128-step tile) round-robin in evaluation-major order,
//      so the tiles of one evaluation run at the same time on neighbouring SMs and its image is read from HBM about once.
//      Each of the two consumer warpgroups owns 64 rows (time steps) of the tile.  A layer is, per K chunk of 64, one
//      m64n64k16 chain per 64-wide N block, into accumulators preloaded with the bias (up to 4 x 32 float32 registers).  The
//      epilogue writes tanh (hi[, lo]) of the warpgroup's own rows back into one shared activation buffer, which is the A
//      operand of the next layer; the observation tile enters through the same buffer.  The last layer's epilogue forms
//      the rewards, action noise, episode means and positions of the tile and writes one partial sum per consumer warp.
//      A producer warp streams the weight blocks (one bulk copy per (K chunk, N block)) through a ring of stages, in the
//      order the consumers use them.
//   3. rollout_tcw_finish_kernel adds the partial sums of every evaluation in a fixed order (tile, warp), so the results do
//      not depend on the grid, the chunking or the order of the pairs.
//
// Shared memory (SPLIT): activations 4 K chunks x 2 pieces x 128 rows x 128 B = 128 KB, weight ring 6 stages x 16 KB = 96 KB.
//
// Choices, and what they were (not) measured against:
//   * m64n64k16 chains per 64-wide N block rather than one m64n{width}k16 chain: one wgmma form and one stage size serve
//     every width from 64 to 256 and the last layer (act <= 32, padded to 64); the accumulators are the same 4 x 32
//     registers either way.  The n{width} form was not built, so the two were not compared.
//   * a ring of 6 stages of one (K chunk of 64, N block of 64) hi + lo block each (16 KB), rather than 3 stages of K 32 x N
//     256 (32 KB): a stage is then the operand of exactly one chain above, in the same 128-byte swizzle (64 float16 per
//     row) as the activation buffer; the bytes in flight are the same 96 KB.  Not compared by measurement.
//   * the separate finish kernel: the tiles of one evaluation run on different CTAs, and adding their sums in a fixed
//     order makes every result independent of the grid, the chunking and the order of the pairs (the tests compare a run
//     with the pairs reversed bit for bit); atomic adds would not.  It costs one small launch per chunk.
//   * the hidden-layer epilogue stores each N block before it touches the next block's accumulators: computed all at
//     once, the tanh and hi / lo values of a 256-wide layer did not fit beside the accumulators (the TC3 kernels spilled
//     about 140 bytes per thread).
//
// Binned-action policies (FFBinned, src/nn/nn.py:99-117; ES_ROLLOUT_TC3 only, rollout_tcw_binned_kernel): the last layer is up
// to four 64-wide N blocks (adim * bins <= 256), and obs-64-64-X binned shapes run here too.  Its tanh outputs go as float32 into
// the warpgroup's rows of the activation buffer, which no MMA reads any more at that point (64 rows x 256 floats = the
// warpgroup's 8 pieces of 8 KB: column n in piece n / 32, at word (n ^ row) mod 32 of its 128-byte row, so that the 32 rows a warp
// reads at one column fall in 32 banks), rather than being reduced across the quads holding a row's columns
// with shuffles: the buffer is free, and one thread per row then takes the arg-max of each dimension in bin order (the first
// maximal bin, as torch.argmax) and forms the action and the float32 reward in index order as rollout_f32.cu does; only the
// float64 sums over the rows and tiles are reassociated.  ES_ROLLOUT_TC refuses binned heads (api.cu): an arg-max over
// float16-grade outputs is not parity grade.
//
// 12 warps (3 warpgroups): warpgroup 0 = warp 0 producer (the other three idle) -> setmaxnreg 24 registers;
// warpgroups 1 and 2: consumers, rows 0-63 / 64-127 of every tile -> setmaxnreg 240 registers.
#include "rollout_tcw.cuh"

namespace {

template <bool SPLIT, bool NOISE>
__global__ void __launch_bounds__(TW_THREADS, 1) rollout_tcw_kernel(const __grid_constant__ TwParams p) { tw_rollout<SPLIT, NOISE, false>(p); }
__global__ void __launch_bounds__(TW_THREADS, 1) rollout_tcw_binned_kernel(const __grid_constant__ TwParams p) {
    tw_rollout<true, false, true>(p);
}

template <bool SPLIT, bool NOISE>
int tw_launch_main(es_ctx* ctx, const TwParams& p, int grid, cudaStream_t stream) {
    constexpr size_t smem = TwCfg<SPLIT>::SMEM;
    ES_CHECK_CUDA(cudaFuncSetAttribute(rollout_tcw_kernel<SPLIT, NOISE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    rollout_tcw_kernel<SPLIT, NOISE><<<grid, TW_THREADS, smem, stream>>>(p);
    ES_LAUNCHED(ctx);
    return ES_OK;
}

// the main kernel of a chunk (tw_run's launch): binned heads (TC3 only), or tanh heads with or without action noise
template <bool SPLIT>
int tw_launch(es_ctx* ctx, const TwParams& p, int grid, cudaStream_t stream) {
    if constexpr (SPLIT) {
        if (p.bins) {
            constexpr size_t smem = TwCfg<true>::SMEM;
            ES_CHECK_CUDA(cudaFuncSetAttribute(rollout_tcw_binned_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            rollout_tcw_binned_kernel<<<grid, TW_THREADS, smem, stream>>>(p);
            ES_LAUNCHED(ctx);
            return ES_OK;
        }
    }
    return p.act_noise ? tw_launch_main<SPLIT, true>(ctx, p, grid, stream) : tw_launch_main<SPLIT, false>(ctx, p, grid, stream);
}

}  // namespace

bool es_tcw_covers(const EsRollout& r) {
    const int* ls = r.dims;
    if (r.n_layers < 3 || r.n_layers > TW_MAX_LAYERS) return false;      // 2 to 4 hidden layers
    if (r.n_layers == 3 && ls[1] == 64 && ls[2] == 64) return false;    // obs-64-64-act: rollout_tc2.cu
    if (ls[0] < 1 || ls[0] > 256 || ls[r.n_layers] < 1 || ls[r.n_layers] > 32) return false;
    for (int l = 1; l < r.n_layers; ++l)
        if (ls[l] % 64 != 0 || ls[l] < 64 || ls[l] > 256) return false;
    return true;
}

// binned heads (ES_ROLLOUT_TC3): 2 to 4 hidden layers of multiples of 64 in [64, 256] (obs-64-64-X included), obs <= 256 and
// adim * bins <= 256 (up to four N blocks in the last layer)
bool es_tcw_covers_binned(const EsRollout& r) {
    const int* ls = r.dims;
    if (r.n_layers < 3 || r.n_layers > TW_MAX_LAYERS) return false;
    if (ls[0] < 1 || ls[0] > 256 || ls[r.n_layers] < 1 || ls[r.n_layers] > 256) return false;
    for (int l = 1; l < r.n_layers; ++l)
        if (ls[l] % 64 != 0 || ls[l] < 64 || ls[l] > 256) return false;
    return true;
}

int es_impl_rollout_tcw(es_ctx* ctx, const EsRollout& r, int split, cudaStream_t stream) {
    if (!split && r.T < TW_TC_MIN_T) {
        es_set_error("es_rollout_openloop(TC): the wide tensor-core path with single float16 products needs T >= %d (shorter "
                     "episodes exceed this mode's error bound of 1e-3 of the reward mass); use ES_ROLLOUT_TC3", TW_TC_MIN_T);
        return ES_ERR_UNSUPPORTED;
    }
    return split ? tw_run<true>(ctx, r, stream, tw_launch<true>) : tw_run<false>(ctx, r, stream, tw_launch<false>);
}
