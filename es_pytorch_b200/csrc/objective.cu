// objective.cu -- the single-objective fitness adaptors of src/gym/training_result.py on the device.
//
// A rollout leaves each evaluation's float64 episode total in column 0 of its fitness row and its float32 final position
// (x, y, z) in behv[e][0..2].  This kernel rewrites column 0 as the adaptor the caller picked would compute it:
//   ES_OBJ_MEAN_REWARD  total / steps                   MeanRewardResult  (training_result.py:67-69)
//   ES_OBJ_DIST         sqrt(x*x + y*y)                 DistResult        np.linalg.norm(positions[-3:-1])  (:72-74)
//   ES_OBJ_XDIST        x                               XDistResult       positions[-3]                      (:77-79)
// Each value equals the host class's get_result bit for bit, by construction:
//   - a float32 value has a 24-bit significand, so its square has at most 48 significant bits and is exact in float64; a
//     float32 square cannot overflow float64 (< 2^256) and a float32 subnormal's square (>= 2^-298) is a float64 normal;
//   - the host's norm is sqrt(dot(v, v)) over the two float64 values: both products are exact, so the sum is rounded once
//     whatever order, blocking or FMA numpy's dot uses, and the kernel's __dadd_rn of the two exact squares is that sum;
//   - CUDA's double sqrt and __ddiv_rn are correctly rounded (IEEE 754), as are numpy's sqrt and python's float division;
//     steps < 2^31 is exact as a double, as python's int-to-float conversion makes it; the reward is sum([total]), which
//     adds the total to 0 (only a -0.0 total changes: to +0.0), and the kernel adds it to 0.0 too;
//   - the float32 -> float64 conversion of x is exact, as float(np.float32) is on the host.
#include "common.cuh"

__global__ void fitness_objective_kernel(int kind, double* __restrict__ fit, int fit_stride, const float* __restrict__ behv,
                                         int n, double steps) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    double* f = fit + (size_t)e * fit_stride;
    if (kind == ES_OBJ_MEAN_REWARD) {
        // sum(rewards) / steps with rewards = [total]: python's sum starts from 0, and 0 + total turns -0.0 into +0.0
        *f = __ddiv_rn(__dadd_rn(0.0, *f), steps);
    } else {
        const double x = (double)behv[(size_t)e * 3 + 0];
        if (kind == ES_OBJ_DIST) {
            const double y = (double)behv[(size_t)e * 3 + 1];
            *f = __dsqrt_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)));
        } else {
            *f = x;
        }
    }
}

// ES_OBJ_MEAN_REWARD with every evaluation's own steps (an env whose episodes end early): total / steps[e], the same operations
__global__ void mean_reward_steps_kernel(double* __restrict__ fit, int fit_stride, const int* __restrict__ steps, int n) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    double* f = fit + (size_t)e * fit_stride;
    *f = __ddiv_rn(__dadd_rn(0.0, *f), (double)steps[e]);
}

int es_impl_fitness_objective(es_ctx* ctx, int kind, double* fit, int fit_stride, const float* behv, int n, int steps,
                              cudaStream_t stream) {
    fitness_objective_kernel<<<es_div_up(n, 256), 256, 0, stream>>>(kind, fit, fit_stride, behv, n, (double)steps);
    ES_LAUNCHED(ctx);
    return ES_OK;
}

int es_impl_mean_reward_steps(es_ctx* ctx, double* fit, int fit_stride, const int* steps, int n, cudaStream_t stream) {
    mean_reward_steps_kernel<<<es_div_up(n, 256), 256, 0, stream>>>(fit, fit_stride, steps, n);
    ES_LAUNCHED(ctx);
    return ES_OK;
}
