// api.cu -- extern "C" surface of libes_b200.so (declared in include/es_b200.h):
// argument validation, context/scratch management, dispatch to the kernels.
#include <math.h>
#include <stdarg.h>
#include <stdlib.h>
#include "common.cuh"

static thread_local char g_err[512] = "";

void es_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int es_ctx_scratch(es_ctx* ctx, size_t bytes, void** out) {
    if (bytes > ctx->scratch_bytes) {
        // growing is rare (first call per shape); it synchronises the device, which is
        // fine outside the steady state.
        if (ctx->scratch) ES_CHECK_CUDA(cudaFree(ctx->scratch));
        ctx->scratch = nullptr;
        ctx->scratch_bytes = 0;
        size_t want = bytes + (bytes >> 2) + 4096;
        cudaError_t e = cudaMalloc(&ctx->scratch, want);
        if (e != cudaSuccess) {
            es_set_error("scratch cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e));
            return ES_ERR_NOMEM;
        }
        ctx->scratch_bytes = want;
    }
    *out = ctx->scratch;
    return ES_OK;
}

int es_ctx_counters(es_ctx* ctx, size_t n, unsigned** out) {
    if (n > ctx->n_counters) {
        if (ctx->counters) ES_CHECK_CUDA(cudaFree(ctx->counters));
        ctx->counters = nullptr;
        ctx->n_counters = 0;
        size_t want = n * 2 + 64;
        cudaError_t e = cudaMalloc((void**)&ctx->counters, want * sizeof(unsigned));
        if (e != cudaSuccess) {
            es_set_error("counter cudaMalloc failed: %s", cudaGetErrorString(e));
            return ES_ERR_NOMEM;
        }
        ES_CHECK_CUDA(cudaMemset(ctx->counters, 0, want * sizeof(unsigned)));
        ctx->n_counters = want;
    }
    *out = ctx->counters;
    return ES_OK;
}

extern "C" {

int es_abi_version(void) { return 1; }

const char* es_last_error(void) { return g_err; }

int es_ctx_create(int device, es_ctx** out) {
    ES_REQUIRE(out != nullptr, "es_ctx_create: out is NULL");
    int n = 0;
    ES_CHECK_CUDA(cudaGetDeviceCount(&n));
    ES_REQUIRE(device >= 0 && device < n, "es_ctx_create: device %d out of range (%d devices)", device, n);
    ES_CHECK_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    ES_CHECK_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
        es_set_error("es_ctx_create: device %d is sm_%d%d; this library is built for sm_90a only", device,
                     prop.major, prop.minor);
        return ES_ERR_UNSUPPORTED;
    }
    es_ctx* c = (es_ctx*)calloc(1, sizeof(es_ctx));
    if (!c) return ES_ERR_NOMEM;
    c->device = device;
    c->sm_count = prop.multiProcessorCount;
    {   // mapped error word for kernel-side argument checks (see es_checked_slice)
        int* h = nullptr;
        if (cudaHostAlloc((void**)&h, sizeof(int), cudaHostAllocMapped) == cudaSuccess) {
            *h = 0;
            int* d = nullptr;
            if (cudaHostGetDevicePointer((void**)&d, h, 0) == cudaSuccess) { c->err_host = h; c->err_dev = d; }
            else cudaFreeHost(h);
        }
        (void)cudaGetLastError();
    }
    *out = c;
    return ES_OK;
}

int es_ctx_destroy(es_ctx* ctx) {
    if (!ctx) return ES_OK;
    cudaSetDevice(ctx->device);
    if (ctx->scratch) cudaFree(ctx->scratch);
    if (ctx->counters) cudaFree(ctx->counters);
    es_tc2_free_shadows(ctx);
    if (ctx->err_host) cudaFreeHost((void*)ctx->err_host);
    free(ctx);
    return ES_OK;
}

int es_noise_table_changed(es_ctx* ctx) {
    if (!ctx) return ES_ERR_INVALID;
    ctx->sh16_src = nullptr;            // the shadows (if any) are rebuilt by the next tensor-core rollout
    ctx->sh16_len = 0;
    return ES_OK;
}

static int es_async_error(es_ctx* ctx, const char* where) {
    if (ctx->err_host && *ctx->err_host) {
        const int code = *ctx->err_host;
        *ctx->err_host = 0;
        if (code == ES_ASYNC_BAD_INDEX)
            es_set_error("%s: a previous kernel was given a noise index outside the table (index < 0 or index + n_params >= "
                         "table length; the reference asserts this in NoiseTable.get, src/core/noisetable.py:34): the "
                         "results of that call are invalid", where);
        else if (code == ES_ASYNC_RNG_OVERFLOW)
            es_set_error("%s: es_draw_noisy consumed more MT19937 words than its jump-ahead pass had generated (a > 12 sigma "
                         "event of the polar method's acceptance count, or a bug): the draws of that call are invalid; set "
                         "ES_MT_JUMP=0 to use the sequential kernel", where);
        else if (code == ES_ASYNC_F16_RANGE)
            es_set_error("%s: a previous ES_ROLLOUT_TC3 rollout met a hidden activation beyond float16 range (|h| > 65504), which its "
                         "split float16 operands cannot hold: the results of that call are invalid; use ES_ROLLOUT_F32 for such "
                         "policies", where);
        else if (code == ES_ASYNC_WALK_OVERFLOW)
            es_set_error("%s: es_rollout_closedloop_terminal_streams walked a stream past the MT19937 words generated for it (a > "
                         "12 sigma event of the polar method's acceptance count, or a bug): the results of that call are invalid",
                         where);
        else if (code == ES_ASYNC_RANDN_OVERFLOW)
            es_set_error("%s: es_randn needed more MT19937 words than its windows had generated (a > 12 sigma event of the "
                         "polar method's acceptance count, or a bug): the values of that call are invalid", where);
        else
            es_set_error("%s: a previous kernel reported error %d", where, code);
        return ES_ERR_INVALID;
    }
    return ES_OK;
}

int es_check_async(es_ctx* ctx) {
    if (!ctx) { es_set_error("es_check_async: ctx is NULL"); return ES_ERR_INVALID; }
    return es_async_error(ctx, "es_check_async");
}

int64_t es_launch_count(const es_ctx* ctx) { return ctx ? ctx->launches : -1; }
int es_sm_count(const es_ctx* ctx) { return ctx ? ctx->sm_count : -1; }

#define ES_ENTER(ctx)                                                        \
    ES_REQUIRE((ctx) != nullptr, "%s: ctx is NULL", __func__);               \
    ES_CHECK_CUDA(cudaSetDevice((ctx)->device));                             \
    do { int _a = es_async_error((ctx), __func__); if (_a) return _a; } while (0)

// the randint bound of es_draw_indices and es_draw_noisy: NoiseTable.sample_idx raises ValueError when upper_bound <= 0
// (noisetable.py:39), and ranges >= 2^32 take numpy's 64-bit draw path
static int es_randint_check(const char* fn, uint64_t upper_bound) {
    ES_REQUIRE(upper_bound >= 1, "%s: upper_bound must be >= 1 (network too large for noise table)", fn);
    if (upper_bound - 1 >= 0xFFFFFFFFull) {
        es_set_error("%s: ranges >= 2^32 use numpy's 64-bit draw path, not implemented", fn);
        return ES_ERR_UNSUPPORTED;
    }
    return ES_OK;
}

int es_draw_indices(es_ctx* ctx, uint32_t* mt_key, int32_t* mt_pos, int n_streams, int n_per_stream,
                    uint64_t upper_bound, int extra_words, int64_t* idx_out, uint32_t* extra_out, void* stream) {
    ES_ENTER(ctx);
    ES_REQUIRE(mt_key && mt_pos && idx_out, "es_draw_indices: NULL pointer");
    ES_REQUIRE(n_streams >= 0 && n_per_stream >= 0, "es_draw_indices: negative count");
    ES_REQUIRE(extra_words >= 0 && extra_words <= 7, "es_draw_indices: extra_words must be in [0,7]");
    const int rc = es_randint_check("es_draw_indices", upper_bound);
    if (rc) return rc;
    if (n_streams == 0 || n_per_stream == 0) return ES_OK;
    return es_impl_draw_indices(ctx, mt_key, mt_pos, n_streams, n_per_stream, upper_bound, extra_words, idx_out,
                                extra_out, (cudaStream_t)stream);
}

int es_mt_skip(es_ctx* ctx, uint32_t* mt_key, int32_t* mt_pos, int n_streams, int n_words, void* stream) {
    ES_ENTER(ctx);
    ES_REQUIRE(mt_key && mt_pos, "es_mt_skip: NULL pointer");
    ES_REQUIRE(n_streams >= 0 && n_words >= 0, "es_mt_skip: negative count");
    if (n_streams == 0 || n_words == 0) return ES_OK;
    return es_impl_mt_skip(ctx, mt_key, mt_pos, n_streams, n_words, (cudaStream_t)stream);
}

int es_perturb(es_ctx* ctx, const float* theta, const float* table, int64_t table_len, const int64_t* idx, int n_idx,
               int P, float sigma, float* out_pos, float* out_neg, void* stream) {
    ES_ENTER(ctx);
    ES_REQUIRE(theta && table && idx && out_pos, "es_perturb: NULL pointer");
    ES_REQUIRE(n_idx >= 0 && P > 0 && table_len > P, "es_perturb: bad sizes");
    if (n_idx == 0) return ES_OK;
    return es_impl_perturb(ctx, theta, table, table_len, idx, n_idx, P, sigma, out_pos, out_neg, (cudaStream_t)stream);
}

int es_normalise_obs(es_ctx* ctx, const float* obs, const double* mean, const double* std, double clip, int rows,
                     int obs_dim, float* out, void* stream) {
    ES_ENTER(ctx);
    ES_REQUIRE(obs && mean && std && out, "es_normalise_obs: NULL pointer");
    ES_REQUIRE(rows >= 0 && obs_dim > 0, "es_normalise_obs: bad sizes");
    if (rows == 0) return ES_OK;
    return es_impl_normalise_obs(ctx, obs, mean, std, clip, rows, obs_dim, out, (cudaStream_t)stream);
}

int es_obs_colsum(es_ctx* ctx, const float* obs, int rows, int obs_dim, float* sum_out, float* sumsq_out, void* stream) {
    ES_ENTER(ctx);
    ES_REQUIRE(obs && sum_out && sumsq_out, "es_obs_colsum: NULL pointer");
    ES_REQUIRE(rows >= 0 && obs_dim > 0, "es_obs_colsum: bad sizes");
    return es_impl_obs_colsum(ctx, obs, rows, obs_dim, sum_out, sumsq_out, (cudaStream_t)stream);
}

int es_obstat_accumulate(es_ctx* ctx, double* sum, double* sumsq, const float* s, const float* ssq, int obs_dim,
                         int n_rollouts, void* stream) {
    ES_ENTER(ctx);
    ES_REQUIRE(sum && sumsq && s && ssq, "es_obstat_accumulate: NULL pointer");
    ES_REQUIRE(obs_dim > 0 && n_rollouts >= 0, "es_obstat_accumulate: bad sizes");
    if (n_rollouts == 0) return ES_OK;
    return es_impl_obstat_accumulate(ctx, sum, sumsq, s, ssq, obs_dim, n_rollouts, (cudaStream_t)stream);
}

int es_obstat_accumulate_coins(es_ctx* ctx, double* sum, double* sumsq, double* count_io, const float* s,
                               const float* ssq, int obs_dim, int rows_per_rollout, const uint32_t* coin_words,
                               int n_coins, double chance, void* stream) {
    ES_ENTER(ctx);
    ES_REQUIRE(sum && sumsq && count_io && s && ssq && (coin_words || n_coins == 0),
               "es_obstat_accumulate_coins: NULL pointer");
    ES_REQUIRE(obs_dim > 0 && n_coins >= 0 && rows_per_rollout >= 0, "es_obstat_accumulate_coins: bad sizes");
    return es_impl_obstat_accumulate_coins(ctx, sum, sumsq, count_io, s, ssq, obs_dim, rows_per_rollout, coin_words,
                                           n_coins, chance, (cudaStream_t)stream);
}

// the checks the open- and closed-loop rollouts share (`ptrs`: the entry point's own pointers are set), then the call's shape
// from the caller's layer sizes into r
static int es_rollout_check(const char* fn, bool ptrs, const int* layer_sizes, EsRollout& r) {
    ES_REQUIRE(ptrs && r.table && r.idx && r.theta && layer_sizes && r.rew_vec && r.fit_pos && r.fit_neg, "%s: NULL pointer", fn);
    ES_REQUIRE(r.n_layers >= 1 && r.n_layers <= ES_MAX_LAYERS, "%s: n_layers must be in [1,%d]", fn, ES_MAX_LAYERS);
    ES_REQUIRE(r.n_pairs >= 0 && r.T >= 1 && r.fit_stride >= 1, "%s: bad sizes", fn);
    ES_REQUIRE((r.behv_pos == nullptr) == (r.behv_neg == nullptr), "%s: behv_pos/behv_neg must both be set or NULL", fn);
    int64_t count = 0;
    for (int l = 0; l < r.n_layers; ++l) {
        ES_REQUIRE(layer_sizes[l] > 0 && layer_sizes[l + 1] > 0, "%s: layer size <= 0", fn);
        count += (int64_t)layer_sizes[l] * layer_sizes[l + 1] + layer_sizes[l + 1];
    }
    ES_REQUIRE(count == r.P, "%s: layer sizes give %lld params, P=%d", fn, (long long)count, r.P);
    ES_REQUIRE(r.table_len > r.P, "%s: table smaller than the network", fn);
    r.dims[0] = layer_sizes[0];
    int at = 0;
    for (int l = 0; l < r.n_layers; ++l) {             // state-dict order (src/core/policy.py:33-35)
        r.dims[l + 1] = layer_sizes[l + 1];
        r.w_off[l] = at; at += r.dims[l] * r.dims[l + 1];
        r.b_off[l] = at; at += r.dims[l + 1];
    }
    // (a binned head with bins < 2 is refused by es_binned_check before any kernel runs)
    const int out = r.dims[r.n_layers];
    r.act = r.bins ? out / r.bins : out;
    r.head_scale = r.bins ? (float)(1.0 / (r.bins - 1.0)) : 0.f;
    return ES_OK;
}

// the head arguments of the binned entry points: bins >= 2 (the reference divides by bins - 1), low / range set, the last layer
// adim * bins <= 256 wide
static int es_binned_check(const char* fn, const EsRollout& r) {
    ES_REQUIRE(r.bins >= 2, "%s: bins must be >= 2 (the action is idx / (bins - 1)), got %d", fn, r.bins);
    ES_REQUIRE(r.head_low && r.head_range, "%s: NULL low / range", fn);
    const int out = r.dims[r.n_layers];
    ES_REQUIRE(out % r.bins == 0, "%s: the last layer's %d outputs are not adim * bins for bins %d", fn, out, r.bins);
    if (out > 256) {
        es_set_error("%s: binned heads up to adim * bins = 256 outputs supported, got %d * %d", fn, out / r.bins, r.bins);
        return ES_ERR_UNSUPPORTED;
    }
    return ES_OK;
}

// the activation arguments of the *_activation entry points
static int es_activation_check(const char* fn, int activation, float act_param) {
    ES_REQUIRE(activation >= ES_ACT_TANH && activation <= ES_ACT_SIGMOID,
               "%s: unknown activation %d (ES_ACT_TANH, ES_ACT_RELU, ES_ACT_LEAKY_RELU, ES_ACT_ELU or ES_ACT_SIGMOID)", fn, activation);
    ES_REQUIRE(isfinite(act_param), "%s: the activation parameter must be finite, got %g", fn, (double)act_param);
    return ES_OK;
}

// the policies an entry point takes: tanh MLPs, binned heads (EsRollout::bins, which es_binned_check refuses below 2),
// es_rollout_closedloop's tanh MLPs (two hidden layers, rollout_closed.cu only), or MLPs with another activation
// (EsRollout::activation)
enum EsHead { ES_HEAD_TANH, ES_HEAD_BINNED, ES_HEAD_TANH_ONE_CTA, ES_HEAD_ACT };

// the part of a shape outside the wide tensor-core kernel's coverage (`max_out`: the widest last layer it takes), into why
static void es_tcw_why(const EsRollout& r, int max_out, char* why, size_t n) {
    const int* dims = r.dims;
    if (r.n_layers < 3 || r.n_layers > 5) {
        snprintf(why, n, "%d hidden layers", r.n_layers - 1);
        return;
    }
    if (dims[0] > 256) {
        snprintf(why, n, "obs %d", dims[0]);
        return;
    }
    for (int l = 1; l < r.n_layers; ++l)
        if (dims[l] % 64 || dims[l] > 256) {
            snprintf(why, n, "hidden layer %d of width %d", l, dims[l]);
            return;
        }
    if (dims[r.n_layers] > max_out) snprintf(why, n, "%d outputs", dims[r.n_layers]);
    else snprintf(why, n, "the shape");
}

// an open-loop entry point after ES_ENTER: its checks in order, then the mode's kernel; `fn` names it in every message
static int es_openloop(es_ctx* ctx, const char* fn, EsRollout r, const int* layer_sizes, EsHead head, int mode, cudaStream_t stream) {
    int rc = es_rollout_check(fn, r.obsn != nullptr, layer_sizes, r);
    if (rc) return rc;
    if (head == ES_HEAD_BINNED) {
        rc = es_binned_check(fn, r);
        if (rc) return rc;
        if (mode == ES_ROLLOUT_TC) {
            es_set_error("%s: ES_ROLLOUT_TC refuses binned heads: an arg-max over float16-grade outputs is not parity grade; use "
                         "ES_ROLLOUT_TC3 or ES_ROLLOUT_F32", fn);
            return ES_ERR_UNSUPPORTED;
        }
        if (mode == ES_ROLLOUT_TC3 && !es_tcw_covers_binned(r)) {
            char why[96];
            es_tcw_why(r, 256, why, sizeof why);
            es_set_error("%s: ES_ROLLOUT_TC3 covers binned heads with 2 to 4 hidden layers of widths in {64, 128, 192, 256} and obs "
                         "<= 256, got %s; use ES_ROLLOUT_F32", fn, why);
            return ES_ERR_UNSUPPORTED;
        }
    } else if (head == ES_HEAD_ACT) {
        if (mode == ES_ROLLOUT_TC) {
            es_set_error("%s: ES_ROLLOUT_TC refuses activations other than tanh (its single float16 products are bounded for "
                         "tanh's outputs only); use ES_ROLLOUT_TC3 or ES_ROLLOUT_F32", fn);
            return ES_ERR_UNSUPPORTED;
        }
        if (mode == ES_ROLLOUT_TC3 && !es_tcw_covers_act(r)) {
            char why[96];
            es_tcw_why(r, 32, why, sizeof why);
            es_set_error("%s: ES_ROLLOUT_TC3 covers activations other than tanh for 2 to 4 hidden layers of widths in {64, 128, 192, "
                         "256}, obs <= 256 and act <= 32, got %s; use ES_ROLLOUT_F32", fn, why);
            return ES_ERR_UNSUPPORTED;
        }
    } else if (r.n_pairs == 0) {
        return ES_OK;                               // a tanh head returns before it looks at the mode, the others after
    }
    if (mode != ES_ROLLOUT_F32 && mode != ES_ROLLOUT_TC && mode != ES_ROLLOUT_TC3) {
        es_set_error("%s: unknown mode %d", fn, mode);
        return ES_ERR_INVALID;
    }
    if (r.n_pairs == 0) return ES_OK;
    if (mode == ES_ROLLOUT_F32) return es_impl_rollout_f32(ctx, r, stream);
    if (head == ES_HEAD_ACT) return es_impl_rollout_tcw_act(ctx, r, stream);
    // tensor cores: binned heads and the shipped configs' wide policies on rollout_tcw.cu; obs-64-64-act and everything else on
    // rollout_tc2.cu
    if (head == ES_HEAD_BINNED || es_tcw_covers(r)) return es_impl_rollout_tcw(ctx, r, mode == ES_ROLLOUT_TC3, stream);
    return es_impl_rollout_tc2(ctx, r, mode == ES_ROLLOUT_TC3, stream);
}

int es_rollout_openloop_episodes(es_ctx* ctx, const float* table, int64_t table_len, const int64_t* idx, int n_pairs,
                                 const float* theta, int P, float sigma, const int* layer_sizes, int n_layers, const float* obsn,
                                 const float* rew_vec, int T, float pos_scale, double* fit_pos, double* fit_neg, int fit_stride,
                                 float* behv_pos, float* behv_neg, const float* act_noise, int n_episodes, int mode, void* stream) {
    ES_ENTER(ctx);
    ES_REQUIRE(n_episodes >= 1, "es_rollout_openloop: n_episodes must be >= 1, got %d", n_episodes);
    // without action noise the episodes are identical and their mean is exactly the one episode (E copies of a float32 value
    // sum exactly in float64, and (E r) / E == r)
    const EsRollout r = {.table = table, .table_len = table_len, .idx = idx, .n_pairs = n_pairs, .theta = theta, .P = P,
                         .sigma = sigma, .n_layers = n_layers, .obsn = obsn, .rew_vec = rew_vec, .T = T, .pos_scale = pos_scale,
                         .fit_pos = fit_pos, .fit_neg = fit_neg, .fit_stride = fit_stride, .behv_pos = behv_pos,
                         .behv_neg = behv_neg, .act_noise = act_noise, .err = ctx->err_dev,
                         .n_episodes = act_noise ? n_episodes : 1};
    return es_openloop(ctx, "es_rollout_openloop", r, layer_sizes, ES_HEAD_TANH, mode, (cudaStream_t)stream);
}

int es_rollout_openloop_noisy(es_ctx* ctx, const float* table, int64_t table_len, const int64_t* idx, int n_pairs,
                              const float* theta, int P, float sigma, const int* layer_sizes, int n_layers, const float* obsn,
                              const float* rew_vec, int T, float pos_scale, double* fit_pos, double* fit_neg, int fit_stride,
                              float* behv_pos, float* behv_neg, const float* act_noise, int mode, void* stream) {
    return es_rollout_openloop_episodes(ctx, table, table_len, idx, n_pairs, theta, P, sigma, layer_sizes, n_layers, obsn, rew_vec, T,
                                        pos_scale, fit_pos, fit_neg, fit_stride, behv_pos, behv_neg, act_noise, 1, mode, stream);
}

int es_rollout_openloop(es_ctx* ctx, const float* table, int64_t table_len, const int64_t* idx, int n_pairs,
                        const float* theta, int P, float sigma, const int* layer_sizes, int n_layers, const float* obsn,
                        const float* rew_vec, int T, float pos_scale, double* fit_pos, double* fit_neg, int fit_stride,
                        float* behv_pos, float* behv_neg, int mode, void* stream) {
    return es_rollout_openloop_noisy(ctx, table, table_len, idx, n_pairs, theta, P, sigma, layer_sizes, n_layers, obsn, rew_vec, T,
                                     pos_scale, fit_pos, fit_neg, fit_stride, behv_pos, behv_neg, nullptr, mode, stream);
}

int es_rollout_openloop_binned(es_ctx* ctx, const float* table, int64_t table_len, const int64_t* idx, int n_pairs,
                               const float* theta, int P, float sigma, const int* layer_sizes, int n_layers, const float* obsn,
                               const float* rew_vec, int T, float pos_scale, double* fit_pos, double* fit_neg, int fit_stride,
                               float* behv_pos, float* behv_neg, int bins, const float* low, const float* range, int mode,
                               void* stream) {
    ES_ENTER(ctx);
    const EsRollout r = {.table = table, .table_len = table_len, .idx = idx, .n_pairs = n_pairs, .theta = theta, .P = P,
                         .sigma = sigma, .n_layers = n_layers, .obsn = obsn, .rew_vec = rew_vec, .T = T, .pos_scale = pos_scale,
                         .fit_pos = fit_pos, .fit_neg = fit_neg, .fit_stride = fit_stride, .behv_pos = behv_pos,
                         .behv_neg = behv_neg, .act_noise = nullptr, .err = ctx->err_dev, .n_episodes = 1, .bins = bins,
                         .head_low = low, .head_range = range};
    return es_openloop(ctx, "es_rollout_openloop_binned", r, layer_sizes, ES_HEAD_BINNED, mode, (cudaStream_t)stream);
}

int es_rollout_openloop_activation(es_ctx* ctx, const float* table, int64_t table_len, const int64_t* idx, int n_pairs,
                                   const float* theta, int P, float sigma, const int* layer_sizes, int n_layers, const float* obsn,
                                   const float* rew_vec, int T, float pos_scale, double* fit_pos, double* fit_neg, int fit_stride,
                                   float* behv_pos, float* behv_neg, const float* act_noise, int n_episodes, int activation,
                                   float act_param, int mode, void* stream) {
    ES_ENTER(ctx);
    const char* fn = "es_rollout_openloop_activation";
    const int rc = es_activation_check(fn, activation, act_param);
    if (rc) return rc;
    if (activation == ES_ACT_TANH)
        return es_rollout_openloop_episodes(ctx, table, table_len, idx, n_pairs, theta, P, sigma, layer_sizes, n_layers, obsn, rew_vec,
                                            T, pos_scale, fit_pos, fit_neg, fit_stride, behv_pos, behv_neg, act_noise, n_episodes,
                                            mode, stream);
    ES_REQUIRE(n_episodes >= 1, "%s: n_episodes must be >= 1, got %d", fn, n_episodes);
    const EsRollout r = {.table = table, .table_len = table_len, .idx = idx, .n_pairs = n_pairs, .theta = theta, .P = P,
                         .sigma = sigma, .n_layers = n_layers, .activation = activation, .obsn = obsn, .rew_vec = rew_vec, .T = T,
                         .pos_scale = pos_scale, .fit_pos = fit_pos, .fit_neg = fit_neg, .fit_stride = fit_stride,
                         .behv_pos = behv_pos, .behv_neg = behv_neg, .act_noise = act_noise, .err = ctx->err_dev,
                         .n_episodes = act_noise ? n_episodes : 1, .act_param = act_param};
    return es_openloop(ctx, fn, r, layer_sizes, ES_HEAD_ACT, mode, (cudaStream_t)stream);
}

// the shapes es_rollout_closedloop's one-CTA kernel (rollout_closed.cu) covers: two hidden layers <= 64, act <= 64, obs <= 384
static bool es_closed_one_cta_covers(const int* dims, int n_layers) {
    return n_layers == 3 && dims[1] <= 64 && dims[2] <= 64 && dims[3] <= 64 && dims[0] <= 384;
}

// a closed-loop entry point after ES_ENTER: its checks in order (the cluster plan refuses a shape whatever n_pairs is;
// rollout_closed.cu checks its own coverage when it runs), the scratch, then the kernel; `fn` names it in every message.
// `term`: es_rollout_closedloop_terminal's early end (steps NULL for the other entry points), always on the cluster kernel
static int es_closedloop(es_ctx* ctx, const char* fn, EsRollout r, const int* layer_sizes, EsClosedEnv env, EsHead head,
                         cudaStream_t stream, const EsTerm& term = EsTerm{}) {
    int rc = es_rollout_check(fn, env.ob_mean && env.ob_std && env.obs0 && env.env_a && env.env_b, layer_sizes, r);
    if (rc) return rc;
    if (head == ES_HEAD_TANH_ONE_CTA && r.n_layers != 3) {
        es_set_error("%s: two hidden layers (n_layers == 3) supported, got %d", fn, r.n_layers);
        return ES_ERR_UNSUPPORTED;
    }
    ES_REQUIRE(env.band >= 1 && env.band <= r.dims[0], "%s: band must be in [1, obs_dim]", fn);
    ES_REQUIRE((env.ob_sum == nullptr) == (env.ob_sumsq == nullptr) && (env.ob_sum == nullptr) == (env.ob_count == nullptr),
               "%s: ob_sum/ob_sumsq/ob_count must all be set or NULL", fn);
    int C = 0;
    size_t smem = 0;
    if (head == ES_HEAD_BINNED) {
        rc = es_binned_check(fn, r);
        if (!rc) rc = es_closedw_binned_plan(r.dims, r.n_layers, env.band, r.bins, &C, &smem);
    } else if (head == ES_HEAD_TANH || head == ES_HEAD_ACT) {
        rc = es_closedw_plan(r.dims, r.n_layers, env.band, &C, &smem);
    }
    if (rc) return rc;
    if (r.n_pairs == 0) return ES_OK;
    // the scratch: the cluster kernel's evaluation counter (dynamic scheduling), then the per-step rows of E > 1 episodes
    void* s = nullptr;
    rc = es_ctx_scratch(ctx, 256 + (r.n_episodes > 1 ? (size_t)2 * ctx->sm_count * r.T * sizeof(double) : 0), &s);
    if (rc) return rc;
    if (r.n_episodes > 1) env.ep_rows = (double*)((char*)s + 256);
    if (!term.steps && (head == ES_HEAD_TANH_ONE_CTA || (head == ES_HEAD_TANH && es_closed_one_cta_covers(r.dims, r.n_layers))))
        return es_impl_rollout_closed(ctx, r, env, stream);
    return es_impl_rollout_closedw(ctx, r, env, term, (unsigned*)s, stream);
}

int es_rollout_closedloop(es_ctx* ctx, const float* table, int64_t table_len, const int64_t* idx, int n_pairs, const float* theta,
                          int P, float sigma, const int* layer_sizes, int n_layers, const double* ob_mean, const double* ob_std,
                          double ob_clip, const float* obs0, const float* env_a, int band, const float* env_b, const float* rew_vec,
                          int T, float pos_scale, const uint32_t* coin_words, double save_obs_chance, double* fit_pos,
                          double* fit_neg, int fit_stride, float* behv_pos, float* behv_neg, double* ob_sum, double* ob_sumsq,
                          double* ob_count, void* stream) {
    ES_ENTER(ctx);
    const EsRollout r = {.table = table, .table_len = table_len, .idx = idx, .n_pairs = n_pairs, .theta = theta, .P = P,
                         .sigma = sigma, .n_layers = n_layers, .obsn = nullptr, .rew_vec = rew_vec, .T = T, .pos_scale = pos_scale,
                         .fit_pos = fit_pos, .fit_neg = fit_neg, .fit_stride = fit_stride, .behv_pos = behv_pos,
                         .behv_neg = behv_neg, .act_noise = nullptr, .err = ctx->err_dev, .n_episodes = 1};
    const EsClosedEnv env = {ob_mean, ob_std, ob_clip, obs0, env_a, band, env_b, coin_words, save_obs_chance, ob_sum, ob_sumsq, ob_count};
    return es_closedloop(ctx, "es_rollout_closedloop", r, layer_sizes, env, ES_HEAD_TANH_ONE_CTA, (cudaStream_t)stream);
}

// the plan entry points after ES_ENTER (`bins`: a binned head's, 0 for the others)
static int es_closedloop_plan(es_ctx* ctx, const char* fn, const int* layer_sizes, int n_layers, int band, EsHead head, int bins,
                              int* cluster_size, int* clusters, int64_t* smem_bytes) {
    ES_REQUIRE(layer_sizes && cluster_size && clusters && smem_bytes, "%s: NULL pointer", fn);
    ES_REQUIRE(n_layers >= 1 && n_layers <= ES_MAX_LAYERS, "%s: n_layers must be in [1,%d]", fn, ES_MAX_LAYERS);
    for (int l = 0; l <= n_layers; ++l) ES_REQUIRE(layer_sizes[l] > 0, "%s: layer size <= 0", fn);
    ES_REQUIRE(band >= 1 && band <= layer_sizes[0], "%s: band must be in [1, obs_dim]", fn);
    const bool binned = head == ES_HEAD_BINNED;
    ES_REQUIRE(!binned || bins >= 2, "%s: bins must be >= 2 (the action is idx / (bins - 1)), got %d", fn, bins);
    int C = 0;
    size_t smem = 0;
    const int rc = binned ? es_closedw_binned_plan(layer_sizes, n_layers, band, bins, &C, &smem)
                          : es_closedw_plan(layer_sizes, n_layers, band, &C, &smem);
    if (rc) return rc;
    if (head == ES_HEAD_TANH && es_closed_one_cta_covers(layer_sizes, n_layers)) {
        *cluster_size = 0; *clusters = ctx->sm_count; *smem_bytes = 0;
        return ES_OK;
    }
    *cluster_size = C; *smem_bytes = (int64_t)smem;
    return es_closedw_max_clusters(n_layers, bins, head == ES_HEAD_ACT, C, smem, clusters);
}

int es_rollout_closedloop_mlp_plan(es_ctx* ctx, const int* layer_sizes, int n_layers, int band, int* cluster_size, int* clusters,
                                   int64_t* smem_bytes) {
    ES_ENTER(ctx);
    return es_closedloop_plan(ctx, "es_rollout_closedloop_mlp_plan", layer_sizes, n_layers, band, ES_HEAD_TANH, 0, cluster_size,
                              clusters, smem_bytes);
}

int es_rollout_closedloop_mlp_episodes(es_ctx* ctx, const float* table, int64_t table_len, const int64_t* idx, int n_pairs,
                                       const float* theta, int P, float sigma, const int* layer_sizes, int n_layers,
                                       const double* ob_mean, const double* ob_std, double ob_clip, const float* obs0,
                                       const float* env_a, int band, const float* env_b, const float* rew_vec, int T, float pos_scale,
                                       const uint32_t* coin_words, double save_obs_chance, double* fit_pos, double* fit_neg,
                                       int fit_stride, float* behv_pos, float* behv_neg, double* ob_sum, double* ob_sumsq,
                                       double* ob_count, const float* act_noise, int n_episodes, void* stream) {
    ES_ENTER(ctx);
    ES_REQUIRE(n_episodes >= 1, "es_rollout_closedloop_mlp: n_episodes must be >= 1, got %d", n_episodes);
    // without action noise the episodes are identical: the noise-free kernels run one (as es_rollout_openloop_episodes)
    const EsRollout r = {.table = table, .table_len = table_len, .idx = idx, .n_pairs = n_pairs, .theta = theta, .P = P,
                         .sigma = sigma, .n_layers = n_layers, .obsn = nullptr, .rew_vec = rew_vec, .T = T, .pos_scale = pos_scale,
                         .fit_pos = fit_pos, .fit_neg = fit_neg, .fit_stride = fit_stride, .behv_pos = behv_pos,
                         .behv_neg = behv_neg, .act_noise = act_noise, .err = ctx->err_dev,
                         .n_episodes = act_noise ? n_episodes : 1};
    const EsClosedEnv env = {ob_mean, ob_std, ob_clip, obs0, env_a, band, env_b, coin_words, save_obs_chance, ob_sum, ob_sumsq, ob_count};
    return es_closedloop(ctx, "es_rollout_closedloop_mlp", r, layer_sizes, env, ES_HEAD_TANH, (cudaStream_t)stream);
}

int es_rollout_closedloop_mlp(es_ctx* ctx, const float* table, int64_t table_len, const int64_t* idx, int n_pairs, const float* theta,
                              int P, float sigma, const int* layer_sizes, int n_layers, const double* ob_mean, const double* ob_std,
                              double ob_clip, const float* obs0, const float* env_a, int band, const float* env_b, const float* rew_vec,
                              int T, float pos_scale, const uint32_t* coin_words, double save_obs_chance, double* fit_pos,
                              double* fit_neg, int fit_stride, float* behv_pos, float* behv_neg, double* ob_sum, double* ob_sumsq,
                              double* ob_count, void* stream) {
    return es_rollout_closedloop_mlp_episodes(ctx, table, table_len, idx, n_pairs, theta, P, sigma, layer_sizes, n_layers, ob_mean,
                                              ob_std, ob_clip, obs0, env_a, band, env_b, rew_vec, T, pos_scale, coin_words,
                                              save_obs_chance, fit_pos, fit_neg, fit_stride, behv_pos, behv_neg, ob_sum, ob_sumsq,
                                              ob_count, nullptr, 1, stream);
}

int es_rollout_closedloop_mlp_binned_plan(es_ctx* ctx, const int* layer_sizes, int n_layers, int band, int bins, int* cluster_size,
                                          int* clusters, int64_t* smem_bytes) {
    ES_ENTER(ctx);
    return es_closedloop_plan(ctx, "es_rollout_closedloop_mlp_binned_plan", layer_sizes, n_layers, band, ES_HEAD_BINNED, bins,
                              cluster_size, clusters, smem_bytes);
}

int es_rollout_closedloop_mlp_binned(es_ctx* ctx, const float* table, int64_t table_len, const int64_t* idx, int n_pairs,
                                     const float* theta, int P, float sigma, const int* layer_sizes, int n_layers, const double* ob_mean,
                                     const double* ob_std, double ob_clip, const float* obs0, const float* env_a, int band,
                                     const float* env_b, const float* rew_vec, int T, float pos_scale, const uint32_t* coin_words,
                                     double save_obs_chance, double* fit_pos, double* fit_neg, int fit_stride, float* behv_pos,
                                     float* behv_neg, double* ob_sum, double* ob_sumsq, double* ob_count, int bins, const float* low,
                                     const float* range, void* stream) {
    ES_ENTER(ctx);
    const EsRollout r = {.table = table, .table_len = table_len, .idx = idx, .n_pairs = n_pairs, .theta = theta, .P = P,
                         .sigma = sigma, .n_layers = n_layers, .obsn = nullptr, .rew_vec = rew_vec, .T = T, .pos_scale = pos_scale,
                         .fit_pos = fit_pos, .fit_neg = fit_neg, .fit_stride = fit_stride, .behv_pos = behv_pos,
                         .behv_neg = behv_neg, .act_noise = nullptr, .err = ctx->err_dev, .n_episodes = 1, .bins = bins,
                         .head_low = low, .head_range = range};
    const EsClosedEnv env = {ob_mean, ob_std, ob_clip, obs0, env_a, band, env_b, coin_words, save_obs_chance, ob_sum, ob_sumsq, ob_count};
    return es_closedloop(ctx, "es_rollout_closedloop_mlp_binned", r, layer_sizes, env, ES_HEAD_BINNED, (cudaStream_t)stream);
}

int es_rollout_closedloop_mlp_activation(es_ctx* ctx, const float* table, int64_t table_len, const int64_t* idx, int n_pairs,
                                         const float* theta, int P, float sigma, const int* layer_sizes, int n_layers,
                                         const double* ob_mean, const double* ob_std, double ob_clip, const float* obs0,
                                         const float* env_a, int band, const float* env_b, const float* rew_vec, int T,
                                         float pos_scale, const uint32_t* coin_words, double save_obs_chance, double* fit_pos,
                                         double* fit_neg, int fit_stride, float* behv_pos, float* behv_neg, double* ob_sum,
                                         double* ob_sumsq, double* ob_count, const float* act_noise, int n_episodes, int activation,
                                         float act_param, void* stream) {
    ES_ENTER(ctx);
    const char* fn = "es_rollout_closedloop_mlp_activation";
    const int rc = es_activation_check(fn, activation, act_param);
    if (rc) return rc;
    if (activation == ES_ACT_TANH)
        return es_rollout_closedloop_mlp_episodes(ctx, table, table_len, idx, n_pairs, theta, P, sigma, layer_sizes, n_layers, ob_mean,
                                                  ob_std, ob_clip, obs0, env_a, band, env_b, rew_vec, T, pos_scale, coin_words,
                                                  save_obs_chance, fit_pos, fit_neg, fit_stride, behv_pos, behv_neg, ob_sum, ob_sumsq,
                                                  ob_count, act_noise, n_episodes, stream);
    ES_REQUIRE(n_episodes >= 1, "%s: n_episodes must be >= 1, got %d", fn, n_episodes);
    const EsRollout r = {.table = table, .table_len = table_len, .idx = idx, .n_pairs = n_pairs, .theta = theta, .P = P,
                         .sigma = sigma, .n_layers = n_layers, .activation = activation, .obsn = nullptr, .rew_vec = rew_vec,
                         .T = T, .pos_scale = pos_scale, .fit_pos = fit_pos, .fit_neg = fit_neg, .fit_stride = fit_stride,
                         .behv_pos = behv_pos, .behv_neg = behv_neg, .act_noise = act_noise, .err = ctx->err_dev,
                         .n_episodes = act_noise ? n_episodes : 1, .act_param = act_param};
    const EsClosedEnv env = {ob_mean, ob_std, ob_clip, obs0, env_a, band, env_b, coin_words, save_obs_chance, ob_sum, ob_sumsq, ob_count};
    return es_closedloop(ctx, fn, r, layer_sizes, env, ES_HEAD_ACT, (cudaStream_t)stream);
}

int es_rollout_closedloop_terminal(es_ctx* ctx, const float* table, int64_t table_len, const int64_t* idx, int n_pairs,
                                   const float* theta, int P, float sigma, const int* layer_sizes, int n_layers, const double* ob_mean,
                                   const double* ob_std, double ob_clip, const float* obs0, const float* env_a, int band,
                                   const float* env_b, const float* rew_vec, int T, float pos_scale, const uint32_t* coin_words,
                                   double save_obs_chance, double* fit_pos, double* fit_neg, int fit_stride, float* behv_pos,
                                   float* behv_neg, double* ob_sum, double* ob_sumsq, double* ob_count, int bins, const float* low,
                                   const float* range, int activation, float act_param, const float* act_noise, int n_episodes,
                                   float fall_height, int32_t* steps, int64_t* noise_used, void* stream) {
    ES_ENTER(ctx);
    const char* fn = "es_rollout_closedloop_terminal";
    ES_REQUIRE(isfinite(fall_height) && fall_height > 0.f, "%s: fall_height must be finite and > 0, got %g", fn, (double)fall_height);
    ES_REQUIRE(steps != nullptr, "%s: NULL steps", fn);
    ES_REQUIRE(n_episodes >= 1, "%s: n_episodes must be >= 1, got %d", fn, n_episodes);
    int rc = es_activation_check(fn, activation, act_param);
    if (rc) return rc;
    ES_REQUIRE(bins == 0 || (activation == ES_ACT_TANH && act_noise == nullptr),
               "%s: a binned head is a tanh stack that draws no action noise (FFBinned.forward ignores rs)", fn);
    // without action noise the episodes are identical: one runs (as es_rollout_closedloop_mlp_episodes)
    const EsRollout r = {.table = table, .table_len = table_len, .idx = idx, .n_pairs = n_pairs, .theta = theta, .P = P,
                         .sigma = sigma, .n_layers = n_layers, .activation = activation, .obsn = nullptr, .rew_vec = rew_vec,
                         .T = T, .pos_scale = pos_scale, .fit_pos = fit_pos, .fit_neg = fit_neg, .fit_stride = fit_stride,
                         .behv_pos = behv_pos, .behv_neg = behv_neg, .act_noise = act_noise, .err = ctx->err_dev,
                         .n_episodes = act_noise ? n_episodes : 1, .bins = bins, .head_low = low, .head_range = range,
                         .act_param = act_param};
    const EsClosedEnv env = {ob_mean, ob_std, ob_clip, obs0, env_a, band, env_b, coin_words, save_obs_chance, ob_sum, ob_sumsq, ob_count};
    const EsTerm term = {fall_height, steps, noise_used};
    return es_closedloop(ctx, fn, r, layer_sizes, env, bins ? ES_HEAD_BINNED : activation == ES_ACT_TANH ? ES_HEAD_TANH : ES_HEAD_ACT,
                         (cudaStream_t)stream, term);
}

int es_rollout_closedloop_terminal_streams(es_ctx* ctx, uint32_t* mt_key, int32_t* mt_pos, int32_t* has_gauss, double* gauss,
                                           int n_streams, int n_per_stream, uint64_t upper_bound, int coins_per_eval, double ac_std,
                                           const float* table, int64_t table_len, const float* theta, int P, float sigma,
                                           const int* layer_sizes, int n_layers, const double* ob_mean, const double* ob_std,
                                           double ob_clip, const float* obs0, const float* env_a, int band, const float* env_b,
                                           const float* rew_vec, int T, float pos_scale, double save_obs_chance, int64_t* idx_out,
                                           uint32_t* coin_out, double* fit_pos, double* fit_neg, int fit_stride, float* behv_pos,
                                           float* behv_neg, double* ob_sum, double* ob_sumsq, double* ob_count, int bins,
                                           int activation, float act_param, int n_episodes, float fall_height, int32_t* steps,
                                           int64_t* noise_used, float* noise_trace, void* stream) {
    ES_ENTER(ctx);
    const char* fn = "es_rollout_closedloop_terminal_streams";
    ES_REQUIRE(mt_key && mt_pos && has_gauss && gauss && idx_out, "%s: NULL stream state or idx_out", fn);
    ES_REQUIRE(n_streams >= 0 && n_per_stream >= 0, "%s: negative count", fn);
    ES_REQUIRE((long long)n_streams * n_per_stream <= 0x3FFFFFFFLL, "%s: %d streams x %d pairs exceed 2^30 pairs", fn, n_streams,
               n_per_stream);
    if (bins != 0) {
        es_set_error("%s: a binned head draws no action noise (FFBinned.forward ignores rs): use es_rollout_closedloop_terminal", fn);
        return ES_ERR_UNSUPPORTED;
    }
    if (coins_per_eval < 0 || coins_per_eval > 1) {
        es_set_error("%s: fit_fns draw at most one save_obs coin per evaluation, got coins_per_eval %d", fn, coins_per_eval);
        return ES_ERR_UNSUPPORTED;
    }
    ES_REQUIRE(coins_per_eval == 0 || coin_out, "%s: coin_out is NULL", fn);
    ES_REQUIRE(isfinite(ac_std) && ac_std != 0.0, "%s: ac_std must be finite and != 0 (without action noise use "
               "es_rollout_closedloop_terminal), got %g", fn, ac_std);
    ES_REQUIRE(isfinite(fall_height) && fall_height > 0.f, "%s: fall_height must be finite and > 0, got %g", fn, (double)fall_height);
    ES_REQUIRE(steps != nullptr, "%s: NULL steps", fn);
    ES_REQUIRE(n_episodes >= 1, "%s: n_episodes must be >= 1, got %d", fn, n_episodes);
    int rc = es_activation_check(fn, activation, act_param);
    if (rc) return rc;
    rc = es_randint_check(fn, upper_bound);
    if (rc) return rc;
    if (upper_bound == 1) {
        es_set_error("%s: upper_bound == 1 is not supported", fn);
        return ES_ERR_UNSUPPORTED;
    }
    const int n_pairs = n_streams * n_per_stream;
    EsRollout r = {.table = table, .table_len = table_len, .idx = idx_out, .n_pairs = n_pairs, .theta = theta, .P = P,
                         .sigma = sigma, .n_layers = n_layers, .activation = activation, .obsn = nullptr, .rew_vec = rew_vec,
                         .T = T, .pos_scale = pos_scale, .fit_pos = fit_pos, .fit_neg = fit_neg, .fit_stride = fit_stride,
                         .behv_pos = behv_pos, .behv_neg = behv_neg, .act_noise = nullptr, .err = ctx->err_dev,
                         .n_episodes = n_episodes, .act_param = act_param};
    rc = es_rollout_check(fn, ob_mean && ob_std && obs0 && env_a && env_b, layer_sizes, r);
    if (rc) return rc;
    ES_REQUIRE(band >= 1 && band <= r.dims[0], "%s: band must be in [1, obs_dim]", fn);
    ES_REQUIRE((ob_sum == nullptr) == (ob_sumsq == nullptr) && (ob_sum == nullptr) == (ob_count == nullptr),
               "%s: ob_sum/ob_sumsq/ob_count must all be set or NULL", fn);
    const EsClosedEnv env = {ob_mean, ob_std, ob_clip, obs0, env_a, band, env_b, nullptr, save_obs_chance, ob_sum, ob_sumsq, ob_count};
    const EsTerm term = {fall_height, steps, noise_used};
    const EsStreamWalk walk = {mt_key, mt_pos, has_gauss, gauss, n_streams, n_per_stream, upper_bound, coins_per_eval, ac_std,
                               idx_out, coin_out, noise_trace};
    if (n_pairs == 0) {
        // (the plan still refuses a shape it does not cover)
        int C = 0;
        size_t smem = 0;
        return es_closedw_plan(r.dims, r.n_layers, band, &C, &smem);
    }
    return es_impl_rollout_closedw_walk(ctx, r, env, term, walk, (cudaStream_t)stream);
}

int es_rollout_closedloop_mlp_activation_plan(es_ctx* ctx, const int* layer_sizes, int n_layers, int band, int activation,
                                              int* cluster_size, int* clusters, int64_t* smem_bytes) {
    ES_ENTER(ctx);
    const char* fn = "es_rollout_closedloop_mlp_activation_plan";
    const int rc = es_activation_check(fn, activation, 0.f);
    if (rc) return rc;
    return es_closedloop_plan(ctx, fn, layer_sizes, n_layers, band, activation == ES_ACT_TANH ? ES_HEAD_TANH : ES_HEAD_ACT, 0,
                              cluster_size, clusters, smem_bytes);
}

int es_draw_noisy(es_ctx* ctx, uint32_t* mt_key, int32_t* mt_pos, int32_t* has_gauss, double* gauss, int n_streams,
                  int n_per_stream, uint64_t upper_bound, int coins_per_eval, int normals_per_eval, double scale,
                  int64_t* idx_out, uint32_t* coin_out, float* noise_out, void* stream) {
    ES_ENTER(ctx);
    ES_REQUIRE(mt_key && mt_pos && has_gauss && gauss && idx_out && noise_out, "es_draw_noisy: NULL pointer");
    ES_REQUIRE(n_streams >= 0 && n_per_stream >= 0 && normals_per_eval >= 0, "es_draw_noisy: negative count");
    ES_REQUIRE(coins_per_eval >= 0 && coins_per_eval <= 8, "es_draw_noisy: coins_per_eval must be in [0,8]");
    ES_REQUIRE(coins_per_eval == 0 || coin_out, "es_draw_noisy: coin_out is NULL");
    const int rc = es_randint_check("es_draw_noisy", upper_bound);
    if (rc) return rc;
    if (n_streams == 0 || n_per_stream == 0) return ES_OK;
    return es_impl_draw_noisy(ctx, mt_key, mt_pos, has_gauss, gauss, n_streams, n_per_stream, upper_bound, coins_per_eval,
                              normals_per_eval, scale, idx_out, coin_out, noise_out, (cudaStream_t)stream);
}

int es_randn(es_ctx* ctx, uint32_t* mt_key, int32_t* mt_pos, int32_t* has_gauss, double* gauss, int64_t n, float* out,
             void* stream) {
    ES_ENTER(ctx);
    ES_REQUIRE(n >= 0, "es_randn: negative count");
    ES_REQUIRE(mt_key && mt_pos && has_gauss && gauss && (out || n == 0), "es_randn: NULL pointer");
    if (n == 0) return ES_OK;
    return es_impl_randn(ctx, mt_key, mt_pos, has_gauss, gauss, n, out, (cudaStream_t)stream);
}

int es_randn_plan(es_ctx* ctx, int64_t n, size_t* scratch_bytes, int* n_windows) {
    ES_REQUIRE(ctx && scratch_bytes && n_windows, "es_randn_plan: NULL pointer");
    ES_REQUIRE(n >= 0, "es_randn_plan: negative count");
    if (n == 0) { *scratch_bytes = 0; *n_windows = 0; return ES_OK; }
    return es_impl_randn_plan(ctx, n, scratch_bytes, n_windows);
}

int es_novelty(es_ctx* ctx, const float* behv, int n, const double* archive, int A, int k, double* out, int out_stride,
               void* stream) {
    ES_ENTER(ctx);
    ES_REQUIRE(behv && archive && out, "es_novelty: NULL pointer");
    ES_REQUIRE(n >= 0 && A >= 1 && k >= 1 && out_stride >= 1, "es_novelty: bad sizes");
    ES_REQUIRE((k < A ? k : A) <= 64, "es_novelty: min(k, archive size) > 64 not supported");
    if (n == 0) return ES_OK;
    return es_impl_novelty(ctx, behv, n, archive, A, k, out, out_stride, (cudaStream_t)stream);
}

int es_fitness_objective(es_ctx* ctx, int kind, double* fit, int fit_stride, const float* behv, int n, int steps,
                         void* stream) {
    ES_ENTER(ctx);
    ES_REQUIRE(kind == ES_OBJ_MEAN_REWARD || kind == ES_OBJ_DIST || kind == ES_OBJ_XDIST,
               "es_fitness_objective: unknown kind %d", kind);
    ES_REQUIRE(n >= 0 && fit_stride >= 1, "es_fitness_objective: bad sizes");
    ES_REQUIRE(kind != ES_OBJ_MEAN_REWARD || steps > 0,
               "es_fitness_objective: the mean reward of an episode with steps = %d (MeanRewardResult divides by zero)", steps);
    if (n == 0) return ES_OK;
    ES_REQUIRE(fit && (kind == ES_OBJ_MEAN_REWARD || behv), "es_fitness_objective: NULL pointer");
    return es_impl_fitness_objective(ctx, kind, fit, fit_stride, behv, n, steps, (cudaStream_t)stream);
}

int es_fitness_objective_steps(es_ctx* ctx, int kind, double* fit, int fit_stride, const float* behv, int n, const int32_t* steps,
                               void* stream) {
    ES_ENTER(ctx);
    if (kind != ES_OBJ_MEAN_REWARD) return es_fitness_objective(ctx, kind, fit, fit_stride, behv, n, 1, stream);
    ES_REQUIRE(n >= 0 && fit_stride >= 1, "es_fitness_objective_steps: bad sizes");
    if (n == 0) return ES_OK;
    ES_REQUIRE(fit && steps, "es_fitness_objective_steps: NULL pointer");
    return es_impl_mean_reward_steps(ctx, fit, fit_stride, steps, n, (cudaStream_t)stream);
}

int es_centered_rank(es_ctx* ctx, const double* fpos, const double* fneg, int K, int n_obj, float w0, float w1,
                     int k_begin, int k_count, float* weights_out, int32_t* ranks_out, void* stream) {
    ES_ENTER(ctx);
    ES_REQUIRE(fpos && fneg && weights_out, "es_centered_rank: NULL pointer");
    // MultiObjectiveRanker asserts exactly two columns (rankers.py:114)
    ES_REQUIRE(n_obj == 1 || n_obj == 2, "es_centered_rank: n_obj must be 1 or 2");
    ES_REQUIRE(K >= 1 && k_begin >= 0 && k_count >= 0 && k_begin + k_count <= K, "es_centered_rank: bad shard");
    if (k_count == 0) return ES_OK;
    return es_impl_rank_transform(ctx, fpos, fneg, K, n_obj, ES_RANK_CENTERED, (double)w0, (double)w1, 0, k_begin, k_count,
                                  nullptr, weights_out, nullptr, ranks_out, nullptr, nullptr, nullptr,
                                  (cudaStream_t)stream);
}

int es_rank_transform(es_ctx* ctx, const double* fpos, const double* fneg, int K, int n_obj, int kind, double w0,
                      double w1, int elite_n, int k_begin, int k_count, const int64_t* noise_idx, float* weights_out,
                      double* weights64_out, int32_t* ranks_out, double* elite_vals_out, int32_t* elite_fit_out,
                      int64_t* elite_idx_out, void* stream) {
    ES_ENTER(ctx);
    ES_REQUIRE(fpos && fneg && weights_out, "es_rank_transform: NULL pointer");
    ES_REQUIRE(kind >= ES_RANK_CENTERED && kind <= ES_RANK_MAX_NORMALIZED, "es_rank_transform: unknown kind");
    ES_REQUIRE(n_obj == 1 || n_obj == 2, "es_rank_transform: n_obj must be 1 or 2");   // rankers.py:114
    ES_REQUIRE(K >= 1 && k_begin >= 0 && k_count >= 0 && k_begin + k_count <= K, "es_rank_transform: bad shard");
    ES_REQUIRE(elite_n >= 0 && elite_n <= 2 * K, "es_rank_transform: elite_n out of range");
    if (elite_n > 0) {
        // EliteRanker(MultiObjectiveRanker) would need a second ranking of the blended values: not provided
        if (n_obj != 1) { es_set_error("es_rank_transform: elite selection needs a single objective"); return ES_ERR_UNSUPPORTED; }
        ES_REQUIRE(!elite_idx_out || noise_idx, "es_rank_transform: elite_idx_out needs noise_idx");
    }
    if (k_count == 0) return ES_OK;
    return es_impl_rank_transform(ctx, fpos, fneg, K, n_obj, kind, w0, w1, elite_n, k_begin, k_count, noise_idx,
                                  weights_out, weights64_out, ranks_out, elite_vals_out, elite_fit_out, elite_idx_out,
                                  (cudaStream_t)stream);
}

int es_grad_reconstruct(es_ctx* ctx, const float* table, int64_t table_len, const int64_t* idx, const float* weights,
                        int n_idx, int P, float* out, void* stream) {
    ES_ENTER(ctx);
    ES_REQUIRE(table && out, "es_grad_reconstruct: NULL pointer");
    ES_REQUIRE(n_idx >= 0 && P > 0 && table_len > P, "es_grad_reconstruct: bad sizes");
    ES_REQUIRE(n_idx == 0 || (idx && weights), "es_grad_reconstruct: NULL idx/weights");
    if (n_idx == 0) {
        ES_CHECK_CUDA(cudaMemsetAsync(out, 0, (size_t)P * sizeof(float), (cudaStream_t)stream));
        return ES_OK;
    }
    return es_impl_grad_reconstruct(ctx, table, table_len, idx, weights, n_idx, P, out, (cudaStream_t)stream);
}

int es_adam_step(es_ctx* ctx, float* theta, float* m, float* v, const float* gsum, float n_ranked, float l2coeff,
                 float neg_a, float beta1, float one_minus_beta1, float beta2, float one_minus_beta2, float epsilon,
                 int P, void* stream) {
    ES_ENTER(ctx);
    ES_REQUIRE(theta && m && v && gsum && P > 0, "es_adam_step: bad arguments");
    return es_impl_adam(ctx, theta, m, v, gsum, n_ranked, l2coeff, neg_a, beta1, one_minus_beta1, beta2,
                        one_minus_beta2, epsilon, P, (cudaStream_t)stream);
}

int es_sgd_step(es_ctx* ctx, float* theta, float* v, const float* gsum, float n_ranked, float l2coeff, float neg_lr,
                float momentum, float one_minus_momentum, int P, void* stream) {
    ES_ENTER(ctx);
    ES_REQUIRE(theta && v && gsum && P > 0, "es_sgd_step: bad arguments");
    return es_impl_sgd(ctx, theta, v, gsum, n_ranked, l2coeff, neg_lr, momentum, one_minus_momentum, P,
                       (cudaStream_t)stream);
}

int es_simple_step(es_ctx* ctx, float* theta, const float* gsum, float n_ranked, float l2coeff, float lr, int P,
                   void* stream) {
    ES_ENTER(ctx);
    ES_REQUIRE(theta && gsum && P > 0, "es_simple_step: bad arguments");
    return es_impl_simple(ctx, theta, gsum, n_ranked, l2coeff, lr, P, (cudaStream_t)stream);
}

}  // extern "C"
