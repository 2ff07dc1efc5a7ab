// mt_draw.cu -- draw the K noise indices on the device, bit-exact with numpy's legacy
// RandomState.randint(0, upper_bound) (reference: NoiseTable.sample_idx,
// src/core/noisetable.py:37-40, called once per antithetic pair from es.py:67-68).
//
// numpy 1.18 legacy path for ranges < 2^32 (numpy/random/src/distributions,
// buffered_bounded_masked_uint32): mask = next_pow2(rng)-1 with rng = upper_bound-1;
// repeat v = mt19937_next32() & mask until v <= rng.  After each accepted index the
// stream optionally consumes `extra` further 32-bit outputs (the rs.random() save_obs
// coins drawn by the fit_fn of simple_example.py:38, two words per double).
//
// One CTA of MT_THREADS threads per virtual-rank stream.  Per 624-word block the CTA (a) regenerates the MT state in
// three dependency-free phases, (b) tempers all words in parallel, (c) runs the accept/skip state machine as a parallel
// scan: every thread composes the transition function of its contiguous chunk for all `extra`+1 entry states (packed in
// registers), a shuffle scan composes them inside each warp and the warp totals are chained through shared memory, and
// each thread then replays its chunk from its true entry state and writes indices/extras at its true output offset.
#include "common.cuh"
#include "mt19937.cuh"

constexpr int MT_MAXS = 8;  // machine states: 0 = seeking an index, j>0 = j extra words still to consume
constexpr int MT_THREADS = 128, MT_WARPS = MT_THREADS / 32;

// transition function of a run of words: entry state s -> (exit state, indices emitted), packed in registers:
// st = 3 bits per entry state, cn = 16 bits per entry state (lo: states 0-3, hi: states 4-7)
struct MtFn {
    uint32_t st;
    unsigned long long lo, hi;
};
__device__ __forceinline__ uint32_t mtfn_st(const MtFn& f, int s) { return (f.st >> (3 * s)) & 7u; }
__device__ __forceinline__ uint32_t mtfn_cn(const MtFn& f, int s) {
    return (uint32_t)(((s & 4) ? f.hi : f.lo) >> (16 * (s & 3))) & 0xFFFFu;
}
__device__ __forceinline__ MtFn mtfn_identity() {
    MtFn r;
    r.st = 0; r.lo = 0; r.hi = 0;
#pragma unroll
    for (int s = 0; s < MT_MAXS; ++s) r.st |= (uint32_t)s << (3 * s);
    return r;
}
// run `a` first, then `b`
__device__ __forceinline__ MtFn mtfn_compose(const MtFn& a, const MtFn& b, int S) {
    MtFn r;
    r.lo = a.lo; r.hi = a.hi;
    uint32_t st = 0;
#pragma unroll
    for (int s = 0; s < MT_MAXS; ++s) {
        if (s < S) {
            const int mid = (int)mtfn_st(a, s);
            st |= mtfn_st(b, mid) << (3 * s);
            const unsigned long long add = (unsigned long long)mtfn_cn(b, mid) << (16 * (s & 3));
            if (s & 4) r.hi += add; else r.lo += add;
        } else {
            st |= (uint32_t)s << (3 * s);
        }
    }
    r.st = st;
    return r;
}
__device__ __forceinline__ MtFn mtfn_shfl_up(const MtFn& f, int d) {
    MtFn r;
    r.st = __shfl_up_sync(0xffffffffu, f.st, d);
    r.lo = __shfl_up_sync(0xffffffffu, f.lo, d);
    r.hi = __shfl_up_sync(0xffffffffu, f.hi, d);
    return r;
}


// next 624-word block of the MT19937 state, by all MT_THREADS threads of the CTA (three dependency-free phases):
// new[i] = x[i+397] ^ twist(old[i], old[i+1]); x is old for i < 227, new after
__device__ __forceinline__ void mt_regenerate(uint32_t* mt, int tid) {
    constexpr int D = MT_DW;
    uint32_t y[(D + MT_THREADS - 1) / MT_THREADS];
    // phase A: i in [0,227)
    for (int c = 0, i = tid; i < D; i += MT_THREADS, ++c) y[c] = mt[i + MT_MW] ^ mt19937_twist(mt[i], mt[i + 1]);
    __syncthreads();
    for (int c = 0, i = tid; i < D; i += MT_THREADS, ++c) mt[i] = y[c];
    __syncthreads();
    // phase B: i in [227,454) uses new[i-227], old[i], old[i+1]
    for (int c = 0, i = D + tid; i < 2 * D; i += MT_THREADS, ++c) y[c] = mt[i - D] ^ mt19937_twist(mt[i], mt[i + 1]);
    __syncthreads();
    for (int c = 0, i = D + tid; i < 2 * D; i += MT_THREADS, ++c) mt[i] = y[c];
    __syncthreads();
    // phase C: i in [454,623) uses new[i-227] (phase B), old[i], old[i+1]
    for (int c = 0, i = 2 * D + tid; i < MT_NW - 1; i += MT_THREADS, ++c) y[c] = mt[i - D] ^ mt19937_twist(mt[i], mt[i + 1]);
    __syncthreads();
    for (int c = 0, i = 2 * D + tid; i < MT_NW - 1; i += MT_THREADS, ++c) mt[i] = y[c];
    __syncthreads();
    if (tid == 0) mt[MT_NW - 1] = mt[MT_MW - 1] ^ mt19937_twist(mt[MT_NW - 1], mt[0]);
    __syncthreads();
}

// Consume `n_words` 32-bit outputs of every stream without using them (the rs.random() coin a fit_fn draws in an
// evaluation whose other effects are computed elsewhere: the noiseless evaluation of es.py:48 still calls the script's
// fit_fn, which draws its save_obs coin first, simple_example.py:38 / obj.py:54).
__global__ void __launch_bounds__(MT_THREADS) mt_skip_kernel(uint32_t* __restrict__ mt_key, int32_t* __restrict__ mt_pos,
                                                             int n_words) {
    __shared__ uint32_t mt[MT_NW];
    const int tid = threadIdx.x;
    uint32_t* key = mt_key + (size_t)blockIdx.x * MT_NW;
    int pos = mt_pos[blockIdx.x];
    if (pos + n_words <= MT_NW) {                       // common case: no regeneration, the key is untouched
        if (tid == 0) mt_pos[blockIdx.x] = pos + n_words;
        return;
    }
    for (int i = tid; i < MT_NW; i += MT_THREADS) mt[i] = key[i];
    __syncthreads();
    int left = n_words;
    while (left > 0) {
        if (pos >= MT_NW) { mt_regenerate(mt, tid); pos = 0; }
        const int take = min(left, MT_NW - pos);
        pos += take; left -= take;
    }
    for (int i = tid; i < MT_NW; i += MT_THREADS) key[i] = mt[i];
    if (tid == 0) mt_pos[blockIdx.x] = pos;
}

// ST > 0: number of machine states (extra + 1) known at compile time (the compositions unroll over ST states only)
template <int ST>
__global__ void __launch_bounds__(MT_THREADS)
mt_draw_kernel(uint32_t* __restrict__ mt_key, int32_t* __restrict__ mt_pos, int n_per_stream, uint32_t rng,
               uint32_t mask, int extra, int64_t* __restrict__ idx_out, uint32_t* __restrict__ extra_out) {
    __shared__ uint32_t mt[MT_NW];
    __shared__ uint32_t tw[MT_NW];
    __shared__ MtFn s_warp[MT_WARPS];          // inclusive function of each warp, then of everything before it
    __shared__ MtFn s_block;
    __shared__ int s_stop[MT_WARPS];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int stream_id = blockIdx.x;
    uint32_t* key = mt_key + (size_t)stream_id * MT_NW;
    int64_t* out = idx_out + (size_t)stream_id * n_per_stream;
    uint32_t* xout = extra_out ? extra_out + (size_t)stream_id * n_per_stream * extra : nullptr;
    const int S = ST > 0 ? ST : extra + 1;

    for (int i = tid; i < MT_NW; i += MT_THREADS) mt[i] = key[i];
    int pos = mt_pos[stream_id];
    __syncthreads();

    int produced = 0;  // indices emitted so far
    int state = 0;     // machine state at `pos`
    while (produced < n_per_stream || state > 0) {
        if (pos >= MT_NW) {
            mt_regenerate(mt, tid);
            pos = 0;
        }
        // temper the available words
        for (int i = pos + tid; i < MT_NW; i += MT_THREADS) tw[i] = mt19937_temper(mt[i]);
        __syncthreads();

        const int avail = MT_NW - pos;
        const int C = (avail + MT_THREADS - 1) / MT_THREADS;  // words per thread (<= 5)
        const int b = pos + tid * C;
        const int e = min(MT_NW, b + C);
        const int len = max(0, e - b);

        // accept bits of this thread's chunk, in a register: bit i <=> word b+i passes the masked rejection test
        uint32_t am = 0;
        for (int i = 0; i < len; ++i) am |= (uint32_t)((tw[b + i] & mask) <= rng) << i;

        // (1) this thread's transition function, from the bit mask alone: skip s words, then repeatedly jump to the
        //     next accept bit and skip `extra` words after it
        MtFn f;
        f.st = 0; f.lo = 0; f.hi = 0;
#pragma unroll
        for (int s = 0; s < MT_MAXS; ++s) {
            int cur = s, cn = 0, st = 0;
            if (s < S) {
                while (cur < len) {
                    const uint32_t m = am >> cur;
                    if (m == 0) { cur = len; break; }
                    cur += __ffs(m) + extra;          // accepted word at cur + ffs - 1, then `extra` words to skip
                    ++cn;
                }
                st = cur - len;                       // words still to skip in the next chunk (0 = seeking)
            } else {
                st = s;
            }
            f.st |= (uint32_t)st << (3 * s);
            if (s & 4) f.hi |= (unsigned long long)cn << (16 * (s & 3)); else f.lo |= (unsigned long long)cn << (16 * (s & 3));
        }
        // (2) inclusive scan of function composition (earlier threads first): shuffles inside a warp ...
        MtFn inc = f;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const MtFn prev = mtfn_shfl_up(inc, d);
            if (lane >= d) inc = mtfn_compose(prev, inc, S);
        }
        if (lane == 31) s_warp[warp] = inc;
        __syncthreads();
        // ... then the (few) warp totals in order: thread 0 leaves the function of everything before each warp, and of the
        // whole block
        if (tid == 0) {
            MtFn run = mtfn_identity();
            for (int w = 0; w < MT_WARPS; ++w) {
                const MtFn tot = s_warp[w];
                s_warp[w] = run;
                run = mtfn_compose(run, tot, S);
            }
            s_block = run;
        }
        __syncthreads();
        const MtFn before = s_warp[warp], blk = s_block;
        // (3) entry state / offset of this thread = exclusive prefix applied to the block entry state
        MtFn exc = mtfn_shfl_up(inc, 1);
        exc = (lane == 0) ? before : mtfn_compose(before, exc, S);
        int st = state, base = produced;
        if (tid > 0) {
            st = (int)mtfn_st(exc, state);
            base = produced + (int)mtfn_cn(exc, state);
        }
        const int blk_state = (int)mtfn_st(blk, state);
        const int blk_count = (int)mtfn_cn(blk, state);
        // (4) replay with the mask; stop where the machine is seeking and everything requested is out
        int stop = MT_NW;  // first unconsumed position if the stream ends inside this thread's chunk
        {
            int cur = 0;
            // leading extra words of the previous thread's last draw
            while (st > 0 && cur < len) {
                if (xout && base - 1 < n_per_stream) xout[(size_t)(base - 1) * extra + (extra - st)] = tw[b + cur];
                --st; ++cur;
            }
            while (cur < len) {                       // st == 0 here
                if (base >= n_per_stream) { stop = b + cur; break; }
                const uint32_t m = am >> cur;
                if (m == 0) { cur = len; break; }
                cur += __ffs(m) - 1;                  // position of the accepted word
                out[base] = (int64_t)(tw[b + cur] & mask);
                ++base; ++cur;
                st = extra;
                while (st > 0 && cur < len) {
                    if (xout && base - 1 < n_per_stream) xout[(size_t)(base - 1) * extra + (extra - st)] = tw[b + cur];
                    --st; ++cur;
                }
            }
        }
        // a thread whose chunk starts after the end also reports its start
        if (b < e && stop == MT_NW && st == 0 && base >= n_per_stream) stop = e;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) stop = min(stop, __shfl_xor_sync(0xffffffffu, stop, o));
        if (lane == 0) s_stop[warp] = stop;
        __syncthreads();
        stop = s_stop[0];
#pragma unroll
        for (int w = 1; w < MT_WARPS; ++w) stop = min(stop, s_stop[w]);

        if (produced + blk_count >= n_per_stream && stop < MT_NW) {
            // the stream finished inside this block at `stop` (state 0 there)
            pos = stop;
            produced = n_per_stream;
            state = 0;
        } else if (produced + blk_count >= n_per_stream && blk_state == 0) {
            pos = MT_NW;  // finished exactly at the block end
            produced = n_per_stream;
            state = 0;
        } else {
            pos = MT_NW;
            produced += blk_count;
            state = blk_state;
        }
        __syncthreads();
    }

    for (int i = tid; i < MT_NW; i += MT_THREADS) key[i] = mt[i];
    if (tid == 0) mt_pos[stream_id] = pos;
}

int es_impl_draw_indices(es_ctx* ctx, uint32_t* mt_key, int32_t* mt_pos, int n_streams, int n_per_stream,
                         uint64_t upper_bound, int extra_words, int64_t* idx_out, uint32_t* extra_out,
                         cudaStream_t stream) {
    const Mt19937Bound bd = mt19937_randint_bound(upper_bound);
    const uint32_t rng = bd.rng, mask = bd.mask;
    if (rng == 0) {
        // numpy returns `low` without consuming any random word when the range is empty
        ES_CHECK_CUDA(cudaMemsetAsync(idx_out, 0, sizeof(int64_t) * (size_t)n_streams * n_per_stream, stream));
        if (extra_words == 0) return ES_OK;
        es_set_error("es_draw_indices: upper_bound == 1 with extra_words > 0 is not supported");
        return ES_ERR_UNSUPPORTED;
    }
    if (extra_words == 0)
        mt_draw_kernel<1><<<n_streams, MT_THREADS, 0, stream>>>(mt_key, mt_pos, n_per_stream, rng, mask, extra_words, idx_out, extra_out);
    else if (extra_words == 4)
        mt_draw_kernel<5><<<n_streams, MT_THREADS, 0, stream>>>(mt_key, mt_pos, n_per_stream, rng, mask, extra_words, idx_out, extra_out);
    else
        mt_draw_kernel<0><<<n_streams, MT_THREADS, 0, stream>>>(mt_key, mt_pos, n_per_stream, rng, mask, extra_words, idx_out, extra_out);
    ES_LAUNCHED(ctx);
    return ES_OK;
}

int es_impl_mt_skip(es_ctx* ctx, uint32_t* mt_key, int32_t* mt_pos, int n_streams, int n_words, cudaStream_t stream) {
    mt_skip_kernel<<<n_streams, MT_THREADS, 0, stream>>>(mt_key, mt_pos, n_words);
    ES_LAUNCHED(ctx);
    return ES_OK;
}
