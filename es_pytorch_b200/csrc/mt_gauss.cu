// mt_gauss.cu -- one generation's draws of a virtual-rank stream when the policy adds action noise (ac_std != 0), bit-exact
// in the MT19937 word stream with numpy's legacy RandomState.
//
// Reference program order per antithetic pair and per rank (src/core/es.py:66-72 with the fit_fn of simple_example.py:37-40 /
// obj.py:53-57, and FeedForward.forward, src/nn/nn.py:47-48):
//     idx  = rs.randint(0, len(table) - P)                      masked rejection on 32-bit words (mt_draw.cu)
//     + :   rs.random() save_obs coin (`coins` doubles, 2 words each),  then T steps x rs.randn(act) * ac_std
//     - :   the same
// rs.randn is the legacy polar method (numpy/random/src/legacy/legacy-distributions.c, legacy_gauss): attempts of two doubles
// (4 words) x1, x2 = 2 u - 1 until r2 = x1^2 + x2^2 is in (0, 1); f = sqrt(-2 log(r2) / r2); returns f*x2 and caches f*x1 for
// the next call.  The number of words a rollout consumes therefore depends on the words themselves, and the indices of all
// later pairs depend on it: the stream has to be walked in order.  Attempts inside one rollout are independent of each other,
// which is the parallelism used here: the CTA of a stream (736 threads) tests 1 472 attempts per step, ranks the accepted ones
// with a ballot scan and records their four words in order; mt_gauss_finish_kernel turns the records into gaussians on the
// whole GPU (float64 log / sqrt off the sequential path).
//
// One CTA per stream.  The state lives in a ring of MG_RING 624-word blocks in shared memory (raw words for the recurrence and
// for the state handed back, tempered words for the attempt windows), regenerated ahead of the cursor by the whole CTA with two
// barriers per block (see `ensure`).  What the time goes to, measured with cycle counters and ncu on the way from
// 109 ms to 72 ms per K = 10 000, T*act = 17 000 generation with 8 streams: the regeneration (69 blocks per rollout) is the
// limiter and it is instruction-issue bound (issue slots 61 %): the textbook three dependent 227-word phases cost ~1 100 cycles
// per block with 4 or 10 warps; ONE pass that recomputes up to three twists per word is as slow (~100 instructions per word);
// sharing the 623 twists through shared memory, warp-aligned ranges, branch-free word expressions and hoisted index arithmetic
// bring a block to ~450 cycles.  Splitting the CTA into producer and consumer warps did not help (the producer alone sets the
// pace), neither did moving the float64 math out (it was not the limiter).  Long streams therefore take the polynomial
// jump-ahead path in the second half of this file, which spreads one stream's regeneration over the whole GPU (8.4 ms for the
// same draw); this kernel stays the path for short streams.
//
// Output noise[((stream * n_pairs + pair) * 2 + sign) * N + t * act + j] = float32(gauss * scale): the float64 product rounded
// once; the rollout kernels add it to the float32 action (the reference forms the float64 sum and the env rounds it to
// float32: identical except when the float32 rounding of the noise term moves the sum across a rounding boundary, 2^-24
// relative on a term that is ~1e-2 of the action).
// log() here is CUDA's (<= 1 ulp), the reference's is glibc's: a gaussian can differ in its last float64 bit, which the
// float32 noise array does not see; the accept/reject arithmetic (the only part that steers the stream) is exact.
#include <math.h>
#include <stdlib.h>
#include <type_traits>
#include <vector>
#include "common.cuh"
#include "mt19937.cuh"

namespace {

constexpr int MG_THREADS = 736, MG_WARPS = MG_THREADS / 32;    // 23 warps: see the word <-> thread map of the regeneration
static_assert(MG_WARPS <= 32, "one shuffle scan over the warp totals");
constexpr int MG_RING = 20;                                    // blocks in the ring (raw + tempered + one block of twists: 102 KB of shared memory)
constexpr int MG_RW = MG_RING * MT_NW, MG_RQ = MG_RW / 4;      // ring words; the tempered ring is stored as 4 quarter rings (see mg_tw_slot)
static_assert(MG_RW % 4 == 0, "quarter rings");
constexpr int MG_APT = 2;                                      // attempts per thread and step (consecutive attempts)
constexpr int MG_WIN = 4 * MG_APT * MG_THREADS;                // words tested per step (5888 = 9.4 blocks)
static_assert((MG_RING - 2) * MT_NW >= MG_WIN + MT_NW, "the ring holds the cursor's block and a whole window ahead of it");

// Where ring word k (0 <= k < MG_RW) of the TEMPERED stream lives: word k sits in quarter ring k % 4 at k / 4, so that the four
// words of consecutive attempts (k = s + 4a + q) are consecutive in shared memory for a fixed q: the attempt windows read
// without bank conflicts (stride-4 or stride-8 word reads were 4- / 8-way conflicts and half of a window step's time)
__device__ __forceinline__ int mg_tw_slot(int k) { return (k & 3) * MG_RQ + (k >> 2); }
struct MgShared {
    int wtot[2][MG_WARPS];
    int end;
};

// is a gaussian cached at the start of evaluation e of a stream?  Every evaluation draws N values; an accepted attempt makes
// two, so the cache state only depends on the parity of N and of e (c0 = the stream's incoming has_gauss)
__device__ __forceinline__ int mg_cached(int c0, int N, int e) { return (N & 1) ? (c0 ^ (e & 1)) : c0; }

// What the finishing kernels write once per evaluation e of a stream (ce = mg_cached(c0, N, e); g0, cache: the stream's
// incoming and outgoing cached gaussian; out: the evaluation's N values)
__device__ __forceinline__ void mg_cache_edges(int e, int n_eval, int c0, int ce, int N, double scale, const double* __restrict__ g0,
                                               float* __restrict__ out, double* __restrict__ cache) {
    if (e == 0 && ce && N > 0) out[0] = (float)__dmul_rn(*g0, scale);              // the stream's incoming cached gaussian
    if (e == n_eval - 1 && !mg_cached(c0, N, n_eval)) *cache = 0.0;                // nothing cached afterwards
    if (N == 0 && e == 0 && c0) *cache = *g0;                                      // no draws at all: the cache is untouched
}
// the pair g of an accepted attempt: values p and p + 1 of the evaluation; a value N is the cache
__device__ __forceinline__ void mg_store_pair(double2 g, int p, int N, bool last_eval, double scale, float* __restrict__ out,
                                              double* __restrict__ cache) {
    out[p] = (float)__dmul_rn(g.x, scale);
    if (p + 1 < N) out[p + 1] = (float)__dmul_rn(g.y, scale);
    else if (!last_eval) out[N] = (float)__dmul_rn(g.y, scale);        // = value 0 of the stream's next evaluation
    else *cache = g.y;                                                 // the cache the stream hands back
}

__global__ void __launch_bounds__(MG_THREADS, 1)
mt_gauss_kernel(uint32_t* __restrict__ mt_key, int32_t* __restrict__ mt_pos, int32_t* __restrict__ has_gauss_io,
                const double* __restrict__ gauss_io, int n_pairs, uint32_t rng, uint32_t mask, int coins, int N,
                int64_t* __restrict__ idx_out, uint32_t* __restrict__ extra_out, uint4* __restrict__ acc4, int a_max,
                int32_t* __restrict__ c0_out, double* __restrict__ gauss0_out) {
    extern __shared__ uint32_t mg_smem[];
    uint32_t* s_raw = mg_smem;                                 // [MG_RING][624] raw state words (the recurrence, the state handed back)
    uint32_t* s_tw = mg_smem + MG_RING * MT_NW;                // [MG_RING][624] tempered words (what the consumers read)
    uint32_t* s_T = mg_smem + 2 * MG_RING * MT_NW;             // [624] twists of the block being regenerated
    __shared__ MgShared sh;

    const int tid = threadIdx.x, lane = tid & 31;
    const int sid = blockIdx.x;
    for (int i = tid; i < MT_NW; i += MG_THREADS) {
        const uint32_t y = mt_key[(size_t)sid * MT_NW + i];
        s_raw[i] = y; s_tw[mg_tw_slot(i)] = mt19937_temper(y);
    }
    const long long cur0 = mt_pos[sid];
    const int c0 = has_gauss_io[sid] ? 1 : 0;
    if (tid == 0) { c0_out[sid] = c0; gauss0_out[sid] = gauss_io[sid]; }     // what the finishing kernel needs of the incoming cache
    __syncthreads();

    // the cursor as (block, offset in the block, offset in the ring): 32-bit bookkeeping, no 64-bit divisions per step
    int gen_b = 0;                                             // newest generated block (block 0 = the incoming state)
    int cblk = (int)(cur0 / MT_NW), coff = (int)(cur0 % MT_NW), cring = (int)(cur0 % (MG_RING * MT_NW));
    auto advance = [&](int n) {
        coff += n;
        while (coff >= MT_NW) { coff -= MT_NW; ++cblk; }
        cring += n;
        if (cring >= MG_RING * MT_NW) cring -= MG_RING * MT_NW;
    };
    // Next block of the recurrence into ring slot (b + 1) % MG_RING by the whole CTA, with two barriers per block instead of the
    // three dependent 227-word phases of the textbook form: the twists of the old block are shared through s_T and every thread
    // forms one new word (Mt19937Regen).  (Recomputing the twists instead of sharing them -- one barrier, ~100 instructions per
    // word -- measured slower.)  Everything that does not depend on the block is computed once.
    Mt19937Regen rg;
    rg.init(tid);
    const int r_tw = rg.my_i >= 0 ? (rg.my_i & 3) * MG_RQ + (rg.my_i >> 2) : 0;   // mg_tw_slot(nslot * 624 + i) = r_tw + nslot * 156
    if (tid == 0) s_T[MT_NW - 1] = 0;
    auto ensure = [&](int n) {                                 // the next n words are in the ring (n uniform over the CTA)
        const int blocks = cblk + (coff + n + MT_NW - 1) / MT_NW;              // blocks [0, blocks) are needed
        while (gen_b + 1 < blocks) {
            const uint32_t* __restrict__ O = s_raw + (gen_b % MG_RING) * MT_NW;
            const int nslot = (gen_b + 1) % MG_RING;
            uint32_t* __restrict__ dst = s_raw + nslot * MT_NW;
            if (tid < MT_NW - 1) s_T[tid] = mt19937_twist(O[tid], O[tid + 1]);
            __syncthreads();
            auto put = [&](uint32_t y) { dst[rg.my_i] = y; s_tw[r_tw + nslot * (MT_NW / 4)] = mt19937_temper(y); };
            if (rg.plain) put(rg.word(O, s_T));
            else if (rg.my_i == MT_NW - 1) put(mt19937_last_word(O, s_T));
            __syncthreads();
            ++gen_b;
        }
    };
    auto word = [&](int ahead) -> uint32_t {                   // the word `ahead` positions after the cursor
        int a = cring + ahead;
        if (a >= MG_RW) a -= MG_RW;
        return s_tw[mg_tw_slot(a)];
    };
    const int warp = tid >> 5;
    int64_t* idx_o = idx_out + (size_t)sid * n_pairs;
    uint32_t* ext_o = extra_out ? extra_out + (size_t)sid * n_pairs * 4 * coins : nullptr;
    unsigned step = 0;

    for (int pair = 0; pair < n_pairs; ++pair) {
        // ---- rs.randint: masked rejection, every thread walks the same few words ----
        uint32_t w;
        do {
            ensure(1);
            w = word(0) & mask;
            advance(1);
        } while (w > rng);
        if (tid == 0) idx_o[pair] = (int64_t)w;
        for (int sgn = 0; sgn < 2; ++sgn) {
            // ---- the fit_fn's save_obs coin(s) ----
            ensure(2 * coins);
            if (ext_o && tid < 2 * coins) ext_o[(size_t)pair * 4 * coins + sgn * 2 * coins + tid] = word(tid);
            advance(2 * coins);
            // ---- T x randn(act): N gaussians = the cached one (if any) + accepted attempts, two values each.  Only the accept /
            //      reject arithmetic steers the stream: the accepted attempts' words are recorded in order and turned into
            //      gaussians by mt_gauss_finish_kernel on the whole GPU ----
            const int e = pair * 2 + sgn;
            uint4* rec = acc4 + ((size_t)sid * 2 * n_pairs + e) * a_max;
            int need = (N - mg_cached(c0, N, e) + 1) >> 1;            // accepted attempts still to find
            int found = 0;
            while (need > 0) {
                // only as many words as the remaining attempts can use at the usual acceptance rate are regenerated up front
                ensure(MG_WIN);
                // this thread's MG_APT consecutive attempts (4 words each)
                uint32_t wd[MG_APT][4];
                bool acc[MG_APT];
                unsigned bal[MG_APT];
                const int ph = cring & 3;                      // the cursor's phase: word q of every attempt sits in quarter ring (ph + q) & 3
#pragma unroll
                for (int j = 0; j < MG_APT; ++j) {
                    const int b4 = (cring >> 2) + MG_APT * tid + j;            // (ring offset of the attempt's first word) / 4, before wrapping
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        int k4 = b4 + ((ph + q) >> 2);
                        if (k4 >= MG_RQ) k4 -= MG_RQ;
                        wd[j][q] = s_tw[((ph + q) & 3) * MG_RQ + k4];
                    }
                    acc[j] = mt19937_polar_accept(wd[j][0], wd[j][1], wd[j][2], wd[j][3]);
                    bal[j] = __ballot_sync(0xffffffffu, acc[j]);
                }
                const unsigned buf = step & 1;
                ++step;
                int wsum = 0, below = 0;                       // accepted in this warp; accepted by lower lanes
#pragma unroll
                for (int j = 0; j < MG_APT; ++j) { wsum += __popc(bal[j]); below += __popc(bal[j] & ((1u << lane) - 1u)); }
                if (lane == 0) sh.wtot[buf][warp] = wsum;
                __syncthreads();
                int scan = (lane < MG_WARPS) ? sh.wtot[buf][lane] : 0;      // inclusive scan of the warp totals
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const int up = __shfl_up_sync(0xffffffffu, scan, d);
                    if (lane >= d) scan += up;
                }
                const int total = __shfl_sync(0xffffffffu, scan, MG_WARPS - 1);
                const int before = warp ? __shfl_sync(0xffffffffu, scan, warp - 1) : 0;
                int rank = before + below;                     // rank of this thread's first attempt among the accepted ones
#pragma unroll
                for (int j = 0; j < MG_APT; ++j) {
                    if (acc[j] && rank < need) {
                        rec[found + rank] = make_uint4(wd[j][0], wd[j][1], wd[j][2], wd[j][3]);
                        if (rank == need - 1) sh.end = MG_APT * tid + j + 1;
                    }
                    rank += acc[j] ? 1 : 0;
                }
                if (total >= need) {
                    __syncthreads();                           // sh.end is written
                    advance(4 * sh.end);
                    need = 0;
                    __syncthreads();                           // ... and read by everyone before the next rollout can write it
                } else {
                    advance(MG_WIN);
                    need -= total;
                    found += total;
                }
            }
        }
    }
    // ---- hand the state back: the block the cursor is in (position 624 = block exhausted), and its position ----
    const bool at_end = coff == 0 && (cblk > 0);
    const int b_last = at_end ? cblk - 1 : cblk;
    ensure(0);                                                 // (block b_last is in the ring: the cursor has been there)
    const uint32_t* last = s_raw + (b_last % MG_RING) * MT_NW;
    for (int i = tid; i < MT_NW; i += MG_THREADS) mt_key[(size_t)sid * MT_NW + i] = last[i];
    if (tid == 0) {
        mt_pos[sid] = at_end ? MT_NW : coff;
        has_gauss_io[sid] = mg_cached(c0, N, 2 * n_pairs);     // (the cached VALUE is written by the finishing kernel)
    }
}

// The recorded attempts -> gaussians, on the whole GPU: attempt r of evaluation e gives values c_e + 2r and c_e + 2r + 1.
__global__ void __launch_bounds__(256)
mt_gauss_finish_kernel(const uint4* __restrict__ acc4, int a_max, const int32_t* __restrict__ c0_in, const double* __restrict__ gauss0,
                       int n_streams, int n_pairs, int N, double scale, float* __restrict__ noise_out, double* __restrict__ gauss_io) {
    const long long per_eval = a_max;
    const long long total = (long long)n_streams * 2 * n_pairs * per_eval;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int r = (int)(i % per_eval);
        const long long ge = i / per_eval;                     // evaluation, stream-major
        const int e = (int)(ge % (2 * n_pairs)), sid = (int)(ge / (2 * n_pairs));
        const int c0 = c0_in[sid];
        const int ce = mg_cached(c0, N, e);
        const int need = (N - ce + 1) >> 1;
        float* out = noise_out + (size_t)ge * N;
        if (r == 0) mg_cache_edges(e, 2 * n_pairs, c0, ce, N, scale, gauss0 + sid, out, gauss_io + sid);
        if (r >= need) continue;
        const uint4 w = acc4[i];
        mg_store_pair(mt19937_polar_pair(w.x, w.y, w.z, w.w), ce + 2 * r, N, e == 2 * n_pairs - 1, scale, out, gauss_io + sid);
    }
}

// =====================================================================================================================
// Jump-ahead: ONE stream regenerated by many CTAs.
//
// The state transition of MT19937 is linear over GF(2); with g(x) = x^(624 * B) mod phi(x) (phi = its characteristic
// polynomial, tools/mt_jump/make_jump_polys.py) every word of the raw sequence obeys x[n + 624 * B] = XOR_{i : g_i = 1}
// x[n + i].  So the state 2^r blocks ahead is, word by word, an XOR of ~10 000 words out of the next 20 560: independent per
// word, no recurrence to follow.  mt_fill_kernel gives every CTA one segment of 2^lb blocks of one stream: it jumps from the
// stream's current state to its segment's first block (one jump per non-zero hexadecimal digit of the block index: the polynomials of B = m * 16^q, m = 1 .. 15, q = 0 .. 4, are precomputed), regenerates the segment and
// writes the TEMPERED words to global memory.  What follows no longer touches the recurrence: mt_flags_kernel computes the accept
// bit of every possible attempt (all four phases) with per-chunk counts, mt_scan_kernel their prefixes; mt_walk_kernel -- the only
// sequential step left, one warp per stream -- follows the reference's order with two table look-ups per rollout ("the next
// `need` accepted attempts of this phase end at word ..."); mt_emit_kernel turns every rollout's accepted attempts into its
// gaussians, one CTA per rollout.
// =====================================================================================================================
constexpr int MJ_NQ = 5, MJ_BITS_RANGE = 4 * MJ_NQ;              // hex digits of a block index that have polynomials: 2^20 blocks
constexpr int MJ_NPOLY = 15 * MJ_NQ;                            // x^(624 * m * 16^q) mod phi at [q * 15 + m - 1], m = 1 .. 15
constexpr int MJ_WIN_BLOCKS = 33;                              // the state block + 32 more: 20 592 words >= 19 937 + 624
// Layout in global memory (per stream): the tempered words in stream order; per phase ph = 0..3 (an attempt starts at a word
// index = ph mod 4) one accept bit per attempt (attempt a of phase ph = words 4 a + ph .. 4 a + ph + 3), in chunks of
// MJ_CA = 1024 attempts (32 mask words) with the number of accepted attempts of every chunk and its exclusive prefix.
constexpr int MJ_CA = 1024, MJ_CW = 4 * MJ_CA;                  // attempts / words per chunk
__device__ const uint32_t mj_polys[MJ_NPOLY][MT_NW] = {
#include "mt_jump_polys.inc"
};

// the set bits of every jump polynomial as a list of word offsets (built once per device by mj_lists_kernel): applying a jump
// is then "XOR the window words at these offsets", 8 offsets per 16-byte load, with independent loads in flight
constexpr int MJ_BITS = MT_NW * 32;
__device__ __align__(16) uint16_t mj_idx[MJ_NPOLY][MJ_BITS];
__device__ int mj_cnt[MJ_NPOLY];

__global__ void __launch_bounds__(640) mj_lists_kernel() {
    __shared__ int s_w[20];
    const int r = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint32_t g = tid < MT_NW ? mj_polys[r][tid] : 0u;
    int inc = __popc(g);
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int up = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc += up;
    }
    if (lane == 31) s_w[warp] = inc;
    __syncthreads();
    int before = 0;
    for (int w = 0; w < warp; ++w) before += s_w[w];
    int at = before + inc - __popc(g);
    while (g) {
        mj_idx[r][at++] = (uint16_t)(tid * 32 + __ffs(g) - 1);
        g &= g - 1;
    }
    if (tid == 639) mj_cnt[r] = before + inc;
}

// Thread <-> word map of the fill: warp w, lane l looks at word 31 w + l and OWNS it when l < 31 (the last lane of a warp only
// supplies its word to its neighbour, so no lane has to form a second word); word 623, whose expression differs, sits right
// after word 622 in warp 20.  One barrier per block: a thread forms its new word N[i] from the old block O and O's twists T
// (see mt19937.cuh), takes N[i + 1] from the next lane and stores N[i] AND the new block's twist T'[i] = tw(N[i], N[i + 1]) --
// so the next block can start right after the barrier.  T[623] stays 0 in both twist buffers.  The main loop is unrolled over
// the two block / twist buffers so that every shared-memory address is a per-thread register plus an immediate (the first
// version recomputed them and issued ~110 instructions per warp and block; the kernel is issue-bound).
constexpr int MF_WARPS = 21, MF_THREADS = 32 * MF_WARPS;

// segments in the order the CTAs should start: most jumps first, so that the long CTAs do not end up in the last wave
__device__ __forceinline__ int mj_jumps(unsigned block) {       // non-zero hexadecimal digits = jumps to reach the block
    int n = 0;
    for (; block; block >>= 4) n += (block & 15u) ? 1 : 0;
    return n;
}
__global__ void __launch_bounds__(1024) mj_order_kernel(int n_seg, int lb_log2, uint16_t* __restrict__ order) {
    for (int k = threadIdx.x; k < n_seg; k += 1024) {
        const int pc = mj_jumps((unsigned)k << lb_log2);
        int rank = 0;
        for (int j = 0; j < n_seg; ++j) {
            const int pj = mj_jumps((unsigned)j << lb_log2);
            rank += (pj > pc || (pj == pc && j < k)) ? 1 : 0;
        }
        order[rank] = (uint16_t)k;
    }
}

__global__ void __launch_bounds__(MF_THREADS, 2)
mt_fill_kernel(const uint32_t* __restrict__ mt_key, int n_streams, int n_seg, int lb_log2, const uint16_t* __restrict__ order,
               uint32_t* __restrict__ words, size_t stride_words) {
    extern __shared__ uint32_t mj_smem[];
    uint32_t* xs = mj_smem;                                    // [33][624] raw words: the jump window; blocks 0 / 1: ping-pong of the fill
    uint32_t* s_T = mj_smem + MJ_WIN_BLOCKS * MT_NW;           // [2][624] twists of the block being read / being written
    uint32_t* s_P = s_T + 2 * MT_NW;                           // [4][624] partial sums of a jump (one per quarter of the polynomial)
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int sid = blockIdx.x % n_streams, k = order[blockIdx.x / n_streams];
    const int iw = 31 * warp + lane;                           // the word this thread looks at
    const bool last = iw == MT_NW - 1;
    const bool owner = (lane < 31 && iw < MT_NW - 1) || last;
    const bool tail_warp = warp == MF_WARPS - 1;
    const int i = iw < MT_NW - 1 ? iw : MT_NW - 2;             // (clamped: whole warps take part in the shuffle)
    const Mt19937Taps tp = mt19937_taps(i);
    uint32_t* __restrict__ out = words + (size_t)sid * stride_words;
    for (int j = tid; j < MT_NW; j += MF_THREADS) {
        const uint32_t y = mt_key[(size_t)sid * MT_NW + j];
        xs[j] = y;
        if (k == 0) out[j] = mt19937_temper(y);               // block 0 = the incoming state: its unread words belong to the stream
    }
    if (tid < 2) s_T[tid * MT_NW + MT_NW - 1] = 0;
    __syncthreads();
    // one block: O, T -> D (raw words), Tn (its twists), opw (this thread's tempered word in global memory, when OUT)
    const bool owner_t = owner && !last;
    auto regen = [&](auto out_tag, const uint32_t* __restrict__ O, const uint32_t* __restrict__ T, uint32_t* __restrict__ D,
                     uint32_t* __restrict__ Tn, uint32_t* __restrict__ opw) {
        constexpr bool OUT = decltype(out_tag)::value;
        uint32_t n = O[tp.o] ^ T[tp.a] ^ T[tp.b] ^ T[tp.c];
        if (tail_warp) {
            if (last) n = mt19937_last_word(O, T);
        }
        const uint32_t nx = __shfl_down_sync(0xffffffffu, n, 1);
        const uint32_t tw = mt19937_twist(n, nx);
        if (owner) D[iw] = n;
        if (owner_t) Tn[iw] = tw;
        if (OUT) {
            const uint32_t y = mt19937_temper(n);
            if (owner) *opw = y;
        }
        __syncthreads();
    };
    using Yes = std::true_type;
    using No = std::false_type;
    auto twists_of = [&](const uint32_t* __restrict__ O, uint32_t* __restrict__ T) {
        if (tid < MT_NW - 1) T[tid] = mt19937_twist(O[tid], O[tid + 1]);
        __syncthreads();
    };
    uint32_t* const T0 = s_T;
    uint32_t* const T1 = s_T + MT_NW;
    // ---- jump to block k << lb_log2 ----
    const unsigned target = (unsigned)k << lb_log2;
    for (int q = MJ_NQ - 1; q >= 0; --q) {                     // (one jump per non-zero hex digit of the first block's index)
        const unsigned m = (target >> (4 * q)) & 15u;
        if (m == 0u) continue;
        const int r = q * 15 + (int)m - 1;
        twists_of(xs, T0);
        for (int b = 1; b < MJ_WIN_BLOCKS; b += 2) {           // 32 more blocks: the window of the jump
            regen(No(), xs + (b - 1) * MT_NW, T0, xs + b * MT_NW, T1, nullptr);
            regen(No(), xs + b * MT_NW, T1, xs + (b + 1) * MT_NW, T0, nullptr);
        }
        // four output words per thread (j, j + 156, j + 312, j + 468: the offsets are decoded once for four loads), and the
        // polynomial's set bits in four quarters, one per group of 156 threads; the partial sums meet in shared memory
        if (tid < MT_NW) {
            const int grp = tid / (MT_NW / 4), j = tid - grp * (MT_NW / 4);
            const uint16_t* __restrict__ L = mj_idx[r];
            const int n = mj_cnt[r];
            const int per = ((n + 3) / 4 + 7) & ~7;            // a quarter of the list, whole 16-byte loads
            const int lo = min(n, grp * per), hi = min(n, lo + per);
            const uint32_t* __restrict__ xb = xs + j;
            uint32_t acc[4] = {0u, 0u, 0u, 0u}, alt[4] = {0u, 0u, 0u, 0u};
            auto tap = [&](uint32_t off, uint32_t* a) {
                const uint32_t* __restrict__ q = xb + off;
                a[0] ^= q[0]; a[1] ^= q[MT_NW / 4]; a[2] ^= q[2 * (MT_NW / 4)]; a[3] ^= q[3 * (MT_NW / 4)];
            };
            int e = lo;
            for (; e + 8 <= hi; e += 8) {
                const uint4 q = __ldg(reinterpret_cast<const uint4*>(L + e));
                tap(q.x & 0xFFFFu, acc); tap(q.x >> 16, alt);
                tap(q.y & 0xFFFFu, acc); tap(q.y >> 16, alt);
                tap(q.z & 0xFFFFu, acc); tap(q.z >> 16, alt);
                tap(q.w & 0xFFFFu, acc); tap(q.w >> 16, alt);
            }
            for (; e < hi; ++e) tap(L[e], acc);
#pragma unroll
            for (int c = 0; c < 4; ++c) s_P[grp * MT_NW + j + c * (MT_NW / 4)] = acc[c] ^ alt[c];
        }
        __syncthreads();
        if (tid < MT_NW)                                       // (word 0: only its top bit is state, and that bit is right)
            xs[tid] = s_P[tid] ^ s_P[MT_NW + tid] ^ s_P[2 * MT_NW + tid] ^ s_P[3 * MT_NW + tid];
        __syncthreads();
    }
    twists_of(xs, T0);
    // ---- regenerate the segment: blocks target + 1 .. target + 2^lb, two per iteration (buffers 0 -> 1 -> 0) ----
    const int Lb = 1 << lb_log2;
    uint32_t* __restrict__ opw = out + (size_t)(1 + target) * MT_NW + iw;
    uint32_t* const X0 = xs;
    uint32_t* const X1 = xs + MT_NW;
    int b = 0;
    for (; b + 2 <= Lb; b += 2) {
        regen(Yes(), X0, T0, X1, T1, opw);
        regen(Yes(), X1, T1, X0, T0, opw + MT_NW);
        opw += 2 * MT_NW;
    }
    if (b < Lb) regen(Yes(), X0, T0, X1, T1, opw);
}

// ---- the accept bit of every possible attempt, in parallel ----
// One WARP per chunk (4096 words = 1024 attempts of each phase): 32 steps of 128 words; lane l holds words 4 l .. 4 l + 3 of a step
// (one 16-byte load), takes the next three from lane l + 1 (lane 31: from the next step's first load, which is already in
// flight), and tests the four attempts that start at its words; lane s keeps the ballots of step s, so the 32 mask words of a
// phase leave as one 128-byte store and the chunk's counts need no shared memory and no barrier.
constexpr int MFL_WARPS = 8;
__global__ void __launch_bounds__(32 * MFL_WARPS)
mt_flags_kernel(const uint32_t* __restrict__ words, size_t stride_words, int n_chunks, uint32_t* __restrict__ masks,
                uint32_t* __restrict__ counts) {
    const int lane = threadIdx.x & 31, sid = blockIdx.y;
    const int c = blockIdx.x * MFL_WARPS + (threadIdx.x >> 5);
    if (c >= n_chunks) return;
    const uint4* __restrict__ w4 = reinterpret_cast<const uint4*>(words + (size_t)sid * stride_words + (size_t)c * MJ_CW) + lane;
    uint32_t keep[4] = {0u, 0u, 0u, 0u};
    uint4 cur = __ldg(w4), nxt1 = __ldg(w4 + 32), nxt2 = __ldg(w4 + 64), nxt3 = __ldg(w4 + 96);   // (the buffer is padded by a chunk)
#pragma unroll 4
    for (int s = 0; s < 32; ++s) {
        const uint4 far = __ldg(w4 + (s + 4) * 32);           // (reads up to 4 steps past the chunk: inside the next chunk / the padding)
        uint4 b;
        b.x = __shfl_down_sync(0xffffffffu, cur.x, 1);
        b.y = __shfl_down_sync(0xffffffffu, cur.y, 1);
        b.z = __shfl_down_sync(0xffffffffu, cur.z, 1);
        const uint32_t n0 = __shfl_sync(0xffffffffu, nxt1.x, 0), n1 = __shfl_sync(0xffffffffu, nxt1.y, 0), n2 = __shfl_sync(0xffffffffu, nxt1.z, 0);
        if (lane == 31) { b.x = n0; b.y = n1; b.z = n2; }
        const unsigned b0 = __ballot_sync(0xffffffffu, mt19937_polar_accept(cur.x, cur.y, cur.z, cur.w));
        const unsigned b1 = __ballot_sync(0xffffffffu, mt19937_polar_accept(cur.y, cur.z, cur.w, b.x));
        const unsigned b2 = __ballot_sync(0xffffffffu, mt19937_polar_accept(cur.z, cur.w, b.x, b.y));
        const unsigned b3 = __ballot_sync(0xffffffffu, mt19937_polar_accept(cur.w, b.x, b.y, b.z));
        if (lane == s) { keep[0] = b0; keep[1] = b1; keep[2] = b2; keep[3] = b3; }
        cur = nxt1; nxt1 = nxt2; nxt2 = nxt3; nxt3 = far;
    }
    uint32_t* mk = masks + ((size_t)sid * 4 * n_chunks + c) * 32 + lane;              // + ph * n_chunks * 32
#pragma unroll
    for (int ph = 0; ph < 4; ++ph) {
        mk[(size_t)ph * n_chunks * 32] = keep[ph];
        const int cnt = __reduce_add_sync(0xffffffffu, __popc(keep[ph]));
        if (lane == 0) counts[((size_t)sid * 4 + ph) * n_chunks + c] = (uint32_t)cnt;
    }
}

// exclusive prefix of the chunk counts of every (stream, phase): one CTA each
__global__ void __launch_bounds__(1024) mt_scan_kernel(uint32_t* __restrict__ counts, int n_chunks) {
    __shared__ uint32_t s_part[1024];
    uint32_t* v = counts + (size_t)blockIdx.x * n_chunks;
    const int per = (n_chunks + 1023) / 1024, lo = threadIdx.x * per, hi = min(n_chunks, lo + per);
    uint32_t sum = 0;
    for (int i = lo; i < hi; ++i) sum += v[i];
    s_part[threadIdx.x] = sum;
    __syncthreads();
    for (int d = 1; d < 1024; d <<= 1) {                          // inclusive scan of the partial sums
        const uint32_t add = threadIdx.x >= d ? s_part[threadIdx.x - d] : 0;
        __syncthreads();
        s_part[threadIdx.x] += add;
        __syncthreads();
    }
    uint32_t run = threadIdx.x ? s_part[threadIdx.x - 1] : 0;
    for (int i = lo; i < hi; ++i) { const uint32_t t = v[i]; v[i] = run; run += t; }
}

// ---- the walk: ONE WARP per stream follows the reference's order; a rollout's N gaussians are "the next `need` accepted
//      attempts of phase ph from word s on", i.e. two look-ups in the prefix tables instead of a pass over the words ----
__global__ void __launch_bounds__(32)
mt_walk_kernel(uint32_t* __restrict__ mt_key, int32_t* __restrict__ mt_pos, int32_t* __restrict__ has_gauss_io,
               const double* __restrict__ gauss_io, int n_pairs, uint32_t rng, uint32_t mask, int coins, int N,
               int64_t* __restrict__ idx_out, uint32_t* __restrict__ extra_out, uint32_t* __restrict__ reg_start,
               int32_t* __restrict__ c0_out, double* __restrict__ gauss0_out, const uint32_t* __restrict__ words,
               size_t stride_words, int n_chunks, const uint32_t* __restrict__ masks, const uint32_t* __restrict__ cumul,
               uint32_t limit, int* __restrict__ err) {
    const int lane = threadIdx.x, sid = blockIdx.x;
    const uint32_t* __restrict__ gw = words + (size_t)sid * stride_words;
    const uint32_t* __restrict__ mk = masks + (size_t)sid * 4 * n_chunks * 32;
    const uint32_t* __restrict__ cu = cumul + (size_t)sid * 4 * n_chunks;
    uint32_t cpos = (uint32_t)mt_pos[sid];
    const int c0 = has_gauss_io[sid] ? 1 : 0;
    if (lane == 0) { c0_out[sid] = c0; gauss0_out[sid] = gauss_io[sid]; }
    int64_t* idx_o = idx_out + (size_t)sid * n_pairs;
    uint32_t* ext_o = extra_out ? extra_out + (size_t)sid * n_pairs * 4 * coins : nullptr;
    uint32_t* rs = reg_start + (size_t)sid * 2 * n_pairs;
    const unsigned FULL = 0xffffffffu;
    const uint32_t nc_u = (uint32_t)n_chunks;                     // (host: n_chunks * 128 < 2^32, every table index fits 32 bits)
    bool overflow = false;
    for (int pair = 0; pair < n_pairs && !overflow; ++pair) {
        // the index: the first of the next words that passes the masked rejection (32 candidates at a time)
        uint32_t w = 0;
        for (;;) {
            if (cpos + 1 > limit) { overflow = true; break; }
            const uint32_t v = __ldg(gw + cpos + lane) & mask;          // (the buffer is padded by a chunk past `limit`)
            const unsigned ok = __ballot_sync(FULL, v <= rng);
            if (ok) {
                const int f = __ffs((int)ok) - 1;
                w = __shfl_sync(FULL, v, f);
                cpos += (uint32_t)f + 1u;
                break;
            }
            cpos += 32u;
        }
        if (overflow || cpos > limit) { overflow = true; break; }
        if (lane == 0) idx_o[pair] = (int64_t)w;
        for (int sgn = 0; sgn < 2; ++sgn) {
            if (cpos + 2 * coins + 8 > limit) { overflow = true; break; }
            if (ext_o && lane < 2 * coins) ext_o[(size_t)pair * 4 * coins + sgn * 2 * coins + lane] = __ldg(gw + cpos + lane);
            cpos += 2 * coins;
            const int e = pair * 2 + sgn;
            if (lane == 0) rs[e] = cpos;
            const int need = (N - mg_cached(c0, N, e) + 1) >> 1;
            if (need == 0) continue;
            const int ph = cpos & 3;
            const uint32_t a0 = cpos >> 2;                        // first attempt of the rollout, in phase ph's numbering
            const uint32_t* __restrict__ mph = mk + (size_t)ph * n_chunks * 32;
            const uint32_t* __restrict__ cph = cu + (size_t)ph * n_chunks;
            // everything the rollout needs is loaded at once (one memory latency per rollout): the mask row and prefix of the
            // chunk it starts in, the prefixes of a window of 32 chunks around the expected end (acceptance pi / 4; the spread
            // of the end is ~sqrt(need) attempts, a window is 32 768), and the mask rows of the three likeliest end chunks.
            // (32-bit arithmetic throughout: one warp per stream leaves every instruction's latency exposed)
            const uint32_t ch0 = a0 >> 10, r0 = a0 & 1023;
            const uint32_t span = (uint32_t)need + (uint32_t)(((uint64_t)(uint32_t)need * 1173554908u) >> 32);      // need * 4 / pi
            const uint32_t a_est = a0 + span;
            uint32_t est = a_est >> 10;
            if (est > nc_u - 1u) est = nc_u - 1u;
            uint32_t wlo = est > ch0 + 12u ? est - 12u : ch0;
            if (wlo + 32u > nc_u) wlo = nc_u > 32u ? nc_u - 32u : 0u;
            uint32_t ci = wlo + lane;
            const uint32_t m0 = __ldg(mph + ch0 * 32u + lane);
            const uint32_t base0 = __ldg(cph + ch0);
            uint32_t pre = (ci < nc_u) ? __ldg(cph + ci) : 0xFFFFFFFFu;
            const uint32_t e0 = est > 0u ? est - 1u : 0u, e2 = est + 1u < nc_u ? est + 1u : est;
            const uint32_t mc0 = __ldg(mph + e0 * 32u + lane), mc1 = __ldg(mph + est * 32u + lane), mc2 = __ldg(mph + e2 * 32u + lane);
            // pull what the NEXT draws will touch towards L2 while this rollout is resolved: the words around the expected end
            // (the next index / coins); for the next rollout, whose phase is not known yet, in all four phases: the mask rows
            // around its start (= this end) and around its expected end, and the prefix windows around its expected end
            {
                const uint32_t a_pf = a_est + (uint32_t)(lane - 12) * 8u;
                if (a_pf < (limit >> 2)) asm volatile("prefetch.global.L2 [%0];" ::"l"(gw + 4u * a_pf));
                const uint32_t est2 = (a_est + span) >> 10;
                if (lane < 24) {
                    const uint32_t l12 = lane < 12 ? lane : lane - 12;
                    const uint32_t nc = (lane < 12 ? est : est2) + (l12 % 3u) - 1u;
                    if (nc < nc_u) asm volatile("prefetch.global.L2 [%0];" ::"l"(mk + ((size_t)(l12 / 3u) * nc_u + nc) * 32));
                } else {
                    const uint32_t nc = (est2 > 12u ? est2 - 12u : 0u) + ((lane & 1) ? 31u : 0u);
                    if (nc < nc_u) asm volatile("prefetch.global.L2 [%0];" ::"l"(cu + (size_t)((lane - 24) >> 1) * nc_u + nc));
                }
            }
            // accepted attempts of the phase before a0
            const int below = __reduce_add_sync(FULL, (lane < (int)(r0 >> 5)) ? __popc(m0)
                                                      : (lane == (int)(r0 >> 5) ? __popc(m0 & ((1u << (r0 & 31)) - 1u)) : 0));
            const uint32_t target = base0 + (uint32_t)below + (uint32_t)need;      // accepted attempts before the END of the rollout
            // the chunk that contains the target-th accepted attempt: the last one whose prefix is < target
            unsigned lt = __ballot_sync(FULL, pre < target);
            if (lt == 0u || (lt == 0xFFFFFFFFu && wlo + 32u < nc_u)) {
                // outside the window (tens of sigma away from the estimate): bisect the prefixes, then look again from there
                uint32_t lo = ch0, hi = nc_u - 1u;                          // invariant: prefix[lo] < target
                while (lo < hi) {
                    const uint32_t mid = (lo + hi + 1u) >> 1;
                    if (__ldg(cph + mid) < target) lo = mid; else hi = mid - 1u;
                }
                wlo = lo;
                ci = wlo + lane;
                pre = (ci < nc_u) ? __ldg(cph + ci) : 0xFFFFFFFFu;
                lt = __ballot_sync(FULL, pre < target);
            }
            const int sel = 31 - __clz((int)lt);                  // last lane with prefix < target (prefixes are non-decreasing)
            const uint32_t c1 = wlo + (uint32_t)sel, pre1 = __shfl_sync(FULL, pre, sel);
            const uint32_t m1 = c1 == est ? mc1 : (c1 == e0 ? mc0 : (c1 == e2 ? mc2 : __ldg(mph + c1 * 32u + lane)));
            int inc = __popc(m1);
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int up = __shfl_up_sync(FULL, inc, d);
                if (lane >= d) inc += up;
            }
            const uint32_t want = target - pre1;                  // the want-th (1-based) accepted attempt of chunk c1 ends the rollout
            const unsigned ge = __ballot_sync(FULL, (uint32_t)inc >= want);
            if (ge == 0u) { overflow = true; break; }
            const int L = __ffs((int)ge) - 1;
            const uint32_t mL = __shfl_sync(FULL, m1, L);
            const int incL = __shfl_sync(FULL, inc, L);
            const int kth = (int)want - (incL - __popc(mL));      // 1-based among the set bits of lane L's word
            // the kth set bit of mL: the lane whose bit is set with kth - 1 set bits below it
            const unsigned hit = __ballot_sync(FULL, ((mL >> lane) & 1u) && __popc(mL & ((1u << lane) - 1u)) == kth - 1);
            const int bit = __ffs((int)hit) - 1;
            const uint32_t a1 = (c1 << 10) + 32u * (uint32_t)L + (uint32_t)bit;
            cpos = 4u * (a1 + 1u) + (uint32_t)ph;
            if (cpos > limit) { overflow = true; break; }
        }
    }
    if (overflow) {
        if (lane == 0 && err) *(volatile int*)err = ES_ASYNC_RNG_OVERFLOW;
        return;
    }
    // ---- hand the state back: the raw words behind the tempered words of the cursor's block ----
    const uint32_t blk = cpos / MT_NW, off = cpos % MT_NW;
    const bool at_end = off == 0 && blk > 0;
    const uint32_t b_last = at_end ? blk - 1 : blk;
    for (int i = lane; i < MT_NW; i += 32) mt_key[(size_t)sid * MT_NW + i] = mt19937_untemper(__ldg(gw + (size_t)b_last * MT_NW + i));
    if (lane == 0) {
        mt_pos[sid] = at_end ? MT_NW : (int32_t)off;
        has_gauss_io[sid] = mg_cached(c0, N, 2 * n_pairs);
    }
}

// ---- the gaussians of one rollout per CTA: attempts from the rollout's first word on, accepted ones ranked by a block scan ----
__global__ void __launch_bounds__(1024)
mt_emit_kernel(const uint32_t* __restrict__ words, size_t stride_words, const uint32_t* __restrict__ reg_start,
               const int32_t* __restrict__ c0_in, const double* __restrict__ gauss0, int n_pairs, int N, double scale,
               float* __restrict__ noise_out, double* __restrict__ gauss_io) {
    __shared__ int s_wt[2][32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int ge = blockIdx.x;                                    // evaluation, stream-major
    const int e = ge % (2 * n_pairs), sid = ge / (2 * n_pairs);
    const int c0 = c0_in[sid], ce = mg_cached(c0, N, e);
    const int need = (N - ce + 1) >> 1;
    float* out = noise_out + (size_t)ge * N;
    if (tid == 0) mg_cache_edges(e, 2 * n_pairs, c0, ce, N, scale, gauss0 + sid, out, gauss_io + sid);
    const uint32_t* __restrict__ gw = words + (size_t)sid * stride_words + reg_start[ge];
    int found = 0;
    for (unsigned it = 0; found < need; ++it) {
        const uint32_t* __restrict__ wp = gw + (size_t)4 * (it * 1024u + tid);
        const uint32_t w0 = __ldg(wp), w1 = __ldg(wp + 1), w2 = __ldg(wp + 2), w3 = __ldg(wp + 3);
        const bool acc = mt19937_polar_accept(w0, w1, w2, w3);
        const unsigned bal = __ballot_sync(0xffffffffu, acc);
        if (lane == 0) s_wt[it & 1][warp] = __popc(bal);
        __syncthreads();
        int scan = s_wt[it & 1][lane];
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int up = __shfl_up_sync(0xffffffffu, scan, d);
            if (lane >= d) scan += up;
        }
        const int total = __shfl_sync(0xffffffffu, scan, 31);
        const int rank = found + (warp ? __shfl_sync(0xffffffffu, scan, warp - 1) : 0) + __popc(bal & ((1u << lane) - 1u));
        if (acc && rank < need)
            mg_store_pair(mt19937_polar_pair(w0, w1, w2, w3), ce + 2 * rank, N, e == 2 * n_pairs - 1, scale, out, gauss_io + sid);
        found += total;
    }
}

// ---- how one es_draw_noisy call runs: the sequential kernel, or the jump-ahead path and the sizes of its buffers ----
struct MgPlan {
    bool jump;
    int lb_log2;                  // segments of 2^lb_log2 blocks, n_seg per stream
    long long n_seg, n_chunks;    // n_chunks chunks of MJ_CW words per stream
    size_t gen_words, stride_words;
};

// log2 of the jump-ahead segment length in blocks: the shortest segments that leave at most ~4 segments per SM over all
// streams (ES_MT_JUMP_LB overrides it, for tests)
int mj_segment_lb(long long n_streams, long long blocks, int sm_count) {
    int lb = 3;
    const char* el = getenv("ES_MT_JUMP_LB");
    if (el) lb = atoi(el);
    else
        while (lb < MJ_BITS_RANGE - 1 && n_streams * ((blocks + (1LL << lb) - 1) >> lb) > 4LL * sm_count) ++lb;
    if (lb < 0) lb = 0;
    if (lb > MJ_BITS_RANGE - 1) lb = MJ_BITS_RANGE - 1;
    return lb;
}

// How many words can a stream consume?  Per rollout ceil(N / 2) accepted attempts at acceptance pi / 4 (a negative binomial
// count), 4 words each; per pair one index draw (~1.08 words with rejections, bounded generously) and the coins.  The
// jump-ahead pass generates the mean + 12 sigma of the total (+ slack); the walk flags an overflow.
long long mg_blocks_needed(int n_pairs, int coins, int N) {
    const double p_acc = 0.78539816339744830962, n_acc = (N + 1) / 2;
    const double att_mean = n_acc / p_acc, att_sd = sqrt(n_acc * (1.0 - p_acc)) / p_acc;
    const double evals = 2.0 * n_pairs;
    const double words_max = 624.0 + n_pairs * (8.0 + 4.0 * coins) + 4.0 * (evals * att_mean + 12.0 * sqrt(evals) * att_sd + 64.0) +
                             2.0 * MG_WIN + 16.0 * MT_NW;
    return (long long)(words_max / MT_NW) + 1;
}

int mg_plan(const es_ctx* ctx, int n_streams, int n_pairs, int coins, int N, MgPlan& pl) {
    const long long blocks_needed = mg_blocks_needed(n_pairs, coins, N);
    // jump-ahead when a stream is long enough to be worth splitting (ES_MT_JUMP=0 / 1 overrides; ES_MT_JUMP_LB: log2 of the
    // segment length in blocks, for tests)
    const char* ej = getenv("ES_MT_JUMP");
    const bool forced = ej && atoi(ej) != 0;
    pl = MgPlan{};
    if (!(ej ? forced : blocks_needed >= 2048)) return ES_OK;
    const int lb = mj_segment_lb(n_streams, blocks_needed, ctx->sm_count);
    const long long n_seg = (blocks_needed + (1LL << lb) - 1) >> lb;
    if (((n_seg << lb) >> MJ_BITS_RANGE) != 0 || (double)(n_seg << lb) * MT_NW > 4.0e9 || n_seg > 65535) {
        // the block index of a segment start must fit the available jumps (2^20 blocks = 654 M words per stream) and a
        // 32-bit word index: longer streams take the sequential kernel unless the jump-ahead path was asked for explicitly
        if (!forced) return ES_OK;
        es_set_error("es_draw_noisy: %lld blocks per stream exceed the jump-ahead range (2^%d blocks)", n_seg << lb, MJ_BITS_RANGE);
        return ES_ERR_UNSUPPORTED;
    }
    pl.jump = true;
    pl.lb_log2 = lb;
    pl.n_seg = n_seg;
    // (whole chunks of MJ_CW words, + one chunk of padding: the flags kernel reads 4 words past every attempt start)
    pl.gen_words = (size_t)(1 + (n_seg << lb)) * MT_NW;
    pl.n_chunks = (long long)((pl.gen_words + MJ_CW - 1) / MJ_CW);
    pl.stride_words = (size_t)(pl.n_chunks + 1) * MJ_CW;
    return ES_OK;
}

struct MgDraw {                   // the arguments of one es_draw_noisy call
    uint32_t* mt_key; int32_t* mt_pos; int32_t* has_gauss; double* gauss;
    int n_streams, n_pairs;
    uint32_t rng, mask;
    int coins, N;
    double scale;
    int64_t* idx_out; uint32_t* extra_out; float* noise_out;
};

size_t mg_pad(size_t b) { return (b + 255) & ~(size_t)255; }

// the tempered words of blocks 0 .. n_seg << lb_log2 of every stream, from the streams' keys (block 0), into words
int mj_launch_fill(es_ctx* ctx, const uint32_t* mt_key, int n_streams, int n_seg, int lb_log2, uint16_t* order, uint32_t* words,
                   size_t stride_words, cudaStream_t stream) {
    if (!ctx->mj_lists_ready) {
        mj_lists_kernel<<<MJ_NPOLY, 640, 0, stream>>>();
        ES_LAUNCHED(ctx);
        ctx->mj_lists_ready = 1;
    }
    mj_order_kernel<<<1, 1024, 0, stream>>>(n_seg, lb_log2, order);
    ES_LAUNCHED(ctx);
    const size_t smem = (size_t)(MJ_WIN_BLOCKS + 6) * MT_NW * sizeof(uint32_t);
    ES_CHECK_CUDA(cudaFuncSetAttribute(mt_fill_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    mt_fill_kernel<<<(unsigned)(n_streams * n_seg), MF_THREADS, smem, stream>>>(mt_key, n_streams, n_seg, lb_log2, order, words,
                                                                               stride_words);
    ES_LAUNCHED(ctx);
    return ES_OK;
}

int mg_launch_jump(es_ctx* ctx, const MgDraw& d, const MgPlan& pl, cudaStream_t stream) {
    // scratch: the streams' words | accept masks [stream][phase][chunk][32] | chunk counts -> prefixes [stream][phase][chunk]
    //          | first word of every rollout [stream][2 n] | incoming cache per stream
    const size_t n_eval = (size_t)d.n_streams * 2 * d.n_pairs;
    const size_t words_bytes = mg_pad((size_t)d.n_streams * pl.stride_words * sizeof(uint32_t));
    const size_t mask_bytes = mg_pad((size_t)d.n_streams * 4 * pl.n_chunks * 32 * sizeof(uint32_t));
    const size_t cnt_bytes = mg_pad((size_t)d.n_streams * 4 * pl.n_chunks * sizeof(uint32_t));
    const size_t reg_bytes = mg_pad(n_eval * sizeof(uint32_t));
    const size_t c0_bytes = mg_pad((size_t)d.n_streams * sizeof(int32_t)), g0_bytes = mg_pad((size_t)d.n_streams * sizeof(double));
    const size_t ord_bytes = mg_pad((size_t)pl.n_seg * sizeof(uint16_t));
    void* scratch = nullptr;
    int rc = es_ctx_scratch(ctx, words_bytes + mask_bytes + cnt_bytes + reg_bytes + c0_bytes + g0_bytes + ord_bytes, &scratch);
    if (rc) return rc;
    char* at = (char*)scratch;
    uint32_t* words = (uint32_t*)at; at += words_bytes;
    uint32_t* masks = (uint32_t*)at; at += mask_bytes;
    uint32_t* counts = (uint32_t*)at; at += cnt_bytes;
    uint32_t* reg_start = (uint32_t*)at; at += reg_bytes;
    int32_t* c0 = (int32_t*)at; at += c0_bytes;
    double* gauss0 = (double*)at; at += g0_bytes;
    uint16_t* order = (uint16_t*)at;
    rc = mj_launch_fill(ctx, d.mt_key, d.n_streams, (int)pl.n_seg, pl.lb_log2, order, words, pl.stride_words, stream);
    if (rc) return rc;
    mt_flags_kernel<<<dim3((unsigned)((pl.n_chunks + MFL_WARPS - 1) / MFL_WARPS), (unsigned)d.n_streams), 32 * MFL_WARPS, 0, stream>>>(
        words, pl.stride_words, (int)pl.n_chunks, masks, counts);
    ES_LAUNCHED(ctx);
    mt_scan_kernel<<<d.n_streams * 4, 1024, 0, stream>>>(counts, (int)pl.n_chunks);
    ES_LAUNCHED(ctx);
    mt_walk_kernel<<<d.n_streams, 32, 0, stream>>>(d.mt_key, d.mt_pos, d.has_gauss, d.gauss, d.n_pairs, d.rng, d.mask, d.coins, d.N,
                                                   d.idx_out, d.extra_out, reg_start, c0, gauss0, words, pl.stride_words,
                                                   (int)pl.n_chunks, masks, counts, (uint32_t)(pl.gen_words - 8), ctx->err_dev);
    ES_LAUNCHED(ctx);
    mt_emit_kernel<<<(unsigned)n_eval, 1024, 0, stream>>>(words, pl.stride_words, reg_start, c0, gauss0, d.n_pairs, d.N, d.scale,
                                                          d.noise_out, d.gauss);
    ES_LAUNCHED(ctx);
    return ES_OK;
}

int mg_launch_sequential(es_ctx* ctx, const MgDraw& d, cudaStream_t stream) {
    // scratch: the accepted attempts' words [stream][evaluation][a_max] (16 bytes per two gaussians), the incoming cache per
    // stream
    const size_t n_eval = (size_t)d.n_streams * 2 * d.n_pairs;
    const int a_max = (d.N + 1) / 2 > 0 ? (d.N + 1) / 2 : 1;
    const size_t acc_bytes = mg_pad(n_eval * a_max * sizeof(uint4));
    const size_t c0_bytes = mg_pad((size_t)d.n_streams * sizeof(int32_t)), g0_bytes = mg_pad((size_t)d.n_streams * sizeof(double));
    void* scratch = nullptr;
    int rc = es_ctx_scratch(ctx, acc_bytes + c0_bytes + g0_bytes, &scratch);
    if (rc) return rc;
    uint4* acc4 = (uint4*)scratch;
    int32_t* c0 = (int32_t*)((char*)scratch + acc_bytes);
    double* gauss0 = (double*)((char*)scratch + acc_bytes + c0_bytes);
    const size_t smem = (size_t)(2 * MG_RING + 1) * MT_NW * sizeof(uint32_t);
    ES_CHECK_CUDA(cudaFuncSetAttribute(mt_gauss_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    mt_gauss_kernel<<<d.n_streams, MG_THREADS, smem, stream>>>(d.mt_key, d.mt_pos, d.has_gauss, d.gauss, d.n_pairs, d.rng, d.mask,
                                                               d.coins, d.N, d.idx_out, d.extra_out, acc4, a_max, c0, gauss0);
    ES_LAUNCHED(ctx);
    const long long total = (long long)n_eval * a_max;
    int blocks = es_div_up(total, 256);
    if (blocks > ctx->sm_count * 16) blocks = ctx->sm_count * 16;
    mt_gauss_finish_kernel<<<blocks, 256, 0, stream>>>(acc4, a_max, c0, gauss0, d.n_streams, d.n_pairs, d.N, d.scale, d.noise_out,
                                                       d.gauss);
    ES_LAUNCHED(ctx);
    return ES_OK;
}

// =====================================================================================================================
// es_randn: n gaussians in a row from ONE stream, rs.randn(n) -- numpy's noise table.  Every attempt of the call starts at
// word p0 + 4 a (p0: the incoming position), so all attempts share the phase ph = p0 & 3 and nothing has to be walked:
// attempt a's values are c0 + 2 r and c0 + 2 r + 1, r = the number of accepted attempts before it (c0: the incoming cache
// bit).  The stream is processed in windows of at most MR_WINDOW_BLOCKS blocks so that the scratch stays bounded; a window
// is the jump-ahead path's fill (block 0 = the window's base state) + the accept masks and chunk prefixes of mt_flags_kernel
// / mt_scan_kernel.  Window w + 1 starts from window w's last block (untempered from its words): the two windows overlap by
// that block, so an attempt that starts in window w's own L blocks but ends in the next block is whole in window w, and no
// window jumps further than its own length.  In its local numbering a window of L blocks owns the attempts a of phase ph
// with a_lo <= a < 156 L (a_lo = p0 >> 2 in window 0, else 0): the next window's first attempt is its attempt 0.
// =====================================================================================================================
constexpr long long MR_WINDOW_BLOCKS = 3LL << 15;               // 98 304 blocks = 61 M words = 245 MB of words per window
constexpr int MR_EMIT_WARPS = 8;

struct MrState {                  // what the windows hand on to each other (device scratch)
    long long base;               // rank among the call's accepted attempts of the window's attempt a = base + cum(a)
    long long next;               // the next window's base
    double g0;                    // the incoming cached gaussian
    int c0, ph, a_lo;             // the incoming cache bit, the attempts' phase, the window's first attempt
};

// accepted attempts of phase ph before attempt a of the window (one warp; mph / cph: the phase's masks and chunk prefixes)
__device__ __forceinline__ uint32_t mr_cum(const uint32_t* __restrict__ mph, const uint32_t* __restrict__ cph, uint32_t a, int lane) {
    const uint32_t c = a >> 10, r = a & 1023u;
    const uint32_t m = mph[(size_t)c * 32 + lane];
    const int below = __reduce_add_sync(0xffffffffu, lane < (int)(r >> 5) ? __popc(m)
                                                     : (lane == (int)(r >> 5) ? __popc(m & ((1u << (r & 31)) - 1u)) : 0));
    return cph[c] + (uint32_t)below;
}

// One warp per window, after the prefixes: the window's rank offsets, the next window's base state; in window 0 the incoming
// cache; in the window that holds the attempt giving value n - 1, the outgoing state (found with the prefix tables as
// mt_walk_kernel does).
__global__ void __launch_bounds__(32)
mr_window_kernel(int w, int last, int64_t L, const uint32_t* __restrict__ words, int n_chunks, const uint32_t* __restrict__ masks,
                 const uint32_t* __restrict__ cumul, uint32_t* __restrict__ key_next, uint32_t* __restrict__ mt_key,
                 int32_t* __restrict__ mt_pos, int32_t* __restrict__ has_gauss, double* __restrict__ gauss, int64_t n,
                 float* __restrict__ out, MrState* __restrict__ st, int* __restrict__ err) {
    const int lane = threadIdx.x;
    const unsigned FULL = 0xffffffffu;
    int c0, ph, a_lo;
    long long base_in = 0;
    if (w == 0) {                                              // the incoming state, read before anything below writes it
        const int p0 = mt_pos[0];
        c0 = has_gauss[0] ? 1 : 0;
        const double g0 = gauss[0];
        ph = p0 & 3;
        a_lo = p0 >> 2;
        __syncwarp();
        if (lane == 0) {
            st->c0 = c0; st->g0 = g0; st->ph = ph;
            if (c0) out[0] = (float)g0;                         // the cached gaussian is value 0 (the host ensures n >= 1)
        }
    } else {
        c0 = st->c0; ph = st->ph; a_lo = 0;
        base_in = st->next;
    }
    const long long A = (n - c0 + 1) >> 1;                     // accepted attempts the call needs
    const uint32_t* __restrict__ mph = masks + (size_t)ph * n_chunks * 32;
    const uint32_t* __restrict__ cph = cumul + (size_t)ph * n_chunks;
    const uint32_t a_hi = (uint32_t)(L * (MT_NW / 4));
    const long long base = w == 0 ? -(long long)mr_cum(mph, cph, (uint32_t)a_lo, lane) : base_in;
    const long long next = base + mr_cum(mph, cph, a_hi, lane);
    if (lane == 0) { st->base = base; st->next = next; st->a_lo = a_lo; }
    if (!last)
        for (int i = lane; i < MT_NW; i += 32) key_next[i] = mt19937_untemper(words[(size_t)L * MT_NW + i]);
    if (A == 0) {                                              // n == 1 served by the cache: nothing cached afterwards
        if (w == 0 && lane == 0) { has_gauss[0] = 0; gauss[0] = 0.0; }
        return;
    }
    if (last && next < A) {                                    // (the host plans the mean + 12 sigma of the words needed)
        if (lane == 0 && err) *(volatile int*)err = ES_ASYNC_RANDN_OVERFLOW;
        return;
    }
    if (!(base <= A - 1 && A - 1 < next)) return;
    // the (k + 1)-th accepted attempt of the window gives value n - 1: its chunk is the last one whose prefix is <= k
    const uint32_t k = (uint32_t)(A - 1 - base);
    uint32_t lo = 0, hi = (uint32_t)n_chunks - 1u;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1u) >> 1;
        if (cph[mid] <= k) lo = mid; else hi = mid - 1u;
    }
    const uint32_t want = k - cph[lo] + 1u;                    // 1-based among the chunk's accepted attempts
    const uint32_t m1 = mph[(size_t)lo * 32 + lane];
    int inc = __popc(m1);
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int up = __shfl_up_sync(FULL, inc, d);
        if (lane >= d) inc += up;
    }
    const int Lw = __ffs((int)__ballot_sync(FULL, (uint32_t)inc >= want)) - 1;
    const uint32_t mL = __shfl_sync(FULL, m1, Lw);
    const int kth = (int)want - (__shfl_sync(FULL, inc, Lw) - __popc(mL));
    const int bit = __ffs((int)__ballot_sync(FULL, ((mL >> lane) & 1u) && __popc(mL & ((1u << lane) - 1u)) == kth - 1)) - 1;
    const uint32_t a1 = (lo << 10) + 32u * (uint32_t)Lw + (uint32_t)bit;
    // the stream after that attempt: the raw words behind the tempered words of the cursor's block, and the position
    const uint32_t end = 4u * a1 + (uint32_t)ph + 4u;
    const uint32_t blk = end / MT_NW, off = end % MT_NW;
    const bool at_end = off == 0 && blk > 0;
    const uint32_t b_last = at_end ? blk - 1 : blk;
    for (int i = lane; i < MT_NW; i += 32) mt_key[i] = mt19937_untemper(words[(size_t)b_last * MT_NW + i]);
    if (lane == 0) {
        const int cached = (int)(c0 + 2 * A - n);              // the last attempt's second value is value n: the cache
        mt_pos[0] = at_end ? MT_NW : (int32_t)off;
        has_gauss[0] = cached;
        if (!cached) gauss[0] = 0.0;                           // (otherwise mr_emit_kernel writes it)
    }
}

// The gaussians of one window, one warp per chunk of 1 024 attempts: lane l takes attempt 32 j + l in step j, its rank is the
// chunk's prefix + the accepted attempts of the chunk's mask words before j + those of lower lanes in word j.
__global__ void __launch_bounds__(32 * MR_EMIT_WARPS)
mr_emit_kernel(const uint32_t* __restrict__ words, int64_t L, int n_chunks, const uint32_t* __restrict__ masks,
               const uint32_t* __restrict__ cumul, const MrState* __restrict__ st, int64_t n, float* __restrict__ out,
               double* __restrict__ gauss) {
    const int lane = threadIdx.x & 31;
    const int c = blockIdx.x * MR_EMIT_WARPS + (threadIdx.x >> 5);
    if (c >= n_chunks) return;
    const int c0 = st->c0, ph = st->ph;
    const uint32_t a_lo = (uint32_t)st->a_lo, a_hi = (uint32_t)(L * (MT_NW / 4));
    const long long A = (n - c0 + 1) >> 1;
    const long long r0 = st->base + cumul[(size_t)ph * n_chunks + c];
    if (r0 >= A) return;                                       // the call's values end before this chunk
    const uint32_t m = masks[((size_t)ph * n_chunks + c) * 32 + lane];
    int inc = __popc(m);
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int up = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc += up;
    }
    const int excl = inc - __popc(m);
    const uint32_t below = (1u << lane) - 1u;
    const uint32_t* __restrict__ wc = words + (size_t)c * MJ_CW + ph + 4 * lane;
    for (int j = 0; j < 32; ++j) {
        const uint32_t mj = __shfl_sync(0xffffffffu, m, j);
        const long long r = r0 + __shfl_sync(0xffffffffu, excl, j) + __popc(mj & below);
        const uint32_t a = ((uint32_t)c << 10) + 32u * (uint32_t)j + (uint32_t)lane;
        if (!((mj >> lane) & 1u) || a < a_lo || a >= a_hi || r < 0 || r >= A) continue;
        const uint32_t* __restrict__ wp = wc + 128 * j;
        const double2 g = mt19937_polar_pair(__ldg(wp), __ldg(wp + 1), __ldg(wp + 2), __ldg(wp + 3));
        const long long v = c0 + 2 * r;
        out[v] = (float)g.x;
        if (v + 1 < n) out[v + 1] = (float)g.y;
        else *gauss = g.y;                                     // value n: the cache the stream hands back
    }
}

// The windows of one es_randn call: each covers L = n_seg << lb blocks of its own; together they cover the mean + 12 sigma of
// the words n values can take (~2.55 words per value), so the last window's prefix shows whether the draw was complete.
struct MrWindow { int n_seg, lb; long long L, n_chunks; };
struct MrPlan {
    std::vector<MrWindow> win;
    // scratch: the window's words (+ a chunk of padding: mt_flags_kernel reads past every attempt start) | accept masks
    //          [phase][chunk][32] | chunk counts -> prefixes [phase][chunk] | the next window's key | segment order | MrState
    size_t words_bytes, mask_bytes, cnt_bytes, key_bytes, ord_bytes, bytes;
};

std::vector<MrWindow> mr_windows(const es_ctx* ctx, int64_t n) {
    const double p_acc = 0.78539816339744830962, n_acc = (double)((n + 1) / 2);
    const double words_max = 2.0 * MT_NW + 4.0 * (n_acc / p_acc + 12.0 * sqrt(n_acc * (1.0 - p_acc)) / p_acc + 64.0);
    long long left = (long long)(words_max / MT_NW) + 1;
    long long per = MR_WINDOW_BLOCKS;
    const char* ew = getenv("ES_RANDN_WINDOW_BLOCKS");          // (tests: many small windows)
    if (ew) per = atoll(ew);
    if (per < 1) per = 1;
    if (per > (1LL << (MJ_BITS_RANGE - 1))) per = 1LL << (MJ_BITS_RANGE - 1);
    std::vector<MrWindow> win;
    while (left > 0) {
        const long long want = left < per ? left : per;
        int lb = mj_segment_lb(1, want, ctx->sm_count);
        while (((want + (1LL << lb) - 1) >> lb) > 65535) ++lb;                 // (mj_order_kernel: 16-bit segment numbers)
        MrWindow wd;
        wd.lb = lb;
        wd.n_seg = (int)((want + (1LL << lb) - 1) >> lb);
        wd.L = (long long)wd.n_seg << lb;
        wd.n_chunks = ((1 + wd.L) * MT_NW + MJ_CW - 1) / MJ_CW;
        win.push_back(wd);
        left -= wd.L;
    }
    return win;
}

MrPlan mr_plan(const es_ctx* ctx, int64_t n) {
    MrPlan pl;
    pl.win = mr_windows(ctx, n);
    long long nc = 0, ns = 0;
    for (const MrWindow& w : pl.win) { nc = w.n_chunks > nc ? w.n_chunks : nc; ns = w.n_seg > ns ? w.n_seg : ns; }
    pl.words_bytes = mg_pad((size_t)(nc + 1) * MJ_CW * sizeof(uint32_t));
    pl.mask_bytes = mg_pad((size_t)4 * nc * 32 * sizeof(uint32_t));
    pl.cnt_bytes = mg_pad((size_t)4 * nc * sizeof(uint32_t));
    pl.key_bytes = mg_pad(MT_NW * sizeof(uint32_t));
    pl.ord_bytes = mg_pad((size_t)ns * sizeof(uint16_t));
    pl.bytes = pl.words_bytes + pl.mask_bytes + pl.cnt_bytes + pl.key_bytes + pl.ord_bytes + mg_pad(sizeof(MrState));
    return pl;
}

}  // namespace

int es_impl_randn_plan(const es_ctx* ctx, int64_t n, size_t* scratch_bytes, int* n_windows) {
    const MrPlan pl = mr_plan(ctx, n);
    *scratch_bytes = pl.bytes;
    *n_windows = (int)pl.win.size();
    return ES_OK;
}

int es_impl_randn(es_ctx* ctx, uint32_t* mt_key, int32_t* mt_pos, int32_t* has_gauss, double* gauss, int64_t n, float* out,
                  cudaStream_t stream) {
    const MrPlan pl = mr_plan(ctx, n);
    const std::vector<MrWindow>& win = pl.win;
    void* scratch = nullptr;
    int rc = es_ctx_scratch(ctx, pl.bytes, &scratch);
    if (rc) return rc;
    char* at = (char*)scratch;
    uint32_t* words = (uint32_t*)at; at += pl.words_bytes;
    uint32_t* masks = (uint32_t*)at; at += pl.mask_bytes;
    uint32_t* counts = (uint32_t*)at; at += pl.cnt_bytes;
    uint32_t* key_next = (uint32_t*)at; at += pl.key_bytes;
    uint16_t* order = (uint16_t*)at; at += pl.ord_bytes;
    MrState* st = (MrState*)at;
    for (size_t w = 0; w < win.size(); ++w) {
        const MrWindow& wd = win[w];
        const int n_chunks = (int)wd.n_chunks;
        rc = mj_launch_fill(ctx, w == 0 ? mt_key : key_next, 1, wd.n_seg, wd.lb, order, words, (size_t)(n_chunks + 1) * MJ_CW, stream);
        if (rc) return rc;
        mt_flags_kernel<<<dim3((unsigned)((n_chunks + MFL_WARPS - 1) / MFL_WARPS), 1), 32 * MFL_WARPS, 0, stream>>>(
            words, (size_t)(n_chunks + 1) * MJ_CW, n_chunks, masks, counts);
        ES_LAUNCHED(ctx);
        mt_scan_kernel<<<4, 1024, 0, stream>>>(counts, n_chunks);                 // (the phase is only known on the device)
        ES_LAUNCHED(ctx);
        mr_window_kernel<<<1, 32, 0, stream>>>((int)w, w + 1 == win.size(), wd.L, words, n_chunks, masks, counts, key_next, mt_key,
                                               mt_pos, has_gauss, gauss, n, out, st, ctx->err_dev);
        ES_LAUNCHED(ctx);
        mr_emit_kernel<<<(unsigned)((n_chunks + MR_EMIT_WARPS - 1) / MR_EMIT_WARPS), 32 * MR_EMIT_WARPS, 0, stream>>>(
            words, wd.L, n_chunks, masks, counts, st, n, out, gauss);
        ES_LAUNCHED(ctx);
    }
    return ES_OK;
}

// The stream walk consumes words only for the steps that run, so its bound is the no-fall consumption: mg_plan's sizing with
// the jump-ahead fill always (the walk reads the words directly, no accept masks or prefixes)
static bool sw_fits(long long blocks, long long n_streams, int sm_count, int* lb, long long* n_seg) {
    *lb = mj_segment_lb(n_streams, blocks, sm_count);
    // mj_segment_lb lengthens the segments until the fill has at most ~4 per SM; with more streams than that it would stop
    // only at its maximum, and every stream would be generated that long.  A segment longer than the stream's need buys no
    // parallelism: at most ceil(log2(blocks)), so the words generated stay under twice the bound
    int need = 0;
    while ((1LL << need) < blocks) ++need;
    if (*lb > need) *lb = need;
    *n_seg = (blocks + (1LL << *lb) - 1) >> *lb;
    return ((*n_seg << *lb) >> MJ_BITS_RANGE) == 0 && *n_seg <= 65535;
}

int es_impl_stream_words_plan(const es_ctx* ctx, const char* fn, int n_streams, int n_pairs, int coins, int N, EsStreamWords* pl) {
    const long long blocks = mg_blocks_needed(n_pairs, coins, N);
    int lb = 0;
    long long n_seg = 0;
    if (!sw_fits(blocks, n_streams, ctx->sm_count, &lb, &n_seg)) {
        int lo = 0, hi = n_pairs;                                  // the most pairs per stream that fit
        while (lo < hi) {
            const int mid = lo + (hi - lo + 1) / 2;
            int l2;
            long long s2;
            if (sw_fits(mg_blocks_needed(mid, coins, N), n_streams, ctx->sm_count, &l2, &s2)) lo = mid; else hi = mid - 1;
        }
        const long long pairs = (long long)n_streams * n_pairs;
        if (lo == 0)
            es_set_error("%s: one pair of %d gaussians per evaluation needs %lld blocks of 624 words, beyond the jump-ahead "
                         "range of 2^%d blocks per stream: no number of streams fits; use fewer episodes or steps", fn, N,
                         mg_blocks_needed(1, coins, N), MJ_BITS_RANGE);
        else
            es_set_error("%s: %d pairs per stream need %lld blocks of 624 words each (%d gaussians per evaluation), beyond the "
                         "jump-ahead range of 2^%d blocks per stream; at most %d pairs per stream fit, so the %lld pairs need "
                         "at least %lld streams", fn, n_pairs, blocks, N, MJ_BITS_RANGE, lo, pairs, (pairs + lo - 1) / lo);
        return ES_ERR_UNSUPPORTED;
    }
    pl->lb_log2 = lb;
    pl->n_seg = (int)n_seg;
    const size_t gen_words = (size_t)(1 + (n_seg << lb)) * MT_NW;
    const size_t n_chunks = (gen_words + MJ_CW - 1) / MJ_CW;
    pl->stride_words = (n_chunks + 1) * MJ_CW;                   // (+ a chunk: the walk stages up to 256 words past its cursor)
    pl->limit = (uint32_t)(gen_words - 8);
    pl->words_bytes = mg_pad((size_t)n_streams * pl->stride_words * sizeof(uint32_t));
    pl->order_bytes = mg_pad((size_t)n_seg * sizeof(uint16_t));
    return ES_OK;
}

int es_impl_stream_words_fill(es_ctx* ctx, const uint32_t* mt_key, int n_streams, const EsStreamWords& pl, uint32_t* words,
                              uint16_t* order, cudaStream_t stream) {
    return mj_launch_fill(ctx, mt_key, n_streams, pl.n_seg, pl.lb_log2, order, words, pl.stride_words, stream);
}

int es_impl_draw_noisy(es_ctx* ctx, uint32_t* mt_key, int32_t* mt_pos, int32_t* has_gauss, double* gauss, int n_streams,
                       int n_per_stream, uint64_t upper_bound, int coins, int normals_per_eval, double scale, int64_t* idx_out,
                       uint32_t* extra_out, float* noise_out, cudaStream_t stream) {
    const Mt19937Bound bd = mt19937_randint_bound(upper_bound);
    if (bd.rng == 0) {
        es_set_error("es_draw_noisy: upper_bound == 1 is not supported");
        return ES_ERR_UNSUPPORTED;
    }
    MgPlan pl;
    const int rc = mg_plan(ctx, n_streams, n_per_stream, coins, normals_per_eval, pl);
    if (rc) return rc;
    const MgDraw d = {mt_key, mt_pos, has_gauss, gauss, n_streams, n_per_stream, bd.rng, bd.mask, coins, normals_per_eval, scale,
                      idx_out, extra_out, noise_out};
    return pl.jump ? mg_launch_jump(ctx, d, pl, stream) : mg_launch_sequential(ctx, d, stream);
}
