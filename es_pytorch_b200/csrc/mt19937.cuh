// mt19937.cuh -- the MT19937 generator and the legacy numpy RandomState draws built on it, bit-exact with numpy (sm_90a): the
// state recurrence and tempering, the randint bound, random_sample and the polar-method gaussian.  Used by mt_draw.cu,
// mt_gauss.cu and by the kernels that read the save_obs coins (elementwise.cu, rollout_closed.cu).
#pragma once
#include <stdint.h>

constexpr int MT_NW = 624, MT_MW = 397, MT_DW = MT_NW - MT_MW;      // state words, middle word, 227

__device__ __forceinline__ uint32_t mt19937_twist(uint32_t u, uint32_t v) {
    const uint32_t y = (u & 0x80000000u) | (v & 0x7FFFFFFFu);
    return (y >> 1) ^ ((y & 1u) ? 0x9908B0DFu : 0u);
}
__device__ __forceinline__ uint32_t mt19937_temper(uint32_t y) {
    y ^= y >> 11;
    y ^= (y << 7) & 0x9D2C5680u;
    y ^= (y << 15) & 0xEFC60000u;
    y ^= y >> 18;
    return y;
}
// the inverse of the tempering (a bijection of 32-bit words): the raw state word behind an output word
__device__ __forceinline__ uint32_t mt19937_untemper(uint32_t y) {
    y ^= y >> 18;
    y ^= (y << 15) & 0xEFC60000u;
    uint32_t t = y;                                   // undo y ^= (y << 7) & B: 7 bits are recovered per round
    t = y ^ ((t << 7) & 0x9D2C5680u);
    t = y ^ ((t << 7) & 0x9D2C5680u);
    t = y ^ ((t << 7) & 0x9D2C5680u);
    t = y ^ ((t << 7) & 0x9D2C5680u);
    y = t;
    t = y;                                            // undo y ^= y >> 11: 11 bits per round
    t = y ^ (t >> 11);
    t = y ^ (t >> 11);
    return t;
}

// The next block from the old one without the recurrence's three dependent phases.  N[i] = N[i-227] ^ tw(O[i], O[i+1]) is
// XOR-linear in its first term, so with the 623 twists T[k] = tw(O[k], O[k+1]) of the OLD block (and T[623] = 0) every new
// word is a few XORs of old words and twists:
//   i <  227:  N[i] = O[i+397] ^ T[i]
//   i <  454:  N[i] = O[i+170] ^ T[i-227] ^ T[i]
//   i <  623:  N[i] = O[i-57]  ^ T[i-454] ^ T[i-227] ^ T[i]
//   N[623] = N[396] ^ tw(O[623], N[0])
// N[i] = O[o] ^ T[a] ^ T[b] ^ T[c] for 0 <= i <= 622 (an unused twist index points at T[623]); plain == false: no word, the
// taps O[0] ^ T[623] ^ T[623] ^ T[623]
struct Mt19937Taps { int o, a, b, c; };
__device__ __forceinline__ Mt19937Taps mt19937_taps(int i, bool plain = true) {
    Mt19937Taps m;
    m.o = !plain ? 0 : (i < MT_DW ? i + MT_MW : i < 2 * MT_DW ? i + MT_MW - MT_DW : i + MT_MW - 2 * MT_DW);
    m.a = plain ? i : MT_NW - 1;
    m.b = (plain && i >= MT_DW) ? i - MT_DW : MT_NW - 1;
    m.c = (plain && i >= 2 * MT_DW) ? i - 2 * MT_DW : MT_NW - 1;
    return m;
}
__device__ __forceinline__ uint32_t mt19937_last_word(const uint32_t* __restrict__ O, const uint32_t* __restrict__ T) {   // N[623]
    const uint32_t n0 = O[MT_MW] ^ T[0];
    const uint32_t n396 = O[396 + MT_MW - MT_DW] ^ T[396 - MT_DW] ^ T[396];
    return n396 ^ mt19937_twist(O[MT_NW - 1], n0);
}

// Thread <-> word map of the two-barrier block regeneration by one CTA (needs >= 705 threads): every warp stays inside one of
// the three ranges above and all three ranges run the SAME code; the odd word out has a warp of its own: threads
// 0-226 | 256-482 | 512-680 | 704.  init() once per kernel: the taps stay in registers.
struct Mt19937Regen {
    int my_i;                                         // the word this thread forms, -1: none
    bool plain;                                       // my_i < 623
    Mt19937Taps tp;
    __device__ __forceinline__ void init(int tid) {
        my_i = (tid < 256) ? (tid < MT_DW ? tid : -1) : (tid < 512) ? (tid - 256 < MT_DW ? tid - 256 + MT_DW : -1)
             : (tid < 704) ? (tid - 512 < MT_NW - 1 - 2 * MT_DW ? tid - 512 + 2 * MT_DW : -1) : (tid == 704 ? MT_NW - 1 : -1);
        plain = my_i >= 0 && my_i < MT_NW - 1;
        tp = mt19937_taps(my_i, plain);
    }
    // the new word of a plain thread after the twists of O are in T (thread 704: mt19937_last_word); call between two barriers
    __device__ __forceinline__ uint32_t word(const uint32_t* __restrict__ O, const uint32_t* __restrict__ T) const {
        return O[tp.o] ^ T[tp.a] ^ T[tp.b] ^ T[tp.c];
    }
};

// randint(0, upper_bound) for ranges < 2^32 (numpy's buffered_bounded_masked_uint32): rng = upper_bound - 1 and the smallest
// all-ones mask >= rng; a word w gives the index w & mask when that is <= rng, otherwise the next word is tried
struct Mt19937Bound { uint32_t rng, mask; };
inline Mt19937Bound mt19937_randint_bound(uint64_t upper_bound) {
    Mt19937Bound b;
    b.rng = (uint32_t)(upper_bound - 1);
    uint32_t mask = b.rng;
    mask |= mask >> 1; mask |= mask >> 2; mask |= mask >> 4; mask |= mask >> 8; mask |= mask >> 16;
    b.mask = mask;
    return b;
}

// random_sample (numpy's legacy_double): two words -> (a >> 5) * 2^26 + (b >> 6), a 53-bit integer, over 2^53: [0, 1)
__device__ __forceinline__ double mt19937_random_sample(uint32_t a, uint32_t b) {
    return ((double)(a >> 5) * 67108864.0 + (double)(b >> 6)) / 9007199254740992.0;
}

// randn, numpy's legacy_gauss (the polar method): an attempt is four words, two doubles u; x1, x2 = 2 u - 1 until
// r2 = x1^2 + x2^2 is in (0, 1).  The 53-bit integer of u converts exactly and one fused multiply-add rounds the exact value
// of 2 u - 1 once, like the reference's (2.0 * u) - 1.0 (2 u is exact); r2 with two roundings as in C.
struct Mt19937Polar { double x1, x2, r2; };
__device__ __forceinline__ Mt19937Polar mt19937_polar(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3) {
    Mt19937Polar p;
    const double v1 = fma((double)(w0 >> 5), 67108864.0, (double)(w1 >> 6));
    const double v2 = fma((double)(w2 >> 5), 67108864.0, (double)(w3 >> 6));
    p.x1 = fma(v1, 1.0 / 4503599627370496.0, -1.0);
    p.x2 = fma(v2, 1.0 / 4503599627370496.0, -1.0);
    p.r2 = __dadd_rn(__dmul_rn(p.x1, p.x1), __dmul_rn(p.x2, p.x2));
    return p;
}
__device__ __forceinline__ bool mt19937_polar_accept(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3) {
    const Mt19937Polar p = mt19937_polar(w0, w1, w2, w3);
    return p.r2 < 1.0 && p.r2 != 0.0;
}
// the two gaussians of an accepted attempt, f = sqrt(-2 log(r2) / r2): .x = f x2 is returned first, .y = f x1 is the one numpy
// caches for the next call
__device__ __forceinline__ double2 mt19937_polar_pair(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3) {
    const Mt19937Polar p = mt19937_polar(w0, w1, w2, w3);
    const double f = sqrt(__ddiv_rn(__dmul_rn(-2.0, log(p.r2)), p.r2));
    return make_double2(__dmul_rn(f, p.x2), __dmul_rn(f, p.x1));
}
