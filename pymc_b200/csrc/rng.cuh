// Device random streams.
//
//  * Pcg64: bit-exact replica of NumPy's PCG64 (128-bit LCG, XSL-RR output) so the on-device tree
//    consumes the chain's `step` stream exactly as `rng.random()` does in the reference
//    (hmc/nuts.py:215, :371, :466 -- the order is specified in SURVEY.md 8a row a15).
//    numpy.random.Generator.random() == (next_uint64 >> 11) * 2^-53.
//  * philox_normal: Philox4x32-10 + Box-Muller for the momentum noise when the caller does not supply
//    NumPy normals (NumPy's 256-layer ziggurat is not replicated on device; see DESIGN.md).
#pragma once
#include <stdint.h>

namespace b200 {

struct Pcg64 {
    unsigned __int128 state;
    unsigned __int128 inc;

    __host__ __device__ __forceinline__ void load(uint64_t shi, uint64_t slo, uint64_t ihi, uint64_t ilo) {
        state = ((unsigned __int128)shi << 64) | slo;
        inc = ((unsigned __int128)ihi << 64) | ilo;
    }
    __host__ __device__ __forceinline__ uint64_t next_u64() {
        // PCG_DEFAULT_MULTIPLIER_128 = 0x2360ED051FC65DA4 4385DF649FCCF645
        const unsigned __int128 mult =
            ((unsigned __int128)0x2360ED051FC65DA4ULL << 64) | 0x4385DF649FCCF645ULL;
        state = state * mult + inc;
        const uint64_t hi = (uint64_t)(state >> 64), lo = (uint64_t)state;
        const uint64_t x = hi ^ lo;
        const unsigned rot = (unsigned)(hi >> 58);
        return (x >> rot) | (x << ((-rot) & 63));
    }
    __host__ __device__ __forceinline__ double next_double() {
        return (double)(next_u64() >> 11) * (1.0 / 9007199254740992.0);
    }
};

// ---- Philox4x32-10 (Salmon et al. 2011) ------------------------------------------------------
__host__ __device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                                       uint32_t k0, uint32_t k1, uint32_t out[4]) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint64_t p0 = (uint64_t)M0 * c0, p1 = (uint64_t)M1 * c2;
        const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0;
        const uint32_t n1 = (uint32_t)p1;
        const uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
        const uint32_t n3 = (uint32_t)p0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += W0; k1 += W1;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// One standard normal for (chain, draw, element) under a 64-bit key: counter-based, so any team
// layout produces the same stream.  u1 in (0,1], u2 in [0,1): z = sqrt(-2 ln u1) cos(2 pi u2).
__device__ __forceinline__ double philox_normal(uint64_t key, uint32_t chain, uint32_t draw, uint32_t elem) {
    uint32_t o[4];
    philox4x32_10(elem, draw, chain, 0x4e555453u /* "NUTS" */, (uint32_t)key, (uint32_t)(key >> 32), o);
    const uint64_t a = ((uint64_t)o[0] << 32) | o[1], b = ((uint64_t)o[2] << 32) | o[3];
    const double u1 = ((double)(a >> 11) + 1.0) * (1.0 / 9007199254740992.0);
    const double u2 = (double)(b >> 11) * (1.0 / 9007199254740992.0);
    double s, c;
    sincospi(2.0 * u2, &s, &c);
    return sqrt(-2.0 * log(u1)) * c;
}

// The same draw from one out-of-line copy: a caller that unrolls its element loop holds the Philox rounds, log, sincospi
// and sqrt once instead of once per element.
__device__ __noinline__ double philox_normal_call(uint64_t key, uint32_t chain, uint32_t draw, uint32_t elem) {
    return philox_normal(key, chain, draw, elem);
}

}  // namespace b200
