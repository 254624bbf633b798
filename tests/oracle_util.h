/* oracle_util.h -- the pure helpers the C oracles under tests/ share: fp16 to float, float bit casts, the device's affine product and a
 * three-term dot product; test infrastructure only.  static inline, so that an oracle that uses only some of them compiles without
 * unused-function warnings. */
#ifndef ORACLE_UTIL_H
#define ORACLE_UTIL_H

#include <math.h>
#include <stdint.h>
#include <string.h>

/* IEEE half -> float, exact */
static inline float half_to_float(uint16_t h)
{
    const uint32_t sign = (uint32_t)(h & 0x8000u) << 16, exp = (h >> 10) & 0x1fu, man = h & 0x3ffu;
    uint32_t bits;
    if (exp == 0) {
        if (man == 0) bits = sign;
        else {                                              /* subnormal: man * 2^-24, exact in float */
            const float f = (float)man * (1.0f / 16777216.0f);
            memcpy(&bits, &f, 4);
            bits |= sign;
        }
    } else if (exp == 31) bits = sign | 0x7f800000u | (man << 13);
    else bits = sign | ((exp + 112u) << 23) | (man << 13);
    float out;
    memcpy(&out, &bits, 4);
    return out;
}

static inline uint32_t float_bits(float f)
{
    uint32_t u;
    memcpy(&u, &f, 4);
    return u;
}

static inline float bits_float(uint32_t u)
{
    float f;
    memcpy(&f, &u, 4);
    return f;
}

/* a12: R row-major then t; out = R p + t as the device's aff_mul forms it: fma(r.x, p.x, fma(r.y, p.y, r.z * p.z)) + t */
static inline void aff_apply(const float *a12, const float *p, float *out)
{
    for (int c = 0; c < 3; ++c) out[c] = fmaf(a12[3 * c], p[0], fmaf(a12[3 * c + 1], p[1], a12[3 * c + 2] * p[2])) + a12[9 + c];
}

static inline float dot(const float *a, const float *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

#endif
