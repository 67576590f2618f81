// Host float -> e4m3 (OCP FP8 E4M3 "fn": bias 7, no infinities, S.1111.111 = NaN, largest finite 448) for the packed
// weights of PE_PREC_E4M3X1.  Round to nearest, ties to even.  Where the result stays within +-448 it equals torch's
// float8_e4m3fn cast bit for bit; larger magnitudes saturate to +-448, as cvt.rn.satfinite does on the device (torch gives
// NaN there).  Plain C++ without CUDA, so that a CPU test compiles it on its own.
#pragma once
#include <math.h>
#include <stdint.h>

namespace pe {

inline uint8_t float_to_e4m3(float x) {
    const uint8_t sign = signbit(x) ? 0x80 : 0x00;
    if (isnan(x)) return sign | 0x7F;
    const double a = fabs((double)x);
    if (a >= 448.0) return sign | 0x7E;   // saturation (also the values that round up to 448 from below)
    // quantum of the binade: 2^(e - 3) for normal values (e >= -6), 2^-9 for the subnormals
    int e = 0;
    frexp(a, &e);                         // a = f * 2^e, f in [0.5, 1): the binade [2^(e-1), 2^e)
    const int q = (a == 0.0 || e - 1 < -6) ? -9 : e - 1 - 3;
    const double m = nearbyint(ldexp(a, -q));   // ties to even (default rounding mode); exact: m < 2^5
    const double r = ldexp(m, q);
    if (r >= 448.0) return sign | 0x7E;   // [448, 464) rounds to 448; 464 (a tie) goes to the even 448
    if (r < 0.015625) return sign | (uint8_t)m;   // subnormal (m = 0..7), or m = 8 = 2^-6, encoded as 0x08 all the same
    int re = 0;
    const double f = frexp(r, &re);       // r = f * 2^re, f in [0.5, 1)
    const int exp_field = re - 1 + 7;
    const int mant = (int)ldexp(f * 2.0 - 1.0, 3);
    return sign | (uint8_t)((exp_field << 3) | mant);
}

}  // namespace pe
