// Python's repr() of a float32 widened to double, as device code: the shortest decimal that reads back as the same
// double (the closest such decimal when there are several), printed the way float.__repr__ prints it.
//
//   digits:  Ryu's d2d (Ulf Adams, "Ryu: fast float-to-string conversion", PLDI 2018) on the 53-bit mantissa, with
//            128-bit products from two 64x64 multiplies (__umul64hi on the device). The power-of-5 multipliers cover
//            only the binary exponents a float32 can reach (pow5_tables.cuh, written by make_pow5_tables.py).
//   layout:  float_repr_style 'short' with the 'r' format code: scientific notation when the decimal point position
//            decpt (value = 0.D * 10^decpt) is <= -4 or > 16, i.e. below 1e-4 and from 1e16 up; otherwise positional
//            with at least one digit after the point ("1.0", "0.0001"). The exponent has a sign and at least two
//            digits ("1e-05", "1e+16"). Zeros print as "0.0" / "-0.0", infinities as "inf" / "-inf", every NaN as
//            "nan".
//
// Header-only and __host__ __device__ so that a host build of the same code can be checked against CPython on whole
// binades (tests/test_sinks_text.py); the shared library itself only instantiates it in device code.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define V2E_HD __host__ __device__ __forceinline__
#define V2E_TABLE __device__
#else
#define V2E_HD static inline
#define V2E_TABLE static
#endif

#include "pow5_tables.cuh"

namespace v2e_repr {

V2E_HD uint64_t umulhi(uint64_t a, uint64_t b) {
#ifdef __CUDA_ARCH__
    return __umul64hi(a, b);
#else
    return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}

V2E_HD uint32_t pow5bits(int32_t e) { return (uint32_t)(((e * 1217359) >> 19) + 1); }   // bit length of 5^e
V2E_HD uint32_t log10_pow2(int32_t e) { return (uint32_t)((e * 78913) >> 18); }         // floor(e log10 2)
V2E_HD uint32_t log10_pow5(int32_t e) { return (uint32_t)((e * 732923) >> 20); }        // floor(e log10 5)

V2E_HD bool multiple_of_pow5(uint64_t v, uint32_t p) {
    uint32_t count = 0;
    while (v % 5 == 0 && v != 0) {
        v /= 5;
        ++count;
    }
    return count >= p;
}

V2E_HD bool multiple_of_pow2(uint64_t v, uint32_t p) { return (v & ((1ull << p) - 1)) == 0; }

// (m * mul) >> j for a 128-bit mul = {lo, hi}; m < 2^55 and 64 < j < 128 over the float32 range
V2E_HD uint64_t mul_shift(uint64_t m, const uint64_t *mul, int32_t j) {
    const uint64_t b0_hi = umulhi(m, mul[0]);
    const uint64_t b2_lo = m * mul[1], b2_hi = umulhi(m, mul[1]);
    const uint64_t s_lo = b2_lo + b0_hi;
    const uint64_t s_hi = b2_hi + (s_lo < b0_hi);
    const int32_t d = j - 64;
    return (s_hi << (64 - d)) | (s_lo >> d);
}

// Shortest decimal digits of a finite, nonzero, positive double given by its biased exponent and 52-bit mantissa:
// value ~ output * 10^e10, output < 10^17.
V2E_HD void d2d(uint64_t ieee_mantissa, uint32_t ieee_exponent, uint64_t *output_out, int32_t *e10_out) {
    int32_t e2;
    uint64_t m2;
    if (ieee_exponent == 0) {
        e2 = 1 - 1023 - 52 - 2;
        m2 = ieee_mantissa;
    } else {
        e2 = (int32_t)ieee_exponent - 1023 - 52 - 2;
        m2 = (1ull << 52) | ieee_mantissa;
    }
    const bool accept_bounds = (m2 & 1) == 0;
    const uint64_t mv = 4 * m2;
    const uint32_t mm_shift = ieee_mantissa != 0 || ieee_exponent <= 1;
    uint64_t vr, vp, vm;
    int32_t e10;
    bool vm_trailing_zeros = false, vr_trailing_zeros = false;
    if (e2 >= 0) {
        const uint32_t q = log10_pow2(e2) - (e2 > 3);
        e10 = (int32_t)q;
        const int32_t k = V2E_POW5_INV_BITCOUNT + (int32_t)pow5bits((int32_t)q) - 1;
        const int32_t i = -e2 + (int32_t)q + k;
        const uint64_t *mul = V2E_POW5_INV_SPLIT[q];
        vr = mul_shift(4 * m2, mul, i);
        vp = mul_shift(4 * m2 + 2, mul, i);
        vm = mul_shift(4 * m2 - 1 - mm_shift, mul, i);
        if (q <= 21) {
            const uint32_t mv_mod5 = (uint32_t)(mv % 5);
            if (mv_mod5 == 0) vr_trailing_zeros = multiple_of_pow5(mv, q);
            else if (accept_bounds) vm_trailing_zeros = multiple_of_pow5(mv - 1 - mm_shift, q);
            else vp -= multiple_of_pow5(mv + 2, q);
        }
    } else {
        const uint32_t q = log10_pow5(-e2) - (-e2 > 1);
        e10 = (int32_t)q + e2;
        const int32_t i = -e2 - (int32_t)q;
        const int32_t k = (int32_t)pow5bits(i) - V2E_POW5_BITCOUNT;
        const int32_t j = (int32_t)q - k;
        const uint64_t *mul = V2E_POW5_SPLIT[i];
        vr = mul_shift(4 * m2, mul, j);
        vp = mul_shift(4 * m2 + 2, mul, j);
        vm = mul_shift(4 * m2 - 1 - mm_shift, mul, j);
        if (q <= 1) {
            vr_trailing_zeros = true;
            if (accept_bounds) vm_trailing_zeros = mm_shift == 1;
            else --vp;
        } else if (q < 63) {
            vr_trailing_zeros = multiple_of_pow2(mv, q);
        }
    }
    // drop digits while the interval (vm, vp) still holds a shorter number
    int32_t removed = 0;
    uint8_t last_removed = 0;
    uint64_t output;
    if (vm_trailing_zeros || vr_trailing_zeros) {
        for (;;) {
            const uint64_t vp10 = vp / 10, vm10 = vm / 10;
            if (vp10 <= vm10) break;
            const uint32_t vm_mod10 = (uint32_t)(vm - 10 * vm10);
            const uint64_t vr10 = vr / 10;
            const uint32_t vr_mod10 = (uint32_t)(vr - 10 * vr10);
            vm_trailing_zeros &= vm_mod10 == 0;
            vr_trailing_zeros &= last_removed == 0;
            last_removed = (uint8_t)vr_mod10;
            vr = vr10;
            vp = vp10;
            vm = vm10;
            ++removed;
        }
        if (vm_trailing_zeros) {
            for (;;) {
                const uint64_t vm10 = vm / 10;
                const uint32_t vm_mod10 = (uint32_t)(vm - 10 * vm10);
                if (vm_mod10 != 0) break;
                const uint64_t vp10 = vp / 10, vr10 = vr / 10;
                const uint32_t vr_mod10 = (uint32_t)(vr - 10 * vr10);
                vr_trailing_zeros &= last_removed == 0;
                last_removed = (uint8_t)vr_mod10;
                vr = vr10;
                vp = vp10;
                vm = vm10;
                ++removed;
            }
        }
        if (vr_trailing_zeros && last_removed == 5 && vr % 2 == 0) last_removed = 4;   // exact half: round to even
        output = vr + ((vr == vm && (!accept_bounds || !vm_trailing_zeros)) || last_removed >= 5);
    } else {
        bool round_up = false;
        const uint64_t vp100 = vp / 100, vm100 = vm / 100;
        if (vp100 > vm100) {
            const uint64_t vr100 = vr / 100;
            round_up = (uint32_t)(vr - 100 * vr100) >= 50;
            vr = vr100;
            vp = vp100;
            vm = vm100;
            removed += 2;
        }
        for (;;) {
            const uint64_t vp10 = vp / 10, vm10 = vm / 10;
            if (vp10 <= vm10) break;
            const uint64_t vr10 = vr / 10;
            round_up = (uint32_t)(vr - 10 * vr10) >= 5;
            vr = vr10;
            vp = vp10;
            vm = vm10;
            ++removed;
        }
        output = vr + (vr == vm || round_up);
    }
    *output_out = output;
    *e10_out = e10 + removed;
}

V2E_HD uint32_t decimal_length17(uint64_t v) {
    uint32_t n = 1;
    for (uint64_t p = 10; n < 17 && v >= p; p *= 10) ++n;
    return n;
}

enum Kind : uint8_t { FINITE = 0, ZERO = 1, INF = 2, NAN_ = 3 };

// What repr() prints for one double: its sign, kind and (finite, nonzero) digits with the decimal point position.
struct Repr {
    uint64_t digits;     // shortest digits, no trailing zeros
    int32_t ndigits;     // 1..17
    int32_t decpt;       // value = 0.<digits> * 10^decpt
    uint8_t kind;
    uint8_t neg;
};

V2E_HD Repr repr_prepare(uint64_t bits) {
    Repr r;
    r.neg = (uint8_t)(bits >> 63);
    const uint64_t mant = bits & ((1ull << 52) - 1);
    const uint32_t expo = (uint32_t)((bits >> 52) & 0x7ff);
    r.digits = 0;
    r.ndigits = 1;
    r.decpt = 1;
    if (expo == 0x7ff) {
        r.kind = mant ? NAN_ : INF;
        if (mant) r.neg = 0;                 // repr(float('-nan')) == 'nan'
    } else if (expo == 0 && mant == 0) {
        r.kind = ZERO;
    } else {
        int32_t e10;
        r.kind = FINITE;
        d2d(mant, expo, &r.digits, &e10);
        r.ndigits = (int32_t)decimal_length17(r.digits);
        r.decpt = r.ndigits + e10;
    }
    return r;
}

V2E_HD bool repr_scientific(const Repr &r) { return r.decpt <= -4 || r.decpt > 16; }

V2E_HD int32_t uint_length(uint32_t v) {
    int32_t n = 1;
    while (v >= 10) {
        v /= 10;
        ++n;
    }
    return n;
}

// Bytes repr() prints (at most 24).
V2E_HD int32_t repr_length(const Repr &r) {
    const int32_t s = r.neg;
    if (r.kind == ZERO) return s + 3;                    // 0.0
    if (r.kind == INF || r.kind == NAN_) return s + 3;
    const int32_t n = r.ndigits, d = r.decpt;
    if (repr_scientific(r)) {
        const int32_t x = d - 1 < 0 ? 1 - d : d - 1;
        return s + n + (n > 1) + 2 + (x < 10 ? 2 : uint_length((uint32_t)x));
    }
    if (d <= 0) return s + 2 - d + n;                    // 0.000ddd
    if (d < n) return s + n + 1;                         // dd.ddd
    return s + d + 2;                                    // ddd000.0
}

// Writes the n decimal digits of v ending just before dst + n.
template <typename Out>
V2E_HD void put_digits(Out dst, uint64_t v, int32_t n) {
    for (int32_t k = n - 1; k >= 0; --k) {
        const uint64_t q = v / 10;
        dst[k] = (char)('0' + (uint32_t)(v - 10 * q));
        v = q;
    }
}

// Writes repr_length(r) bytes at dst (a char pointer into any memory space).
template <typename Out>
V2E_HD int32_t repr_write(const Repr &r, Out dst) {
    int32_t o = 0;
    if (r.neg) dst[o++] = '-';
    if (r.kind == ZERO) {
        dst[o] = '0'; dst[o + 1] = '.'; dst[o + 2] = '0';
        return o + 3;
    }
    if (r.kind == INF) {
        dst[o] = 'i'; dst[o + 1] = 'n'; dst[o + 2] = 'f';
        return o + 3;
    }
    if (r.kind == NAN_) {
        dst[o] = 'n'; dst[o + 1] = 'a'; dst[o + 2] = 'n';
        return o + 3;
    }
    const int32_t n = r.ndigits, d = r.decpt;
    if (repr_scientific(r)) {
        // d.ddde[+-]xx: the digits go to [o, o + n + 1) with the point after the first one
        put_digits(dst + o + 1, r.digits, n);
        dst[o] = dst[o + 1];
        if (n > 1) {
            dst[o + 1] = '.';
            o += n + 1;
        } else {
            o += 1;
        }
        dst[o++] = 'e';
        const int32_t x = d - 1;
        dst[o++] = x < 0 ? '-' : '+';
        const uint32_t ax = (uint32_t)(x < 0 ? -x : x);
        const int32_t xl = ax < 10 ? 2 : uint_length(ax);
        put_digits(dst + o, ax, xl);
        return o + xl;
    }
    if (d <= 0) {
        dst[o++] = '0';
        dst[o++] = '.';
        for (int32_t k = 0; k < -d; ++k) dst[o++] = '0';
        put_digits(dst + o, r.digits, n);
        return o + n;
    }
    if (d < n) {
        // the first d digits, the point, the rest: write all n digits one place right, then pull the first d back
        put_digits(dst + o + 1, r.digits, n);
        for (int32_t k = 0; k < d; ++k) dst[o + k] = dst[o + k + 1];
        dst[o + d] = '.';
        return o + n + 1;
    }
    put_digits(dst + o, r.digits, n);
    o += n;
    for (int32_t k = n; k < d; ++k) dst[o++] = '0';
    dst[o] = '.';
    dst[o + 1] = '0';
    return o + 2;
}

// '{}'.format of an int32 (numpy's astype(np.int32) value): optional '-', decimal digits.
V2E_HD int32_t int_length(int32_t v) {
    const uint32_t a = v < 0 ? 0u - (uint32_t)v : (uint32_t)v;
    return (v < 0) + uint_length(a);
}

template <typename Out>
V2E_HD int32_t int_write(int32_t v, Out dst) {
    int32_t o = 0;
    uint32_t a = (uint32_t)v;
    if (v < 0) {
        dst[o++] = '-';
        a = 0u - a;
    }
    const int32_t n = uint_length(a);
    put_digits(dst + o, a, n);
    return o + n;
}

}  // namespace v2e_repr
