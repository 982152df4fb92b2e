// kb_numparse.cuh — Rust's `str::parse::<f64>()` and `str::parse::<i32>()` of one string, as __host__ __device__ code: the device
// numeric side table (kb_numeric.cu) and a host build of the same code (tests/test_numparse_cpu.py, g++) run exactly these lines.
//
// f64: the grammar of `engine.rust_parse_f64` — an optional sign, then inf / infinity / nan in any case, or digits[.digits] / .digits /
// digits. with an optional e|E[+-]digits; nothing else. The value is the nearest double, ties to even, for input of any length:
//   1. scan: up to 19 significant digits into a u64 w, the decimal exponent q (saturated), and whether a non-zero digit was dropped;
//   2. Clinger's fast path (w <= 2^53, |q| small, nothing dropped): one correctly rounded multiply or divide by an exact power of ten;
//   3. Eisel–Lemire with a 128-bit power of five (kb_pow5.inc); with dropped digits, w and w + 1 must round to the same double;
//   4. what step 3 cannot decide (the two bracketing results differ, or a near-halfway product) is NUM_SLOW: slow_f64 resolves it
//      exactly with a decimal of up to 768 digits plus a non-zero-tail flag, shifted by powers of two (the simple decimal conversion).
// i32: `[+-]?[0-9]+` within [-2^31, 2^31).
#pragma once
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define KB_NP_HD __host__ __device__ __forceinline__
#define KB_NP_HD_SLOW __host__ __device__ __noinline__
#else
#define KB_NP_HD inline
#define KB_NP_HD_SLOW inline
#endif

namespace kb_np {

constexpr int POW5_MIN_Q = -342, POW5_MAX_Q = 308;
constexpr int POW5_N = POW5_MAX_Q - POW5_MIN_Q + 1;

struct Tables {
    uint64_t pow5[POW5_N][2];  // {hi, lo} of 5^q, row q - POW5_MIN_Q
    double pow10[23];          // 10^0 .. 10^22, exact doubles
    uint64_t ipow10[16];       // 10^0 .. 10^15
};

// the initializer of a Tables: { { #include "kb_pow5.inc" }, KB_NP_POW10_INIT, KB_NP_IPOW10_INIT }
#define KB_NP_POW10_INIT {1e0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 1e8, 1e9, 1e10, 1e11, 1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22}
#define KB_NP_IPOW10_INIT {1ull, 10ull, 100ull, 1000ull, 10000ull, 100000ull, 1000000ull, 10000000ull, 100000000ull, 1000000000ull, 10000000000ull, \
                           100000000000ull, 1000000000000ull, 10000000000000ull, 100000000000000ull, 1000000000000000ull}

// How parse_f64 decided (the CPU test checks that a corpus reaches every one)
enum Route : uint32_t {
    NUM_REJECT = 0,        // not a number
    NUM_SPECIAL,           // inf / infinity / nan
    NUM_CLINGER,           // w * 10^q or w / 10^-q, |q| <= 22
    NUM_CLINGER_DISGUISED, // w * 10^(q-22) still exact below 2^53, times 10^22
    NUM_LEMIRE_LIMIT,      // w == 0, or q outside [-342, 308]: zero or infinity without a product
    NUM_LEMIRE_SUBNORMAL,  // Eisel–Lemire, subnormal result (or zero by underflow)
    NUM_LEMIRE,            // Eisel–Lemire, all significant digits in w
    NUM_LEMIRE_MANY,       // Eisel–Lemire, digits dropped, and w and w + 1 give the same double
    NUM_SLOW,              // undecided: slow_f64
    NUM_ROUTES
};

KB_NP_HD uint8_t ld(const uint8_t* p) {
#if defined(__CUDA_ARCH__)
    return __ldg(p);
#else
    return *p;
#endif
}
KB_NP_HD uint64_t ld64(const uint64_t* p) {
#if defined(__CUDA_ARCH__)
    return __ldg(reinterpret_cast<const unsigned long long*>(p));
#else
    return *p;
#endif
}
KB_NP_HD double ldd(const double* p) {
#if defined(__CUDA_ARCH__)
    return __ldg(p);
#else
    return *p;
#endif
}
KB_NP_HD uint64_t to_bits(double d) {
#if defined(__CUDA_ARCH__)
    return (uint64_t)__double_as_longlong(d);
#else
    uint64_t b;
    memcpy(&b, &d, sizeof b);
    return b;
#endif
}
KB_NP_HD void mul128(uint64_t a, uint64_t b, uint64_t* lo, uint64_t* hi) {
#if defined(__CUDA_ARCH__)
    *hi = __umul64hi(a, b);
    *lo = a * b;
#else
    const unsigned __int128 r = (unsigned __int128)a * b;
    *hi = (uint64_t)(r >> 64);
    *lo = (uint64_t)r;
#endif
}
KB_NP_HD int clz64(uint64_t x) {
#if defined(__CUDA_ARCH__)
    return __clzll((long long)x);
#else
    return __builtin_clzll(x);
#endif
}
// correctly rounded, never contracted into an FMA
KB_NP_HD double dmul(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
KB_NP_HD double ddiv(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}
KB_NP_HD double u64_to_double(uint64_t x) {  // exact for x <= 2^53
#if defined(__CUDA_ARCH__)
    return __ull2double_rn(x);
#else
    return (double)x;
#endif
}

KB_NP_HD bool is_digit(uint8_t c) { return (uint8_t)(c - '0') < 10; }
// a byte a number can start with: sign, digit, '.', or the first letter of inf / nan
KB_NP_HD bool can_start(uint8_t c) { return is_digit(c) || c == '+' || c == '-' || c == '.' || (c | 0x20) == 'i' || (c | 0x20) == 'n'; }

constexpr uint64_t EXP_SAT = 0x10000;  // exponent digits stop accumulating here: any larger exponent is 0 or inf already
constexpr uint64_t SIGN = 1ull << 63;
constexpr uint64_t INF_BITS = 0x7FF0000000000000ull, NAN_BITS = 0x7FF8000000000000ull;

// the binary exponent of 10^q, floor(q * log2(10)) + 63 (Lemire, section 5)
KB_NP_HD int32_t power(int32_t q) { return (((152170 + 65536) * q) >> 16) + 63; }

// Eisel–Lemire of w * 10^q for binary64: the biased exponent (e) and the explicit mantissa bits (f); e = -1 when the 128-bit product
// cannot decide the rounding. *route = NUM_LEMIRE_LIMIT / NUM_LEMIRE_SUBNORMAL / NUM_LEMIRE.
KB_NP_HD void lemire(int64_t q, uint64_t w, const Tables* T, uint64_t* f, int32_t* e, uint32_t* route) {
    *route = NUM_LEMIRE_LIMIT;
    *f = 0;
    if (w == 0 || q < POW5_MIN_Q) { *e = 0; return; }
    if (q > POW5_MAX_Q) { *e = 0x7FF; return; }
    *route = NUM_LEMIRE;
    const int lz = clz64(w);
    w <<= lz;
    const int idx = (int)(q - POW5_MIN_Q);
    const uint64_t mask = 0xFFFFFFFFFFFFFFFFull >> 55;  // 52 explicit bits + 3
    uint64_t lo, hi;
    mul128(w, ld64(&T->pow5[idx][0]), &lo, &hi);
    if ((hi & mask) == mask) {  // the truncated product may be off by one in its low bits: take the next 64 bits of 5^q too
        uint64_t lo2, hi2;
        mul128(w, ld64(&T->pow5[idx][1]), &lo2, &hi2);
        lo += hi2;
        if (hi2 > lo) hi++;
    }
    if (lo == 0xFFFFFFFFFFFFFFFFull && !(q >= -27 && q <= 55)) { *e = -1; return; }
    const int upper = (int)(hi >> 63);
    const int shift = upper + 64 - 52 - 3;
    uint64_t m = hi >> shift;
    int32_t p2 = power((int32_t)q) + upper - lz + 1023;
    if (p2 <= 0) {  // subnormal
        *route = NUM_LEMIRE_SUBNORMAL;
        if (-p2 + 1 >= 64) { *e = 0; return; }
        m >>= -p2 + 1;
        m += m & 1;
        m >>= 1;
        *e = m < (1ull << 52) ? 0 : 1;
        *f = m & ((1ull << 52) - 1);
        return;
    }
    // exactly halfway between two doubles (possible only while 5^q fits in 64 bits): round to even
    if (lo <= 1 && q >= -4 && q <= 23 && (m & 3) == 1 && (m << shift) == hi) m &= ~1ull;
    m += m & 1;
    m >>= 1;
    if (m >= (2ull << 52)) { m = 1ull << 52; p2++; }
    m &= ~(1ull << 52);
    if (p2 >= 0x7FF) { *e = 0x7FF; return; }
    *e = p2;
    *f = m;
}

// str::parse::<f64>() of s[0, len). Returns the Route; *bits = the double's bits except for NUM_REJECT (0) and NUM_SLOW (unset).
KB_NP_HD uint32_t parse_f64(const uint8_t* s, uint64_t len, const Tables* T, uint64_t* bits) {
    *bits = 0;
    if (len == 0) return NUM_REJECT;
    uint8_t c = ld(s);
    if (!can_start(c)) return NUM_REJECT;  // most terms: IRIs and names, one byte read
    uint64_t i = 0;
    bool neg = false;
    if (c == '+' || c == '-') {
        neg = c == '-';
        if (++i == len) return NUM_REJECT;
        c = ld(s + i);
    }
    const uint64_t sign = neg ? SIGN : 0;
    if ((c | 0x20) == 'i' || (c | 0x20) == 'n') {
        const uint64_t rest = len - i;
        if (rest != 3 && rest != 8) return NUM_REJECT;
        const char* word = (c | 0x20) == 'n' ? "nan" : "infinity";
        if ((c | 0x20) == 'n' && rest != 3) return NUM_REJECT;
        for (uint64_t k = 0; k < rest; k++)
            if ((ld(s + i + k) | 0x20) != (uint8_t)word[k]) return NUM_REJECT;
        *bits = ((c | 0x20) == 'n' ? NAN_BITS : INF_BITS) | sign;
        return NUM_SPECIAL;
    }
    uint64_t w = 0;
    int64_t q = 0;
    int nd = 0;          // significant digits in w
    bool any = false, dropped = false;
    for (; i < len; i++) {  // integer part
        c = ld(s + i);
        if (!is_digit(c)) break;
        any = true;
        const uint32_t d = c - '0';
        if (nd == 0 && d == 0) continue;
        if (nd < 19) { w = w * 10 + d; nd++; }
        else { q++; dropped |= d != 0; }
    }
    if (i < len && c == '.') {
        for (i++; i < len; i++) {  // fraction
            c = ld(s + i);
            if (!is_digit(c)) break;
            any = true;
            const uint32_t d = c - '0';
            if (nd == 0 && d == 0) { q--; continue; }
            if (nd < 19) { w = w * 10 + d; nd++; q--; }
            else dropped |= d != 0;
        }
    }
    if (!any) return NUM_REJECT;
    if (i < len) {
        if ((c | 0x20) != 'e') return NUM_REJECT;
        if (++i == len) return NUM_REJECT;
        c = ld(s + i);
        bool eneg = false;
        if (c == '+' || c == '-') {
            eneg = c == '-';
            if (++i == len) return NUM_REJECT;
        }
        uint64_t ev = 0;
        for (; i < len; i++) {
            c = ld(s + i);
            if (!is_digit(c)) return NUM_REJECT;
            if (ev < EXP_SAT) ev = ev * 10 + (c - '0');
        }
        q += eneg ? -(int64_t)ev : (int64_t)ev;
    }
    if (!dropped && q >= -22 && q <= 22 + 15 && w <= (1ull << 53)) {  // Clinger
        if (q <= 22) {
            const double v = u64_to_double(w);
            const double r = q < 0 ? ddiv(v, ldd(&T->pow10[-q])) : dmul(v, ldd(&T->pow10[q]));
            *bits = to_bits(r) | sign;
            return NUM_CLINGER;
        }
        const uint64_t p = ld64(&T->ipow10[q - 22]);
        if (w <= 0xFFFFFFFFFFFFFFFFull / p && w * p <= (1ull << 53)) {
            const double r = dmul(u64_to_double(w * p), ldd(&T->pow10[22]));
            *bits = to_bits(r) | sign;
            return NUM_CLINGER_DISGUISED;
        }
    }
    uint64_t f;
    int32_t e;
    uint32_t route;
    lemire(q, w, T, &f, &e, &route);
    if (e >= 0 && dropped) {  // the value lies in (w, w + 1) * 10^q: both ends must round alike
        uint64_t f1;
        int32_t e1;
        uint32_t r1;
        lemire(q, w + 1, T, &f1, &e1, &r1);
        if (f1 != f || e1 != e) return NUM_SLOW;
        if (route == NUM_LEMIRE) route = NUM_LEMIRE_MANY;
    }
    if (e < 0) return NUM_SLOW;
    *bits = f | ((uint64_t)e << 52) | sign;
    return route;
}

// ------------------------------------------------------------------------------------------------ the exact slow path
constexpr int DEC_MAX = 768;                // digits kept; a non-zero digit beyond them sets `truncated`
constexpr int DEC_ROOM = DEC_MAX + 20;      // + room for the digits a left shift by <= 60 bits adds

struct Decimal {
    int32_t nd;        // digits held
    int32_t dp;        // value = 0.d[0]d[1]... * 10^dp
    bool truncated;    // a non-zero digit beyond d[nd - 1] was dropped
    uint8_t d[DEC_ROOM];
};

KB_NP_HD void dec_trim(Decimal* x) {
    while (x->nd > 0 && x->d[x->nd - 1] == 0) x->nd--;
}

// x *= 2^shift, shift <= 60: the product is written right-aligned 19 places up (a shift by <= 60 bits adds <= 19 digits), then moved down
KB_NP_HD void dec_left_shift(Decimal* x, int shift) {
    if (x->nd == 0) return;
    int r = x->nd, wi = x->nd + 19;
    uint64_t n = 0;
    while (r > 0) {
        r--;
        wi--;
        n += (uint64_t)x->d[r] << shift;
        const uint64_t qq = n / 10;
        x->d[wi] = (uint8_t)(n - 10 * qq);
        n = qq;
    }
    while (n > 0) {
        wi--;
        const uint64_t qq = n / 10;
        x->d[wi] = (uint8_t)(n - 10 * qq);
        n = qq;
    }
    const int count = x->nd + 19 - wi;
    for (int k = 0; k < count; k++) x->d[k] = x->d[wi + k];
    x->dp += count - x->nd;
    x->nd = count;
    if (x->nd > DEC_MAX) {
        for (int k = DEC_MAX; k < x->nd; k++) x->truncated |= x->d[k] != 0;
        x->nd = DEC_MAX;
    }
    dec_trim(x);
}

// x /= 2^shift, shift <= 60
KB_NP_HD void dec_right_shift(Decimal* x, int shift) {
    int r = 0, wi = 0;
    uint64_t n = 0;
    while ((n >> shift) == 0) {
        if (r < x->nd) {
            n = 10 * n + x->d[r++];
        } else if (n == 0) {
            return;
        } else {
            while ((n >> shift) == 0) { n *= 10; r++; }
            break;
        }
    }
    x->dp -= r - 1;
    if (x->dp < -2047) { x->nd = 0; x->dp = 0; x->truncated = false; return; }
    const uint64_t mask = (1ull << shift) - 1;
    while (r < x->nd) {
        const uint8_t nd_ = (uint8_t)(n >> shift);
        n = 10 * (n & mask) + x->d[r++];
        x->d[wi++] = nd_;
    }
    while (n > 0) {
        const uint8_t nd_ = (uint8_t)(n >> shift);
        n = 10 * (n & mask);
        if (wi < DEC_MAX) x->d[wi++] = nd_;
        else if (nd_ > 0) x->truncated = true;
    }
    x->nd = wi;
    dec_trim(x);
}

// the integer part, rounded half to even (a dropped non-zero tail breaks the tie upward)
KB_NP_HD uint64_t dec_round(const Decimal* x) {
    if (x->nd == 0 || x->dp < 0) return 0;
    if (x->dp > 18) return 0xFFFFFFFFFFFFFFFFull;
    const int dp = x->dp;
    uint64_t n = 0;
    for (int k = 0; k < dp; k++) n = 10 * n + (k < x->nd ? x->d[k] : 0);
    bool up = false;
    if (dp < x->nd) {
        up = x->d[dp] >= 5;
        if (x->d[dp] == 5 && dp + 1 == x->nd) up = x->truncated || (dp != 0 && (x->d[dp - 1] & 1));
    }
    return n + (up ? 1 : 0);
}

KB_NP_HD int dec_shift_for(int n) { return n < 19 ? (n * 217706) >> 16 : 60; }  // floor(n * log2(10)), at most 60

// the exact value of a string parse_f64 accepted with NUM_SLOW, as the bits of the nearest double (ties to even)
KB_NP_HD_SLOW uint64_t slow_f64(const uint8_t* s, uint64_t len, Decimal* x) {
    uint64_t i = 0;
    bool neg = false;
    if (ld(s) == '+' || ld(s) == '-') { neg = ld(s) == '-'; i = 1; }
    const uint64_t sign = neg ? SIGN : 0;
    x->nd = 0;
    x->truncated = false;
    int64_t total = 0, last_nz = -1, dp = 0, lead_frac_zeros = 0;
    uint8_t c = 0;
    bool frac = false;
    for (; i < len; i++) {
        c = ld(s + i);
        if (c == '.') { frac = true; continue; }
        if (!is_digit(c)) break;
        const uint8_t d = c - '0';
        if (total == 0 && d == 0) { if (frac) lead_frac_zeros++; continue; }
        if (!frac) dp++;
        if (total < DEC_MAX) x->d[total] = d;
        if (d != 0) last_nz = total;
        total++;
    }
    dp -= lead_frac_zeros;
    if (i < len) {  // exponent ('e' already checked by parse_f64)
        i++;
        bool eneg = false;
        if (ld(s + i) == '+' || ld(s + i) == '-') { eneg = ld(s + i) == '-'; i++; }
        uint64_t ev = 0;
        for (; i < len; i++)
            if (ev < EXP_SAT) ev = ev * 10 + (ld(s + i) - '0');
        dp += eneg ? -(int64_t)ev : (int64_t)ev;
    }
    const int64_t nd = last_nz + 1;  // trailing zeros dropped
    if (nd == 0 || dp < -324) return sign;
    if (dp >= 310) return INF_BITS | sign;
    x->nd = (int32_t)(nd > DEC_MAX ? DEC_MAX : nd);
    x->truncated = nd > DEC_MAX;
    x->dp = (int32_t)dp;
    int32_t exp2 = 0;
    while (x->dp > 0) {  // toward [1/2, 1)
        const int sh = dec_shift_for(x->dp);
        dec_right_shift(x, sh);
        if (x->dp < -2047) return sign;
        exp2 += sh;
    }
    while (x->dp <= 0) {
        int sh;
        if (x->dp == 0) {
            if (x->d[0] >= 5) break;
            sh = x->d[0] < 2 ? 2 : 1;
        } else {
            sh = dec_shift_for(-x->dp);
        }
        dec_left_shift(x, sh);
        if (x->dp > 2047) return INF_BITS | sign;
        exp2 -= sh;
    }
    exp2--;  // [1/2, 1) -> [1, 2)
    while (-1023 + 1 > exp2) {
        int n = (-1023 + 1) - exp2;
        if (n > 60) n = 60;
        dec_right_shift(x, n);
        exp2 += n;
    }
    if (exp2 + 1023 >= 0x7FF) return INF_BITS | sign;
    dec_left_shift(x, 53);
    uint64_t m = dec_round(x);
    if (m >= (1ull << 53)) {  // rounding carried into a new bit
        dec_right_shift(x, 1);
        exp2++;
        m = dec_round(x);
        if (exp2 + 1023 >= 0x7FF) return INF_BITS | sign;
    }
    int32_t p2 = exp2 + 1023;
    if (m < (1ull << 52)) p2--;
    m &= (1ull << 52) - 1;
    return m | ((uint64_t)p2 << 52) | sign;
}

// str::parse::<i32>(): [+-]?[0-9]+ within range
KB_NP_HD bool parse_i32(const uint8_t* s, uint64_t len, int32_t* out) {
    *out = 0;
    if (len == 0) return false;
    uint64_t i = 0;
    const uint8_t c0 = ld(s);
    if (!is_digit(c0) && c0 != '+' && c0 != '-') return false;
    const bool neg = c0 == '-';
    if (c0 == '+' || c0 == '-') i = 1;
    if (i == len) return false;
    int64_t v = 0;
    for (; i < len; i++) {
        const uint8_t c = ld(s + i);
        if (!is_digit(c)) return false;
        if (v <= 2147483648ll) v = v * 10 + (c - '0');
    }
    if (neg) v = -v;
    if (v < -2147483648ll || v > 2147483647ll) return false;
    *out = (int32_t)v;
    return true;
}

}  // namespace kb_np
