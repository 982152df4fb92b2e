// kb_numrank.cuh — the value order of the numeric side table, as __host__ __device__ code: the device (the rank fills of the store
// index, kb_store.cu), the host (a FILTER resolved to a rank range, kb_api.cu) and a host build of the same lines
// (tests/test_numrank_cpu.py, g++) run exactly these lines.
//
// V = the sorted distinct non-NaN values of num_or0 over all ids, -0.0 folded into +0.0, 0.0 always included (num_of answers 0.0 for
// an id past the table). A value x of the table has the rank lower_bound(V, x): two values compare (<, <=, >, >=) exactly as their
// ranks do, so FILTER(?o <cmp> c) over num_of(o) (cmp_num, kb_device.cuh) is `rank in [lo, hi)` for the [lo, hi) below. NaN compares
// false with everything: its rank is NAN_RANK, which no range of a V smaller than 2^32 - 1 values holds.
#pragma once
#include <stdint.h>
#include <string.h>

#include "../../include/kolibrie_b200.h"

#if defined(__CUDACC__)
#define KB_NR_HD __host__ __device__ __forceinline__
#else
#define KB_NR_HD inline
#endif
#if defined(__CUDA_ARCH__)
#define KB_NR_UNROLL _Pragma("unroll")
#else
#define KB_NR_UNROLL
#endif

namespace kb_nr {

constexpr uint32_t NAN_RANK = 0xFFFFFFFFu;

// -0.0 == +0.0 in every comparison: one entry of V stands for both
KB_NR_HD double fold(double x) { return x == 0.0 ? 0.0 : x; }

// how V is built (kb_numeric.cu): every value as an order-preserving u64 (sign set: all bits flipped, else the sign bit set; NaN takes
// 0.0's key, which V holds anyway), a radix sort, the distinct keys, back to doubles
KB_NR_HD uint64_t order_key(double x) {
    x = x != x ? 0.0 : fold(x);
    uint64_t b;
    memcpy(&b, &x, sizeof b);
    return (b >> 63) ? ~b : (b | (1ull << 63));
}
// ORDER BY's order of numbers (kb_order.cu): as order_key, except that every NaN takes one key of its own above +inf (a key column that
// holds NaN and another number is refused, so where NaN sits never matters), and 0, which no number takes, is left for ""
KB_NR_HD uint64_t order_key_total(double x) {
    if (x != x) return ~0ull;
    x = fold(x);
    uint64_t b;
    memcpy(&b, &x, sizeof b);
    return (b >> 63) ? ~b : (b | (1ull << 63));
}
KB_NR_HD double order_value(uint64_t k) {
    const uint64_t b = (k >> 63) ? (k & ~(1ull << 63)) : ~k;
    double x;
    memcpy(&x, &b, sizeof x);
    return x;
}

// first i in [0, n) with !(v[i] < x), else n
KB_NR_HD uint32_t lower_bound(const double* v, uint32_t n, double x) {
    uint32_t lo = 0, len = n;
    while (len > 0) {
        const uint32_t h = len >> 1;
        if (v[lo + h] < x) { lo += h + 1; len -= h + 1; }
        else len = h;
    }
    return lo;
}
// first i in [0, n) with x < v[i], else n
KB_NR_HD uint32_t upper_bound(const double* v, uint32_t n, double x) {
    uint32_t lo = 0, len = n;
    while (len > 0) {
        const uint32_t h = len >> 1;
        if (!(x < v[lo + h])) { lo += h + 1; len -= h + 1; }
        else len = h;
    }
    return lo;
}

// ranks of N values of the table at once (each is in V unless it is NaN). A branchless lower bound: every search takes the same
// ceil(log2 n) steps, set by n alone, so the N searches advance side by side and their dependent loads overlap instead of queuing
// behind each other (on the device each step is an L2 round trip)
template <int N>
KB_NR_HD void rank_of_n(const double* v, uint32_t n, const double* x, uint32_t* out) {
    uint32_t base[N];
    KB_NR_UNROLL
    for (int k = 0; k < N; k++) base[k] = 0;
    for (uint32_t len = n; len > 1;) {
        const uint32_t half = len >> 1;
        KB_NR_UNROLL
        for (int k = 0; k < N; k++) base[k] = v[base[k] + half] < x[k] ? base[k] + half : base[k];
        len -= half;
    }
    KB_NR_UNROLL
    for (int k = 0; k < N; k++) out[k] = x[k] != x[k] ? NAN_RANK : n == 0 ? 0u : base[k] + (v[base[k]] < x[k] ? 1u : 0u);
}
KB_NR_HD uint32_t rank_of(const double* v, uint32_t n, double x) {
    uint32_t r;
    rank_of_n<1>(v, n, &x, &r);
    return r;
}

// the ranks whose values satisfy `value <cmp> c`: [lo, hi), empty (lo == hi == 0) for a NaN constant or a non-ordering cmp
struct Range {
    uint32_t lo, hi;
};
KB_NR_HD Range cmp_range(uint32_t cmp, const double* v, uint32_t n, double c) {
    if (c != c) return Range{0u, 0u};
    switch (cmp) {
        case KB_CMP_GT: return Range{upper_bound(v, n, c), n};
        case KB_CMP_GE: return Range{lower_bound(v, n, c), n};
        case KB_CMP_LT: return Range{0u, lower_bound(v, n, c)};
        case KB_CMP_LE: return Range{0u, upper_bound(v, n, c)};
        default: return Range{0u, 0u};
    }
}
// unsigned: one compare, and NAN_RANK is outside every range
KB_NR_HD bool in_range(uint32_t rank, uint32_t lo, uint32_t hi) { return rank - lo < hi - lo; }

// The 16-bit rank columns of the store index: a rank r of a V of n values is stored as r >> rank_shift(n), the smallest shift that
// keeps every rank below NAN_RANK16 (0 while n <= 65535: the stored rank is exact). A rank range [lo, hi) then covers the stored
// ranks [lo >> s, (hi - 1) >> s]; every stored rank strictly inside is wholly in the range, and only the two at its ends can hold
// values on both sides of the constant, which the reader decides from the value itself.
constexpr uint32_t NAN_RANK16 = 0xFFFFu;
KB_NR_HD uint32_t rank_shift(uint32_t n) {
    uint32_t s = 0;
    while (n > 0 && ((n - 1) >> s) >= NAN_RANK16) s++;
    return s;
}
KB_NR_HD uint16_t rank16(uint32_t rank, uint32_t shift) { return (uint16_t)(rank == NAN_RANK ? NAN_RANK16 : rank >> shift); }
struct Range16 {
    uint32_t lo, hi;  // stored ranks [lo, hi], inclusive (lo > hi: empty)
};
KB_NR_HD Range16 range16(Range r, uint32_t shift) {
    if (r.lo >= r.hi) return Range16{1u, 0u};
    return Range16{r.lo >> shift, (r.hi - 1u) >> shift};
}

}  // namespace kb_nr
