// The 16-bit rank columns of kb_numrank.cuh (rank_shift, rank16, range16) against the exact rank range: for V sizes on both sides of
// 65535 and random rank ranges [lo, hi) (empty ones included), every rank stored strictly inside the stored range must be in [lo, hi),
// every rank stored outside it must not be, and with shift 0 the stored range is exact. Prints "checks <n>"; exits 1 on a mismatch.
#include <cstdio>
#include <cstdlib>
#include <random>

#include "kb_numrank.cuh"

int main(int argc, char** argv) {
    const unsigned seed = argc > 1 ? (unsigned)atoi(argv[1]) : 1u;
    std::mt19937_64 rng(seed);
    const uint32_t sizes[] = {1, 2, 3, 1000, 65534, 65535, 65536, 65537, 131070, 131071, 131072, 120001, 1u << 20, (1u << 31) - 1};
    unsigned long long checks = 0;
    for (uint32_t n : sizes) {
        const uint32_t s = kb_nr::rank_shift(n);
        if (((n - 1) >> s) >= kb_nr::NAN_RANK16 || (s > 0 && ((n - 1) >> (s - 1)) < kb_nr::NAN_RANK16)) {
            printf("rank_shift(%u) = %u is not the smallest shift below the NaN code\n", n, s);
            return 1;
        }
        for (int t = 0; t < 400; t++) {
            uint32_t lo = (uint32_t)(rng() % ((uint64_t)n + 1)), hi = (uint32_t)(rng() % ((uint64_t)n + 1));
            if (t % 7 == 0) hi = lo;  // empty
            if (lo > hi) { const uint32_t x = lo; lo = hi; hi = x; }
            const kb_nr::Range16 q = kb_nr::range16(kb_nr::Range{lo, hi}, s);
            for (int k = 0; k < 2000; k++) {
                uint32_t r = k == 0 ? kb_nr::NAN_RANK : k < 8 ? (uint32_t)((int64_t)lo + k - 4) : k < 16 ? (uint32_t)((int64_t)hi + k - 12) : (uint32_t)(rng() % n);
                if (r != kb_nr::NAN_RANK && r >= n) continue;
                const uint32_t c = kb_nr::rank16(r, s);
                const bool exact = kb_nr::in_range(r, lo, hi);
                const bool in = c >= q.lo && c <= q.hi;
                const bool end = in && (c == q.lo || c == q.hi);
                if ((exact && !in) || (in && !end && !exact) || (s == 0 && in != exact)) {
                    printf("n %u shift %u range [%u, %u) rank %u stored %u: stored range [%u, %u]\n", n, s, lo, hi, r, c, q.lo, q.hi);
                    return 1;
                }
                checks++;
            }
        }
    }
    printf("checks %llu\n", checks);
    return 0;
}
