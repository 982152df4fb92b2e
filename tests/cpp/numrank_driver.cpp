// Host build of kolibrie_b200/csrc/kb_numrank.cuh (the value order the table-mode index probe filters on), for tests/test_numrank_cpu.py.
// argv[1]: random seed, argv[2]: trials. Every trial draws a numeric side table from a pool of edge values (signed zeros, infinities,
// NaNs, subnormals, neighbours of each other) and random doubles, builds V twice (the device's route: order keys, sort, distinct,
// back to doubles; and a plain sort of the folded non-NaN values plus 0.0) and checks, for every constant of the pool, of the table,
// their nextafter neighbours and values beyond both ends, and every comparison, that `rank in cmp_range` equals the direct double
// comparison on every value of the table. stdout: "checks <n> failures <m>" and up to 20 failing cases; exit code 1 on a failure.
#include <algorithm>
#include <cfloat>
#include <cinttypes>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>

#include "kb_numrank.cuh"

static bool direct(uint32_t cmp, double a, double b) {  // cmp_num (kb_device.cuh)
    switch (cmp) {
        case KB_CMP_GT: return a > b;
        case KB_CMP_GE: return a >= b;
        case KB_CMP_LT: return a < b;
        case KB_CMP_LE: return a <= b;
        default: return false;
    }
}

int main(int argc, char** argv) {
    const uint64_t seed = argc > 1 ? strtoull(argv[1], nullptr, 10) : 1;
    const int trials = argc > 2 ? atoi(argv[2]) : 200;
    std::mt19937_64 rng(seed);
    const double inf = HUGE_VAL, nan_ = std::nan(""), dmin = std::numeric_limits<double>::denorm_min();
    std::vector<double> pool = {0.0, -0.0, inf, -inf, nan_, -nan_, dmin, -dmin, 2 * dmin, DBL_MIN, -DBL_MIN, std::nextafter(DBL_MIN, 0.0),
                                DBL_MAX, -DBL_MAX, 1.0, -1.0, 0.5, 100000.0, 100001.0, 99999.5, -100000.0, 1e300, -1e-300, 3.0, 7.0};
    {
        const size_t n0 = pool.size();
        for (size_t i = 0; i < n0; i++) {
            pool.push_back(std::nextafter(pool[i], inf));
            pool.push_back(std::nextafter(pool[i], -inf));
        }
    }
    uint64_t checks = 0, failures = 0;
    auto fail = [&](const char* what, uint32_t cmp, double x, double c, uint32_t rank, kb_nr::Range r) {
        if (failures++ < 20)
            printf("FAIL %s cmp=%u x=%a c=%a rank=%u range=[%u,%u)\n", what, cmp, x, c, rank, r.lo, r.hi);
    };
    for (int t = 0; t < trials; t++) {
        // the table: a mix of pool values and random doubles (a few trials: only zeros / NaNs, so V = {0.0}; one trial: no ids)
        std::vector<double> num;
        const int mode = t % 10;
        const size_t n = t == 0 ? 0 : 1 + rng() % 300;
        for (size_t i = 0; i < n; i++) {
            double x;
            if (mode == 0) x = (rng() & 1) ? -0.0 : ((rng() & 1) ? nan_ : 0.0);
            else if (mode < 4) x = pool[rng() % pool.size()];
            else if (mode < 7) x = (double)((int64_t)(rng() % 2001) - 1000) * ((rng() & 3) == 0 ? 0.25 : 1.0);
            else {
                uint64_t b = rng();
                memcpy(&x, &b, sizeof x);
            }
            num.push_back(x);
        }
        // V the device's way
        std::vector<uint64_t> keys;
        for (double x : num) keys.push_back(kb_nr::order_key(x));
        keys.push_back(kb_nr::order_key(0.0));
        std::sort(keys.begin(), keys.end());
        keys.erase(std::unique(keys.begin(), keys.end()), keys.end());
        std::vector<double> V;
        for (uint64_t k : keys) V.push_back(kb_nr::order_value(k));
        // and the plain way: they must be the same bits
        std::vector<double> W = {0.0};
        for (double x : num) if (x == x) W.push_back(x == 0.0 ? 0.0 : x);
        std::sort(W.begin(), W.end());
        W.erase(std::unique(W.begin(), W.end()), W.end());
        bool same = V.size() == W.size();
        for (size_t i = 0; same && i < V.size(); i++) same = memcmp(&V[i], &W[i], sizeof(double)) == 0;
        checks++;
        if (!same) {
            if (failures++ < 20) printf("FAIL value order: %zu values, expected %zu\n", V.size(), W.size());
            continue;
        }
        for (size_t i = 0; i < V.size(); i++) {  // V: strictly ascending, no NaN, no -0.0
            checks++;
            if (V[i] != V[i] || (std::signbit(V[i]) && V[i] == 0.0) || (i && !(V[i - 1] < V[i]))) {
                if (failures++ < 20) printf("FAIL V[%zu] = %a\n", i, V[i]);
            }
        }
        const uint32_t nv = (uint32_t)V.size();
        std::vector<double> consts = pool;
        for (double x : num) {
            consts.push_back(x);
            consts.push_back(std::nextafter(x, inf));
            consts.push_back(std::nextafter(x, -inf));
        }
        consts.push_back(V.front() - 1.0);
        consts.push_back(V.back() + 1.0);
        for (int i = 0; i < 20; i++) {
            uint64_t b = rng();
            double c;
            memcpy(&c, &b, sizeof c);
            consts.push_back(c);
        }
        std::vector<double> xs = num;  // the values the filter sees: the table's, and num_of's 0.0 past the table
        xs.push_back(0.0);
        // the branchless batched search (the device's) against the plain lower bound, four values at a time
        for (size_t i = 0; i < xs.size(); i += 4) {
            double x4[4];
            uint32_t r4[4];
            for (int k = 0; k < 4; k++) x4[k] = kb_nr::fold(xs[(i + k) % xs.size()]);
            kb_nr::rank_of_n<4>(V.data(), nv, x4, r4);
            for (int k = 0; k < 4; k++) {
                checks++;
                const uint32_t want = x4[k] != x4[k] ? kb_nr::NAN_RANK : kb_nr::lower_bound(V.data(), nv, x4[k]);
                if (r4[k] != want) fail("batched rank", 0, x4[k], 0.0, r4[k], kb_nr::Range{want, want});
            }
        }
        for (double c : consts) {
            for (uint32_t cmp = KB_CMP_GT; cmp <= KB_CMP_NE; cmp++) {
                const kb_nr::Range r = kb_nr::cmp_range(cmp, V.data(), nv, c);
                if (r.lo > r.hi || r.hi > nv) { fail("range bounds", cmp, 0.0, c, 0, r); continue; }
                for (double x : xs) {
                    const uint32_t rank = kb_nr::rank_of(V.data(), nv, kb_nr::fold(x));
                    checks++;
                    if (x == x && (rank >= nv || !(V[rank] == x))) { fail("rank", cmp, x, c, rank, r); continue; }
                    if (kb_nr::in_range(rank, r.lo, r.hi) != direct(cmp, x, c)) fail("compare", cmp, x, c, rank, r);
                }
            }
        }
    }
    printf("checks %" PRIu64 " failures %" PRIu64 "\n", checks, failures);
    return failures ? 1 : 0;
}
