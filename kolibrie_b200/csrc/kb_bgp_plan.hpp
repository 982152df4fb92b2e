// kb_bgp_plan.hpp — the host-side plan of kb_bgp_execute's component route (kb_bgp.cu): connected components over shared variables,
// GYO acyclicity with a join tree, and the join order inside a component. Header-only and free of CUDA, so that the library and a
// host build of the same lines (tests/cpp/bgp_plan_driver.cpp, g++) run exactly this code.
//
// A BGP is a hypergraph: the patterns are edges over their variables. Two patterns are joined only when they share a variable, so
// a join inside a component is never keyless; components are cross-joined by the caller.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <vector>

namespace kb_bgp {

using Vars = std::vector<std::vector<uint32_t>>;  // the distinct variables of every pattern

inline bool shares(const std::vector<uint32_t>& a, const std::vector<uint32_t>& b) {
    for (uint32_t x : a) if (std::find(b.begin(), b.end(), x) != b.end()) return true;
    return false;
}

// Connected components: patterns ascending inside a component, components in the order of their first pattern. A pattern without
// variables is a component of its own.
inline std::vector<std::vector<uint32_t>> components(const Vars& pv) {
    const uint32_t n = (uint32_t)pv.size();
    std::vector<int> comp(n, -1);
    std::vector<std::vector<uint32_t>> out;
    for (uint32_t s = 0; s < n; s++) {
        if (comp[s] >= 0) continue;
        const int c = (int)out.size();
        out.push_back({});
        std::vector<uint32_t> stack{s};
        comp[s] = c;
        while (!stack.empty()) {
            const uint32_t k = stack.back();
            stack.pop_back();
            out[c].push_back(k);
            for (uint32_t j = 0; j < n; j++)
                if (comp[j] < 0 && shares(pv[k], pv[j])) { comp[j] = c; stack.push_back(j); }
        }
        std::sort(out[c].begin(), out[c].end());
    }
    return out;
}

// GYO reduction of the patterns `comp`: repeatedly drop a variable that only one remaining pattern holds, and a pattern whose
// remaining variables another remaining pattern holds too (its join-tree parent). Acyclic iff at most one pattern remains.
// parent[i] = the pattern comp[i] hangs off in the join tree (-1: the last one standing); filled only when the result is true.
inline bool gyo(const Vars& pv, const std::vector<uint32_t>& comp, std::vector<int>* parent) {
    const size_t m = comp.size();
    std::vector<std::vector<uint32_t>> e(m);
    for (size_t i = 0; i < m; i++) e[i] = pv[comp[i]];
    std::vector<bool> alive(m, true);
    std::vector<int> par(m, -1);
    size_t left = m;
    for (bool changed = true; changed && left > 1;) {
        changed = false;
        for (size_t i = 0; i < m; i++) {
            if (!alive[i]) continue;
            std::vector<uint32_t> keep;
            for (uint32_t v : e[i]) {
                bool other = false;
                for (size_t j = 0; j < m && !other; j++)
                    if (j != i && alive[j] && std::find(e[j].begin(), e[j].end(), v) != e[j].end()) other = true;
                if (other) keep.push_back(v);
            }
            if (keep.size() != e[i].size()) { e[i] = keep; changed = true; }
        }
        for (size_t i = 0; i < m && left > 1; i++) {
            if (!alive[i]) continue;
            for (size_t j = 0; j < m; j++) {
                if (j == i || !alive[j]) continue;
                bool sub = true;
                for (uint32_t v : e[i]) if (std::find(e[j].begin(), e[j].end(), v) == e[j].end()) sub = false;
                if (sub) { alive[i] = false; par[i] = (int)comp[j]; left--; changed = true; break; }
            }
        }
    }
    if (left > 1) return false;
    parent->assign(par.begin(), par.end());
    return true;
}

// The join order of a component, rows[k] = rows of pattern k's (reduced) relation. It starts at the smallest relation. Acyclic
// (parent from gyo): each step adds the smallest relation adjacent in the join tree to those joined so far. Cyclic: each step adds
// the smallest relation that shares a variable with those joined so far. Ties go to the lower pattern index.
inline std::vector<uint32_t> join_order(const Vars& pv, const std::vector<uint32_t>& comp, const std::vector<uint64_t>& rows, bool acyclic,
                                        const std::vector<int>& parent) {
    const size_t m = comp.size();
    auto adjacent = [&](size_t i, size_t j) {  // may comp[j] join comp[i]?
        if (!acyclic) return shares(pv[comp[i]], pv[comp[j]]);
        return parent[i] == (int)comp[j] || parent[j] == (int)comp[i];
    };
    std::vector<bool> in(m, false);
    std::vector<uint32_t> order;
    size_t first = 0;
    for (size_t i = 1; i < m; i++) if (rows[comp[i]] < rows[comp[first]]) first = i;
    in[first] = true;
    order.push_back(comp[first]);
    std::vector<size_t> joined{first};
    while (order.size() < m) {
        int best = -1;
        for (size_t j = 0; j < m; j++) {
            if (in[j]) continue;
            bool adj = false;
            for (size_t i : joined) if (adjacent(i, j)) { adj = true; break; }
            if (adj && (best < 0 || rows[comp[j]] < rows[comp[best]])) best = (int)j;
        }
        if (best < 0) break;  // (not connected: the caller's components are)
        in[best] = true;
        joined.push_back((size_t)best);
        order.push_back(comp[best]);
    }
    return order;
}

}  // namespace kb_bgp
