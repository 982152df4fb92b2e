// Host build of kolibrie_b200/csrc/kb_bgp_plan.hpp (the component split, GYO and join order of kb_bgp_execute), for
// tests/test_bgp_plan_cpu.py. stdin: one BGP hypergraph per line, "n  m_0 v.. m_1 v.. ..  rows_0 .. rows_{n-1}" (m_k = variables of
// pattern k). stdout: one line per BGP, "n_comp" then per component "size k.. acyclic parent.. order.." (parent -1: root; the
// parents are written only for an acyclic component, the order always).
#include <cstdio>
#include <iostream>
#include <string>
#include <vector>

#include "kb_bgp_plan.hpp"

int main() {
    size_t n;
    while (std::cin >> n) {
        kb_bgp::Vars pv(n);
        for (size_t k = 0; k < n; k++) {
            size_t m;
            std::cin >> m;
            pv[k].resize(m);
            for (auto& v : pv[k]) std::cin >> v;
        }
        std::vector<uint64_t> rows(n);
        for (auto& r : rows) std::cin >> r;
        const auto comps = kb_bgp::components(pv);
        std::string line = std::to_string(comps.size());
        for (const auto& c : comps) {
            std::vector<int> parent;
            const bool acyclic = kb_bgp::gyo(pv, c, &parent);
            const auto order = kb_bgp::join_order(pv, c, rows, acyclic, parent);
            line += " " + std::to_string(c.size());
            for (uint32_t k : c) line += " " + std::to_string(k);
            line += acyclic ? " 1" : " 0";
            if (acyclic) for (int p : parent) line += " " + std::to_string(p);
            line += " " + std::to_string(order.size());
            for (uint32_t k : order) line += " " + std::to_string(k);
        }
        std::puts(line.c_str());
    }
    return 0;
}
