// bc_tests.cpp — three of the reference's backward-chaining tests (datalog/tests/reasoning_tests.rs:446-476, 511-539, 639-654) written
// against the C++ host mirror's Reasoner::backward_chaining, so they read like the reference's own. Built and run by
// tests/test_gpu_backward.py. Exit code = number of failed checks.
#include <cstdio>
#include <string>

#include "../../kolibrie_b200/host/kolibrie_host.hpp"

using namespace kolibrie;
static int g_failed = 0;
#define CHECK(cond, msg) do { if (!(cond)) { g_failed++; std::fprintf(stderr, "FAILED %s:%d %s\n", __func__, __LINE__, msg); } } while (0)

static std::shared_ptr<Device> g_dev;
static Term V(const char* n) { return Term::Variable(n); }
static Term C(uint32_t c) { return Term::Constant(c); }
static bool bc_has(const std::vector<std::map<std::string, Term>>& res, const char* var, uint32_t val) {
    for (auto& b : res) {
        auto it = b.find(var);
        if (it != b.end() && !it->second.is_var && it->second.id == val) return true;
    }
    return false;
}
static void ancestor_rules(Reasoner& r, uint32_t parent, uint32_t ancestor) {
    r.add_rule(Rule{{{V("X"), C(parent), V("Y")}}, {}, {{V("X"), C(ancestor), V("Y")}}});
    r.add_rule(Rule{{{V("X"), C(ancestor), V("Y")}, {V("Y"), C(ancestor), V("Z")}}, {}, {{V("X"), C(ancestor), V("Z")}}});
}

static void bc_2hop_transitive() {
    Reasoner r(g_dev);
    r.add_abox_triple("A", "parent", "B");
    r.add_abox_triple("B", "parent", "C");
    auto parent = r.dictionary.encode("parent"), ancestor = r.dictionary.encode("ancestor");
    auto a = r.dictionary.encode("A"), b = r.dictionary.encode("B"), c = r.dictionary.encode("C");
    ancestor_rules(r, parent, ancestor);
    auto res = r.backward_chaining({C(a), C(ancestor), V("Y")});
    CHECK(bc_has(res, "Y", b), "A ancestor B");
    CHECK(bc_has(res, "Y", c), "A ancestor C");
    CHECK(res.size() == 2, "each binding once");
}
static void bc_specific_target() {
    Reasoner r(g_dev);
    r.add_abox_triple("A", "parent", "B");
    r.add_abox_triple("B", "parent", "C");
    auto parent = r.dictionary.encode("parent"), ancestor = r.dictionary.encode("ancestor");
    auto a = r.dictionary.encode("A"), c = r.dictionary.encode("C");
    ancestor_rules(r, parent, ancestor);
    CHECK(!r.backward_chaining({C(a), C(ancestor), C(c)}).empty(), "A ancestor C derivable");
    CHECK(r.last_bc_stats.stopped_early == 1, "a ground query stops at its triple");
}
static void bc_no_spurious_negative() {
    Reasoner r(g_dev);
    r.add_abox_triple("A", "parent", "B");
    auto unknown = r.dictionary.encode("unknown");
    CHECK(r.backward_chaining({V("X"), C(unknown), V("Y")}).empty(), "nothing for an unknown predicate");
}

int main() {
    g_dev = std::make_shared<Device>(0);
    bc_2hop_transitive();
    bc_specific_target();
    bc_no_spurious_negative();
    std::printf("bc_tests: %d failed\n", g_failed);
    return g_failed;
}
