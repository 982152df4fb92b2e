// repair_tests.cpp — the reference's two query_with_repairs examples (kolibrie/examples/sparql_syntax/knowledge_graph/contradictions.rs:15-53
// and knowledge_graph.rs:228-272) and a free fact beside a conflict, written against the C++ host mirror's Reasoner::query_with_repairs.
// Built and run by tests/test_gpu_repairs.py. Exit code = number of failed checks.
#include <cstdio>
#include <string>

#include "../../kolibrie_b200/host/kolibrie_host.hpp"

using namespace kolibrie;
static int g_failed = 0;
#define CHECK(cond, msg) do { if (!(cond)) { g_failed++; std::fprintf(stderr, "FAILED %s:%d %s\n", __func__, __LINE__, msg); } } while (0)

static std::shared_ptr<Device> g_dev;
static Term V(const char* n) { return Term::Variable(n); }
static Term C(uint32_t c) { return Term::Constant(c); }

// no one is both a professor and a student (the examples' constraint; its conclusion is a dummy the reasoner never reads)
static void prof_and_student(Reasoner& r) {
    auto isa = r.dictionary.encode("isA"), prof = r.dictionary.encode("professor"), student = r.dictionary.encode("student");
    r.add_constraint(Rule{{{V("X"), C(isa), C(prof)}, {V("X"), C(isa), C(student)}}, {}, {{C(0), C(0), C(0)}}});
}

static void contradictions() {
    Reasoner r(g_dev);
    r.add_abox_triple("john", "isA", "professor");
    r.add_abox_triple("john", "isA", "student");
    r.add_abox_triple("john", "teaches", "math101");
    r.add_abox_triple("john", "enrolledIn", "physics101");
    prof_and_student(r);
    auto john = r.dictionary.encode("john"), isa = r.dictionary.encode("isA"), teaches = r.dictionary.encode("teaches");
    CHECK(r.query_with_repairs({C(john), C(isa), V("Role")}).empty(), "both roles are in the conflict");
    CHECK(r.last_repair_stats.minimal_conflicts == 1 && r.last_repair_stats.conflicted_facts == 2, "one conflict of two facts");
    auto res = r.query_with_repairs({C(john), C(teaches), V("Course")});
    CHECK(res.size() == 1 && res[0]["Course"] == r.dictionary.encode("math101"), "a fact outside the conflict is answered");
}
static void inconsistency() {
    Reasoner r(g_dev);
    r.add_abox_triple("john", "isA", "professor");
    r.add_abox_triple("john", "isA", "student");
    prof_and_student(r);
    auto isa = r.dictionary.encode("isA");
    CHECK(r.query_with_repairs({V("X"), C(isa), V("Y")}).empty(), "only consistent results");
    r.add_abox_triple("mary", "isA", "student");
    auto res = r.query_with_repairs({V("X"), C(isa), V("Y")});
    CHECK(res.size() == 1 && res[0]["X"] == r.dictionary.encode("mary"), "mary's role is certain");
    auto mary = r.dictionary.encode("mary"), student = r.dictionary.encode("student");
    CHECK(r.query_with_repairs({C(mary), C(isa), C(student)}).size() == 1, "a ground query that holds gives one empty map");
}

int main() {
    g_dev = std::make_shared<Device>(0);
    contradictions();
    inconsistency();
    std::printf("repair_tests: %d failed\n", g_failed);
    return g_failed;
}
