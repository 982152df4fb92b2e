// kolibrie_host.hpp — header-only C++ mirror of the reference's host-side interfaces for the hot path, on top of the C ABI
// (include/kolibrie_b200.h). The reference is compiled code (Rust); with no Rust toolchain in the image this is the host side
// a maintainer can read next to the reference: same names, argument meaning and error behaviour.
//
//   Dictionary                shared/src/dictionary.rs:17-51
//   Term / TriplePattern      shared/src/terms.rs:13-23
//   Rule / FilterCondition    shared/src/rule.rs:14-25
//   Reasoner                  datalog/src/reasoning.rs:31-100, materialisation/semi_naive.rs:89, my_naive.rs:74
//   PhysicalOperator          kolibrie/src/streamertail_optimizer/operators/physical.rs:16-76 (hot-path variants)
//   Condition                 kolibrie/src/streamertail_optimizer/types.rs:110-186
//   SparqlDatabase            kolibrie/src/sparql_database.rs:49-60, 215-258, 3364-3394
//   ExecutionEngine           kolibrie/src/streamertail_optimizer/execution/engine.rs:27, 54
//   PreparedStarJoin          (new) a StarJoin resolved once, submitted asynchronously: kb_star_join_prepare / kb_plan_submit / kb_plan_collect
//   WindowStore               the R2R store maintenance of kolibrie/src/rsp/simple_r2r.rs:95-142 on the device (append / evict by tag)
//
// All data-touching work happens in libkolibrie_b200.so; a kb_status other than KB_OK becomes a kolibrie::GpuError whose
// `unsupported()` tells the caller to take the reference's CPU path (KB_E_UNSUPPORTED).
#pragma once
#include <algorithm>
#include <cctype>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <map>
#include <memory>
#include <optional>
#include <set>
#include <stdexcept>
#include <string>
#include <tuple>
#include <unordered_map>
#include <vector>

#include "../../include/kolibrie_b200.h"

namespace kolibrie {

struct GpuError : std::runtime_error {
    kb_status status;
    GpuError(kb_status s, const std::string& m) : std::runtime_error(m), status(s) {}
    bool unsupported() const { return status == KB_E_UNSUPPORTED; }
};

// Rust `str::parse::<f64>()` acceptance (no whitespace, no '_', no hex; inf/infinity/nan in any case; "5.", ".5", "1e5")
inline std::optional<double> rust_parse_f64(const std::string& s) {
    size_t i = 0, n = s.size();
    if (n == 0) return std::nullopt;
    bool neg = false;
    if (s[0] == '+' || s[0] == '-') { neg = s[0] == '-'; i = 1; }
    if (i >= n) return std::nullopt;
    std::string rest = s.substr(i);
    std::string low = rest;
    for (auto& c : low) c = (char)std::tolower((unsigned char)c);
    if (low == "inf" || low == "infinity") return neg ? -INFINITY : INFINITY;
    if (low == "nan") return NAN;
    size_t j = i, nd = 0;
    while (j < n && std::isdigit((unsigned char)s[j])) { j++; nd++; }
    if (j < n && s[j] == '.') { j++; while (j < n && std::isdigit((unsigned char)s[j])) { j++; nd++; } }
    if (nd == 0) return std::nullopt;
    if (j < n && (s[j] == 'e' || s[j] == 'E')) {
        j++;
        if (j < n && (s[j] == '+' || s[j] == '-')) j++;
        size_t ne = 0;
        while (j < n && std::isdigit((unsigned char)s[j])) { j++; ne++; }
        if (ne == 0) return std::nullopt;
    }
    if (j != n) return std::nullopt;
    return std::strtod(s.c_str(), nullptr);
}

struct Dictionary {
    std::unordered_map<std::string, uint32_t> string_to_id;
    std::vector<std::string> id_to_string;
    uint32_t encode(const std::string& v) {
        auto it = string_to_id.find(v);
        if (it != string_to_id.end()) return it->second;
        uint32_t id = (uint32_t)id_to_string.size();
        if (id >= 0x80000000u) throw std::runtime_error("Dictionary ID space exhausted");  // dictionary.rs:36-40
        string_to_id.emplace(v, id);
        id_to_string.push_back(v);
        return id;
    }
    std::optional<uint32_t> lookup(const std::string& v) const {
        auto it = string_to_id.find(v);
        if (it == string_to_id.end()) return std::nullopt;
        return it->second;
    }
    const std::string* decode(uint32_t id) const { return id < id_to_string.size() ? &id_to_string[id] : nullptr; }
    void numeric_table(std::vector<double>* num, std::vector<uint8_t>* isn) const {
        num->assign(id_to_string.size(), 0.0);
        isn->assign(id_to_string.size(), 0);
        for (size_t i = 0; i < id_to_string.size(); i++)
            if (auto v = rust_parse_f64(id_to_string[i])) { (*num)[i] = *v; (*isn)[i] = 1; }
    }
};

struct Term {
    bool is_var = false;
    std::string name;
    uint32_t id = 0;
    static Term Variable(const std::string& n) { Term t; t.is_var = true; t.name = (!n.empty() && n[0] == '?') ? n.substr(1) : n; return t; }
    static Term Constant(uint32_t c) { Term t; t.id = c; return t; }
};
using TriplePattern = std::tuple<Term, Term, Term>;
struct Triple {
    uint32_t subject, predicate, object;
    bool operator<(const Triple& t) const { return std::tie(subject, predicate, object) < std::tie(t.subject, t.predicate, t.object); }
    bool operator==(const Triple& t) const { return subject == t.subject && predicate == t.predicate && object == t.object; }
};
struct FilterCondition { std::string variable, op, value; };
struct Rule {
    std::vector<TriplePattern> premise;
    std::vector<FilterCondition> filters;
    std::vector<TriplePattern> conclusion;
};

class SlotMap {
  public:
    uint32_t of(const std::string& raw) {
        std::string n = (!raw.empty() && raw[0] == '?') ? raw.substr(1) : raw;
        auto it = slot_.find(n);
        if (it != slot_.end()) return it->second;
        uint32_t s = (uint32_t)names.size();
        slot_.emplace(n, s);
        names.push_back(n);
        return s;
    }
    bool has(const std::string& n) const { return slot_.count(n) != 0; }
    kb_term term(const Term& t) { return t.is_var ? kb_term{1, of(t.name)} : kb_term{0, t.id}; }
    kb_pattern pattern(const TriplePattern& p) { return kb_pattern{term(std::get<0>(p)), term(std::get<1>(p)), term(std::get<2>(p))}; }
    std::vector<std::string> names;

  private:
    std::unordered_map<std::string, uint32_t> slot_;
};

class Device {  // RAII kb_ctx
  public:
    explicit Device(int device = 0) {
        kb_status rc = kb_ctx_create(device, &ctx_);
        if (rc != KB_OK) throw GpuError(rc, kb_last_error(nullptr));
    }
    ~Device() { kb_ctx_destroy(ctx_); }
    Device(const Device&) = delete;
    kb_ctx* get() const { return ctx_; }
    void check(kb_status rc) const { if (rc != KB_OK) throw GpuError(rc, kb_last_error(ctx_)); }

  private:
    kb_ctx* ctx_ = nullptr;
};

struct RelHandle {
    const Device* dev;
    kb_rel* r;
    RelHandle(const Device* d, kb_rel* rel) : dev(d), r(rel) {}
    ~RelHandle() { if (r) kb_rel_free(dev->get(), r); }
    RelHandle(const RelHandle&) = delete;
};
using Rel = std::unique_ptr<RelHandle>;

inline std::vector<std::vector<uint32_t>> download(const Device& dev, const kb_rel* r, std::vector<uint32_t>* slots) {
    uint64_t n = 0;
    uint32_t nc = 0, sl[KB_MAX_COLS];
    dev.check(kb_rel_info(r, &n, &nc, sl));
    slots->assign(sl, sl + nc);
    std::vector<std::vector<uint32_t>> cols(nc, std::vector<uint32_t>(n));
    for (uint32_t c = 0; c < nc; c++) dev.check(kb_rel_download(dev.get(), r, c, cols[c].data()));
    return cols;
}

// ------------------------------------------------------------------------------------------------------------- Reasoner
class Reasoner {
  public:
    Dictionary dictionary;
    std::vector<Rule> rules;
    std::vector<Rule> constraints;
    kb_fixpoint_stats last_stats{};
    explicit Reasoner(std::shared_ptr<Device> dev = std::make_shared<Device>(0)) : dev_(std::move(dev)) {}

    void add_abox_triple(const std::string& s, const std::string& p, const std::string& o) {
        Triple t{dictionary.encode(s), dictionary.encode(p), dictionary.encode(o)};
        if (fact_set_.insert(t).second) { facts_.push_back(t); dirty_ = true; }  // index_manager.insert dedups (index_manager.rs:41-57)
    }
    void add_rule(const Rule& r) { rules.push_back(r); }
    // reasoning.rs:95-98: a denial constraint; only its premises are read (its filters and conclusion are ignored)
    void add_constraint(const Rule& r) { constraints.push_back(r); }
    std::vector<Triple> infer_new_facts_semi_naive() { return infer(KB_SEMI_NAIVE); }
    std::vector<Triple> infer_new_facts_naive() { return infer(KB_NAIVE); }
    std::vector<Triple> infer_new_facts() { return infer_new_facts_naive(); }  // my_naive.rs:78-80

    // reasoning.rs:79-93 — like the reference, querying ENCODES unknown strings (they match nothing)
    std::vector<Triple> query_abox(const std::optional<std::string>& s, const std::optional<std::string>& p, const std::optional<std::string>& o) {
        sync();
        const std::optional<std::string>* in[3] = {&s, &p, &o};
        kb_term t[3];
        uint32_t fixed[3] = {0, 0, 0};
        for (int k = 0; k < 3; k++) {
            if (in[k]->has_value()) { fixed[k] = dictionary.encode(**in[k]); t[k] = kb_term{0, fixed[k]}; }
            else t[k] = kb_term{1, (uint32_t)k};
        }
        kb_pattern pat{t[0], t[1], t[2]};
        kb_rel* r = nullptr;
        dev_->check(kb_scan(dev_->get(), &pat, 1, nullptr, nullptr, &r));
        RelHandle h(dev_.get(), r);
        std::vector<uint32_t> slots;
        auto cols = download(*dev_, r, &slots);
        uint64_t n = 0;
        kb_rel_info(r, &n, nullptr, nullptr);
        std::vector<Triple> out(n);
        for (uint64_t i = 0; i < n; i++) {
            uint32_t v[3] = {fixed[0], fixed[1], fixed[2]};
            for (size_t c = 0; c < slots.size(); c++) v[slots[c]] = cols[c][i];
            out[i] = Triple{v[0], v[1], v[2]};
        }
        return out;
    }

    // backward_chaining.rs:165-171 on the device (kb_datalog_query): the distinct bindings of the query's variables over the facts with a
    // proof of height <= max_depth, each once, without the reference's renamed rule variables (quirk Q12); a ground query gives one empty
    // map when it holds, none when it does not. The store is only read.
    std::vector<std::map<std::string, Term>> backward_chaining(const TriplePattern& query, uint32_t max_depth = KB_BC_MAX_DEPTH) {
        sync();
        CompiledRules cr = compile_rules(rules);
        SlotMap sm;
        const kb_pattern q = sm.pattern(query);
        kb_rel* out = nullptr;
        dev_->check(kb_datalog_query(dev_->get(), cr.kr.data(), (uint32_t)cr.kr.size(), &q, max_depth, &out, &last_bc_stats));
        RelHandle h(dev_.get(), out);
        std::vector<uint32_t> slots;
        auto cols = download(*dev_, out, &slots);
        uint64_t n = 0;
        dev_->check(kb_rel_info(out, &n, nullptr, nullptr));
        std::vector<std::map<std::string, Term>> res(n);
        for (uint64_t i = 0; i < n; i++)
            for (size_t c = 0; c < slots.size(); c++) res[i][sm.names[slots[c]]] = Term::Constant(cols[c][i]);
        return res;
    }
    kb_bc_stats last_bc_stats{};

    // repairs.rs:10-43 on the device (kb_datalog_query_repairs), under IAR semantics: the distinct bindings of the query's variables, as
    // ids, over the facts that lie in no minimal conflict of the constraints. The reference's answer can be a strict subset when its
    // search keeps a non-maximal repair (quirk Q13). A ground query gives one empty map when it holds. The store is only read.
    std::vector<std::map<std::string, uint32_t>> query_with_repairs(const TriplePattern& query) {
        sync();
        CompiledRules cr = compile_rules(constraints);
        SlotMap sm;
        const kb_pattern q = sm.pattern(query);
        kb_rel* out = nullptr;
        dev_->check(kb_datalog_query_repairs(dev_->get(), cr.kr.data(), (uint32_t)cr.kr.size(), &q, &out, &last_repair_stats));
        RelHandle h(dev_.get(), out);
        std::vector<uint32_t> slots;
        auto cols = download(*dev_, out, &slots);
        uint64_t n = 0;
        dev_->check(kb_rel_info(out, &n, nullptr, nullptr));
        std::vector<std::map<std::string, uint32_t>> res(n);
        for (uint64_t i = 0; i < n; i++)
            for (size_t c = 0; c < slots.size(); c++) res[i][sm.names[slots[c]]] = cols[c][i];
        return res;
    }
    kb_repair_stats last_repair_stats{};

  private:
    static uint32_t cmp_of(const std::string& op) {
        if (op == ">") return KB_CMP_GT;
        if (op == ">=") return KB_CMP_GE;
        if (op == "<") return KB_CMP_LT;
        if (op == "<=") return KB_CMP_LE;
        if (op == "=") return KB_CMP_EQ;
        if (op == "!=") return KB_CMP_NE;
        return 0;  // e.g. "OR:>" is a no-op in the reference (rules.rs:133-165)
    }
    void sync() {
        if (dirty_) {
            std::vector<uint32_t> s(facts_.size()), p(facts_.size()), o(facts_.size());
            for (size_t i = 0; i < facts_.size(); i++) { s[i] = facts_[i].subject; p[i] = facts_[i].predicate; o[i] = facts_[i].object; }
            dev_->check(kb_store_load(dev_->get(), s.data(), p.data(), o.data(), s.size()));
            dirty_ = false;
        }
        // the numeric side table the rule filters read, parsed on the device from the dictionary's strings (uploaded when the device
        // dictionary does not hold as many)
        uint32_t n_dev = 0;
        dev_->check(kb_dict_strings_info(dev_->get(), &n_dev, nullptr));
        if (n_dev != dictionary.id_to_string.size()) {
            std::vector<uint64_t> off(dictionary.id_to_string.size() + 1, 0);
            std::string bytes;
            for (size_t i = 0; i < dictionary.id_to_string.size(); i++) { bytes += dictionary.id_to_string[i]; off[i + 1] = bytes.size(); }
            dev_->check(kb_dict_strings_load(dev_->get(), off.data(), reinterpret_cast<const uint8_t*>(bytes.data()), (uint32_t)dictionary.id_to_string.size()));
        }
        dev_->check(kb_dict_numeric_derive(dev_->get(), KB_NUMERIC_F64, 0, nullptr));
    }
    struct CompiledRules {  // kb_rule views over their own pattern and filter arrays
        std::vector<std::vector<kb_pattern>> prem, conc;
        std::vector<std::vector<kb_rule_filter>> fl;
        std::vector<kb_rule> kr;
    };
    CompiledRules compile_rules(const std::vector<Rule>& rs) const {
        CompiledRules c;
        auto& prem = c.prem; auto& conc = c.conc; auto& fl = c.fl; auto& kr = c.kr;
        prem.resize(rs.size()); conc.resize(rs.size()); fl.resize(rs.size()); kr.resize(rs.size());
        for (size_t r = 0; r < rs.size(); r++) {
            SlotMap sm;
            for (auto& p : rs[r].premise) prem[r].push_back(sm.pattern(p));
            for (auto& p : rs[r].conclusion) conc[r].push_back(sm.pattern(p));
            for (auto& f : rs[r].filters) {
                if (!sm.has(f.variable)) continue;  // unbound lhs: the reference skips the filter (rules.rs:139)
                kb_rule_filter k{sm.of(f.variable), cmp_of(f.op), 0, 0, 0.0};
                if (sm.has(f.value)) { k.rhs_is_var = 1; k.rhs_slot = sm.of(f.value); }
                else k.rhs_value = rust_parse_f64(f.value).value_or(0.0);
                fl[r].push_back(k);
            }
            kr[r] = kb_rule{prem[r].data(), (uint32_t)prem[r].size(), fl[r].data(), (uint32_t)fl[r].size(), conc[r].data(), (uint32_t)conc[r].size()};
        }
        return c;
    }
    std::vector<Triple> infer(uint32_t strategy) {
        sync();
        CompiledRules cr = compile_rules(rules);
        kb_rel* out = nullptr;
        dev_->check(kb_datalog_fixpoint(dev_->get(), cr.kr.data(), (uint32_t)cr.kr.size(), strategy, &out, &last_stats));
        RelHandle h(dev_.get(), out);
        std::vector<uint32_t> slots;
        auto cols = download(*dev_, out, &slots);
        std::vector<Triple> res(cols.empty() ? 0 : cols[0].size());
        for (size_t i = 0; i < res.size(); i++) res[i] = Triple{cols[0][i], cols[1][i], cols[2][i]};
        for (auto& t : res) if (fact_set_.insert(t).second) facts_.push_back(t);  // the device appended them to its store too
        return res;
    }
    std::shared_ptr<Device> dev_;
    std::vector<Triple> facts_;
    std::set<Triple> fact_set_;
    bool dirty_ = true;
};

// ------------------------------------------------------------------------------------------------------ FILTER conditions
struct FilterExpression {
    enum Kind { Comparison, And, Or, Not } kind = Comparison;
    std::string var, op, value;                  // Comparison(var, op, value)
    std::shared_ptr<FilterExpression> left, right;  // And / Or (Not uses left)
    static FilterExpression Cmp(std::string v, std::string o, std::string val) { FilterExpression e; e.var = std::move(v); e.op = std::move(o); e.value = std::move(val); return e; }
    static FilterExpression AndOf(FilterExpression a, FilterExpression b) { FilterExpression e; e.kind = And; e.left = std::make_shared<FilterExpression>(std::move(a)); e.right = std::make_shared<FilterExpression>(std::move(b)); return e; }
    static FilterExpression OrOf(FilterExpression a, FilterExpression b) { FilterExpression e; e.kind = Or; e.left = std::make_shared<FilterExpression>(std::move(a)); e.right = std::make_shared<FilterExpression>(std::move(b)); return e; }
    static FilterExpression NotOf(FilterExpression a) { FilterExpression e; e.kind = Not; e.left = std::make_shared<FilterExpression>(std::move(a)); return e; }
};
struct Condition {
    FilterExpression expression;
    void compile(const FilterExpression& e, SlotMap& sm, const Dictionary& d, std::vector<kb_filter_op>* ops) const {
        switch (e.kind) {
            case FilterExpression::Comparison: {
                kb_filter_op op{};
                op.slot = sm.of(e.var);
                if (e.op == "=" || e.op == "!=") {  // decoded == literal <=> id == encode(literal) (types.rs:131-132)
                    op.op = e.op == "=" ? KB_F_EQ_ID : KB_F_NE_ID;
                    op.id = d.lookup(e.value).value_or(KB_ID_NONE);
                } else {
                    op.op = KB_F_CMP_NUM;
                    op.cmp = e.op == ">" ? KB_CMP_GT : e.op == ">=" ? KB_CMP_GE : e.op == "<" ? KB_CMP_LT : e.op == "<=" ? KB_CMP_LE : 0;
                    if (!op.cmp) throw GpuError(KB_E_UNSUPPORTED, "operator " + e.op + ": the reference evaluates it to false");
                    op.value = rust_parse_f64(e.value).value_or(0.0);  // types.rs:133-148 unwrap_or(0.0) — also for "?other" (quirk Q10)
                }
                ops->push_back(op);
            } break;
            case FilterExpression::And: case FilterExpression::Or: {
                compile(*e.left, sm, d, ops); compile(*e.right, sm, d, ops);
                kb_filter_op op{}; op.op = e.kind == FilterExpression::And ? KB_F_AND : KB_F_OR; ops->push_back(op);
            } break;
            case FilterExpression::Not: {
                compile(*e.left, sm, d, ops);
                kb_filter_op op{}; op.op = KB_F_NOT; ops->push_back(op);
            } break;
        }
    }
};

// ---------------------------------------------------------------------------------------------------- PhysicalOperator
struct PhysicalOperator {
    enum Kind { TableScan, IndexScan, Filter, Projection, HashJoin, OptimizedHashJoin, NestedLoopJoin, ParallelJoin, StarJoin } kind;
    TriplePattern pattern;                      // scans
    std::shared_ptr<PhysicalOperator> input, left, right;
    Condition condition;                        // Filter
    std::vector<std::string> variables;         // Projection
    std::string join_var;                       // StarJoin
    std::vector<TriplePattern> patterns;        // StarJoin
    static PhysicalOperator Scan(Kind k, TriplePattern p) { PhysicalOperator o; o.kind = k; o.pattern = std::move(p); return o; }
    static PhysicalOperator FilterOf(PhysicalOperator in, Condition c) { PhysicalOperator o; o.kind = Filter; o.input = std::make_shared<PhysicalOperator>(std::move(in)); o.condition = std::move(c); return o; }
    static PhysicalOperator ProjectionOf(PhysicalOperator in, std::vector<std::string> v) { PhysicalOperator o; o.kind = Projection; o.input = std::make_shared<PhysicalOperator>(std::move(in)); o.variables = std::move(v); return o; }
    static PhysicalOperator Join(Kind k, PhysicalOperator l, PhysicalOperator r) { PhysicalOperator o; o.kind = k; o.left = std::make_shared<PhysicalOperator>(std::move(l)); o.right = std::make_shared<PhysicalOperator>(std::move(r)); return o; }
    static PhysicalOperator Star(std::string jv, std::vector<TriplePattern> ps) { PhysicalOperator o; o.kind = StarJoin; o.join_var = std::move(jv); o.patterns = std::move(ps); return o; }
};

class SparqlDatabase {
  public:
    Dictionary dictionary;
    std::set<Triple> triples;  // BTreeSet<Triple>: set semantics, (s,p,o) order
    explicit SparqlDatabase(std::shared_ptr<Device> dev = std::make_shared<Device>(0)) : dev_(std::move(dev)) {}
    void add_triple_parts(const std::string& s, const std::string& p, const std::string& o) { add_triple(Triple{dictionary.encode(s), dictionary.encode(p), dictionary.encode(o)}); }
    void add_triple(const Triple& t) { if (triples.insert(t).second) version_++; }        // sparql_database.rs:215-226
    bool delete_triple(const Triple& t) { if (triples.erase(t)) { version_++; return true; } return false; }  // :229-242
    // the reference builds six hash indexes here (:3364-3394); we (re)upload the store and partition it by predicate on the device
    void build_all_indexes() { sync(); dev_->check(kb_store_build_index(dev_->get(), nullptr, nullptr)); }
    void sync() {
        if (uploaded_ == version_) return;
        std::vector<uint32_t> s, p, o;
        for (auto& t : triples) { s.push_back(t.subject); p.push_back(t.predicate); o.push_back(t.object); }
        dev_->check(kb_store_load(dev_->get(), s.data(), p.data(), o.data(), s.size()));
        // the strings themselves: the final id -> string step of execute() runs on the device (kb_rel_decode), and the numeric side
        // table is parsed from them there (kb_dict_numeric_derive)
        upload_strings();
        dev_->check(kb_dict_numeric_derive(dev_->get(), KB_NUMERIC_F64, 0, nullptr));
        uploaded_ = version_;
    }
    const Device& device() const { return *dev_; }
    // the per-term encode loop of a bulk load (sparql_database.rs:1000-1013 -> dictionary.rs:32-48) as one device call: `terms` holds
    // three strings per triple in document order; the ids are those of the sequential loop, the host dictionary learns the new strings
    // from the positions that introduced them, the triples join the set
    void add_triples_bulk(const std::vector<std::string>& terms) {
        if (terms.size() % 3) throw std::invalid_argument("three terms per triple");
        uint32_t n_dev = 0;
        dev_->check(kb_dict_strings_info(dev_->get(), &n_dev, nullptr));
        if (n_dev != dictionary.id_to_string.size()) upload_strings();
        std::vector<uint64_t> off(terms.size() + 1, 0);
        std::string bytes;
        for (size_t i = 0; i < terms.size(); i++) { bytes += terms[i]; off[i + 1] = bytes.size(); }
        std::vector<uint32_t> ids(terms.size());
        std::vector<uint64_t> first(terms.size());
        uint32_t n_new = 0;
        dev_->check(kb_dict_encode(dev_->get(), off.data(), reinterpret_cast<const uint8_t*>(bytes.data()), terms.size(), ids.data(), &n_new, first.data()));
        for (uint32_t k = 0; k < n_new; k++) dictionary.encode(terms[first[k]]);  // same order => same ids
        for (size_t i = 0; i + 2 < ids.size(); i += 3) add_triple(Triple{ids[i], ids[i + 1], ids[i + 2]});
    }

  private:
    void upload_strings() {
        std::vector<uint64_t> off(dictionary.id_to_string.size() + 1, 0);
        std::string bytes;
        for (size_t i = 0; i < dictionary.id_to_string.size(); i++) { bytes += dictionary.id_to_string[i]; off[i + 1] = bytes.size(); }
        dev_->check(kb_dict_strings_load(dev_->get(), off.data(), reinterpret_cast<const uint8_t*>(bytes.data()), (uint32_t)dictionary.id_to_string.size()));
    }
    std::shared_ptr<Device> dev_;
    long version_ = 0, uploaded_ = -1;
};

// A StarJoin resolved once and submitted asynchronously (the headline path of bench.py): submit() is one kernel launch, collect() waits
// for that ticket only; up to `ring` tickets may be in flight. The plan is bound to the store / index version it was prepared on.
class PreparedStarJoin {
  public:
    PreparedStarJoin(SparqlDatabase& db, const std::string& join_var, const std::vector<TriplePattern>& patterns, const Condition* filter = nullptr, uint32_t ring = 4)
        : dev_(&db.device()) {
        db.build_all_indexes();
        std::vector<kb_pattern> ps;
        for (auto& p : patterns) ps.push_back(sm_.pattern(p));
        std::vector<kb_filter_op> ops;
        if (filter) filter->compile(filter->expression, sm_, db.dictionary, &ops);
        dev_->check(kb_star_join_prepare(dev_->get(), sm_.of(join_var), ps.data(), (uint32_t)ps.size(), ops.data(), (uint32_t)ops.size(), nullptr, 0, nullptr, 0, ring, &plan_));
    }
    ~PreparedStarJoin() { if (plan_) kb_plan_free(dev_->get(), plan_); }
    PreparedStarJoin(const PreparedStarJoin&) = delete;
    PreparedStarJoin& operator=(const PreparedStarJoin&) = delete;
    uint64_t submit() { uint64_t t = 0; dev_->check(kb_plan_submit(dev_->get(), plan_, &t)); return t; }
    uint64_t collect(uint64_t ticket) { uint64_t n = 0; dev_->check(kb_plan_collect(dev_->get(), plan_, ticket, &n, nullptr, nullptr)); return n; }  // rows of that step
    const SlotMap& slots() const { return sm_; }

  private:
    const Device* dev_;
    SlotMap sm_;
    kb_plan* plan_ = nullptr;
};

// SimpleR2R::add / remove (kolibrie/src/rsp/simple_r2r.rs:95-128) for whole window slides: a slide is a store segment with a tag; the
// store index built once stays valid across slides (kb_store_append / kb_store_evict maintain it in place).
class WindowStore {
  public:
    explicit WindowStore(std::shared_ptr<Device> dev) : dev_(std::move(dev)) {}
    void append_slide(uint64_t tag, const std::vector<Triple>& slide) {
        std::vector<uint32_t> s, p, o;
        for (auto& t : slide) { s.push_back(t.subject); p.push_back(t.predicate); o.push_back(t.object); }
        dev_->check(kb_store_append(dev_->get(), s.data(), p.data(), o.data(), s.size(), tag));
    }
    void evict_slide(uint64_t tag) { dev_->check(kb_store_evict(dev_->get(), tag)); }
    void build_index() { dev_->check(kb_store_build_index(dev_->get(), nullptr, nullptr)); }
    uint64_t star_join_rows(uint32_t join_slot, const std::vector<kb_pattern>& ps) {
        kb_rel* out = nullptr;
        dev_->check(kb_star_join(dev_->get(), join_slot, ps.data(), (uint32_t)ps.size(), nullptr, 0, &out));
        uint64_t n = 0;
        kb_rel_info(out, &n, nullptr, nullptr);
        kb_rel_free(dev_->get(), out);
        return n;
    }

  private:
    std::shared_ptr<Device> dev_;
};

struct ExecutionEngine {
    static Rel run(const PhysicalOperator& op, SparqlDatabase& db, SlotMap& sm) {
        const Device& dev = db.device();
        kb_rel* out = nullptr;
        switch (op.kind) {
            case PhysicalOperator::TableScan: case PhysicalOperator::IndexScan: {
                kb_pattern p = sm.pattern(op.pattern);
                dev.check(kb_scan(dev.get(), &p, 1, nullptr, nullptr, &out));
            } break;
            case PhysicalOperator::Filter: {
                std::vector<kb_filter_op> ops;
                if (op.input->kind == PhysicalOperator::StarJoin) {  // Selection over a star: conjuncts are pushed into its scans
                    std::vector<kb_pattern> ps;
                    for (auto& p : op.input->patterns) ps.push_back(sm.pattern(p));
                    op.condition.compile(op.condition.expression, sm, db.dictionary, &ops);
                    dev.check(kb_star_join(dev.get(), sm.of(op.input->join_var), ps.data(), (uint32_t)ps.size(), ops.data(), (uint32_t)ops.size(), &out));
                } else {
                    Rel in = run(*op.input, db, sm);
                    op.condition.compile(op.condition.expression, sm, db.dictionary, &ops);
                    dev.check(kb_filter(dev.get(), in->r, ops.data(), (uint32_t)ops.size(), &out));
                }
            } break;
            case PhysicalOperator::Projection: {
                Rel in = run(*op.input, db, sm);
                std::vector<uint32_t> slots;
                for (auto& v : op.variables) slots.push_back(sm.of(v));
                dev.check(kb_project(dev.get(), in->r, slots.data(), (uint32_t)slots.size(), &out));
            } break;
            case PhysicalOperator::ParallelJoin:
                // ParallelJoin with a scan on the right = bind join (engine.rs:926-949 -> 840-885): every left row is substituted into the
                // right pattern and looked up in the index; relationally the natural join of the two (the fallback when the device says
                // the pattern's shape has no lookup)
                if (op.right->kind == PhysicalOperator::TableScan || op.right->kind == PhysicalOperator::IndexScan) {
                    Rel l = run(*op.left, db, sm);
                    kb_pattern p = sm.pattern(op.right->pattern);
                    const kb_status st = kb_bind_join(dev.get(), l->r, &p, &out);
                    if (st == KB_OK) break;
                    if (st != KB_E_UNSUPPORTED) dev.check(st);
                    Rel r = run(*op.right, db, sm);
                    dev.check(kb_hash_join(dev.get(), l->r, r->r, &out));
                    break;
                }
                [[fallthrough]];
            case PhysicalOperator::HashJoin: case PhysicalOperator::OptimizedHashJoin: case PhysicalOperator::NestedLoopJoin: {
                Rel l = run(*op.left, db, sm), r = run(*op.right, db, sm);
                dev.check(kb_hash_join(dev.get(), l->r, r->r, &out));
            } break;
            case PhysicalOperator::StarJoin: {
                std::vector<kb_pattern> ps;
                for (auto& p : op.patterns) ps.push_back(sm.pattern(p));
                dev.check(kb_star_join(dev.get(), sm.of(op.join_var), ps.data(), (uint32_t)ps.size(), nullptr, 0, &out));
            } break;
        }
        return std::make_unique<RelHandle>(&dev, out);
    }
    // engine.rs:54
    static std::vector<std::unordered_map<std::string, uint32_t>> execute_with_ids(const PhysicalOperator& op, SparqlDatabase& db) {
        db.sync();
        SlotMap sm;
        Rel rel = run(op, db, sm);
        std::vector<uint32_t> slots;
        auto cols = download(db.device(), rel->r, &slots);
        uint64_t n = 0;
        kb_rel_info(rel->r, &n, nullptr, nullptr);
        std::vector<std::unordered_map<std::string, uint32_t>> rows(n);
        for (uint64_t i = 0; i < n; i++) for (size_t c = 0; c < slots.size(); c++) rows[i][sm.names[slots[c]]] = cols[c][i];
        return rows;
    }
    // engine.rs:27-51 — ids all the way, decoded only at the final step: kb_rel_decode gathers each column's strings on the device
    static std::vector<std::unordered_map<std::string, std::string>> execute(const PhysicalOperator& op, SparqlDatabase& db) {
        db.sync();
        SlotMap sm;
        Rel rel = run(op, db, sm);
        uint64_t n = 0;
        uint32_t n_cols = 0, slots[KB_MAX_COLS];
        db.device().check(kb_rel_info(rel->r, &n, &n_cols, slots));
        std::vector<std::unordered_map<std::string, std::string>> out(n);
        for (uint32_t c = 0; c < n_cols; c++) {
            kb_strings* h = nullptr;
            db.device().check(kb_rel_decode(db.device().get(), rel->r, c, &h));
            uint64_t cnt = 0, total = 0;
            kb_strings_info(h, &cnt, &total);
            std::vector<uint64_t> off(cnt + 1);
            std::string bytes(total, '\0');
            const kb_status st = kb_strings_download(db.device().get(), h, off.data(), reinterpret_cast<uint8_t*>(&bytes[0]));
            kb_strings_free(db.device().get(), h);
            db.device().check(st);
            for (uint64_t i = 0; i < cnt; i++) out[i][sm.names[slots[c]]] = bytes.substr(off[i], off[i + 1] - off[i]);
        }
        return out;
    }
};

}  // namespace kolibrie
