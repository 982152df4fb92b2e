//! `InferenceStrategy` that runs the whole fixpoint on the device in its first round (infer_generic.rs:27-53 then sees an empty
//! second round and stops): rounds, per-round deltas and the inferred set are those of `SemiNaiveStrategy` (semi_naive.rs:17-85).
use crate::ffi::*;
use crate::{DeviceStore, SlotMap};
use datalog::reasoning::materialisation::infer_generic::InferenceStrategy;
use shared::dictionary::Dictionary;
use shared::rule::Rule;
use shared::triple::Triple;
use std::collections::HashSet;
use std::ptr;

pub struct GpuSemiNaiveStrategy<'a> { pub dev: &'a mut DeviceStore, pub strategy: u32, done: bool }

impl<'a> GpuSemiNaiveStrategy<'a> {
    pub fn new(dev: &'a mut DeviceStore) -> Self { Self { dev, strategy: KB_SEMI_NAIVE, done: false } }
}

/// `Rule` -> (patterns, filters) in slot form; FilterCondition semantics of rules.rs:133-165
pub(crate) fn compile_rule(rule: &Rule) -> Option<(Vec<KbPattern>, Vec<KbRuleFilter>, Vec<KbPattern>)> {
    let mut slots = SlotMap::default();
    let prem: Option<Vec<KbPattern>> = rule.premise.iter().map(|p| slots.pattern(p)).collect();
    let conc: Option<Vec<KbPattern>> = rule.conclusion.iter().map(|p| slots.pattern(p)).collect();
    let mut fl = Vec::new();
    for f in &rule.filters {
        let name = f.variable.strip_prefix('?').unwrap_or(&f.variable);
        let Some(&lhs) = slots.slot.get(name) else { continue };  // unbound lhs: the reference skips the filter (rules.rs:139)
        let cmp = match f.operator.as_str() { ">" => KB_CMP_GT, ">=" => KB_CMP_GE, "<" => KB_CMP_LT, "<=" => KB_CMP_LE, "=" => KB_CMP_EQ, "!=" => KB_CMP_NE, _ => 0 };
        let rhs = f.value.strip_prefix('?').unwrap_or(&f.value);
        if let Some(&r) = slots.slot.get(rhs) { fl.push(KbRuleFilter { lhs_slot: lhs, cmp, rhs_is_var: 1, rhs_slot: r, rhs_value: 0.0 }); }
        else { fl.push(KbRuleFilter { lhs_slot: lhs, cmp, rhs_is_var: 0, rhs_slot: 0, rhs_value: f.value.parse::<f64>().unwrap_or(0.0) }); }
    }
    Some((prem?, fl, conc?))
}

impl<'a> InferenceStrategy for GpuSemiNaiveStrategy<'a> {
    fn infer_round(&mut self, dictionary: &mut Dictionary, rules: &Vec<Rule>, all_facts: &Vec<Triple>, _known: &HashSet<Triple>) -> HashSet<Triple> {
        if self.done { return HashSet::new(); }
        self.done = true;
        let ctx = self.dev.ctx;
        let n = all_facts.len();
        let (mut s, mut p, mut o) = (Vec::with_capacity(n), Vec::with_capacity(n), Vec::with_capacity(n));
        for t in all_facts { s.push(t.subject); p.push(t.predicate); o.push(t.object); }
        let nd = dictionary.id_to_string.len();
        let (mut num, mut isn) = (vec![0f64; nd], vec![0u8; nd]);
        for (i, st) in dictionary.id_to_string.iter().enumerate() { if let Ok(v) = st.parse::<f64>() { num[i] = v; isn[i] = 1; } }
        unsafe {
            if kb_store_load(ctx, s.as_ptr(), p.as_ptr(), o.as_ptr(), n as u64) != KB_OK { return HashSet::new(); }
            if kb_dict_numeric_load(ctx, num.as_ptr(), isn.as_ptr(), nd as u32) != KB_OK { return HashSet::new(); }
        }
        self.dev.invalidate();
        let compiled: Option<Vec<_>> = rules.iter().map(compile_rule).collect();
        let Some(compiled) = compiled else { return HashSet::new() };  // quoted-triple terms in a rule: the CPU strategy
        let kr: Vec<KbRule> = compiled.iter().map(|(pr, fl, co)| KbRule { premise: pr.as_ptr(), n_premise: pr.len() as u32, filters: fl.as_ptr(),
            n_filters: fl.len() as u32, conclusion: co.as_ptr(), n_conclusion: co.len() as u32 }).collect();
        let mut rel: *mut KbRel = ptr::null_mut();
        let mut st = std::mem::MaybeUninit::<KbFixpointStats>::zeroed();
        if unsafe { kb_datalog_fixpoint(ctx, kr.as_ptr(), kr.len() as u32, self.strategy, &mut rel, st.as_mut_ptr()) } != KB_OK {
            return HashSet::new();  // KB_E_UNSUPPORTED (unsafe head, variable head predicate ...): the caller retries with SemiNaiveStrategy
        }
        let mut nrows = 0u64;
        unsafe { kb_rel_info(rel, &mut nrows, ptr::null_mut(), ptr::null_mut()) };
        let mut cols = [vec![0u32; nrows as usize], vec![0u32; nrows as usize], vec![0u32; nrows as usize]];
        for c in 0..3 { unsafe { kb_rel_download(ctx, rel, c as u32, cols[c].as_mut_ptr()) }; }
        unsafe { kb_rel_free(ctx, rel) };
        (0..nrows as usize).map(|i| Triple { subject: cols[0][i], predicate: cols[1][i], object: cols[2][i] }).collect()
    }
}

/// `Reasoner::backward_chaining` (backward_chaining.rs:165-171) on the device: `all_facts` become the store and kb_datalog_query answers
/// `query` over the facts with a proof of height <= `max_depth` (KB_BC_MAX_DEPTH = the reference's MAX_DEPTH). Each distinct binding of
/// the query's own variables comes once, without the renamed rule variables (quirk Q12); a ground query gives one empty map when it
/// holds. None: the device refuses the shape (a quoted term, a rule without premises, a variable premise predicate): the caller runs
/// the reference's own method.
pub fn backward_chaining(dev: &mut DeviceStore, all_facts: &[Triple], rules: &[Rule], query: &shared::terms::TriplePattern, max_depth: u32)
                         -> Option<Vec<std::collections::HashMap<String, shared::terms::Term>>> {
    let ctx = dev.ctx;
    let n = all_facts.len();
    let (mut s, mut p, mut o) = (Vec::with_capacity(n), Vec::with_capacity(n), Vec::with_capacity(n));
    for t in all_facts { s.push(t.subject); p.push(t.predicate); o.push(t.object); }
    if unsafe { kb_store_load(ctx, s.as_ptr(), p.as_ptr(), o.as_ptr(), n as u64) } != KB_OK { return None; }
    dev.invalidate();
    let compiled: Option<Vec<_>> = rules.iter().map(compile_rule).collect();
    let compiled = compiled?;
    let kr: Vec<KbRule> = compiled.iter().map(|(pr, fl, co)| KbRule { premise: pr.as_ptr(), n_premise: pr.len() as u32, filters: fl.as_ptr(),
        n_filters: fl.len() as u32, conclusion: co.as_ptr(), n_conclusion: co.len() as u32 }).collect();
    let mut slots = SlotMap::default();
    let q = slots.pattern(query)?;
    let mut rel: *mut KbRel = ptr::null_mut();
    let mut st = std::mem::MaybeUninit::<KbBcStats>::zeroed();
    if unsafe { kb_datalog_query(ctx, kr.as_ptr(), kr.len() as u32, &q, max_depth, &mut rel, st.as_mut_ptr()) } != KB_OK { return None; }
    let (mut nrows, mut ncols) = (0u64, 0u32);
    let mut sl = [0u32; KB_MAX_COLS as usize];
    unsafe { kb_rel_info(rel, &mut nrows, &mut ncols, sl.as_mut_ptr()) };
    let mut cols = vec![vec![0u32; nrows as usize]; ncols as usize];
    for c in 0..ncols as usize { unsafe { kb_rel_download(ctx, rel, c as u32, cols[c].as_mut_ptr()) }; }
    unsafe { kb_rel_free(ctx, rel) };
    Some((0..nrows as usize).map(|i| (0..ncols as usize).map(|c| (slots.names[sl[c] as usize].clone(), shared::terms::Term::Constant(cols[c][i]))).collect()).collect())
}

/// `Reasoner::query_with_repairs` (repairs.rs:10-43) on the device, under IAR semantics: `all_facts` become the store and
/// kb_datalog_query_repairs answers `query` over the facts that lie in no minimal conflict of `constraints` (their premises are read,
/// their filters and conclusions are not). Each distinct binding comes once, as ids; the reference's answer can be a strict subset of it
/// when its search keeps a non-maximal repair (quirk Q13). A ground query gives one empty map when it holds. None: the device refuses
/// the shape (a quoted term, more than KB_MAX_PREMISES premises): the caller runs the reference's own method.
pub fn query_with_repairs(dev: &mut DeviceStore, all_facts: &[Triple], constraints: &[Rule], query: &shared::terms::TriplePattern)
                          -> Option<Vec<std::collections::HashMap<String, u32>>> {
    let ctx = dev.ctx;
    let n = all_facts.len();
    let (mut s, mut p, mut o) = (Vec::with_capacity(n), Vec::with_capacity(n), Vec::with_capacity(n));
    for t in all_facts { s.push(t.subject); p.push(t.predicate); o.push(t.object); }
    if unsafe { kb_store_load(ctx, s.as_ptr(), p.as_ptr(), o.as_ptr(), n as u64) } != KB_OK { return None; }
    dev.invalidate();
    let compiled: Option<Vec<_>> = constraints.iter().map(compile_rule).collect();
    let compiled = compiled?;
    let kr: Vec<KbRule> = compiled.iter().map(|(pr, fl, co)| KbRule { premise: pr.as_ptr(), n_premise: pr.len() as u32, filters: fl.as_ptr(),
        n_filters: fl.len() as u32, conclusion: co.as_ptr(), n_conclusion: co.len() as u32 }).collect();
    let mut slots = SlotMap::default();
    let q = slots.pattern(query)?;
    let mut rel: *mut KbRel = ptr::null_mut();
    let mut st = std::mem::MaybeUninit::<KbRepairStats>::zeroed();
    if unsafe { kb_datalog_query_repairs(ctx, kr.as_ptr(), kr.len() as u32, &q, &mut rel, st.as_mut_ptr()) } != KB_OK { return None; }
    let (mut nrows, mut ncols) = (0u64, 0u32);
    let mut sl = [0u32; KB_MAX_COLS as usize];
    unsafe { kb_rel_info(rel, &mut nrows, &mut ncols, sl.as_mut_ptr()) };
    let mut cols = vec![vec![0u32; nrows as usize]; ncols as usize];
    for c in 0..ncols as usize { unsafe { kb_rel_download(ctx, rel, c as u32, cols[c].as_mut_ptr()) }; }
    unsafe { kb_rel_free(ctx, rel) };
    Some((0..nrows as usize).map(|i| (0..ncols as usize).map(|c| (slots.names[sl[c] as usize].clone(), cols[c][i])).collect()).collect())
}
