//! `R2ROperator` over the device store: a window firing is `remove(previous window)` + `add(current window)` + `materialize()` +
//! `execute_query(plan)` (rsp_engine.rs:94-109; simple_r2r.rs:95-142). The adds of one firing become ONE store segment tagged with the
//! firing number, the removes evict the segment of the firing they were added in; the store index is maintained across both (one chunk
//! per segment), so that the per-slide query keeps the one-kernel index path.
//!
//! Rules run on the device. The first firing evicts the inferred segment and runs `kb_datalog_fixpoint` over the window; from then on
//! the store is closed under the rules and every firing is ONE `kb_datalog_maintain` call (the segments that left the window, the
//! firing's adds): delete-and-rederive from the slide instead of a closure from scratch per firing (simple_r2r.rs:103-128).
//!
//! The device store is this operator's: `DeviceStore::segmented` keeps `execute_query` from replacing it with `inner.item.triples`
//! (which would drop the firing tags and the inferred segment); the dictionary's tables are still mirrored before every firing and query
//! (a numeric-table load voids the closed token only when a rule filter compares numbers). The derived triples are mirrored into
//! `inner.item`, so the host's query path (shapes the device does not take) sees them too.
//!
//! `with_stream_operator` moves the Relation-to-Stream operator (r2s.rs:37-58) onto the device as well: `execute_query` then runs
//! `kb_r2s_eval` on the firing's device result and downloads and decodes only the rows it emits. Register such an engine with RSTREAM,
//! whose operator is a passthrough (r2s.rs:39): the composition is the reference's ISTREAM / DSTREAM.
use crate::ffi::*;
use crate::reasoner::compile_rule;
use crate::{try_execute, try_execute_rel, DeviceStore};
use kolibrie::rsp::r2r::{AsAnyMut, R2ROperator};
use kolibrie::rsp::r2s::StreamOperator;
use kolibrie::rsp::simple_r2r::SimpleR2R;
use kolibrie::streamertail_optimizer::PhysicalOperator;
use shared::triple::Triple;
use std::any::Any;
use std::collections::{HashMap, HashSet};
use std::ptr;

pub struct GpuR2R {
    pub inner: SimpleR2R,       // parsing, rules, dictionary: unchanged host logic
    pub dev: DeviceStore,
    pending: Vec<Triple>,       // adds of the current firing, not yet on the device
    evicted: Vec<u64>,          // segments whose triples all left the window since the last firing, not yet evicted on the device
    firing: u64,
    tag_of: HashMap<Triple, u64>,
    live: HashMap<u64, usize>,  // tag -> triples of that segment still in the window
    closed: bool,               // the device store is closed under the rules (the last materialize succeeded, nothing changed since)
    derived: HashSet<Triple>,   // the inferred segment, mirrored on the host (what materialize returns)
    stream: Option<DeviceStream>,  // with_stream_operator: the R2S operator runs on the device result
}

/// The device R2S operator of a `GpuR2R`. Its rows are the query's variables in name order: slot i is `names[i]`, whichever slots the
/// query's own relation used, so that device results and host fallbacks feed one state.
struct DeviceStream {
    kind: u32,
    op: *mut kb_r2s,      // created at the first firing, when the variables are known
    names: Vec<String>,
}

fn triples_of(dev: &DeviceStore, rel: *mut KbRel) -> Vec<Triple> {
    let mut n = 0u64;
    unsafe { kb_rel_info(rel, &mut n, ptr::null_mut(), ptr::null_mut()) };
    let mut cols = [vec![0u32; n as usize], vec![0u32; n as usize], vec![0u32; n as usize]];
    for c in 0..3 { unsafe { kb_rel_download(dev.ctx, rel, c as u32, cols[c].as_mut_ptr()) }; }
    unsafe { kb_rel_free(dev.ctx, rel) };
    (0..n as usize).map(|i| Triple { subject: cols[0][i], predicate: cols[1][i], object: cols[2][i] }).collect()
}

impl GpuR2R {
    pub fn new(inner: SimpleR2R, device: i32) -> Result<Self, String> {
        let mut dev = DeviceStore::new(device)?;
        dev.segmented = true;
        Ok(Self { inner, dev, pending: Vec::new(), evicted: Vec::new(), firing: 1, tag_of: HashMap::new(), live: HashMap::new(),
                  closed: false, derived: HashSet::new(), stream: None })
    }
    /// Opt in to the device R2S operator: `execute_query` returns what `stream_operator` emits for the firing, not the whole result.
    pub fn with_stream_operator(mut self, stream_operator: StreamOperator) -> Self {
        let kind = match stream_operator { StreamOperator::RSTREAM => KB_RSTREAM, StreamOperator::ISTREAM => KB_ISTREAM, StreamOperator::DSTREAM => KB_DSTREAM };
        self.stream = Some(DeviceStream { kind, op: ptr::null_mut(), names: Vec::new() });
        self
    }
    /// `kb_r2s_eval` on a firing's result (`names[c]` = variable of column c), then the emitted rows decoded. None: the result has
    /// other variables than the operator's, or a device error (the operator's state is then unchanged).
    fn stream_eval(&mut self, rel: *const KbRel, names: &[String]) -> Option<Vec<Vec<(String, String)>>> {
        let ctx = self.dev.ctx;
        let st = self.stream.as_mut()?;
        if st.op.is_null() {
            let mut sorted = names.to_vec();
            sorted.sort();
            let slots: Vec<u32> = (0..sorted.len() as u32).collect();
            if unsafe { kb_r2s_create(ctx, st.kind, slots.as_ptr(), slots.len() as u32, &mut st.op) } != KB_OK { return None; }
            st.names = sorted;
        }
        // the same columns under the operator's slots (a view, no copy)
        let (mut n, mut sl, mut cols) = (0u64, Vec::new(), Vec::new());
        unsafe { kb_rel_info(rel, &mut n, ptr::null_mut(), ptr::null_mut()) };
        for (c, k) in names.iter().enumerate() {
            sl.push(st.names.iter().position(|x| x == k)? as u32);
            let mut p: *const u32 = ptr::null();
            unsafe { kb_rel_device_col(rel, c as u32, &mut p) };
            cols.push(p as *mut u32);
        }
        let mut view: *mut KbRel = ptr::null_mut();
        if unsafe { kb_rel_wrap_device(ctx, sl.as_ptr(), sl.len() as u32, cols.as_ptr(), n, &mut view) } != KB_OK { return None; }
        let mut emitted: *mut KbRel = ptr::null_mut();
        let rc = unsafe { kb_r2s_eval(ctx, st.op, view, &mut emitted) };
        unsafe { kb_rel_free(ctx, view) };
        if rc != KB_OK { return None; }
        let out_names = if st.kind == KB_RSTREAM { names.to_vec() } else { st.names.clone() };  // RSTREAM: the response's own columns
        let rows = crate::download_rows(&self.dev, emitted, &out_names);
        unsafe { kb_rel_free(ctx, emitted) };
        let dict = self.inner.item.dictionary.read().unwrap();
        Some(rows?.into_iter().map(|r| {
            let mut r: Vec<(String, String)> = r.into_iter().map(|(k, v)| (k, dict.decode(v).unwrap_or("unknown").to_string())).collect();
            r.sort();
            r
        }).collect())
    }
    /// a host fallback's rows, encoded back to ids and passed through the same device operator
    fn stream_eval_host(&mut self, rows: Vec<Vec<(String, String)>>) -> Option<Vec<Vec<(String, String)>>> {
        let names: Vec<String> = match (rows.first(), self.stream.as_ref()) {
            (_, Some(st)) if !st.names.is_empty() => st.names.clone(),
            (Some(r), _) => { let mut v: Vec<String> = r.iter().map(|(k, _)| k.clone()).collect(); v.sort(); v }
            (None, _) => return Some(Vec::new()),  // no firing yet told the variables, and nothing to emit
        };
        let cols: Vec<Vec<u32>> = {
            let dict = self.inner.item.dictionary.read().unwrap();
            names.iter().map(|k| rows.iter().map(|r| r.iter().find(|(x, _)| x == k)
                .and_then(|(_, v)| dict.string_to_id.get(v.as_str()).copied()).unwrap_or(KB_ID_NONE)).collect()).collect()
        };
        let slots: Vec<u32> = (0..names.len() as u32).collect();
        let ptrs: Vec<*const u32> = cols.iter().map(|c| c.as_ptr()).collect();
        let mut rel: *mut KbRel = ptr::null_mut();
        if unsafe { kb_rel_from_host(self.dev.ctx, slots.as_ptr(), slots.len() as u32, ptrs.as_ptr(), rows.len() as u64, &mut rel) } != KB_OK { return None; }
        let rel = crate::Rel(rel, self.dev.ctx);
        self.stream_eval(rel.0, &names)
    }
    /// the derived triples as the device now holds them, mirrored into the host database (a derived triple that is also a live streamed
    /// triple stays there when it stops being derived: Q11)
    fn set_derived(&mut self, gone: Vec<Triple>, new: Vec<Triple>) {
        let pending: HashSet<&Triple> = self.pending.iter().collect();
        for t in gone {
            self.derived.remove(&t);
            if !self.tag_of.contains_key(&t) && !pending.contains(&t) { self.inner.item.delete_triple(&t); }
        }
        for t in new { self.inner.item.add_triple(t.clone()); self.derived.insert(t); }
    }
    fn columns(&self) -> (Vec<u32>, Vec<u32>, Vec<u32>) {
        (self.pending.iter().map(|t| t.subject).collect(), self.pending.iter().map(|t| t.predicate).collect(), self.pending.iter().map(|t| t.object).collect())
    }
    fn commit_pending(&mut self) {
        self.live.insert(self.firing, self.pending.len());
        for t in self.pending.drain(..) { self.tag_of.insert(t, self.firing); }
        self.firing += 1;
    }
    /// the window's changes go to the store as plain segment operations (no rules involved): the store is no longer closed
    fn flush(&mut self) {
        for tag in self.evicted.drain(..) { unsafe { kb_store_evict(self.dev.ctx, tag) }; self.closed = false; }
        if self.pending.is_empty() { return; }
        let (s, p, o) = self.columns();
        unsafe { kb_store_append(self.dev.ctx, s.as_ptr(), p.as_ptr(), o.as_ptr(), s.len() as u64, self.firing) };
        self.commit_pending();
        self.closed = false;
    }
    /// one firing's maintenance: Some(()) when the device did it, None when the rules need the host (quoted-triple terms, unsupported shapes)
    fn maintain(&mut self, kr: &[KbRule]) -> Option<()> {
        let ctx = self.dev.ctx;
        let (s, p, o) = self.columns();
        let mut add: *mut KbRel = ptr::null_mut();
        let slots = [0u32, 1, 2];
        let cols = [s.as_ptr(), p.as_ptr(), o.as_ptr()];
        if !self.pending.is_empty() && unsafe { kb_rel_from_host(ctx, slots.as_ptr(), 3, cols.as_ptr(), s.len() as u64, &mut add) } != KB_OK { return None; }
        let (mut gone, mut new): (*mut KbRel, *mut KbRel) = (ptr::null_mut(), ptr::null_mut());
        let mut st = KbMaintainStats::default();
        let rc = unsafe { kb_datalog_maintain(ctx, kr.as_ptr(), kr.len() as u32, KB_SEMI_NAIVE, self.evicted.as_ptr(), self.evicted.len() as u32, add, self.firing,
                                              &mut gone, &mut new, &mut st) };
        if !add.is_null() { unsafe { kb_rel_free(ctx, add) }; }
        if rc != KB_OK {
            // a failure while the store was being rewritten may have stored `add` under this firing's tag already: the fallback's
            // flush appends the pending triples again, so that segment goes first (KB_E_NOT_FOUND when it was not stored)
            unsafe { kb_store_evict(ctx, self.firing) };
            return None;
        }
        self.evicted.clear();
        let (gone, new) = (triples_of(&self.dev, gone), triples_of(&self.dev, new));
        self.set_derived(gone, new);
        if !self.pending.is_empty() { self.commit_pending(); }
        Some(())
    }
    fn fixpoint(&mut self, kr: &[KbRule]) -> Option<()> {
        self.flush();
        unsafe { kb_store_evict(self.dev.ctx, KB_TAG_INFERRED) };
        let mut rel: *mut KbRel = ptr::null_mut();
        let mut st = std::mem::MaybeUninit::<KbFixpointStats>::zeroed();
        if unsafe { kb_datalog_fixpoint(self.dev.ctx, kr.as_ptr(), kr.len() as u32, KB_SEMI_NAIVE, &mut rel, st.as_mut_ptr()) } != KB_OK { return None; }
        let gone: Vec<Triple> = self.derived.iter().cloned().collect();
        let new = triples_of(&self.dev, rel);
        self.set_derived(gone, new);
        Some(())
    }
}

impl Drop for GpuR2R {
    // the operator's state lives in the context's memory: it goes before `dev` destroys the context
    fn drop(&mut self) {
        if let Some(st) = self.stream.take() { unsafe { kb_r2s_free(self.dev.ctx, st.op) }; }
    }
}

impl AsAnyMut for GpuR2R { fn as_any_mut(&mut self) -> &mut dyn Any { self } }

impl R2ROperator<Triple, Vec<(String, String)>, Vec<(String, String)>> for GpuR2R {
    fn load_triples(&mut self, data: &str, syntax: String) -> Result<(), String> { self.inner.load_triples(data, syntax) }
    fn load_rules(&mut self, data: &str) -> Result<(), &'static str> { self.closed = false; self.inner.load_rules(data) }
    fn add(&mut self, data: Triple) { self.inner.add(data.clone()); self.pending.push(data); }
    fn remove(&mut self, data: &Triple) {
        self.inner.remove(data);
        if let Some(tag) = self.tag_of.remove(data) {
            let left = self.live.get_mut(&tag).map(|n| { *n -= 1; *n }).unwrap_or(0);
            if left == 0 { self.live.remove(&tag); self.evicted.push(tag); }  // the whole slide left the window
        }
    }
    fn materialize(&mut self) -> Vec<Triple> {
        if self.inner.rules.is_empty() { self.flush(); return Vec::new(); }
        if self.dev.sync(&self.inner.item).is_err() { self.closed = false; }  // the dictionary's tables (the store itself is ours)
        let compiled: Option<Vec<_>> = self.inner.rules.iter().map(compile_rule).collect();
        let done = compiled.as_ref().and_then(|compiled| {
            let kr: Vec<KbRule> = compiled.iter().map(|(pr, fl, co)| KbRule { premise: pr.as_ptr(), n_premise: pr.len() as u32, filters: fl.as_ptr(),
                n_filters: fl.len() as u32, conclusion: co.as_ptr(), n_conclusion: co.len() as u32 }).collect();
            // the first firing (or the first after a plain store change): evict the inferred segment, closure from scratch; then DRed
            let r = if self.closed { self.maintain(&kr).or_else(|| self.fixpoint(&kr)) } else { self.fixpoint(&kr) };
            self.closed = r.is_some();
            r
        });
        if done.is_none() {  // rules the device does not take: the host's SimpleR2R materialises (simple_r2r.rs:103-128)
            self.flush();
            unsafe { kb_store_evict(self.dev.ctx, KB_TAG_INFERRED) };
            let old: Vec<Triple> = self.derived.drain().collect();
            for t in old { if !self.tag_of.contains_key(&t) { self.inner.item.delete_triple(&t); } }
            let derived = self.inner.materialize();
            // the device store holds what the host derived, as its inferred segment, for the device query path
            let (s, p, o): (Vec<u32>, Vec<u32>, Vec<u32>) = (derived.iter().map(|t| t.subject).collect(), derived.iter().map(|t| t.predicate).collect(),
                                                             derived.iter().map(|t| t.object).collect());
            if !derived.is_empty() { unsafe { kb_store_append(self.dev.ctx, s.as_ptr(), p.as_ptr(), o.as_ptr(), s.len() as u64, KB_TAG_INFERRED) }; }
            self.closed = false;
            return derived;
        }
        self.derived.iter().cloned().collect()
    }
    fn execute_query(&mut self, op: &PhysicalOperator) -> Vec<Vec<(String, String)>> {
        self.flush();
        if self.stream.is_some() {
            let emitted = match try_execute_rel(op, &self.inner.item, &mut self.dev) {
                Some(res) => self.stream_eval(res.rel.0, &res.names),
                None => { let rows = self.inner.execute_query(op); self.stream_eval_host(rows) }
            };
            return emitted.unwrap_or_else(|| {
                eprintln!("kb_r2s_eval failed: {}", self.dev.last_error());
                Vec::new()
            });
        }
        match try_execute(op, &self.inner.item, &mut self.dev) {
            Some(rows) => {
                let dict = self.inner.item.dictionary.read().unwrap();
                rows.into_iter().map(|r| r.into_iter().map(|(k, v)| (k, dict.decode(v).unwrap_or("unknown").to_string())).collect()).collect()
            }
            None => self.inner.execute_query(op),
        }
    }
    fn parse_data(&mut self, data: &str) -> Vec<Triple> { self.inner.parse_data(data) }
}
