//! kolibrie-gpu-b200 — the three seams through which Kolibrie hands its hot path to libkolibrie_b200.so:
//!
//! * [`try_execute`]            for `ExecutionEngine::execute_with_ids` (kolibrie/src/streamertail_optimizer/execution/engine.rs:54);
//!                              [`try_execute_mut`] also runs `Bind` (engine.rs:144-277) and `Values` (engine.rs:279-308) and
//!                              grows the database's dictionary and quoted-triple store as the reference does
//! * [`GpuSemiNaiveStrategy`]   for `Reasoner::infer_with_strategy`    (datalog/src/reasoning/materialisation/infer_generic.rs:27-53)
//! * [`GpuR2R`]                 for the RSP engine's `R2ROperator`      (kolibrie/src/rsp/r2r.rs:17-30), optionally with the
//!                              Relation-to-Stream operator on the device (`GpuR2R::with_stream_operator`, kolibrie/src/rsp/r2s.rs:37-58)
//!
//! plus [`planner`]: the device operators' cost constants for Streamertail's estimator (cost/estimator.rs:17-29).
//!
//! STATUS: written against the reference's types (commit 1d7c306c) and the C header of this repository; NOT compiled or tested in the
//! repository's build image, which has no Rust toolchain. The Python (`kolibrie_b200/engine.py`, `planner.py`) and C++
//! (`kolibrie_b200/host/kolibrie_host.hpp`) mirrors implement the same logic and ARE tested against the same C ABI.
pub mod ffi;
pub mod planner;
pub mod r2r;
pub mod reasoner;

use ffi::*;
use kolibrie::sparql_database::SparqlDatabase;
use kolibrie::streamertail_optimizer::{Condition, PhysicalOperator};
use shared::query::{ArithmeticExpression, FilterExpression};
use shared::terms::{Term, TriplePattern};
use shared::triple::Triple;
use std::collections::HashMap;
use std::ffi::CStr;
use std::ptr;

/// One device context + the store version it mirrors. Kolibrie holds `&mut SparqlDatabase` around every call, so no locking here.
pub struct DeviceStore {
    pub ctx: *mut KbCtx,
    synced_triples: usize,
    synced_dict: usize,
    synced_quoted: usize,
    indexed: bool,
    /// the store is maintained segment by segment by its owner (GpuR2R: one segment per firing, the inferred segment): `sync` then
    /// mirrors the dictionary only and never replaces the store with `database.triples`
    pub segmented: bool,
}
unsafe impl Send for DeviceStore {}

impl DeviceStore {
    pub fn new(device: i32) -> Result<Self, String> {
        let mut ctx: *mut KbCtx = ptr::null_mut();
        let rc = unsafe { kb_ctx_create(device, &mut ctx) };
        if rc != KB_OK {
            return Err(unsafe { CStr::from_ptr(kb_last_error(ptr::null())) }.to_string_lossy().into_owned());
        }
        Ok(Self { ctx, synced_triples: usize::MAX, synced_dict: usize::MAX, synced_quoted: usize::MAX, indexed: false, segmented: false })
    }

    pub fn last_error(&self) -> String {
        unsafe { CStr::from_ptr(kb_last_error(self.ctx)) }.to_string_lossy().into_owned()
    }

    /// Mirror `database.triples` (BTreeSet iteration = (s,p,o) order) and the numeric side table on the device when they changed.
    /// The reference has no store version counter; `len()` of the set and of the dictionary is the cheap change signal used here —
    /// a caller that mutates without changing the sizes must call `invalidate()`.
    pub fn sync(&mut self, database: &SparqlDatabase) -> Result<(), String> {
        let dict = database.dictionary.read().unwrap();
        if dict.id_to_string.len() != self.synced_dict {
            let n = dict.id_to_string.len();
            let mut offs = Vec::with_capacity(n + 1);
            let mut bytes = Vec::new();
            offs.push(0u64);
            for s in dict.id_to_string.iter() { bytes.extend_from_slice(s.as_bytes()); offs.push(bytes.len() as u64); }
            if unsafe { kb_dict_strings_load(self.ctx, offs.as_ptr(), bytes.as_ptr(), n as u32) } != KB_OK { return Err(self.last_error()); }
            // the numeric side table (`s.parse::<f64>()`, types.rs:133-148 / 163-167) parsed on the device from those strings
            if unsafe { kb_dict_numeric_derive(self.ctx, KB_NUMERIC_F64, 0, ptr::null_mut()) } != KB_OK { return Err(self.last_error()); }
            self.synced_dict = n;
        }
        // the quoted-triple table (kb_quoted_load) when the store's size changed; an empty store clears it (n = 0), so that a table
        // never outlives the database it came from
        let qt = database.quoted_triple_store.read().unwrap();
        if qt.id_to_components.len() != self.synced_quoted {
            let n = qt.id_to_components.len();
            let (mut ids, mut s, mut p, mut o) = (Vec::with_capacity(n), Vec::with_capacity(n), Vec::with_capacity(n), Vec::with_capacity(n));
            for (&id, &(a, b, c)) in qt.id_to_components.iter() { ids.push(id); s.push(a); p.push(b); o.push(c); }
            if unsafe { kb_quoted_load(self.ctx, ids.as_ptr(), s.as_ptr(), p.as_ptr(), o.as_ptr(), n as u64) } != KB_OK { return Err(self.last_error()); }
            self.synced_quoted = n;
        }
        if !self.segmented && database.triples.len() != self.synced_triples {
            let n = database.triples.len();
            let (mut s, mut p, mut o) = (Vec::with_capacity(n), Vec::with_capacity(n), Vec::with_capacity(n));
            for t in database.triples.iter() { s.push(t.subject); p.push(t.predicate); o.push(t.object); }
            if unsafe { kb_store_load(self.ctx, s.as_ptr(), p.as_ptr(), o.as_ptr(), n as u64) } != KB_OK { return Err(self.last_error()); }
            self.synced_triples = n;
            self.indexed = false;
        }
        Ok(())
    }

    /// `SparqlDatabase::build_all_indexes` (sparql_database.rs:3364-3394) on the device; appends / evictions maintain it afterwards.
    pub fn build_all_indexes(&mut self) -> Result<(), String> {
        if unsafe { kb_store_build_index(self.ctx, ptr::null_mut(), ptr::null_mut()) } != KB_OK { return Err(self.last_error()); }
        self.indexed = true;
        Ok(())
    }

    pub fn invalidate(&mut self) { self.synced_triples = usize::MAX; self.synced_dict = usize::MAX; self.synced_quoted = usize::MAX; }

    /// The per-term `Dictionary::encode` loop of a bulk load (sparql_database.rs:1000-1013) as one device call. Returns the ids of
    /// `terms` (those the sequential loop would hand out, dictionary.rs:32-48) and, for every NEW string in id order, the index of the
    /// term that introduced it: the caller replays `dict.encode(terms[p])` for those positions only. The device dictionary must hold
    /// the host dictionary's strings (`sync` uploads them; afterwards the two grow in lock step through this call).
    pub fn encode_bulk(&mut self, terms: &[&str]) -> Result<(Vec<u32>, Vec<u64>), String> {
        let n = terms.len();
        let mut offs = Vec::with_capacity(n + 1);
        let mut bytes = Vec::new();
        offs.push(0u64);
        for t in terms { bytes.extend_from_slice(t.as_bytes()); offs.push(bytes.len() as u64); }
        let mut ids = vec![0u32; n];
        let mut first = vec![0u64; n];
        let mut n_new = 0u32;
        let rc = unsafe { kb_dict_encode(self.ctx, offs.as_ptr(), bytes.as_ptr(), n as u64, ids.as_mut_ptr(), &mut n_new, first.as_mut_ptr()) };
        if rc != KB_OK { return Err(self.last_error()); }
        first.truncate(n_new as usize);
        if self.synced_dict != usize::MAX { self.synced_dict += n_new as usize; }
        Ok((ids, first))
    }

    /// `add_triple` of each triple in order (sparql_database.rs:215-218) on `database` and on the device store together
    /// (kb_store_insert, into a segment tagged `tag`): returns whether each triple was new. `sync` first, so that the device holds the
    /// set the batch applies to; the sync counter then moves with the set, so the next `sync` uploads no triples.
    pub fn insert(&mut self, database: &mut SparqlDatabase, triples: &[Triple], tag: u64) -> Result<Vec<bool>, String> {
        self.write(database, triples, Some(tag))
    }

    /// `delete_triple` of each triple in order (sparql_database.rs:220-226) on `database` and on the device store together
    /// (kb_store_remove): returns what each `delete_triple` returns
    pub fn remove(&mut self, database: &mut SparqlDatabase, triples: &[Triple]) -> Result<Vec<bool>, String> {
        self.write(database, triples, None)
    }

    fn write(&mut self, database: &mut SparqlDatabase, triples: &[Triple], insert_tag: Option<u64>) -> Result<Vec<bool>, String> {
        if triples.is_empty() { return Ok(Vec::new()); }
        if self.segmented { return Err("the store is maintained segment by segment by its owner".into()); }
        self.sync(database)?;
        let s: Vec<u32> = triples.iter().map(|t| t.subject).collect();
        let p: Vec<u32> = triples.iter().map(|t| t.predicate).collect();
        let o: Vec<u32> = triples.iter().map(|t| t.object).collect();
        let mut flags = vec![0u8; triples.len()];
        let mut n = 0u64;
        let rc = unsafe {
            match insert_tag {
                Some(tag) => kb_store_insert(self.ctx, s.as_ptr(), p.as_ptr(), o.as_ptr(), s.len() as u64, tag, flags.as_mut_ptr(), &mut n),
                None => kb_store_remove(self.ctx, s.as_ptr(), p.as_ptr(), o.as_ptr(), s.len() as u64, flags.as_mut_ptr(), &mut n),
            }
        };
        if rc != KB_OK { return Err(self.last_error()); }
        let mut host = Vec::with_capacity(triples.len());
        for t in triples {
            host.push(match insert_tag {
                Some(_) => { let new = !database.triples.contains(t); database.add_triple(t.clone()); new }
                None => database.delete_triple(t),
            });
        }
        if host.iter().zip(flags.iter()).any(|(h, &d)| *h != (d != 0)) {
            self.invalidate();  // the next sync uploads the host set again
            return Err("the device store and the host set disagree on a batch write".into());
        }
        self.synced_triples = database.triples.len();
        Ok(host)
    }

    /// DELETE { template } WHERE { ... } (execute_query.rs:354-413) once the WHERE's rows are `rel` on the device (`try_execute_rel`):
    /// kb_store_remove_template fills `template` from every row and removes the triples from the device store, and `database` loses
    /// the same triples. Returns the triples removed, or None where the device refuses a binding (KB_E_UNSUPPORTED: one that
    /// `encode_term_star` would not map back to its own id, or a template variable the WHERE leaves unbound): the caller then runs the
    /// reference's loop, and both stores are as they were.
    pub fn remove_template(&mut self, database: &mut SparqlDatabase, rel: &Rel, names: &[String], template: &[KbPattern]) -> Result<Option<u64>, String> {
        let mut n = 0u64;
        let rc = unsafe { kb_store_remove_template(self.ctx, rel.0, template.as_ptr(), template.len() as u32, &mut n) };
        if rc == KB_E_UNSUPPORTED { return Ok(None); }
        if rc != KB_OK { return Err(self.last_error()); }
        let rows = download_rows(self, rel.0, names).ok_or_else(|| self.last_error())?;
        let (_, slots) = rel_slots(rel).ok_or_else(|| self.last_error())?;  // names[c] is the variable of column c, slots[c] its slot
        let value = |t: &KbTerm, row: &HashMap<String, u32>| if t.is_var == 1 {
            slots.iter().position(|&s| s == t.value).and_then(|c| names.get(c)).and_then(|k| row.get(k)).copied()
        } else { Some(t.value) };
        let mut gone = 0u64;
        for row in &rows {
            for pt in template {
                if let (Some(s), Some(p), Some(o)) = (value(&pt.s, row), value(&pt.p, row), value(&pt.o, row)) {
                    if database.delete_triple(&Triple { subject: s, predicate: p, object: o }) { gone += 1; }
                }
            }
        }
        if gone != n {
            self.invalidate();
            return Err("the device store and the host set disagree on a DELETE WHERE".into());
        }
        self.synced_triples = database.triples.len();
        Ok(Some(n))
    }

    /// `SparqlDatabase::handle_update` (sparql_database.rs:3091-3117) with the store written as one batch: the reference's loop
    /// encodes every term with `encode_term_star` in its order, then the triples are inserted or removed on `database` and on the
    /// device together. Returns the reference's strings.
    pub fn handle_update(&mut self, database: &mut SparqlDatabase, update: &str) -> Result<String, String> {
        use kolibrie::parser::{parse_delete, parse_insert};
        let trimmed = update.trim();
        let (insert, terms) = if trimmed.starts_with("INSERT") {
            match parse_insert(trimmed) { Ok((_, c)) => (true, c.triples), Err(_) => return Ok("Update Failed".into()) }
        } else if trimmed.starts_with("DELETE") {
            match parse_delete(trimmed) { Ok((_, c)) => (false, c.triples), Err(_) => return Ok("Update Failed".into()) }
        } else {
            return Ok("Update Failed".into());
        };
        let triples: Vec<Triple> = terms.iter().map(|(s, p, o)| Triple {
            subject: database.encode_term_star(s), predicate: database.encode_term_star(p), object: database.encode_term_star(o),
        }).collect();
        if insert { self.insert(database, &triples, 0)?; } else { self.remove(database, &triples)?; }
        Ok("Update Successful".into())
    }

    /// `SparqlDatabase::generate_ntriples` (`turtle` false) or `generate_turtle` (sparql_database.rs:301-382) of the device store
    /// (`sync` first), written on the device: `sink` receives the text in pieces of whole lines / triples, each at most `capacity`
    /// bytes (at least the largest unit, `kb_serialize_info.max_unit_bytes`). `prefixes` are the Turtle header's (name, uri) pairs
    /// in the order given.
    pub fn serialize(&mut self, turtle: bool, prefixes: &[(&str, &str)], capacity: usize, mut sink: impl FnMut(&[u8])) -> Result<kb_serialize_info, String> {
        let mut offs = vec![0u64];
        let mut bytes = Vec::new();
        for (name, uri) in prefixes {
            for x in [name, uri] { bytes.extend_from_slice(x.as_bytes()); offs.push(bytes.len() as u64); }
        }
        let mut ser: *mut kb_serializer = ptr::null_mut();
        let mut info = KbSerializeInfo::default();
        let fmt = if turtle { KB_SER_TURTLE } else { KB_SER_NTRIPLES };
        if unsafe { kb_serialize_begin(self.ctx, fmt, offs.as_ptr(), bytes.as_ptr(), prefixes.len() as u32, &mut ser, &mut info) } != KB_OK {
            return Err(self.last_error());
        }
        let mut buf = vec![0u8; capacity.min(info.total_bytes as usize).max(1)];
        let result = loop {
            let mut got = 0u64;
            if unsafe { kb_serialize_next(self.ctx, ser, buf.as_mut_ptr(), buf.len() as u64, &mut got) } != KB_OK { break Err(self.last_error()); }
            if got == 0 { break Ok(info); }
            sink(&buf[..got as usize]);
        };
        unsafe { kb_serialize_free(ser) };
        result
    }

    /// `DatabaseStats::gather_stats_fast` (database_stats.rs:43-105) of the device store (`sync` first): `max_sample` 100 000 is the
    /// reference's sampling, 0 counts every triple. The maps carry the sampling step already; INTEGRATION.md shows how they fill the
    /// reference's `DatabaseStats` for `Streamertail::with_cached_stats`.
    pub fn gather_stats(&mut self, max_sample: u64) -> Result<StoreStats, String> {
        let mut st: *mut kb_db_stats = ptr::null_mut();
        let mut info = KbDbStatsInfo::default();
        if unsafe { kb_store_gather_stats(self.ctx, max_sample, &mut st, &mut info) } != KB_OK { return Err(self.last_error()); }
        let mut maps: [HashMap<u32, u64>; 3] = Default::default();
        for (pos, map) in maps.iter_mut().enumerate() {
            let (mut ids, mut counts, mut n): (*const u32, *const u64, u64) = (ptr::null(), ptr::null(), 0);
            if unsafe { kb_db_stats_counts(st, pos as u32, &mut ids, &mut counts, &mut n) } != KB_OK {
                unsafe { kb_db_stats_free(st) };
                return Err("kb_db_stats_counts refused a position".into());
            }
            if n > 0 {
                let (ids, counts) = unsafe { (std::slice::from_raw_parts(ids, n as usize), std::slice::from_raw_parts(counts, n as usize)) };
                map.extend(ids.iter().copied().zip(counts.iter().copied()));
            }
        }
        unsafe { kb_db_stats_free(st) };
        let [subject, predicate, object] = maps;
        Ok(StoreStats { info, subject, predicate, object })
    }
}

/// One position filter of a device QueryBuilder query (`TripleFilter` without `Custom`): `Exact` takes the id the caller's dictionary
/// gives the string (`KB_ID_NONE` when it lacks it), the others the pattern's text.
pub enum QbFilter<'a> { Exact(u32), Contains(&'a str), StartsWith(&'a str), EndsWith(&'a str) }

/// A device QueryBuilder result: the rows in `BTreeSet<Triple>` order (`kb_qb_triples`), owned until dropped.
pub struct QbRows { ctx: *mut KbCtx, rel: *mut KbRel, pub info: KbQbInfo }
impl Drop for QbRows {
    fn drop(&mut self) { unsafe { kb_rel_free(self.ctx, self.rel) } }
}

impl DeviceStore {
    /// `QueryBuilder::apply_filters` (query_builder.rs:486-568) on the device store (`sync` first), for a query without closures:
    /// `filters` per position, `join` the `KB_QB_ON_*` bits against `right`'s store (a context on the same device, `self` for a
    /// self-join; `None`: no join), rows [offset, offset + limit) of the set order. `count_only` gives no rows, only `info.n_rows`
    /// (`count()`). `get_triples` reads the rows with `QbRows::triples`; `get_decoded_triples` / `get_subjects` & co. with `query_terms`.
    /// Err(KB_E_UNSUPPORTED's message) means: run the reference's loop.
    pub fn query_triples(&mut self, filters: [Option<QbFilter>; 3], join: u32, right: Option<&DeviceStore>, offset: u64, limit: Option<u64>,
                         count_only: bool) -> Result<Option<QbRows>, String> {
        let mut spec = KbQbSpec { join, offset, limit: limit.unwrap_or(KB_QB_NO_LIMIT), ..Default::default() };
        for (k, f) in filters.iter().enumerate() {
            spec.pos[k] = match f {
                None => KbQbFilter::default(),
                Some(QbFilter::Exact(id)) => KbQbFilter { mode: KB_QB_EXACT, id: *id, ..Default::default() },
                Some(QbFilter::Contains(t)) => KbQbFilter { mode: KB_QB_CONTAINS, pattern: t.as_ptr(), len: t.len() as u64, id: 0 },
                Some(QbFilter::StartsWith(t)) => KbQbFilter { mode: KB_QB_STARTS, pattern: t.as_ptr(), len: t.len() as u64, id: 0 },
                Some(QbFilter::EndsWith(t)) => KbQbFilter { mode: KB_QB_ENDS, pattern: t.as_ptr(), len: t.len() as u64, id: 0 },
            };
        }
        let slots = [0u32, 1, 2];
        let mut rel: *mut KbRel = ptr::null_mut();
        let mut info = KbQbInfo::default();
        let r = right.map_or(ptr::null(), |d| d.ctx as *const KbCtx);
        let out = if count_only { ptr::null_mut() } else { &mut rel as *mut *mut KbRel };
        if unsafe { kb_qb_triples(self.ctx, &spec, r, slots.as_ptr(), out, &mut info) } != KB_OK { return Err(self.last_error()); }
        Ok(if count_only { None } else { Some(QbRows { ctx: self.ctx, rel, info }) })
    }

    /// column `col` (0 subject, 1 predicate, 2 object) of a `query_triples` result as `Dictionary::decode(id).unwrap_or("")` renders it:
    /// `KB_QB_TERMS_EMPTY` every row (`get_decoded_triples`), `KB_QB_TERMS_DROP` the rows that decode (`get_subjects` & co.),
    /// `KB_QB_TERMS_DISTINCT` their distinct strings in byte order (the same with `distinct()`)
    pub fn query_terms(&mut self, rows: &QbRows, col: u32, mode: u32) -> Result<Vec<String>, String> {
        let mut s: *mut KbStrings = ptr::null_mut();
        if unsafe { kb_qb_terms(self.ctx, rows.rel, col, mode, &mut s) } != KB_OK { return Err(self.last_error()); }
        let (mut n, mut total) = (0u64, 0u64);
        unsafe { kb_strings_info(s, &mut n, &mut total) };
        let mut offs = vec![0u64; n as usize + 1];
        let mut bytes = vec![0u8; total as usize + 1];
        let rc = unsafe { kb_strings_download(self.ctx, s, offs.as_mut_ptr(), bytes.as_mut_ptr()) };
        unsafe { kb_strings_free(self.ctx, s) };
        if rc != KB_OK { return Err(self.last_error()); }
        Ok((0..n as usize).map(|i| String::from_utf8_lossy(&bytes[offs[i] as usize..offs[i + 1] as usize]).into_owned()).collect())
    }
}

impl DeviceStore {
    /// `SparqlDatabase::union(self, other)` (sparql_database.rs:1874-1933) on the device: both stores `sync`ed first, the result in a new
    /// context on `device` (the same as both). Its store, device dictionary and quoted-triple table are the union's: the new database's
    /// dictionary is a clone of `database`'s extended with the `info.dict_new` strings from id `info.dict_first` on
    /// (`kb_dict_strings_download`), its triples the set `kb_store_download` reads. An id of `other`'s triples that its dictionary does
    /// not map (the reference panics) is an Err.
    pub fn union(&mut self, database: &SparqlDatabase, other: &mut DeviceStore, other_db: &SparqlDatabase, device: i32)
                 -> Result<(DeviceStore, KbUnionInfo), String> {
        self.sync(database)?;
        other.sync(other_db)?;
        let mut out = DeviceStore::new(device)?;
        let mut info = KbUnionInfo::default();
        if unsafe { kb_store_union(out.ctx, self.ctx, other.ctx, &mut info) } != KB_OK { return Err(out.last_error()); }
        Ok((out, info))
    }

    /// `SparqlDatabase::par_join(self, other, predicate)` (sparql_database.rs:1935-2005) for `predicate_id`, the predicate as `database`'s
    /// dictionary encodes it (the caller encodes it first, as the reference does): the result in a new context on `device`, whose
    /// dictionary and quoted-triple table are copies of this one's, as the result shares `database`'s.
    pub fn par_join(&mut self, database: &SparqlDatabase, other: &mut DeviceStore, other_db: &SparqlDatabase, predicate_id: u32, device: i32)
                    -> Result<(DeviceStore, KbParJoinInfo), String> {
        self.sync(database)?;
        other.sync(other_db)?;
        let mut out = DeviceStore::new(device)?;
        let mut info = KbParJoinInfo::default();
        if unsafe { kb_store_par_join(out.ctx, self.ctx, other.ctx, predicate_id, &mut info) } != KB_OK { return Err(out.last_error()); }
        Ok((out, info))
    }
}

impl QbRows {
    /// the rows as `Triple`s, in set order (collect them into the `BTreeSet` `get_triples` returns)
    pub fn triples(&self) -> Result<Vec<Triple>, String> {
        let n = self.info.n_rows as usize;
        let mut cols = [vec![0u32; n], vec![0u32; n], vec![0u32; n]];
        for (c, v) in cols.iter_mut().enumerate() {
            if n > 0 && unsafe { kb_rel_download(self.ctx, self.rel, c as u32, v.as_mut_ptr()) } != KB_OK {
                return Err("kb_rel_download refused the result".into());
            }
        }
        Ok((0..n).map(|i| Triple { subject: cols[0][i], predicate: cols[1][i], object: cols[2][i] }).collect())
    }
}

/// What `DeviceStore::gather_stats` returns: the totals (`info.total_triples`, `info.quoted_triple_count`) and the three cardinality maps
/// of `DatabaseStats` (database_stats.rs:17-26), counts already scaled by the sampling step.
pub struct StoreStats {
    pub info: KbDbStatsInfo,
    pub subject: HashMap<u32, u64>,
    pub predicate: HashMap<u32, u64>,
    pub object: HashMap<u32, u64>,
}

impl Drop for DeviceStore {
    fn drop(&mut self) { unsafe { kb_ctx_destroy(self.ctx) } }
}

/// variable name (without '?', as engine.rs strips it everywhere) <-> slot
#[derive(Default)]
pub struct SlotMap { pub slot: HashMap<String, u32>, pub names: Vec<String> }
impl SlotMap {
    pub fn of(&mut self, name: &str) -> u32 {
        let name = name.strip_prefix('?').unwrap_or(name);
        if let Some(&s) = self.slot.get(name) { return s; }
        let s = self.names.len() as u32;
        self.slot.insert(name.to_string(), s);
        self.names.push(name.to_string());
        s
    }
    pub fn term(&mut self, t: &Term) -> Option<KbTerm> {
        match t {
            Term::Variable(v) => Some(KbTerm { is_var: 1, value: self.of(v) }),
            Term::Constant(c) => Some(KbTerm { is_var: 0, value: *c }),
            Term::QuotedTriple(_) => None,  // only a TableScan / IndexScan takes `<< s p o >>` terms: see quoted_pattern
        }
    }
    pub fn pattern(&mut self, p: &TriplePattern) -> Option<KbPattern> {
        Some(KbPattern { s: self.term(&p.0)?, p: self.term(&p.1)?, o: self.term(&p.2)? })
    }
    /// kb_quoted_pattern of a scan with a quoted subject and/or object (kb_scan_quoted); inside a quoted term, a nested one is
    /// KB_TERM_QUOTED: "any quoted-triple id", as match_term checks it (engine.rs:1100-1105). None for a quoted predicate.
    pub fn quoted_pattern(&mut self, p: &TriplePattern) -> Option<KbQuotedPattern> {
        const ANY: KbTerm = KbTerm { is_var: KB_TERM_QUOTED, value: 0 };
        fn inner(m: &mut SlotMap, t: &Term) -> Option<KbTerm> { if t.is_quoted_triple() { Some(ANY) } else { m.term(t) } }
        fn position(m: &mut SlotMap, t: &Term) -> Option<(KbTerm, KbPattern)> {
            match t {
                Term::QuotedTriple(q) => {
                    let (s, p, o) = &**q;
                    Some((ANY, KbPattern { s: inner(m, s)?, p: inner(m, p)?, o: inner(m, o)? }))
                }
                _ => Some((m.term(t)?, KbPattern::default())),
            }
        }
        if p.1.is_quoted_triple() { return None; }
        let (s, inner_s) = position(self, &p.0)?;
        let pt = self.term(&p.1)?;
        let (o, inner_o) = position(self, &p.2)?;
        Some(KbQuotedPattern { outer: KbPattern { s, p: pt, o }, inner_s, inner_o })
    }
}

/// `Condition` -> postfix filter program with the semantics of `evaluate_with_ids` (types.rs:110-186). None: a construct the device
/// does not evaluate (the caller falls back to the CPU operator).
pub fn compile_condition(cond: &Condition, slots: &mut SlotMap, database: &SparqlDatabase) -> Option<Vec<KbFilterOp>> {
    fn op(op: u32, slot: u32, cmp: u32, id: u32, value: f64) -> KbFilterOp { KbFilterOp { op, slot, cmp, id, value } }
    fn arith(e: &ArithmeticExpression, slots: &mut SlotMap, out: &mut Vec<KbFilterOp>) -> Option<()> {
        match e {
            ArithmeticExpression::Operand(s) => {
                if s.starts_with('?') { out.push(op(KB_F_PUSH_VAR, slots.of(s), 0, 0, 0.0)); }
                else { out.push(op(KB_F_PUSH_CONST, 0, 0, 0, s.parse::<f64>().ok()?)); }
            }
            ArithmeticExpression::Add(l, r) => { arith(l, slots, out)?; arith(r, slots, out)?; out.push(op(KB_F_ADD, 0, 0, 0, 0.0)); }
            ArithmeticExpression::Subtract(l, r) => { arith(l, slots, out)?; arith(r, slots, out)?; out.push(op(KB_F_SUB, 0, 0, 0, 0.0)); }
            ArithmeticExpression::Multiply(l, r) => { arith(l, slots, out)?; arith(r, slots, out)?; out.push(op(KB_F_MUL, 0, 0, 0, 0.0)); }
            ArithmeticExpression::Divide(l, r) => { arith(l, slots, out)?; arith(r, slots, out)?; out.push(op(KB_F_DIV, 0, 0, 0, 0.0)); }
        }
        Some(())
    }
    fn rec(e: &FilterExpression, slots: &mut SlotMap, db: &SparqlDatabase, out: &mut Vec<KbFilterOp>) -> Option<()> {
        match e {
            FilterExpression::Comparison(var, o, value) => {
                let slot = slots.of(var);
                match *o {
                    "=" | "!=" => {
                        // decoded == literal  <=>  id == lookup(literal); a literal the dictionary does not hold equals nothing
                        let id = db.dictionary.read().unwrap().string_to_id.get(*value).copied().unwrap_or(KB_ID_NONE);
                        out.push(op(if *o == "=" { KB_F_EQ_ID } else { KB_F_NE_ID }, slot, 0, id, 0.0));
                    }
                    ">" | ">=" | "<" | "<=" => {
                        let cmp = match *o { ">" => KB_CMP_GT, ">=" => KB_CMP_GE, "<" => KB_CMP_LT, _ => KB_CMP_LE };
                        out.push(op(KB_F_CMP_NUM, slot, cmp, 0, value.parse::<f64>().unwrap_or(0.0)));
                    }
                    _ => return None,
                }
            }
            FilterExpression::And(l, r) => { rec(l, slots, db, out)?; rec(r, slots, db, out)?; out.push(op(KB_F_AND, 0, 0, 0, 0.0)); }
            FilterExpression::Or(l, r) => { rec(l, slots, db, out)?; rec(r, slots, db, out)?; out.push(op(KB_F_OR, 0, 0, 0, 0.0)); }
            FilterExpression::Not(i) => { rec(i, slots, db, out)?; out.push(op(KB_F_NOT, 0, 0, 0, 0.0)); }
            FilterExpression::ArithmeticExpr(a) => { arith(a, slots, out)?; out.push(op(KB_F_TRUTHY, 0, 0, 0, 0.0)); }
            FilterExpression::FunctionCall(name, args) => {
                if *name == "isTRIPLE" && !args.is_empty() { out.push(op(KB_F_IS_TRIPLE, slots.of(args[0]), 0, 0, 0.0)); } else { return None; }
            }
        }
        Some(())
    }
    let mut out = Vec::new();
    rec(&cond.expression, slots, database, &mut out)?;
    Some(out)
}

/// a device relation owned by the shim (freed on drop)
pub struct Rel(pub *mut KbRel, pub *mut KbCtx);
impl Drop for Rel { fn drop(&mut self) { unsafe { kb_rel_free(self.1, self.0) } } }

fn is_quoted(p: &TriplePattern) -> bool { p.0.is_quoted_triple() || p.1.is_quoted_triple() || p.2.is_quoted_triple() }

fn run(op: &PhysicalOperator, dev: &DeviceStore, db: &SparqlDatabase, slots: &mut SlotMap) -> Option<Rel> {
    let ctx = dev.ctx;
    let mut out: *mut KbRel = ptr::null_mut();
    let ok = |rc: kb_status, out: *mut KbRel| if rc == KB_OK { Some(Rel(out, ctx)) } else { None };
    match op {
        PhysicalOperator::TableScan { pattern } | PhysicalOperator::IndexScan { pattern } => {
            if is_quoted(pattern) {  // resolve_quoted_triple_scan (engine.rs:1111-1188) on the device
                let q = slots.quoted_pattern(pattern)?;
                return ok(unsafe { kb_scan_quoted(ctx, &q, &mut out) }, out);
            }
            let p = slots.pattern(pattern)?;
            ok(unsafe { kb_scan(ctx, &p, 1, ptr::null(), ptr::null(), &mut out) }, out)
        }
        PhysicalOperator::Filter { input, condition } => {
            let prog = compile_condition(condition, slots, db)?;
            if let PhysicalOperator::StarJoin { join_var, patterns } = input.as_ref() {
                // Selection over a star: the fused operator pushes the conjuncts into its scans / probe
                let pats: Option<Vec<KbPattern>> = patterns.iter().map(|p| slots.pattern(p)).collect();
                let pats = pats?;
                let js = slots.of(join_var);
                return ok(unsafe { kb_star_join(ctx, js, pats.as_ptr(), pats.len() as u32, prog.as_ptr(), prog.len() as u32, &mut out) }, out);
            }
            let r = run(input, dev, db, slots)?;
            ok(unsafe { kb_filter(ctx, r.0, prog.as_ptr(), prog.len() as u32, &mut out) }, out)
        }
        PhysicalOperator::Projection { input, variables } => {
            let r = run(input, dev, db, slots)?;
            let sl: Vec<u32> = variables.iter().map(|v| slots.of(v)).collect();
            ok(unsafe { kb_project(ctx, r.0, sl.as_ptr(), sl.len() as u32, &mut out) }, out)
        }
        PhysicalOperator::HashJoin { left, right } | PhysicalOperator::OptimizedHashJoin { left, right } | PhysicalOperator::NestedLoopJoin { left, right } => {
            let (l, r) = (run(left, dev, db, slots)?, run(right, dev, db, slots)?);
            ok(unsafe { kb_hash_join(ctx, l.0, r.0, &mut out) }, out)
        }
        PhysicalOperator::ParallelJoin { left, right } => {
            let l = run(left, dev, db, slots)?;
            match right.as_ref() {  // a scan on the right is a bind join (engine.rs:935-937): the index's persistent table answers it
                PhysicalOperator::TableScan { pattern } | PhysicalOperator::IndexScan { pattern } if !is_quoted(pattern) => {
                    let p = slots.pattern(pattern)?;
                    ok(unsafe { kb_bind_join(ctx, l.0, &p, &mut out) }, out)
                }
                // anything else, a quoted scan included (kb_scan_quoted, then the natural join)
                _ => { let r = run(right, dev, db, slots)?; ok(unsafe { kb_hash_join(ctx, l.0, r.0, &mut out) }, out) }
            }
        }
        PhysicalOperator::StarJoin { join_var, patterns } => {
            let pats: Option<Vec<KbPattern>> = patterns.iter().map(|p| slots.pattern(p)).collect();
            let pats = pats?;
            let js = slots.of(join_var);
            ok(unsafe { kb_star_join(ctx, js, pats.as_ptr(), pats.len() as u32, ptr::null(), 0, &mut out) }, out)
        }
        PhysicalOperator::InMemoryBuffer { content, .. } => {
            let mut names: Vec<String> = content.iter().flat_map(|r| r.keys().cloned()).collect();
            names.sort(); names.dedup();
            let cols: Vec<Vec<u32>> = names.iter().map(|k| content.iter().map(|r| *r.get(k).unwrap_or(&KB_ID_NONE)).collect()).collect();
            let ptrs: Vec<*const u32> = cols.iter().map(|c| c.as_ptr()).collect();
            let sl: Vec<u32> = names.iter().map(|k| slots.of(k)).collect();
            ok(unsafe { kb_rel_from_host(ctx, sl.as_ptr(), sl.len() as u32, ptrs.as_ptr(), content.len() as u64, &mut out) }, out)
        }
        _ => None,  // Bind and Values (see run_mut), MLPredict, Subquery: the reference's CPU path
    }
}

/// The device dictionary's ids [first, first + n) join the host dictionary, in the order the device created them (no lookup of its own).
fn take_new_strings(dev: &mut DeviceStore, db: &mut SparqlDatabase, first: u32, n: u32) -> Option<()> {
    if n == 0 { return Some(()); }
    let ctx = dev.ctx;
    let mut offs = vec![0u64; n as usize + 1];
    if unsafe { kb_dict_strings_download(ctx, first, n, offs.as_mut_ptr(), ptr::null_mut()) } != KB_OK { return None; }
    let mut bytes = vec![0u8; offs[n as usize] as usize];
    if unsafe { kb_dict_strings_download(ctx, first, n, offs.as_mut_ptr(), bytes.as_mut_ptr()) } != KB_OK { return None; }
    let mut dict = db.dictionary.write().unwrap();
    for k in 0..n as usize {
        dict.encode(std::str::from_utf8(&bytes[offs[k] as usize..offs[k + 1] as usize]).ok()?);
    }
    dev.synced_dict = dict.id_to_string.len();
    Some(())
}

fn has_values(op: &PhysicalOperator) -> bool {
    match op {
        PhysicalOperator::Values { .. } => true,
        PhysicalOperator::Filter { input, .. } | PhysicalOperator::Projection { input, .. } => has_values(input),
        PhysicalOperator::HashJoin { left, right } | PhysicalOperator::OptimizedHashJoin { left, right }
        | PhysicalOperator::NestedLoopJoin { left, right } | PhysicalOperator::ParallelJoin { left, right } => has_values(left) || has_values(right),
        _ => false,
    }
}

fn rel_slots(r: &Rel) -> Option<(u64, Vec<u32>)> {
    let (mut n, mut nc, mut rs) = (0u64, 0u32, [0u32; KB_MAX_COLS]);
    if unsafe { kb_rel_info(r.0, &mut n, &mut nc, rs.as_mut_ptr()) } != KB_OK { return None; }
    Some((n, rs[..nc as usize].to_vec()))
}

#[derive(Clone, Copy, PartialEq)]
enum JoinKind { Hash, OptimizedHash, NestedLoop, Parallel }

/// One join operator of the reference over device relations whose `ragged` slots may hold KB_ID_NONE (a VALUES block's UNDEF cells),
/// as engine.py's ExecutionEngine._join: without KB_ID_NONE in a shared slot every operator is kb_hash_join; NestedLoopJoin is the join
/// of mappings (kb_natural_join, engine.rs:814-837); the hash joins and the merge join pair rows on the shared variables bound in row 0
/// of both sides (kb_hash_join_keyed, engine.rs:710-811, 970-1039), the other shared variables left-first, except the probe side of
/// OptimizedHashJoin (the right side when the left is the smaller or equal one) and the cartesian product (engine.rs:1054-1071), which
/// are right-first. A key cell a row leaves unbound is refused (None: the CPU path, where the reference panics). Row 0 is the device
/// relation's: below a join that is the join's device order, not the reference's hash order.
fn join_ragged(ctx: *mut KbCtx, kind: JoinKind, l: &Rel, r: &Rel, ragged: &[u32]) -> Option<Rel> {
    let mut out: *mut KbRel = ptr::null_mut();
    let (nl, ls) = rel_slots(l)?;
    let (nr, rs) = rel_slots(r)?;
    let shared: Vec<u32> = ls.iter().copied().filter(|s| rs.contains(s)).collect();
    let rc = if !shared.iter().any(|s| ragged.contains(s)) {
        unsafe { kb_hash_join(ctx, l.0, r.0, &mut out) }
    } else if kind == JoinKind::NestedLoop {
        unsafe { kb_natural_join(ctx, l.0, r.0, &mut out) }
    } else {
        let mut key = Vec::new();
        if nl > 0 && nr > 0 {
            let row0 = |rel: &Rel, slots: &[u32]| -> Option<Vec<u32>> {
                let mut v: *mut KbRel = ptr::null_mut();
                if unsafe { kb_order_by(ctx, rel.0, ptr::null(), 0, 1, &mut v, ptr::null_mut()) } != KB_OK { return None; }
                let v = Rel(v, ctx);
                let mut row = vec![KB_ID_NONE; slots.len()];
                for c in 0..slots.len() {
                    if unsafe { kb_rel_download(ctx, v.0, c as u32, &mut row[c]) } != KB_OK { return None; }
                }
                Some(row)
            };
            let (l0, r0) = (row0(l, &ls)?, row0(r, &rs)?);
            for &s in &shared {
                let (i, j) = (ls.iter().position(|&x| x == s)?, rs.iter().position(|&x| x == s)?);
                if l0[i] != KB_ID_NONE && r0[j] != KB_ID_NONE { key.push(s); }
            }
        }
        let right_first = key.is_empty() || (kind == JoinKind::OptimizedHash && nl <= nr);
        let merge = if right_first { KB_MERGE_RIGHT_FIRST } else { KB_MERGE_LEFT_FIRST };
        unsafe { kb_hash_join_keyed(ctx, l.0, r.0, key.as_ptr(), key.len() as u32, merge, &mut out) }
    };
    if rc == KB_OK { Some(Rel(out, ctx)) } else { None }
}

/// `run` plus `Bind` with the built-in functions (engine.rs:144-277) through kb_bind. The plan builder puts every Bind above the join and
/// filter tree (utils.rs:101-191), so only Projection and Bind are looked at here: a Bind anywhere else, or an operator reading a Bind
/// output, goes through `run`, which returns None. `bind_out` collects the output slots (KB_ID_NONE there = the variable is unbound).
fn run_mut(op: &PhysicalOperator, dev: &mut DeviceStore, db: &mut SparqlDatabase, slots: &mut SlotMap, bind_out: &mut Vec<u32>) -> Option<Rel> {
    let ctx = dev.ctx;
    let mut out: *mut KbRel = ptr::null_mut();
    match op {
        PhysicalOperator::Projection { input, variables } => {
            let r = run_mut(input, dev, db, slots, bind_out)?;
            let sl: Vec<u32> = variables.iter().map(|v| slots.of(v)).collect();
            if unsafe { kb_project(ctx, r.0, sl.as_ptr(), sl.len() as u32, &mut out) } != KB_OK { return None; }
            Some(Rel(out, ctx))
        }
        // VALUES (engine.rs:279-308) through kb_values: every defined cell encoded verbatim, in row-major order, into the device
        // dictionary, which the host dictionary then follows; an UNDEF cell is KB_ID_NONE, so its slots join `bind_out`
        PhysicalOperator::Values { variables, values } => {
            let sl: Vec<u32> = variables.iter().map(|v| slots.of(v)).collect();
            let nv = sl.len();
            let mut undef = vec![1u8; values.len() * nv];
            let mut offs = vec![0u64; values.len() * nv + 1];
            let mut bytes: Vec<u8> = Vec::new();
            for (r, row) in values.iter().enumerate() {
                for v in 0..nv {
                    let i = r * nv + v;
                    if let Some(Some(t)) = row.get(v) {  // value_row.get(i): a missing trailing cell is UNDEF
                        undef[i] = 0;
                        bytes.extend_from_slice(t.as_bytes());
                    }
                    offs[i + 1] = bytes.len() as u64;
                }
            }
            let mut info = KbValuesInfo::default();
            if unsafe { kb_values(ctx, sl.as_ptr(), nv as u32, values.len() as u64, undef.as_ptr(), offs.as_ptr(), bytes.as_ptr(), &mut out, &mut info) } != KB_OK {
                return None;
            }
            let res = Rel(out, ctx);
            take_new_strings(dev, db, info.dict_first, info.dict_new)?;
            for s in sl { if !bind_out.contains(&s) { bind_out.push(s); } }
            Some(res)
        }
        // the plan builder puts a VALUES block at the base of the join chain (utils.rs:110-171): the operators above it come here
        PhysicalOperator::Filter { input, condition } if has_values(input) => {
            let r = run_mut(input, dev, db, slots, bind_out)?;
            let prog = compile_condition(condition, slots, db)?;
            if unsafe { kb_filter(ctx, r.0, prog.as_ptr(), prog.len() as u32, &mut out) } != KB_OK { return None; }
            Some(Rel(out, ctx))
        }
        PhysicalOperator::HashJoin { left, right } | PhysicalOperator::OptimizedHashJoin { left, right }
        | PhysicalOperator::NestedLoopJoin { left, right } if has_values(left) || has_values(right) => {
            let kind = match op {
                PhysicalOperator::HashJoin { .. } => JoinKind::Hash,
                PhysicalOperator::OptimizedHashJoin { .. } => JoinKind::OptimizedHash,
                _ => JoinKind::NestedLoop,
            };
            let l = run_mut(left, dev, db, slots, bind_out)?;
            let r = run_mut(right, dev, db, slots, bind_out)?;
            join_ragged(ctx, kind, &l, &r, bind_out)
        }
        PhysicalOperator::ParallelJoin { left, right } if has_values(left) || has_values(right) => {
            let l = run_mut(left, dev, db, slots, bind_out)?;
            match right.as_ref() {
                // a bind join (engine.rs:840-923): bind_pattern leaves a variable the row lacks free, which is the join of mappings
                PhysicalOperator::TableScan { pattern } | PhysicalOperator::IndexScan { pattern } if !is_quoted(pattern) => {
                    let p = slots.pattern(pattern)?;
                    let (_, ls) = rel_slots(&l)?;
                    let ragged = [p.s, p.p, p.o].iter().any(|t| t.is_var == 1 && ls.contains(&t.value) && bind_out.contains(&t.value));
                    if !ragged {
                        if unsafe { kb_bind_join(ctx, l.0, &p, &mut out) } != KB_OK { return None; }
                        return Some(Rel(out, ctx));
                    }
                    if unsafe { kb_scan(ctx, &p, 1, ptr::null(), ptr::null(), &mut out) } != KB_OK { return None; }
                    let m = Rel(out, ctx);
                    let mut j: *mut KbRel = ptr::null_mut();
                    if unsafe { kb_natural_join(ctx, l.0, m.0, &mut j) } != KB_OK { return None; }
                    Some(Rel(j, ctx))
                }
                _ => { let r = run_mut(right, dev, db, slots, bind_out)?; join_ragged(ctx, JoinKind::Parallel, &l, &r, bind_out) }
            }
        }
        PhysicalOperator::Bind { input, function_name, arguments, output_variable } => {
            if db.udfs.contains_key(function_name.as_str()) { return None; }  // a UDF shadows the built-ins (engine.rs:183)
            let function = match function_name.as_str() {
                "SUBJECT" => KB_BIND_SUBJECT, "PREDICATE" => KB_BIND_PREDICATE, "OBJECT" => KB_BIND_OBJECT,
                "isTRIPLE" => KB_BIND_IS_TRIPLE, "TRIPLE" => KB_BIND_TRIPLE, "CONCAT" => KB_BIND_CONCAT,
                _ => return None,
            };
            let r = run_mut(input, dev, db, slots, bind_out)?;
            let (mut n, mut nc, mut rs) = (0u64, 0u32, [0u32; KB_MAX_COLS]);
            if unsafe { kb_rel_info(r.0, &mut n, &mut nc, rs.as_mut_ptr()) } != KB_OK { return None; }
            let column = |slots: &SlotMap, a: &str| slots.slot.get(a.strip_prefix('?').unwrap_or(a)).copied().filter(|s| rs[..nc as usize].contains(s));
            let mut args: Vec<KbTerm> = Vec::new();
            let mut consts: Vec<u8> = Vec::new();
            let mut const_offsets: Vec<u64> = vec![0];
            match function {
                KB_BIND_CONCAT => for a in arguments {
                    match column(slots, a).filter(|_| a.starts_with('?')) {
                        Some(s) => args.push(KbTerm { is_var: 1, value: s }),
                        None => {  // a constant: arg.trim_matches('"'); a variable the rows lack contributes ""
                            args.push(KbTerm { is_var: 0, value: (const_offsets.len() - 1) as u32 });
                            if !a.starts_with('?') { consts.extend_from_slice(a.trim_matches('"').as_bytes()); }
                            const_offsets.push(consts.len() as u64);
                        }
                    }
                },
                KB_BIND_TRIPLE => {
                    if arguments.len() != 3 { return None; }
                    // constants are encoded inside the reference's row loop: in argument order, and only when there is a row
                    let constant: Vec<&str> = arguments.iter().filter(|a| !a.starts_with('?')).map(|a| a.as_str()).collect();
                    let ids = if n > 0 && !constant.is_empty() {
                        let (ids, first) = dev.encode_bulk(&constant).ok()?;
                        let mut dict = db.dictionary.write().unwrap();
                        for &p in &first { dict.encode(constant[p as usize]); }
                        ids
                    } else { vec![0; constant.len()] };
                    let mut k = 0;
                    for a in arguments {
                        if a.starts_with('?') { args.push(KbTerm { is_var: 1, value: column(slots, a)? }); }
                        else { args.push(KbTerm { is_var: 0, value: ids[k] }); k += 1; }
                    }
                }
                _ => {
                    if arguments.len() != 1 { return None; }
                    args.push(KbTerm { is_var: 1, value: column(slots, &arguments[0])? });
                }
            }
            let out_slot = slots.of(output_variable);
            let next_qt_id = db.quoted_triple_store.read().unwrap().next_qt_id;
            let spec = KbBindSpec { function, n_args: args.len() as u32, args: args.as_ptr(), n_const: (const_offsets.len() - 1) as u32,
                                    const_offsets: const_offsets.as_ptr(), const_bytes: consts.as_ptr(), out_slot, next_qt_id };
            let mut info = KbBindInfo::default();
            if unsafe { kb_bind(ctx, r.0, &spec, &mut out, &mut info) } != KB_OK { return None; }
            let res = Rel(out, ctx);
            // the host takes the device's new entries in the order the device created them (no lookup of its own)
            take_new_strings(dev, db, info.dict_first, info.dict_new)?;
            if info.quoted_new > 0 {
                let m = info.quoted_new as usize;
                let (mut s, mut p, mut o) = (vec![0u32; m], vec![0u32; m], vec![0u32; m]);
                if unsafe { kb_quoted_download(ctx, info.quoted_first, info.quoted_new, s.as_mut_ptr(), p.as_mut_ptr(), o.as_mut_ptr()) } != KB_OK { return None; }
                let mut qt = db.quoted_triple_store.write().unwrap();
                for k in 0..m {
                    let id = info.quoted_first + k as u32;
                    qt.id_to_components.insert(id, (s[k], p[k], o[k]));
                    qt.components_to_id.insert((s[k], p[k], o[k]), id);
                }
                qt.next_qt_id = info.quoted_first + info.quoted_new;
                dev.synced_quoted = qt.id_to_components.len();  // the device table holds them: no reload (it would drop the reverse index)
            }
            bind_out.push(out_slot);
            Some(res)
        }
        _ => run(op, dev, db, slots),
    }
}

/// The hook for `ExecutionEngine::execute_with_ids`:
/// ```ignore
/// #[cfg(feature = "cuda")]
/// if shared::GPU_MODE_ENABLED.load(Ordering::Relaxed) {
///     if let Some(rows) = kolibrie_gpu_b200::try_execute(operator, database, &mut DEVICE.lock().unwrap()) { return rows; }
/// }
/// ```
/// None means "shape not handled on the device" (KB_E_UNSUPPORTED or an operator outside the hot path): run the CPU path.
pub fn try_execute(op: &PhysicalOperator, database: &SparqlDatabase, dev: &mut DeviceStore) -> Option<Vec<HashMap<String, u32>>> {
    let res = try_execute_rel(op, database, dev)?;
    download_rows(dev, res.rel.0, &res.names)
}

/// [`try_execute`] for a plan that may hold `Bind` operators with the built-in functions (engine.rs:144-277): they run on the device
/// (kb_bind) and the dictionary and quoted-triple store of `database` take the strings and quoted triples the device created, in its
/// order. A variable a Bind left unbound is not a key of the row, as in the reference. [`try_execute`] keeps returning None for a Bind.
pub fn try_execute_mut(op: &PhysicalOperator, database: &mut SparqlDatabase, dev: &mut DeviceStore) -> Option<Vec<HashMap<String, u32>>> {
    dev.sync(database).ok()?;
    let mut slots = SlotMap::default();
    let mut bind_out = Vec::new();
    let rel = run_mut(op, dev, database, &mut slots, &mut bind_out)?;
    let mut nc = 0u32;
    let mut rs = [0u32; KB_MAX_COLS];
    if unsafe { kb_rel_info(rel.0, ptr::null_mut(), &mut nc, rs.as_mut_ptr()) } != KB_OK { return None; }
    let names: Vec<String> = (0..nc as usize).map(|c| slots.names[rs[c] as usize].clone()).collect();
    let mut rows = download_rows(dev, rel.0, &names)?;
    for c in 0..nc as usize {
        if bind_out.contains(&rs[c]) {
            for row in rows.iter_mut() { if row.get(&names[c]) == Some(&KB_ID_NONE) { row.remove(&names[c]); } }
        }
    }
    Some(rows)
}

/// The operator's result on the device, before any download: the relation and the variable name of each of its columns.
pub struct DeviceResult { pub rel: Rel, pub names: Vec<String> }

/// The device half of [`try_execute`]. None: shape not handled on the device.
pub fn try_execute_rel(op: &PhysicalOperator, database: &SparqlDatabase, dev: &mut DeviceStore) -> Option<DeviceResult> {
    dev.sync(database).ok()?;
    let mut slots = SlotMap::default();
    let rel = run(op, dev, database, &mut slots)?;
    let mut nc = 0u32;
    let mut rs = [0u32; KB_MAX_COLS];
    if unsafe { kb_rel_info(rel.0, ptr::null_mut(), &mut nc, rs.as_mut_ptr()) } != KB_OK { return None; }
    let names = (0..nc as usize).map(|c| slots.names[rs[c] as usize].clone()).collect();
    Some(DeviceResult { rel, names })
}

/// Every row of a device relation as a (variable -> id) map; `names[c]` is the variable of column c.
pub fn download_rows(dev: &DeviceStore, rel: *const KbRel, names: &[String]) -> Option<Vec<HashMap<String, u32>>> {
    let mut n = 0u64;
    if unsafe { kb_rel_info(rel, &mut n, ptr::null_mut(), ptr::null_mut()) } != KB_OK { return None; }
    let mut cols: Vec<Vec<u32>> = Vec::with_capacity(names.len());
    for c in 0..names.len() {
        let mut v = vec![0u32; n as usize];
        if unsafe { kb_rel_download(dev.ctx, rel, c as u32, v.as_mut_ptr()) } != KB_OK { return None; }
        cols.push(v);
    }
    Some((0..n as usize).map(|i| names.iter().enumerate().map(|(c, k)| (k.clone(), cols[c][i])).collect()).collect())
}
