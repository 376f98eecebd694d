//! UNVERIFIED SOURCE — never compiled (no rustc in the build image).
//!
//! Thin Rust host layer keeping the hnsw_rs API surface (`Hnsw<f32, D>`, `AnnT`, `FilterT`, `Neighbour`)
//! on top of the C ABI of libhnsw_b200.so (include/hnsw_b200.h).  Names, argument order and meaning follow
//! hnsw_rs 0.3.4: `src/hnsw.rs:771-777,1069-1071,1224-1238,1487-1635`, `src/api.rs:13-38`, `src/filter.rs:7-24`.
#![allow(non_camel_case_types)]
use std::marker::PhantomData;
use std::os::raw::{c_int, c_void};

pub type DataId = usize;

#[repr(C)]
pub struct HnswApif32 {
    _private: [u8; 0],
}
#[repr(C)]
#[derive(Clone, Copy)]
pub struct Neighbour_api {
    pub id: usize,
    pub d: f32,
}
#[repr(C)]
pub struct Neighbourhood_api {
    pub nbgh: i64,
    pub neighbours: *const Neighbour_api,
}
#[repr(C)]
pub struct Vec_api<T> {
    pub len: i64,
    pub ptr: *const T,
}

extern "C" {
    fn new_hnsw_f32(max_nb_conn: usize, ef_const: usize, namelen: usize, cdistname: *const u8, max_elements: usize,
                    max_layer: usize) -> *const HnswApif32;
    fn drop_hnsw_f32(p: *const HnswApif32);
    fn insert_f32(h: *mut HnswApif32, len: usize, data: *const f32, id: usize);
    fn parallel_insert_f32(h: *mut HnswApif32, nb_vec: usize, vec_len: usize, datas: *mut *const f32, ids: *const usize);
    fn parallel_search_neighbours_f32(h: *const HnswApif32, nb_vec: usize, vec_len: i64, data: *mut *const f32,
                                      knbn: usize, ef_search: usize) -> *const Vec_api<Neighbourhood_api>;
    fn hnsw_b200_free_vec_api(p: *const Vec_api<Neighbourhood_api>);
    fn hnsw_b200_search_flat(h: *const HnswApif32, queries: *const f32, nq: u64, dim: u64, knbn: u64, ef: u64,
                             filter_mode: c_int, filter_ids: *const u64, nfilter: u64,
                             f: Option<extern "C" fn(u64, *mut c_void) -> c_int>, ctx: *mut c_void, out_ids: *mut u64,
                             out_dist: *mut f32, out_internal: *mut u32, out_pid: *mut i32, out_counts: *mut i32) -> c_int;
    fn hnsw_b200_set_extend_candidates(h: *mut HnswApif32, flag: c_int) -> c_int;
    fn hnsw_b200_set_keeping_pruned(h: *mut HnswApif32, flag: c_int) -> c_int;
    fn hnsw_b200_modify_level_scale(h: *mut HnswApif32, scale: f64) -> c_int;
    fn hnsw_b200_set_searching_mode(h: *mut HnswApif32, flag: c_int) -> c_int;
    // reverse-link layer of later inserts (include/hnsw_b200.h): 0 the reference's rule, 1 per layer
    fn hnsw_b200_set_link_mode(h: *mut HnswApif32, mode: c_int) -> c_int;
    fn hnsw_b200_get_link_mode(h: *const HnswApif32) -> c_int;
    fn hnsw_b200_get_nb_point(h: *const HnswApif32) -> u64;
    // multi-GPU (include/hnsw_b200.h "Multi-GPU search"): one process drives several devices
    fn hnsw_b200_replicate(h: *mut HnswApif32, ndev: c_int, devices: *const c_int) -> c_int;
    fn hnsw_b200_replica_count(h: *const HnswApif32) -> c_int;
    // partitioned index (include/hnsw_b200.h "Partitioned index"): the points split over several devices
    fn hnsw_b200_partition(h: *mut HnswApif32, nparts: c_int, devices: *const c_int) -> c_int;
    // saved indexes (include/hnsw_b200.h "Saved indexes"): dir and basename are NUL-terminated
    fn hnsw_b200_save(h: *const HnswApif32, dir: *const u8, basename: *const u8, overwrite: c_int, used_basename: *mut u8,
                      used_cap: usize) -> c_int;
    fn hnsw_b200_restore(dir: *const u8, basename: *const u8, ndev: c_int, devices: *const c_int) -> *mut c_void;
    fn hnsw_b200_partition_count(h: *const HnswApif32) -> c_int;
    // resident filters (include/hnsw_b200.h "Resident filters"): a FilterT materialised once, passed by id
    fn hnsw_b200_filter_new(h: *const HnswApif32, filter_mode: c_int, filter_ids: *const u64, nfilter: u64,
                            f: Option<extern "C" fn(u64, *mut c_void) -> c_int>, ctx: *mut c_void) -> i64;
    fn hnsw_b200_filter_free(h: *const HnswApif32, filter: i64) -> c_int;
    fn hnsw_b200_search_flat_filtered(h: *const HnswApif32, filter: i64, queries: *const f32, nq: u64, dim: u64, knbn: u64,
                                      ef: u64, out_ids: *mut u64, out_dist: *mut f32, out_internal: *mut u32,
                                      out_pid: *mut i32, out_counts: *mut i32) -> c_int;
    fn hnsw_b200_search_flat_submit_filtered(h: *const HnswApif32, filter: i64, queries: *const f32, nq: u64, dim: u64,
                                             knbn: u64, ef: u64, out_ids: *mut u64, out_dist: *mut f32,
                                             out_internal: *mut u32, out_pid: *mut i32, out_counts: *mut i32) -> i64;
    fn hnsw_b200_search_device_filtered(h: *const HnswApif32, filter: i64, d_queries: *const c_void, nq: u64, knbn: u64,
                                        ef: u64, d_out: *mut c_void, d_counts: *mut i32, sync: c_int,
                                        kernel_ms: *mut f32) -> c_int;
    // exact search (include/hnsw_b200.h "Exact search"): filter = a resident filter's id, or -1 for every point
    fn hnsw_b200_search_exact(h: *const HnswApif32, filter: i64, queries: *const f32, nq: u64, dim: u64, knbn: u64,
                              out_ids: *mut u64, out_dist: *mut f32, out_internal: *mut u32, out_pid: *mut i32,
                              out_counts: *mut i32) -> c_int;
    fn hnsw_b200_search_exact_device(h: *const HnswApif32, filter: i64, d_queries: *const c_void, nq: u64, knbn: u64,
                                     d_out: *mut c_void, d_counts: *mut i32, sync: c_int, kernel_ms: *mut f32) -> c_int;
    // a filter per query (include/hnsw_b200.h "A filter per query"): filters[i] = a resident filter's id, or -1
    fn hnsw_b200_search_flat_per_query(h: *const HnswApif32, filters: *const i64, queries: *const f32, nq: u64, dim: u64,
                                       knbn: u64, ef: u64, out_ids: *mut u64, out_dist: *mut f32, out_internal: *mut u32,
                                       out_pid: *mut i32, out_counts: *mut i32) -> c_int;
    fn hnsw_b200_search_exact_per_query(h: *const HnswApif32, filters: *const i64, queries: *const f32, nq: u64, dim: u64,
                                        knbn: u64, out_ids: *mut u64, out_dist: *mut f32, out_internal: *mut u32,
                                        out_pid: *mut i32, out_counts: *mut i32) -> c_int;
    // point labels (include/hnsw_b200.h "Point labels"): qlabels[i] = a label, or LABEL_NONE for every point
    fn hnsw_b200_set_labels(h: *mut HnswApif32, first: u64, n: u64, labels: *const u32) -> c_int;
    fn hnsw_b200_get_labels(h: *const HnswApif32, first: u64, n: u64, out: *mut u32) -> c_int;
    fn hnsw_b200_search_flat_labeled(h: *const HnswApif32, qlabels: *const u32, queries: *const f32, nq: u64, dim: u64,
                                     knbn: u64, ef: u64, out_ids: *mut u64, out_dist: *mut f32, out_internal: *mut u32,
                                     out_pid: *mut i32, out_counts: *mut i32) -> c_int;
    fn hnsw_b200_search_exact_labeled(h: *const HnswApif32, qlabels: *const u32, queries: *const f32, nq: u64, dim: u64,
                                      knbn: u64, out_ids: *mut u64, out_dist: *mut f32, out_internal: *mut u32,
                                      out_pid: *mut i32, out_counts: *mut i32) -> c_int;
    // label sets (include/hnsw_b200.h "Label sets"): query i's set is qset[qset_off[i] .. qset_off[i + 1]]
    fn hnsw_b200_search_flat_label_sets(h: *const HnswApif32, qset_off: *const u64, qset: *const u32, queries: *const f32,
                                        nq: u64, dim: u64, knbn: u64, ef: u64, out_ids: *mut u64, out_dist: *mut f32,
                                        out_internal: *mut u32, out_pid: *mut i32, out_counts: *mut i32) -> c_int;
    fn hnsw_b200_search_exact_label_sets(h: *const HnswApif32, qset_off: *const u64, qset: *const u32, queries: *const f32,
                                         nq: u64, dim: u64, knbn: u64, out_ids: *mut u64, out_dist: *mut f32,
                                         out_internal: *mut u32, out_pid: *mut i32, out_counts: *mut i32) -> c_int;
    // attribute ranges (include/hnsw_b200.h "Attribute ranges"): query i's range is qrange[2i] ..= qrange[2i + 1]
    fn hnsw_b200_set_attributes(h: *mut HnswApif32, first: u64, n: u64, values: *const i64) -> c_int;
    fn hnsw_b200_get_attributes(h: *const HnswApif32, first: u64, n: u64, out: *mut i64) -> c_int;
    fn hnsw_b200_search_flat_ranges(h: *const HnswApif32, qrange: *const i64, qset_off: *const u64, qset: *const u32,
                                    queries: *const f32, nq: u64, dim: u64, knbn: u64, ef: u64, out_ids: *mut u64,
                                    out_dist: *mut f32, out_internal: *mut u32, out_pid: *mut i32, out_counts: *mut i32) -> c_int;
    fn hnsw_b200_search_exact_ranges(h: *const HnswApif32, qrange: *const i64, qset_off: *const u64, qset: *const u32,
                                     queries: *const f32, nq: u64, dim: u64, knbn: u64, out_ids: *mut u64, out_dist: *mut f32,
                                     out_internal: *mut u32, out_pid: *mut i32, out_counts: *mut i32) -> c_int;
    // search by stored point (include/hnsw_b200.h "Search by stored point"): qids are insertion ranks; filter -1 and
    // qrange, qset_off, qset null is no restriction
    fn hnsw_b200_get_vectors(h: *const HnswApif32, ranks: *const u64, n: u64, out: *mut f32) -> c_int;
    fn hnsw_b200_search_flat_by_id(h: *const HnswApif32, qids: *const u64, nq: u64, knbn: u64, ef: u64, exclude_self: c_int,
                                   filter: i64, qrange: *const i64, qset_off: *const u64, qset: *const u32,
                                   out_ids: *mut u64, out_dist: *mut f32, out_internal: *mut u32, out_pid: *mut i32,
                                   out_counts: *mut i32) -> c_int;
    fn hnsw_b200_search_exact_by_id(h: *const HnswApif32, qids: *const u64, nq: u64, knbn: u64, exclude_self: c_int,
                                    filter: i64, qrange: *const i64, qset_off: *const u64, qset: *const u32,
                                    out_ids: *mut u64, out_dist: *mut f32, out_internal: *mut u32, out_pid: *mut i32,
                                    out_counts: *mut i32) -> c_int;
    fn hnsw_b200_search_device_by_id(h: *const HnswApif32, exact: c_int, filter: i64, d_qids: *const u64, nq: u64,
                                     knbn: u64, ef: u64, exclude_self: c_int, d_out: *mut c_void, d_counts: *mut i32,
                                     sync: c_int, kernel_ms: *mut f32) -> c_int;
    fn hnsw_b200_search_exact_radius(h: *const HnswApif32, filter: i64, qrange: *const i64, qset_off: *const u64,
                                     qset: *const u32, queries: *const c_void, nq: u64, dim: u64, radius: *const f32,
                                     knbn: u64, out_ids: *mut u64, out_dist: *mut f32, out_internal: *mut u32,
                                     out_pid: *mut i32, out_counts: *mut i32, out_total: *mut u64) -> c_int;
    fn hnsw_b200_search_exact_radius_by_id(h: *const HnswApif32, qids: *const u64, nq: u64, radius: *const f32,
                                           knbn: u64, exclude_self: c_int, filter: i64, qrange: *const i64,
                                           qset_off: *const u64, qset: *const u32, out_ids: *mut u64,
                                           out_dist: *mut f32, out_internal: *mut u32, out_pid: *mut i32,
                                           out_counts: *mut i32, out_total: *mut u64) -> c_int;
}

/// The attribute of a point that has none (include/hnsw_b200.h HNSW_B200_ATTR_NONE): no range admits it.
pub const ATTR_NONE: i64 = i64::MIN;
/// The range of a request that has none: every point, also those without an attribute.
pub const RANGE_ALL: (i64, i64) = (i64::MIN, i64::MAX);

/// The label of a point that has none (include/hnsw_b200.h HNSW_B200_LABEL_NONE): no label admits it.
pub const LABEL_NONE: u32 = 0xFFFF_FFFF;

/// hnsw.rs:46
#[derive(Debug, Clone, Copy, Default, PartialEq, Eq)]
pub struct PointId(pub u8, pub i32);

/// hnsw.rs:98-107
#[derive(Debug, Clone, Copy, Default)]
pub struct Neighbour {
    pub d_id: DataId,
    pub distance: f32,
    pub p_id: PointId,
}

/// filter.rs:7-9
pub trait FilterT {
    fn hnsw_filter(&self, id: &DataId) -> bool;
}
impl FilterT for Vec<usize> {
    fn hnsw_filter(&self, id: &DataId) -> bool {
        self.binary_search(id).is_ok()
    }
}
impl<F: Fn(&DataId) -> bool> FilterT for F {
    fn hnsw_filter(&self, id: &DataId) -> bool {
        self(id)
    }
}

/// Distance marker types: the kernels are selected by NAME, as in libext.rs:468-520.
pub trait DistName {
    const NAME: &'static str;
}
macro_rules! dist { ($t:ident) => { #[derive(Default, Clone, Copy)] pub struct $t; impl DistName for $t { const NAME: &'static str = stringify!($t); } } }
dist!(DistL1); dist!(DistL2); dist!(DistDot); dist!(DistCosine); dist!(DistHellinger); dist!(DistJeffreys); dist!(DistJensenShannon);

pub struct Hnsw<D: DistName> {
    h: *mut HnswApif32,
    _d: PhantomData<D>,
}
unsafe impl<D: DistName> Send for Hnsw<D> {}
unsafe impl<D: DistName> Sync for Hnsw<D> {}

extern "C" fn filter_trampoline(id: u64, ctx: *mut c_void) -> c_int {
    let f: &&dyn FilterT = unsafe { &*(ctx as *const &dyn FilterT) };
    f.hnsw_filter(&(id as usize)) as c_int
}

impl<D: DistName> Hnsw<D> {
    /// Hnsw::new, hnsw.rs:771-777
    pub fn new(max_nb_connection: usize, max_elements: usize, max_layer: usize, ef_construction: usize, _f: D) -> Self {
        let name = D::NAME.as_bytes();
        let h = unsafe { new_hnsw_f32(max_nb_connection, ef_construction, name.len(), name.as_ptr(), max_elements, max_layer) };
        assert!(!h.is_null(), "libhnsw_b200: no usable CUDA device or bad parameters (there is no CPU fallback)");
        Hnsw { h: h as *mut HnswApif32, _d: PhantomData }
    }
    pub fn get_nb_point(&self) -> usize { unsafe { hnsw_b200_get_nb_point(self.h) as usize } }
    pub fn set_extend_candidates(&mut self, flag: bool) { unsafe { hnsw_b200_set_extend_candidates(self.h, flag as c_int); } }
    pub fn set_keeping_pruned(&mut self, flag: bool) { unsafe { hnsw_b200_set_keeping_pruned(self.h, flag as c_int); } }
    pub fn modify_level_scale(&mut self, s: f64) { unsafe { hnsw_b200_modify_level_scale(self.h, s); } }
    pub fn set_searching_mode(&mut self, flag: bool) { unsafe { hnsw_b200_set_searching_mode(self.h, flag as c_int); } }
    /// Extension: 0 files every back-link of a later insert under the new point's level, as hnsw.rs:1257 does; 1 files
    /// it in the layer where the link was made.  Err on any other mode.
    pub fn set_link_mode(&mut self, mode: i32) -> Result<(), i32> {
        let r = unsafe { hnsw_b200_set_link_mode(self.h, mode as c_int) };
        if r == 0 { Ok(()) } else { Err(r) }
    }
    pub fn get_link_mode(&self) -> i32 { unsafe { hnsw_b200_get_link_mode(self.h) as i32 } }
    /// Extension: copy the index to `devices[1..]` (devices[0] = the device it lives on); `parallel_search` then shards its
    /// batch over all of them, one call as on the CPU (hnsw.rs:1612-1635).
    pub fn replicate(&mut self, devices: &[i32]) -> Result<(), i32> {
        let r = unsafe { hnsw_b200_replicate(self.h, devices.len() as c_int, devices.as_ptr()) };
        if r == 0 { Ok(()) } else { Err(r) }
    }
    pub fn replica_count(&self) -> usize { unsafe { hnsw_b200_replica_count(self.h) as usize } }
    /// Extension (uncompiled, like the rest of this shim): split this EMPTY index into `devs.len()` partitions, partition p
    /// on `devs[p]` (devs[0] = the device it lives on; a device may repeat).  Point g goes to partition g % P; every
    /// search runs on all partitions and merges their answers, so the index may exceed one device's memory.
    pub fn partition(&mut self, devs: &[i32]) -> Result<(), i32> {
        let r = unsafe { hnsw_b200_partition(self.h, devs.len() as c_int, devs.as_ptr()) };
        if r == 0 { Ok(()) } else { Err(r) }
    }
    pub fn partition_count(&self) -> usize { unsafe { hnsw_b200_partition_count(self.h) as usize } }
    /// Extension: save the index with its insertion ranks, labels, attributes, deleted points, settings and level RNG
    /// (<basename>.hnsw.graph / .hnsw.data, one pair <basename>-p<i> per partition, and the manifest
    /// <basename>.hnsw.b200 under `dir`).  Returns the basename used: a unique one when `overwrite` is false and a file
    /// of the set exists.
    pub fn save(&self, dir: &str, basename: &str, overwrite: bool) -> Result<String, i32> {
        let (d, b) = (format!("{}\0", dir), format!("{}\0", basename));
        let mut used = vec![0u8; 4096];
        let r = unsafe { hnsw_b200_save(self.h, d.as_ptr(), b.as_ptr(), overwrite as c_int, used.as_mut_ptr(), used.len()) };
        if r != 0 { return Err(r); }
        let len = used.iter().position(|&c| c == 0).unwrap_or(used.len());
        Ok(String::from_utf8_lossy(&used[..len]).into_owned())
    }
    /// Extension: the index `save` wrote, the same ranks, columns and settings; `devices`: empty for the current device,
    /// or one device per saved partition.  None when the files are refused.  This shim serves f32 only: the saved index
    /// must hold f32 vectors under the distance D.
    pub fn restore(dir: &str, basename: &str, devices: &[i32]) -> Option<Self> {
        let (d, b) = (format!("{}\0", dir), format!("{}\0", basename));
        let h = unsafe { hnsw_b200_restore(d.as_ptr(), b.as_ptr(), devices.len() as c_int, devices.as_ptr()) };
        if h.is_null() { None } else { Some(Hnsw { h: h as *mut HnswApif32, _d: PhantomData }) }
    }

    /// hnsw.rs:1069-1071
    pub fn insert(&self, datav_with_id: (&[f32], usize)) {
        unsafe { insert_f32(self.h, datav_with_id.0.len(), datav_with_id.0.as_ptr(), datav_with_id.1) }
    }
    /// hnsw.rs:1224-1230
    pub fn parallel_insert(&self, datas: &[(&Vec<f32>, usize)]) {
        if datas.is_empty() { return; }
        let mut ptrs: Vec<*const f32> = datas.iter().map(|d| d.0.as_ptr()).collect();
        let ids: Vec<usize> = datas.iter().map(|d| d.1).collect();
        unsafe { parallel_insert_f32(self.h, datas.len(), datas[0].0.len(), ptrs.as_mut_ptr(), ids.as_ptr()) }
    }
    /// hnsw.rs:1597-1599
    pub fn search(&self, data: &[f32], knbn: usize, ef_arg: usize) -> Vec<Neighbour> {
        self.search_filter(data, knbn, ef_arg, None)
    }
    /// hnsw.rs:1487-1580.  Closures are evaluated once per stored origin id by the library (device bitmap).
    pub fn search_filter(&self, data: &[f32], knbn: usize, ef_arg: usize, filter: Option<&dyn FilterT>) -> Vec<Neighbour> {
        let mut ids = vec![0u64; knbn];
        let mut ds = vec![0f32; knbn];
        let mut pid = vec![0i32; 2 * knbn];
        let mut cnt = 0i32;
        let (mode, cb, ctx) = match filter.as_ref() {
            None => (0, None, std::ptr::null_mut()),
            Some(f) => (2, Some(filter_trampoline as extern "C" fn(u64, *mut c_void) -> c_int), f as *const &dyn FilterT as *mut c_void),
        };
        let r = unsafe {
            hnsw_b200_search_flat(self.h, data.as_ptr(), 1, data.len() as u64, knbn as u64, ef_arg as u64, mode,
                                  std::ptr::null(), 0, cb, ctx, ids.as_mut_ptr(), ds.as_mut_ptr(), std::ptr::null_mut(),
                                  pid.as_mut_ptr(), &mut cnt)
        };
        assert_eq!(r, 0, "hnsw_b200_search_flat failed");
        (0..cnt as usize).map(|j| Neighbour { d_id: ids[j] as usize, distance: ds[j], p_id: PointId(pid[2 * j] as u8, pid[2 * j + 1]) }).collect()
    }
    /// Extension: materialise `filter` once, over the points stored now (the closure runs once per stored origin id,
    /// here).  Searches with the returned filter answer exactly as `search_filter` with `filter` does, without
    /// re-evaluating it; after an insert they are refused.
    pub fn make_filter(&self, filter: &dyn FilterT) -> Result<ResidentFilter<'_, D>, i64> {
        let ctx = &filter as *const &dyn FilterT as *mut c_void;
        let id = unsafe { hnsw_b200_filter_new(self.h, 2, std::ptr::null(), 0, Some(filter_trampoline), ctx) };
        if id >= 0 { Ok(ResidentFilter { index: self, id }) } else { Err(id) }
    }
    /// search_filter with a resident filter
    pub fn search_resident(&self, data: &[f32], knbn: usize, ef_arg: usize, filter: &ResidentFilter<'_, D>) -> Vec<Neighbour> {
        let mut ids = vec![0u64; knbn];
        let mut ds = vec![0f32; knbn];
        let mut pid = vec![0i32; 2 * knbn];
        let mut cnt = 0i32;
        let r = unsafe {
            hnsw_b200_search_flat_filtered(self.h, filter.id, data.as_ptr(), 1, data.len() as u64, knbn as u64, ef_arg as u64,
                                           ids.as_mut_ptr(), ds.as_mut_ptr(), std::ptr::null_mut(), pid.as_mut_ptr(), &mut cnt)
        };
        assert_eq!(r, 0, "hnsw_b200_search_flat_filtered failed");
        (0..cnt as usize).map(|j| Neighbour { d_id: ids[j] as usize, distance: ds[j], p_id: PointId(pid[2 * j] as u8, pid[2 * j + 1]) }).collect()
    }
    /// Extension: the exact `knbn` nearest among the points `filter` admits (None: every stored point)
    pub fn search_exact(&self, data: &[f32], knbn: usize, filter: Option<&ResidentFilter<'_, D>>) -> Vec<Neighbour> {
        let mut ids = vec![0u64; knbn];
        let mut ds = vec![0f32; knbn];
        let mut pid = vec![0i32; 2 * knbn];
        let mut cnt = 0i32;
        let r = unsafe {
            hnsw_b200_search_exact(self.h, filter.map_or(-1, |f| f.id), data.as_ptr(), 1, data.len() as u64, knbn as u64,
                                   ids.as_mut_ptr(), ds.as_mut_ptr(), std::ptr::null_mut(), pid.as_mut_ptr(), &mut cnt)
        };
        assert_eq!(r, 0, "hnsw_b200_search_exact failed");
        (0..cnt as usize).map(|j| Neighbour { d_id: ids[j] as usize, distance: ds[j], p_id: PointId(pid[2 * j] as u8, pid[2 * j + 1]) }).collect()
    }
    /// Extension: one batch, request i filtered by `filters[i]` (None: no filter); answer i is what search_resident
    /// (or search, for None) returns for request i.  Graph search with `Some(ef)`, the exact scan with None.
    pub fn search_per_query(&self, datas: &[Vec<f32>], knbn: usize, ef: Option<usize>,
                            filters: &[Option<&ResidentFilter<'_, D>>]) -> Vec<Vec<Neighbour>> {
        assert_eq!(datas.len(), filters.len(), "one filter per request");
        if datas.is_empty() { return Vec::new(); }
        let (nq, dim) = (datas.len(), datas[0].len());
        let flat: Vec<f32> = datas.iter().flat_map(|d| d.iter().copied()).collect();
        let fids: Vec<i64> = filters.iter().map(|f| f.map_or(-1, |f| f.id)).collect();
        let mut ids = vec![0u64; nq * knbn];
        let mut ds = vec![0f32; nq * knbn];
        let mut pid = vec![0i32; 2 * nq * knbn];
        let mut cnt = vec![0i32; nq];
        let r = unsafe {
            match ef {
                Some(ef) => hnsw_b200_search_flat_per_query(self.h, fids.as_ptr(), flat.as_ptr(), nq as u64, dim as u64, knbn as u64,
                                                            ef as u64, ids.as_mut_ptr(), ds.as_mut_ptr(), std::ptr::null_mut(),
                                                            pid.as_mut_ptr(), cnt.as_mut_ptr()),
                None => hnsw_b200_search_exact_per_query(self.h, fids.as_ptr(), flat.as_ptr(), nq as u64, dim as u64, knbn as u64,
                                                         ids.as_mut_ptr(), ds.as_mut_ptr(), std::ptr::null_mut(), pid.as_mut_ptr(),
                                                         cnt.as_mut_ptr()),
            }
        };
        assert_eq!(r, 0, "hnsw_b200_search_flat_per_query / _exact_per_query failed");
        (0..nq).map(|i| (0..cnt[i] as usize).map(|j| {
            let s = i * knbn + j;
            Neighbour { d_id: ids[s] as usize, distance: ds[s], p_id: PointId(pid[2 * s] as u8, pid[2 * s + 1]) }
        }).collect()).collect()
    }
    /// Extension: label the points with insertion ranks `first .. first + labels.len()` (LABEL_NONE clears a label).
    /// Every point starts without one; labels are not written into dumps.  Err when the range passes nb_point.
    pub fn set_labels(&mut self, first: usize, labels: &[u32]) -> Result<(), i32> {
        let r = unsafe { hnsw_b200_set_labels(self.h, first as u64, labels.len() as u64, labels.as_ptr()) };
        if r == 0 { Ok(()) } else { Err(r) }
    }
    /// Extension: the labels of the points `first .. first + n`
    pub fn get_labels(&self, first: usize, n: usize) -> Result<Vec<u32>, i32> {
        let mut out = vec![LABEL_NONE; n];
        let r = unsafe { hnsw_b200_get_labels(self.h, first as u64, n as u64, out.as_mut_ptr()) };
        if r == 0 { Ok(out) } else { Err(r) }
    }
    /// Extension: one batch, request i restricted to the points labelled `labels[i]` (LABEL_NONE: every point); answer i
    /// is what search_resident returns with a filter admitting exactly those points (search, for LABEL_NONE).  Graph
    /// search with `Some(ef)`, the exact scan with None.
    pub fn search_labeled(&self, datas: &[Vec<f32>], knbn: usize, ef: Option<usize>, labels: &[u32]) -> Vec<Vec<Neighbour>> {
        assert_eq!(datas.len(), labels.len(), "one label per request");
        if datas.is_empty() { return Vec::new(); }
        let (nq, dim) = (datas.len(), datas[0].len());
        let flat: Vec<f32> = datas.iter().flat_map(|d| d.iter().copied()).collect();
        let mut ids = vec![0u64; nq * knbn];
        let mut ds = vec![0f32; nq * knbn];
        let mut pid = vec![0i32; 2 * nq * knbn];
        let mut cnt = vec![0i32; nq];
        let r = unsafe {
            match ef {
                Some(ef) => hnsw_b200_search_flat_labeled(self.h, labels.as_ptr(), flat.as_ptr(), nq as u64, dim as u64, knbn as u64,
                                                          ef as u64, ids.as_mut_ptr(), ds.as_mut_ptr(), std::ptr::null_mut(),
                                                          pid.as_mut_ptr(), cnt.as_mut_ptr()),
                None => hnsw_b200_search_exact_labeled(self.h, labels.as_ptr(), flat.as_ptr(), nq as u64, dim as u64, knbn as u64,
                                                       ids.as_mut_ptr(), ds.as_mut_ptr(), std::ptr::null_mut(), pid.as_mut_ptr(),
                                                       cnt.as_mut_ptr()),
            }
        };
        assert_eq!(r, 0, "hnsw_b200_search_flat_labeled / _exact_labeled failed");
        (0..nq).map(|i| (0..cnt[i] as usize).map(|j| {
            let s = i * knbn + j;
            Neighbour { d_id: ids[s] as usize, distance: ds[s], p_id: PointId(pid[2 * s] as u8, pid[2 * s + 1]) }
        }).collect()).collect()
    }
    /// Extension: one batch, request i restricted to the points whose label is one of `sets[i]` (any order, repeats
    /// allowed; `[LABEL_NONE]`: every point; empty: none); answer i is what search_resident returns with a filter
    /// admitting exactly those points.  Graph search with `Some(ef)`, the exact scan with None.
    pub fn search_label_sets(&self, datas: &[Vec<f32>], knbn: usize, ef: Option<usize>, sets: &[Vec<u32>]) -> Vec<Vec<Neighbour>> {
        assert_eq!(datas.len(), sets.len(), "one label set per request");
        if datas.is_empty() { return Vec::new(); }
        let (nq, dim) = (datas.len(), datas[0].len());
        let flat: Vec<f32> = datas.iter().flat_map(|d| d.iter().copied()).collect();
        let mut off = vec![0u64; nq + 1];
        for (i, s) in sets.iter().enumerate() { off[i + 1] = off[i] + s.len() as u64; }
        let mut vals: Vec<u32> = sets.iter().flat_map(|s| s.iter().copied()).collect();
        vals.push(LABEL_NONE);  // never empty, so never a null pointer; past every set's end
        let mut ids = vec![0u64; nq * knbn];
        let mut ds = vec![0f32; nq * knbn];
        let mut pid = vec![0i32; 2 * nq * knbn];
        let mut cnt = vec![0i32; nq];
        let r = unsafe {
            match ef {
                Some(ef) => hnsw_b200_search_flat_label_sets(self.h, off.as_ptr(), vals.as_ptr(), flat.as_ptr(), nq as u64, dim as u64,
                                                             knbn as u64, ef as u64, ids.as_mut_ptr(), ds.as_mut_ptr(),
                                                             std::ptr::null_mut(), pid.as_mut_ptr(), cnt.as_mut_ptr()),
                None => hnsw_b200_search_exact_label_sets(self.h, off.as_ptr(), vals.as_ptr(), flat.as_ptr(), nq as u64, dim as u64,
                                                          knbn as u64, ids.as_mut_ptr(), ds.as_mut_ptr(), std::ptr::null_mut(),
                                                          pid.as_mut_ptr(), cnt.as_mut_ptr()),
            }
        };
        assert_eq!(r, 0, "hnsw_b200_search_flat_label_sets / _exact_label_sets failed");
        (0..nq).map(|i| (0..cnt[i] as usize).map(|j| {
            let s = i * knbn + j;
            Neighbour { d_id: ids[s] as usize, distance: ds[s], p_id: PointId(pid[2 * s] as u8, pid[2 * s + 1]) }
        }).collect()).collect()
    }
    /// Extension: give the points with insertion ranks `first .. first + values.len()` an int64 attribute (ATTR_NONE
    /// clears one).  Every point starts without one; attributes are not written into dumps.  Err when the range passes
    /// nb_point.
    pub fn set_attributes(&mut self, first: usize, values: &[i64]) -> Result<(), i32> {
        let r = unsafe { hnsw_b200_set_attributes(self.h, first as u64, values.len() as u64, values.as_ptr()) };
        if r == 0 { Ok(()) } else { Err(r) }
    }
    /// Extension: the attributes of the points `first .. first + n`
    pub fn get_attributes(&self, first: usize, n: usize) -> Result<Vec<i64>, i32> {
        let mut out = vec![0i64; n];
        let r = unsafe { hnsw_b200_get_attributes(self.h, first as u64, n as u64, out.as_mut_ptr()) };
        if r == 0 { Ok(out) } else { Err(r) }
    }
    /// Extension: one batch, request i restricted to the points whose attribute lies in `ranges[i]` (inclusive;
    /// RANGE_ALL: every point, also those without one) and, with `sets`, whose label is one of `sets[i]` (as
    /// search_label_sets takes it); answer i is what search_resident returns with a filter admitting exactly those
    /// points.  Graph search with `Some(ef)`, the exact scan with None.
    pub fn search_ranges(&self, datas: &[Vec<f32>], knbn: usize, ef: Option<usize>, ranges: &[(i64, i64)],
                         sets: Option<&[Vec<u32>]>) -> Vec<Vec<Neighbour>> {
        assert_eq!(datas.len(), ranges.len(), "one range per request");
        if let Some(s) = sets { assert_eq!(datas.len(), s.len(), "one label set per request"); }
        if datas.is_empty() { return Vec::new(); }
        let (nq, dim) = (datas.len(), datas[0].len());
        let flat: Vec<f32> = datas.iter().flat_map(|d| d.iter().copied()).collect();
        let qrange: Vec<i64> = ranges.iter().flat_map(|&(lo, hi)| [lo, hi]).collect();
        let (mut off, mut vals) = (Vec::new(), Vec::new());
        if let Some(sets) = sets {
            off = vec![0u64; nq + 1];
            for (i, s) in sets.iter().enumerate() { off[i + 1] = off[i] + s.len() as u64; }
            vals = sets.iter().flat_map(|s| s.iter().copied()).collect();
            vals.push(LABEL_NONE);  // never empty, so never a null pointer; past every set's end
        }
        let (po, pv) = if sets.is_some() { (off.as_ptr(), vals.as_ptr()) } else { (std::ptr::null(), std::ptr::null()) };
        let mut ids = vec![0u64; nq * knbn];
        let mut ds = vec![0f32; nq * knbn];
        let mut pid = vec![0i32; 2 * nq * knbn];
        let mut cnt = vec![0i32; nq];
        let r = unsafe {
            match ef {
                Some(ef) => hnsw_b200_search_flat_ranges(self.h, qrange.as_ptr(), po, pv, flat.as_ptr(), nq as u64, dim as u64,
                                                         knbn as u64, ef as u64, ids.as_mut_ptr(), ds.as_mut_ptr(),
                                                         std::ptr::null_mut(), pid.as_mut_ptr(), cnt.as_mut_ptr()),
                None => hnsw_b200_search_exact_ranges(self.h, qrange.as_ptr(), po, pv, flat.as_ptr(), nq as u64, dim as u64,
                                                      knbn as u64, ids.as_mut_ptr(), ds.as_mut_ptr(), std::ptr::null_mut(),
                                                      pid.as_mut_ptr(), cnt.as_mut_ptr()),
            }
        };
        assert_eq!(r, 0, "hnsw_b200_search_flat_ranges / _exact_ranges failed");
        (0..nq).map(|i| (0..cnt[i] as usize).map(|j| {
            let s = i * knbn + j;
            Neighbour { d_id: ids[s] as usize, distance: ds[s], p_id: PointId(pid[2 * s] as u8, pid[2 * s + 1]) }
        }).collect()).collect()
    }
    /// hnsw.rs:1612-1635: one answer per request, in input order
    pub fn parallel_search(&self, datas: &[Vec<f32>], knbn: usize, ef: usize) -> Vec<Vec<Neighbour>> {
        if datas.is_empty() { return Vec::new(); }
        let mut ptrs: Vec<*const f32> = datas.iter().map(|d| d.as_ptr()).collect();
        let res = unsafe { parallel_search_neighbours_f32(self.h, datas.len(), datas[0].len() as i64, ptrs.as_mut_ptr(), knbn, ef) };
        assert!(!res.is_null());
        let v = unsafe { &*res };
        let hoods = unsafe { std::slice::from_raw_parts(v.ptr, v.len as usize) };
        let out = hoods.iter().map(|h| {
            let nb = unsafe { std::slice::from_raw_parts(h.neighbours, h.nbgh as usize) };
            nb.iter().map(|n| Neighbour { d_id: n.id, distance: n.d, p_id: PointId::default() }).collect()
        }).collect();
        unsafe { hnsw_b200_free_vec_api(res) };
        out
    }
}

impl<D: DistName> Drop for Hnsw<D> {
    fn drop(&mut self) { unsafe { drop_hnsw_f32(self.h) } }
}

/// A filter made by `Hnsw::make_filter`; it borrows its index and is freed when dropped (the drop waits for searches that
/// may still read it, so collect this thread's own submitted batches first).
pub struct ResidentFilter<'a, D: DistName> {
    index: &'a Hnsw<D>,
    id: i64,
}
impl<'a, D: DistName> ResidentFilter<'a, D> {
    pub fn id(&self) -> i64 { self.id }
}
impl<'a, D: DistName> Drop for ResidentFilter<'a, D> {
    fn drop(&mut self) { unsafe { hnsw_b200_filter_free(self.index.h, self.id); } }
}

/// api.rs:13-38
pub trait AnnT {
    type Val;
    fn insert_data(&mut self, data: &[Self::Val], id: usize);
    fn search_neighbours(&self, data: &[Self::Val], knbn: usize, ef_s: usize) -> Vec<Neighbour>;
    fn parallel_insert_data(&mut self, data: &[(&Vec<Self::Val>, usize)]);
    fn parallel_search_neighbours(&self, data: &[Vec<Self::Val>], knbn: usize, ef_s: usize) -> Vec<Vec<Neighbour>>;
}
impl<D: DistName> AnnT for Hnsw<D> {
    type Val = f32;
    fn insert_data(&mut self, data: &[f32], id: usize) { self.insert((data, id)) }
    fn search_neighbours(&self, data: &[f32], knbn: usize, ef_s: usize) -> Vec<Neighbour> { self.search(data, knbn, ef_s) }
    fn parallel_insert_data(&mut self, data: &[(&Vec<f32>, usize)]) { self.parallel_insert(data) }
    fn parallel_search_neighbours(&self, data: &[Vec<f32>], knbn: usize, ef_s: usize) -> Vec<Vec<Neighbour>> { self.parallel_search(data, knbn, ef_s) }
}
