//! gpu_shuffle.rs — the vega-side shim over libvega_b200.so (would live at src/gpu/mod.rs).
//!
//! SOURCE ONLY, never compiled: this image has no rustc/cargo and vega needs nightly-2020-05-31 + capnpc.
//! It shows, as code rather than prose, the four call-site specialisations INTEGRATION.md lists.
//! Everything generic (any K/V, serde_closure aggregators) keeps vega's CPU path; only POD rows with a
//! *named* op take the GPU path.
#![allow(dead_code)]
use std::os::raw::c_void;
use std::sync::Arc;

use dashmap::DashMap;
use once_cell::sync::Lazy;

use crate::aggregator::Aggregator;
use crate::dependency::{ShuffleDependency, ShuffleDependencyTrait};
use crate::env;
use crate::error::{Error, Result};
use crate::rdd::{Rdd, RddBase, ShuffledRdd};
use crate::shuffle::ShuffleError;
use crate::split::Split;

mod sys; // rust_shim/vega_b200_sys.rs

/// Named reduce op carried by the aggregator (a serde_closure cannot be inspected):
/// `Aggregator::sum()/min()/max()/count()` set it, `Aggregator::default()` sets Group.
#[derive(Clone, Copy, Debug, Serialize, Deserialize)]
pub enum GpuOp { Group, Sum, Min, Max, Count, CoGroup }

impl GpuOp {
    fn code(self) -> i32 {
        match self {
            GpuOp::Group => sys::VB_AGG_GROUP, GpuOp::Sum => sys::VB_AGG_SUM, GpuOp::Min => sys::VB_AGG_MIN,
            GpuOp::Max => sys::VB_AGG_MAX, GpuOp::Count => sys::VB_AGG_COUNT, GpuOp::CoGroup => sys::VB_AGG_COGROUP,
        }
    }
}

struct Handle(*mut sys::vb_shuf);
unsafe impl Send for Handle {}
unsafe impl Sync for Handle {}

/// Process-wide engine, the analogue of env::SHUFFLE_CACHE (src/env.rs:18-27).
pub struct GpuEngine { ctx: *mut sys::vb_ctx, shuffles: DashMap<usize, Handle> }
unsafe impl Send for GpuEngine {}
unsafe impl Sync for GpuEngine {}

pub static GPU: Lazy<GpuEngine> = Lazy::new(|| {
    let dev = std::env::var("VEGA_GPU_DEVICE").ok().and_then(|s| s.parse().ok()).unwrap_or(0);
    let mut ctx = std::ptr::null_mut();
    check(unsafe { sys::vb_ctx_create(dev, &mut ctx) }).expect("vb_ctx_create");
    GpuEngine { ctx, shuffles: DashMap::new() }
});

fn check(rc: i32) -> std::result::Result<(), ShuffleError> {
    if rc == sys::VB_OK { return Ok(()); }
    let msg = unsafe { std::ffi::CStr::from_ptr(sys::vb_last_error()) }.to_string_lossy().into_owned();
    log::error!("vega_b200 error {}: {}", rc, msg);
    Err(ShuffleError::Other) // src/shuffle/mod.rs:17-57
}

impl GpuEngine {
    /// ShuffleDependency::new + register_shuffle: create on first use, keyed by shuffle_id.
    fn shuffle(&self, shuffle_id: usize, n_map: usize, n_reduce: usize, op: GpuOp, key_width: u32) -> *mut sys::vb_shuf {
        self.shuffles.entry(shuffle_id).or_insert_with(|| {
            let mut s = std::ptr::null_mut();
            check(unsafe { sys::vb_shuffle_create(self.ctx, shuffle_id as u64, n_map as u32, n_reduce as u32, sys::VB_U64,
                                                  sys::VB_U64, op.code(), sys::VB_PART_HASH_METRO64, &mut s) }).expect("vb_shuffle_create");
            if key_width == 4 { check(unsafe { sys::vb_shuffle_set_key_width(s, 4) }).unwrap(); }
            Handle(s)
        }).0
    }
    fn get(&self, shuffle_id: usize) -> *mut sys::vb_shuf { self.shuffles.get(&shuffle_id).expect("unknown shuffle").0 }
    /// called from NativeScheduler::on_event_success next to register_map_outputs (base_scheduler.rs:315)
    pub fn seal(&self, shuffle_id: usize) {
        if let Some(h) = self.shuffles.get(&shuffle_id) { let _ = check(unsafe { sys::vb_shuffle_seal(h.0) }); }
    }
    /// Distributed mode (one executor process per GPU): join the NCCL communicator with the 128-byte id the
    /// master created (`vb_comm_unique_id`) and shipped over the MapOutputTracker channel (map_output_tracker.rs:68-166).
    pub fn comm_init(&self, unique_id: &[u8; 128], rank: u32, world: u32) {
        check(unsafe { sys::vb_ctx_comm_init(self.ctx, unique_id.as_ptr() as *const c_void, rank, world) }).expect("vb_ctx_comm_init");
    }
    /// ShuffleFetcher::fetch for the whole shuffle at once (shuffle_fetcher.rs:16-119): after this executor's map tasks
    /// of `shuffle_id` are registered, swap rows with the other executors inside the library (count all-gather + one
    /// grouped ncclSend/ncclRecv, or the fused peer-memory scatter), then seal.  Collective over the executors.
    pub fn exchange_and_seal(&self, shuffle_id: usize, rank: u32, world: u32) {
        if let Some(h) = self.shuffles.get(&shuffle_id) {
            if world > 1 {
                let _ = check(unsafe { sys::vb_shuffle_set_dist(h.0, rank, world) });       // before the first map call in real code
                let _ = check(unsafe { sys::vb_shuffle_exchange(h.0, 0 /* VB_XCHG_AUTO */) });
            }
            let _ = check(unsafe { sys::vb_shuffle_seal(h.0) });
        }
    }
    /// Drop for ShuffleDependency (the reference never evicts SHUFFLE_CACHE, env.rs:27)
    pub fn free(&self, shuffle_id: usize) {
        if let Some((_, h)) = self.shuffles.remove(&shuffle_id) { unsafe { sys::vb_shuffle_free(h.0) }; }
    }
}

// 1. map side — specialises src/dependency.rs:164-229 (the crate enables `specialization`, src/lib.rs:7)
impl ShuffleDependencyTrait for ShuffleDependency<u64, u64, u64> {
    fn do_shuffle_task(&self, rdd_base: Arc<dyn RddBase>, partition: usize) -> String {
        let op = match self.aggregator.gpu_op { Some(op) => op, None => return self.do_shuffle_task_cpu(rdd_base, partition) };
        let split = rdd_base.splits()[partition].clone();
        // same iterator the CPU path drains (:185-193); Vec<(u64,u64)> already IS the AoS layout the ABI takes
        let rows: Vec<(u64, u64)> = rdd_base.iterator_any(split).unwrap()
            .map(|b| *b.into_any().downcast::<(u64, u64)>().unwrap()).collect();
        let s = GPU.shuffle(self.shuffle_id, rdd_base.number_of_splits(), self.partitioner.get_num_of_partitions(), op, 8);
        check(unsafe { sys::vb_shuffle_map_aos(s, partition as u32, rows.as_ptr() as *const c_void, rows.len() as u64, sys::VB_HOST) })
            .expect("vb_shuffle_map_aos");
        env::Env::get().shuffle_manager.get_server_uri() // unchanged return value (:228)
    }
}

// 3. reduce side — specialises src/rdd/shuffled_rdd.rs:149-170 (reduce ops: C = u64)
impl ShuffledRdd<u64, u64, u64> {
    fn compute_gpu(&self, split: Box<dyn Split>) -> Result<Box<dyn Iterator<Item = (u64, u64)>>> {
        let s = GPU.get(self.shuffle_id);
        let r = split.get_index() as u32;
        let (mut nk, mut nv) = (0u64, 0u64);
        check(unsafe { sys::vb_shuffle_reduce_size(s, r, &mut nk, &mut nv) }).map_err(Error::from)?; // blocks until sealed
        let (mut k, mut c) = (vec![0u64; nk as usize], vec![0u64; nk as usize]);
        check(unsafe { sys::vb_shuffle_reduce(s, r, k.as_mut_ptr() as *mut c_void, c.as_mut_ptr() as *mut c_void,
                                             std::ptr::null_mut(), std::ptr::null_mut(), sys::VB_HOST) }).map_err(Error::from)?;
        Ok(Box::new(k.into_iter().zip(c.into_iter())))
    }
}

//    group_by_key: C = Vec<u64>; the CSR comes back as (keys, offsets, vals)
impl ShuffledRdd<u64, u64, Vec<u64>> {
    fn compute_gpu(&self, split: Box<dyn Split>) -> Result<Box<dyn Iterator<Item = (u64, Vec<u64>)>>> {
        let s = GPU.get(self.shuffle_id);
        let r = split.get_index() as u32;
        let (mut nk, mut nv) = (0u64, 0u64);
        check(unsafe { sys::vb_shuffle_reduce_size(s, r, &mut nk, &mut nv) }).map_err(Error::from)?;
        let (mut k, mut o, mut v) = (vec![0u64; nk as usize], vec![0u64; nk as usize + 1], vec![0u64; nv as usize]);
        check(unsafe { sys::vb_shuffle_reduce(s, r, k.as_mut_ptr() as *mut c_void, std::ptr::null_mut(), o.as_mut_ptr(),
                                             v.as_mut_ptr() as *mut c_void, sys::VB_HOST) }).map_err(Error::from)?;
        let it = (0..nk as usize).map(move |i| (k[i], v[o[i] as usize..o[i + 1] as usize].to_vec()));
        Ok(Box::new(it.collect::<Vec<_>>().into_iter()))
    }
}

// 4. join — replaces CoGroupedRdd::compute + the cross product (co_grouped_rdd.rs:206-249, pair_rdd.rs:104-121)
pub fn join_partition(left_shuffle: usize, right_shuffle: usize, reduce_id: usize) -> Result<Vec<(u64, (u64, u64))>> {
    let (l, r) = (GPU.get(left_shuffle), GPU.get(right_shuffle));
    let mut n = 0u64;
    check(unsafe { sys::vb_join_size(l, r, reduce_id as u32, &mut n) }).map_err(Error::from)?;
    let (mut k, mut v, mut w) = (vec![0u64; n as usize], vec![0u64; n as usize], vec![0u64; n as usize]);
    check(unsafe { sys::vb_join(l, r, reduce_id as u32, k.as_mut_ptr() as *mut c_void, v.as_mut_ptr() as *mut c_void,
                                w.as_mut_ptr() as *mut c_void, sys::VB_HOST) }).map_err(Error::from)?;
    Ok((0..n as usize).map(|i| (k[i], (v[i], w[i]))).collect())
}

// 5. cogroup of any number of parents — replaces CoGroupedRdd::compute (co_grouped_rdd.rs:206-249); each item has the
//    shape of CoGroupedRdd::Item: (K, Vec<Vec<V>>), one list per parent in parent order
pub fn cogroup_partition(shuffles: &[usize], reduce_id: usize) -> Result<Vec<(u64, Vec<Vec<u64>>)>> {
    let sides: Vec<*mut sys::vb_shuf> = shuffles.iter().map(|&id| GPU.get(id)).collect();
    let (n, r) = (sides.len(), reduce_id as u32);
    let (mut nk, mut nv) = (0u64, vec![0u64; n]);
    check(unsafe { sys::vb_cogroup_n_size(sides.as_ptr(), n as u32, r, &mut nk, nv.as_mut_ptr()) }).map_err(Error::from)?;
    let mut k = vec![0u64; nk as usize];
    let mut offs: Vec<Vec<u64>> = (0..n).map(|_| vec![0u64; nk as usize + 1]).collect();
    let mut vals: Vec<Vec<u64>> = nv.iter().map(|&c| vec![0u64; c as usize]).collect();
    let op: Vec<*mut u64> = offs.iter_mut().map(|o| o.as_mut_ptr()).collect();
    let vp: Vec<*mut c_void> = vals.iter_mut().map(|v| v.as_mut_ptr() as *mut c_void).collect();
    check(unsafe { sys::vb_cogroup_n(sides.as_ptr(), n as u32, r, k.as_mut_ptr() as *mut c_void, op.as_ptr(), vp.as_ptr(),
                                     sys::VB_HOST) }).map_err(Error::from)?;
    Ok((0..nk as usize)
        .map(|i| (k[i], (0..n).map(|j| vals[j][offs[j][i] as usize..offs[j][i + 1] as usize].to_vec()).collect()))
        .collect())
}

//    and the inner join of all parents: (k, [v_0, ..., v_{n-1}]) per row
pub fn join_n_partition(shuffles: &[usize], reduce_id: usize) -> Result<Vec<(u64, Vec<u64>)>> {
    let sides: Vec<*mut sys::vb_shuf> = shuffles.iter().map(|&id| GPU.get(id)).collect();
    let (n, r) = (sides.len(), reduce_id as u32);
    let mut rows = 0u64;
    check(unsafe { sys::vb_join_n_size(sides.as_ptr(), n as u32, r, &mut rows) }).map_err(Error::from)?;
    let mut k = vec![0u64; rows as usize];
    let mut vals: Vec<Vec<u64>> = (0..n).map(|_| vec![0u64; rows as usize]).collect();
    let vp: Vec<*mut c_void> = vals.iter_mut().map(|v| v.as_mut_ptr() as *mut c_void).collect();
    check(unsafe { sys::vb_join_n(sides.as_ptr(), n as u32, r, k.as_mut_ptr() as *mut c_void, vp.as_ptr(), sys::VB_HOST) })
        .map_err(Error::from)?;
    Ok((0..rows as usize).map(|i| (k[i], (0..n).map(|j| vals[j][i]).collect())).collect())
}

// 2. "all map outputs registered" — src/scheduler/base_scheduler.rs:315 gains one line:
//        self.map_output_tracker.register_map_outputs(shuffle_id, locs);
//    +   crate::gpu::GPU.seal(shuffle_id);
