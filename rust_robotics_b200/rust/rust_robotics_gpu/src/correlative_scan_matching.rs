//! Correlative scan matching over the GPU engine — mirrors crates/rust_robotics_slam/src/correlative_scan_matching.rs.  Every
//! candidate pose of the window is scored on the device with the reference's result bit for bit (DESIGN §3.13).
//! `correlative_scan_match` keeps the reference's signature (it returns an error where the engine refuses an input the reference
//! accepts: non-finite values, a table or window above the caps, no device); `CorrelativeScanMatcher` keeps the reference points and
//! their lookup table on the device between calls, takes them from an OccupancyGridMap without a host round trip, and matches batches.
use pfgpu_sys as sys;
use rust_robotics_core::{RoboticsError, RoboticsResult};

fn status(rc: i32) -> RoboticsResult<()> {
    if rc == 0 { return Ok(()); }
    let msg = unsafe { std::ffi::CStr::from_ptr(sys::pfgpu_strerror(rc)) }.to_string_lossy().into_owned();
    Err(RoboticsError::InvalidParameter(msg))
}

#[derive(Debug, Clone, Copy)]
pub struct CorrelativeScanMatcherConfig {                                                   // correlative_scan_matching.rs:17-42
    pub linear_search_range: f64,
    pub angular_search_range: f64,
    pub linear_step: f64,
    pub angular_step: f64,
    pub grid_resolution: f64,
}
impl Default for CorrelativeScanMatcherConfig {
    fn default() -> Self {
        Self { linear_search_range: 1.0, angular_search_range: 0.2, linear_step: 0.1, angular_step: 0.02, grid_resolution: 0.05 }
    }
}
impl CorrelativeScanMatcherConfig {
    fn to_c(&self) -> sys::pfgpu_csm_config {
        sys::pfgpu_csm_config { linear_search_range: self.linear_search_range, angular_search_range: self.angular_search_range,
                                linear_step: self.linear_step, angular_step: self.angular_step, grid_resolution: self.grid_resolution }
    }
}

#[derive(Debug, Clone, Copy)]
pub struct ScanMatchResult {                                                                // correlative_scan_matching.rs:44-52
    pub x: f64,
    pub y: f64,
    pub yaw: f64,
    pub score: f64,
    pub converged: bool,
}
impl From<sys::pfgpu_csm_result> for ScanMatchResult {
    fn from(r: sys::pfgpu_csm_result) -> Self { Self { x: r.x, y: r.y, yaw: r.yaw, score: r.score, converged: r.converged != 0 } }
}

pub struct CorrelativeScanMatcher {
    h: *mut sys::pfgpu_csm,
}

impl CorrelativeScanMatcher {
    pub fn new() -> RoboticsResult<Self> { Self::on_device(0) }
    pub fn on_device(device: i32) -> RoboticsResult<Self> {
        let mut h = std::ptr::null_mut();
        status(unsafe { sys::pfgpu_csm_create(device, &mut h) })?;
        Ok(Self { h })
    }
    pub fn set_reference(&mut self, reference_x: &[f64], reference_y: &[f64]) -> RoboticsResult<()> {
        if reference_x.len() != reference_y.len() {
            return Err(RoboticsError::InvalidParameter("reference_x and reference_y differ in length".to_string()));
        }
        status(unsafe { sys::pfgpu_csm_set_reference(self.h, reference_x.as_ptr(), reference_y.as_ptr(), reference_x.len()) })
    }
    /// the centres of the grid's obstacle cells at `threshold`, built on the device; the grid is copied now
    pub fn set_reference_from_grid(&mut self, grid: &crate::occupancy_grid_map::OccupancyGridMap, threshold: f64) -> RoboticsResult<()> {
        status(unsafe { sys::pfgpu_csm_set_reference_grid(self.h, grid.handle(), threshold) })
    }
    pub fn match_scan(&mut self, query_x: &[f64], query_y: &[f64], initial_pose: (f64, f64, f64),
                      config: &CorrelativeScanMatcherConfig) -> RoboticsResult<ScanMatchResult> {
        if query_x.len() != query_y.len() {
            return Err(RoboticsError::InvalidParameter("query_x and query_y differ in length".to_string()));
        }
        let pose = [initial_pose.0, initial_pose.1, initial_pose.2];
        let off = [0u64, query_x.len() as u64];
        let c = config.to_c();
        let mut r = sys::pfgpu_csm_result::default();
        status(unsafe { sys::pfgpu_csm_match(self.h, &c, pose.as_ptr(), 1, query_x.as_ptr(), query_y.as_ptr(), off.as_ptr(), &mut r) })?;
        Ok(r.into())
    }
    /// Q queries in one call: poses[q] = (x, y, yaw); query q's points are query_x[k], query_y[k] for offsets[q] <= k < offsets[q + 1]
    pub fn match_batch(&mut self, poses: &[[f64; 3]], query_x: &[f64], query_y: &[f64], offsets: &[u64],
                       config: &CorrelativeScanMatcherConfig) -> RoboticsResult<Vec<ScanMatchResult>> {
        if offsets.len() != poses.len() + 1 || query_x.len() != query_y.len() || offsets.last().copied() != Some(query_x.len() as u64) {
            return Err(RoboticsError::InvalidParameter("match_batch: offsets of poses.len() + 1, ending at query_x.len()".to_string()));
        }
        let c = config.to_c();
        let mut r = vec![sys::pfgpu_csm_result::default(); poses.len()];
        status(unsafe { sys::pfgpu_csm_match(self.h, &c, poses.as_ptr() as *const f64, poses.len(), query_x.as_ptr(), query_y.as_ptr(),
                                             offsets.as_ptr(), r.as_mut_ptr()) })?;
        Ok(r.into_iter().map(ScanMatchResult::from).collect())
    }
}

impl Drop for CorrelativeScanMatcher {
    fn drop(&mut self) { unsafe { sys::pfgpu_csm_destroy(self.h) } }
}

/// correlative_scan_matching.rs:55-120 with its signature: a one-shot matcher on device 0
pub fn correlative_scan_match(reference_x: &[f64], reference_y: &[f64], query_x: &[f64], query_y: &[f64], initial_pose: (f64, f64, f64),
                              config: &CorrelativeScanMatcherConfig) -> RoboticsResult<ScanMatchResult> {
    let mut m = CorrelativeScanMatcher::new()?;
    m.set_reference(reference_x, reference_y)?;
    m.match_scan(query_x, query_y, initial_pose, config)
}
