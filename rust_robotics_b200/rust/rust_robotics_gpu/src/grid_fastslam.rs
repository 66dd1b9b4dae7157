//! Grid-based FastSLAM over the GPU engine (DESIGN §3.16; no reference counterpart): N particles, each a pose, a weight and its own
//! log-odds grid laid out as `OccupancyGridMap`'s.  `step` moves every particle by two odometry poses, weighs it by the scan's
//! endpoints against its own grid, normalises, fuses the scan into every grid and resamples when N_eff < nth, bit for bit as
//! include/pfgpu.h states.  Every method is one call into libpfgpu.so.
use crate::occupancy_grid_map::{OccupancyGridConfig, OccupancyGridMap};
use pfgpu_sys as sys;
use rust_robotics_core::{RoboticsError, RoboticsResult};

fn status(rc: i32) -> RoboticsResult<()> {
    if rc == 0 { return Ok(()); }
    let msg = unsafe { std::ffi::CStr::from_ptr(sys::pfgpu_strerror(rc)) }.to_string_lossy().into_owned();
    Err(RoboticsError::InvalidParameter(msg))
}

#[derive(Clone, Debug)]
pub struct GridFastSlamConfig {
    pub grid: OccupancyGridConfig,
    pub n_particles: usize,
    /// resample when N_eff < nth (absolute)
    pub nth: f64,
    pub z_hit: f64,
    pub z_rand: f64,
    pub max_range: f64,
    pub max_beams: u32,
    /// R: the window is (2R + 1)^2 cells
    pub search_radius: u32,
}
impl Default for GridFastSlamConfig {
    fn default() -> Self {
        Self { grid: OccupancyGridConfig::default(), n_particles: 100, nth: 50.0, z_hit: 0.95, z_rand: 0.05, max_range: 30.0, max_beams: 60,
               search_radius: 1 }
    }
}

pub struct GridFastSlam {
    h: *mut sys::pfgpu_gs,
    pub config: GridFastSlamConfig,
}

impl GridFastSlam {
    pub fn new(config: GridFastSlamConfig, start_pose: [f64; 3], seed: u64, device: i32) -> RoboticsResult<Self> {
        let g = &config.grid;
        let c = sys::pfgpu_gs_config {
            ogm: sys::pfgpu_ogm_config { resolution: g.resolution, width: g.width as u64, height: g.height as u64,
                                         prior_log_odds: g.prior_log_odds, occupied_log_odds: g.occupied_log_odds,
                                         free_log_odds: g.free_log_odds, max_log_odds: g.max_log_odds, min_log_odds: g.min_log_odds },
            n_particles: config.n_particles as u64, nth: config.nth, z_hit: config.z_hit, z_rand: config.z_rand, max_range: config.max_range,
            max_beams: config.max_beams, search_radius: config.search_radius };
        let mut h = std::ptr::null_mut();
        status(unsafe { sys::pfgpu_gs_create(&c, seed, start_pose.as_ptr(), device, &mut h) })?;
        Ok(Self { h, config })
    }
    pub fn set_odometry_noise(&mut self, alpha: [f64; 4]) -> RoboticsResult<()> { status(unsafe { sys::pfgpu_gs_set_odom_noise(self.h, alpha.as_ptr()) }) }
    pub fn odometry_noise(&self) -> [f64; 4] {
        let mut a = [0.0; 4];
        unsafe { sys::pfgpu_gs_odom_noise(self.h, a.as_mut_ptr()) };
        a
    }
    /// one step with the odometry poses before and after it and the scan taken after it; enqueued, not waited for
    pub fn step(&mut self, odom_prev: [f64; 3], odom_cur: [f64; 3], ranges: &[f64], angle_min: f64, angle_increment: f64) -> RoboticsResult<()> {
        let o = [odom_prev[0], odom_prev[1], odom_prev[2], odom_cur[0], odom_cur[1], odom_cur[2]];
        status(unsafe { sys::pfgpu_gs_step(self.h, o.as_ptr(), ranges.as_ptr(), ranges.len(), angle_min, angle_increment) })
    }
    pub fn particles(&self) -> RoboticsResult<Vec<[f64; 3]>> {
        let mut p = vec![[0.0f64; 3]; self.config.n_particles];
        status(unsafe { sys::pfgpu_gs_download(self.h, p.as_mut_ptr() as *mut f64, std::ptr::null_mut(), p.len()) })?;
        Ok(p)
    }
    pub fn weights(&self) -> RoboticsResult<Vec<f64>> {
        let mut w = vec![0.0; self.config.n_particles];
        status(unsafe { sys::pfgpu_gs_download(self.h, std::ptr::null_mut(), w.as_mut_ptr(), w.len()) })?;
        Ok(w)
    }
    /// (slot, pose) of the largest weight, ties to the lowest slot
    pub fn best(&self) -> RoboticsResult<(usize, [f64; 3])> {
        let (mut s, mut p) = (0usize, [0.0f64; 3]);
        status(unsafe { sys::pfgpu_gs_best(self.h, &mut s, p.as_mut_ptr()) })?;
        Ok((s, p))
    }
    /// slot's grid in the reference's grid[ix][iy] shape
    pub fn grid(&self, slot: usize) -> RoboticsResult<Vec<Vec<f64>>> {
        let (w, h) = (self.config.grid.width, self.config.grid.height);
        let mut flat = vec![0.0; w * h];
        status(unsafe { sys::pfgpu_gs_grid_read(self.h, slot, 0, flat.len(), flat.as_mut_ptr()) })?;
        Ok(flat.chunks(h).map(|c| c.to_vec()).collect())
    }
    /// slot's grid into an OccupancyGridMap of the same config on the same device, without leaving the device
    pub fn copy_grid_to(&self, slot: usize, map: &mut OccupancyGridMap) -> RoboticsResult<()> {
        status(unsafe { sys::pfgpu_gs_grid_to_ogm(self.h, slot, map.handle() as *mut sys::pfgpu_ogm) })
    }
    pub fn last_indices(&self) -> RoboticsResult<Vec<u32>> {
        let mut idx = vec![0u32; self.config.n_particles];
        let mut n = 0usize;
        status(unsafe { sys::pfgpu_gs_last_indices(self.h, idx.as_mut_ptr(), idx.len(), &mut n) })?;
        idx.truncate(n);
        Ok(idx)
    }
    pub fn stats(&self) -> RoboticsResult<sys::pfgpu_gs_stats> {
        let mut s = sys::pfgpu_gs_stats::default();
        status(unsafe { sys::pfgpu_gs_info(self.h, std::ptr::null_mut(), std::ptr::null_mut(), std::ptr::null_mut(), std::ptr::null_mut(), &mut s) })?;
        Ok(s)
    }
    /// the scan-matched proposal (DESIGN §3.17): `Some(p)` enables it with p's parameters (p.enabled is ignored), `None` disables
    /// it; applies from the next step
    pub fn set_proposal(&mut self, p: Option<sys::pfgpu_gs_proposal>) -> RoboticsResult<()> {
        let mut c = sys::pfgpu_gs_proposal::default();
        unsafe { sys::pfgpu_gs_default_proposal(&mut c) };
        if let Some(p) = p { c = p; c.enabled = 1; }
        status(unsafe { sys::pfgpu_gs_set_proposal(self.h, &c) })
    }
    /// the proposal in use, `None` when it is off
    pub fn proposal(&self) -> RoboticsResult<Option<sys::pfgpu_gs_proposal>> {
        let mut c = sys::pfgpu_gs_proposal::default();
        status(unsafe { sys::pfgpu_gs_get_proposal(self.h, &mut c) })?;
        Ok(if c.enabled != 0 { Some(c) } else { None })
    }
    /// the last step's per-slot match winners (x, y, yaw; NaN where no match ran), eta (NaN where no lattice ran) and whether each
    /// particle took the proposal
    pub fn last_proposal(&self) -> RoboticsResult<(Vec<[f64; 3]>, Vec<f64>, Vec<bool>)> {
        let n = self.config.n_particles;
        let (mut xh, mut eta, mut took) = (vec![0.0f64; 3 * n], vec![0.0f64; n], vec![0u8; n]);
        status(unsafe { sys::pfgpu_gs_last_proposal(self.h, xh.as_mut_ptr(), eta.as_mut_ptr(), took.as_mut_ptr(), n) })?;
        Ok((xh.chunks(3).map(|c| [c[0], c[1], c[2]]).collect(), eta, took.into_iter().map(|t| t != 0).collect()))
    }
}

impl Drop for GridFastSlam {
    fn drop(&mut self) { unsafe { sys::pfgpu_gs_destroy(self.h) } }
}
unsafe impl Send for GridFastSlam {}
