//! OccupancyGridMap over the GPU engine — mirrors crates/rust_robotics_mapping/src/occupancy_grid_map.rs.  The log-odds grid lives
//! on the device; scans are fused there with `update_with_scan`'s sequential result bit for bit (DESIGN §3.12), and `grid()`
//! downloads it in the reference's `grid[ix][iy]` shape.
use pfgpu_sys as sys;
use rust_robotics_core::{RoboticsError, RoboticsResult};

fn status(rc: i32) -> RoboticsResult<()> {
    if rc == 0 { return Ok(()); }
    let msg = unsafe { std::ffi::CStr::from_ptr(sys::pfgpu_strerror(rc)) }.to_string_lossy().into_owned();
    Err(RoboticsError::InvalidParameter(msg))
}

#[derive(Clone, Debug)]
pub struct OccupancyGridConfig {                                                            // occupancy_grid_map.rs:6-41
    pub resolution: f64,
    pub width: usize,
    pub height: usize,
    pub prior_log_odds: f64,
    pub occupied_log_odds: f64,
    pub free_log_odds: f64,
    pub max_log_odds: f64,
    pub min_log_odds: f64,
}
impl Default for OccupancyGridConfig {
    fn default() -> Self {
        Self { resolution: 0.5, width: 100, height: 100, prior_log_odds: 0.0, occupied_log_odds: 0.85, free_log_odds: -0.4,
               max_log_odds: 5.0, min_log_odds: -5.0 }
    }
}

pub struct OccupancyGridMap {                                                               // occupancy_grid_map.rs:43-160
    h: *mut sys::pfgpu_ogm,
    pub config: OccupancyGridConfig,
}

impl OccupancyGridMap {
    /// A grid initialised to `config.prior_log_odds` on device 0.  The reference cannot fail here; a config the device engine
    /// refuses (min_log_odds > max_log_odds, on which the reference's clamp panics, or a grid above 65536 x 65536) is an error.
    pub fn new(config: OccupancyGridConfig) -> RoboticsResult<Self> { Self::on_device(config, 0) }
    pub fn on_device(config: OccupancyGridConfig, device: i32) -> RoboticsResult<Self> {
        let c = sys::pfgpu_ogm_config { resolution: config.resolution, width: config.width as u64, height: config.height as u64,
                                        prior_log_odds: config.prior_log_odds, occupied_log_odds: config.occupied_log_odds,
                                        free_log_odds: config.free_log_odds, max_log_odds: config.max_log_odds,
                                        min_log_odds: config.min_log_odds };
        let mut h = std::ptr::null_mut();
        status(unsafe { sys::pfgpu_ogm_create(&c, device, &mut h) })?;
        Ok(Self { h, config })
    }
    pub(crate) fn handle(&self) -> *const sys::pfgpu_ogm { self.h }

    pub fn update_with_scan(&mut self, robot_x: f64, robot_y: f64, robot_yaw: f64, scan_ranges: &[f64], angle_min: f64,
                            angle_increment: f64) -> RoboticsResult<()> {
        let pose = [robot_x, robot_y, robot_yaw];
        status(unsafe { sys::pfgpu_ogm_update_scans(self.h, pose.as_ptr(), 1, scan_ranges.as_ptr(), scan_ranges.len(), angle_min,
                                                    angle_increment) })
    }
    /// S scans in order in one call: poses[s] = (x, y, yaw), scan_ranges S x n_ranges row-major
    pub fn update_with_scans(&mut self, poses: &[[f64; 3]], scan_ranges: &[f64], angle_min: f64, angle_increment: f64) -> RoboticsResult<()> {
        if poses.is_empty() { return Ok(()); }
        if scan_ranges.len() % poses.len() != 0 {
            return Err(RoboticsError::InvalidParameter("update_with_scans: scan_ranges.len() not a multiple of poses.len()".to_string()));
        }
        status(unsafe { sys::pfgpu_ogm_update_scans(self.h, poses.as_ptr() as *const f64, poses.len(), scan_ranges.as_ptr(),
                                                    scan_ranges.len() / poses.len(), angle_min, angle_increment) })
    }
    pub fn get_probability(&self, ix: usize, iy: usize) -> f64 {
        let mut l = 0.0f64;
        let rc = unsafe { sys::pfgpu_ogm_read(self.h, ix * self.config.height + iy, 1, &mut l) };
        assert!(rc == 0, "get_probability: cell ({ix}, {iy}) outside the grid");
        1.0 - 1.0 / (1.0 + l.exp())
    }
    pub fn world_to_grid(&self, x: f64, y: f64) -> Option<(usize, usize)> {
        let ix = (x / self.config.resolution + self.config.width as f64 / 2.0).floor() as i32;
        let iy = (y / self.config.resolution + self.config.height as f64 / 2.0).floor() as i32;
        if ix >= 0 && ix < self.config.width as i32 && iy >= 0 && iy < self.config.height as i32 {
            Some((ix as usize, iy as usize))
        } else {
            None
        }
    }
    pub fn is_occupied(&self, ix: usize, iy: usize, threshold: f64) -> bool { self.get_probability(ix, iy) > threshold }
    /// the log-odds grid, downloaded: grid[ix][iy]
    pub fn grid(&self) -> RoboticsResult<Vec<Vec<f64>>> {
        let (w, h) = (self.config.width, self.config.height);
        let mut flat = vec![0.0f64; w * h];
        status(unsafe { sys::pfgpu_ogm_read(self.h, 0, flat.len(), flat.as_mut_ptr()) })?;
        Ok(flat.chunks(h).map(|c| c.to_vec()).collect())
    }
    /// is_occupied of every cell, on the device: mask[ix * height + iy]
    pub fn obstacles(&self, threshold: f64) -> RoboticsResult<Vec<u8>> {
        let mut m = vec![0u8; self.config.width * self.config.height];
        status(unsafe { sys::pfgpu_ogm_obstacles(self.h, threshold, m.as_mut_ptr(), m.len()) })?;
        Ok(m)
    }
    pub fn stats(&self) -> RoboticsResult<sys::pfgpu_ogm_stats> {
        let mut s = sys::pfgpu_ogm_stats::default();
        status(unsafe { sys::pfgpu_ogm_info(self.h, std::ptr::null_mut(), std::ptr::null_mut(), &mut s) })?;
        Ok(s)
    }
}

impl Drop for OccupancyGridMap {
    fn drop(&mut self) { unsafe { sys::pfgpu_ogm_destroy(self.h) } }
}
