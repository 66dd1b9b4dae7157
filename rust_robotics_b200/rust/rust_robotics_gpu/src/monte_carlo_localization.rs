//! MonteCarloLocalizer over the GPU engine — mirrors crates/rust_robotics_localization/src/monte_carlo_localization.rs.
//! The particle count follows the KLD bound between `min_particles` and `max_particles` (mcl.rs:322-378) exactly like the
//! reference; `particle_count()` therefore changes from step to step.
use nalgebra::{DMatrix, Vector2, Vector4};
use pfgpu_sys as sys;
use rust_robotics_core::{RoboticsError, RoboticsResult, State2D, StateEstimator};

use crate::particle_filter::{PFControl, PFMeasurement, PFState, Particle};

#[derive(Debug, Clone)]
pub struct MonteCarloLocalizationConfig {                                                   // mcl.rs:50-74
    pub min_particles: usize, pub max_particles: usize, pub kld_epsilon: f64, pub kld_z: f64,
    pub range_noise: f64, pub velocity_noise: f64, pub yaw_rate_noise: f64, pub dt: f64,
}
impl Default for MonteCarloLocalizationConfig {
    fn default() -> Self {
        Self { min_particles: 100, max_particles: 5000, kld_epsilon: 0.05, kld_z: 2.326, range_noise: 0.2,
               velocity_noise: 2.0, yaw_rate_noise: 40.0_f64.to_radians(), dt: 0.1 }
    }
}
impl MonteCarloLocalizationConfig {
    fn to_c(&self) -> sys::pfgpu_pf_config {
        sys::pfgpu_pf_config { n_particles: self.min_particles as u64, resample_threshold: 0.0, range_noise: self.range_noise,
            velocity_noise: self.velocity_noise, yaw_rate_noise: self.yaw_rate_noise, dt: self.dt, mode: 1, _pad: 0,
            max_particles: self.max_particles as u64, kld_epsilon: self.kld_epsilon, kld_z: self.kld_z }
    }
    pub fn validate(&self) -> RoboticsResult<()> { status(unsafe { sys::pfgpu_pf_config_validate(&self.to_c()) }) }   // mcl.rs:87-130
}

fn status(rc: i32) -> RoboticsResult<()> {
    if rc == 0 { return Ok(()); }
    let msg = unsafe { std::ffi::CStr::from_ptr(sys::pfgpu_strerror(rc)) }.to_string_lossy().into_owned();
    Err(RoboticsError::InvalidParameter(msg))
}

pub struct MonteCarloLocalizer {
    h: *mut sys::pfgpu_pf,
    state_estimate: PFState,
    covariance_dyn: DMatrix<f64>,
    particles: Vec<Particle>,
    dirty: bool,
}
unsafe impl Send for MonteCarloLocalizer {}

impl MonteCarloLocalizer {
    pub fn try_new(config: MonteCarloLocalizationConfig) -> RoboticsResult<Self> {                  // mcl.rs:150-164
        // the reference draws from rand::rng() (mcl.rs:187,216,338): entropy, not a constant, so that independent localizers
        // (Monte-Carlo trials) are not correlated; try_new_seeded pins the Philox seed for tests
        let t = std::time::SystemTime::now().duration_since(std::time::UNIX_EPOCH).map(|d| d.as_nanos() as u64).unwrap_or(0);
        Self::try_new_seeded(config, t.wrapping_mul(0x9E37_79B9_7F4A_7C15), 0)
    }
    pub fn try_new_seeded(config: MonteCarloLocalizationConfig, seed: u64, device: i32) -> RoboticsResult<Self> {
        let mut h = std::ptr::null_mut();
        status(unsafe { sys::pfgpu_pf_create(&config.to_c(), seed, device, &mut h) })?;
        let mut s = Self { h, state_estimate: PFState::zeros(), covariance_dyn: DMatrix::zeros(4, 4), particles: vec![], dirty: true };
        s.refresh_cache()?;
        Ok(s)
    }
    pub fn new(config: MonteCarloLocalizationConfig) -> Self { Self::try_new(config).expect("invalid MCL configuration") }
    pub fn try_with_initial_state(initial_state: PFState, config: MonteCarloLocalizationConfig) -> RoboticsResult<Self> {   // mcl.rs:176-206
        let mut s = Self::try_new(config)?;
        status(unsafe { sys::pfgpu_pf_init_state(s.h, initial_state.as_ptr()) })?;
        s.refresh_cache()?;
        Ok(s)
    }
    pub fn with_initial_state(initial_state: PFState, config: MonteCarloLocalizationConfig) -> Self {
        Self::try_with_initial_state(initial_state, config).expect("invalid MCL initial state")
    }
    /// Augmented MCL (not in the reference; DESIGN §3.8): random-particle injection for global localisation and kidnapped-robot
    /// recovery.  region = [x0, x1, y0, y1]; alpha_slow = alpha_fast = 0 disables.
    pub fn enable_recovery(&mut self, alpha_slow: f64, alpha_fast: f64, region: [f64; 4]) -> RoboticsResult<()> {
        status(unsafe { sys::pfgpu_pf_recovery_enable(self.h, alpha_slow, alpha_fast, region.as_ptr()) })
    }
    /// (w_slow, w_fast, p, particles injected by the last predict)
    pub fn recovery_state(&self) -> RoboticsResult<(f64, f64, f64, u64)> {
        let (mut w, mut inj) = ([0.0f64; 3], 0u64);
        status(unsafe { sys::pfgpu_pf_recovery_state(self.h, w.as_mut_ptr(), &mut inj) })?;
        Ok((w[0], w[1], w[2], inj))
    }
    /// every particle uniform over region = [x0, x1, y0, y1], yaw uniform in [-pi, pi), v = 0, w = 1/n
    pub fn init_region(&mut self, region: [f64; 4]) -> RoboticsResult<()> {
        status(unsafe { sys::pfgpu_pf_init_region(self.h, region.as_ptr()) })?;
        self.refresh_cache()
    }
    pub fn try_with_region(region: [f64; 4], config: MonteCarloLocalizationConfig) -> RoboticsResult<Self> {
        let mut s = Self::try_new(config)?;
        s.init_region(region)?;
        Ok(s)
    }
    /// Likelihood-field scan model (not in the reference; DESIGN §3.9): obstacles[ix * height + iy], nonzero = obstacle; world
    /// (0, 0) at the grid centre.  Builds the distance field and the per-cell likelihood on the device.
    pub fn set_likelihood_field(&mut self, obstacles: &[u8], width: usize, height: usize, cfg: &sys::pfgpu_lfield_config) -> RoboticsResult<()> {
        if obstacles.len() != width * height {
            return Err(RoboticsError::InvalidParameter("likelihood field: obstacles.len() != width * height".to_string()));
        }
        status(unsafe { sys::pfgpu_pf_lfield_set(self.h, obstacles.as_ptr(), width, height, cfg) })
    }
    pub fn clear_likelihood_field(&mut self) -> RoboticsResult<()> {
        status(unsafe { sys::pfgpu_pf_lfield_clear(self.h) })
    }
    /// the measurement update from a laser scan: ranges[i] at angle_min + i * angle_increment from the heading
    pub fn try_update_with_scan(&mut self, ranges: &[f64], angle_min: f64, angle_increment: f64) -> RoboticsResult<()> {
        status(unsafe { sys::pfgpu_pf_update_scan(self.h, ranges.as_ptr(), ranges.len(), angle_min, angle_increment) })?;
        self.refresh_cache()
    }
    /// try_step with a laser scan in place of the landmark observations
    pub fn try_step_scan(&mut self, control: &PFControl, ranges: &[f64], angle_min: f64, angle_increment: f64) -> RoboticsResult<PFState> {
        let mut est = [0.0f64; 4];
        status(unsafe { sys::pfgpu_pf_step_scan(self.h, control.as_ptr(), ranges.as_ptr(), ranges.len(), angle_min, angle_increment,
                                                est.as_mut_ptr()) })?;
        self.refresh_cache()?;
        Ok(self.state_estimate)
    }
    /// Pose hypotheses (not in the reference; ROS AMCL's pose hypotheses; DESIGN §3.10): the max_count heaviest clusters of the cloud
    /// in xy_res x xy_res x (2 pi / yaw_bins) bins, heaviest first, and the total number of clusters
    pub fn hypotheses(&self, max_count: usize, xy_res: f64, yaw_bins: u32) -> RoboticsResult<(Vec<sys::pfgpu_pf_hypothesis>, usize)> {
        let mut out = vec![sys::pfgpu_pf_hypothesis { mass: 0.0, mean: [0.0; 4], cov: [0.0; 16], count: 0, bins: 0, label: 0 }; max_count];
        let mut total = 0usize;
        status(unsafe { sys::pfgpu_pf_hypotheses(self.h, xy_res, yaw_bins, out.as_mut_ptr(), max_count, &mut total, std::ptr::null_mut()) })?;
        out.truncate(total.min(max_count));
        Ok((out, total))
    }
    /// Beam scan model (not in the reference; DESIGN §3.11): the likelihood field's map conventions, a map of its own.  Every
    /// particle's expected range along every used beam is ray-cast in the map on the device and compared with the measured one.
    pub fn set_beam_model(&mut self, obstacles: &[u8], width: usize, height: usize, cfg: &sys::pfgpu_beam_config) -> RoboticsResult<()> {
        if obstacles.len() != width * height {
            return Err(RoboticsError::InvalidParameter("beam model: obstacles.len() != width * height".to_string()));
        }
        status(unsafe { sys::pfgpu_pf_beam_set(self.h, obstacles.as_ptr(), width, height, cfg) })
    }
    /// set_beam_model with the obstacle mask of an OccupancyGridMap built on the device at `threshold`; the grid is copied now
    pub fn set_beam_model_from_grid(&mut self, grid: &crate::occupancy_grid_map::OccupancyGridMap, threshold: f64,
                                    cfg: &sys::pfgpu_beam_config) -> RoboticsResult<()> {
        status(unsafe { sys::pfgpu_pf_beam_set_grid(self.h, grid.handle(), threshold, cfg) })
    }
    /// set_likelihood_field with the obstacle mask of an OccupancyGridMap built on the device at `threshold`
    pub fn set_likelihood_field_from_grid(&mut self, grid: &crate::occupancy_grid_map::OccupancyGridMap, threshold: f64,
                                          cfg: &sys::pfgpu_lfield_config) -> RoboticsResult<()> {
        status(unsafe { sys::pfgpu_pf_lfield_set_grid(self.h, grid.handle(), threshold, cfg) })
    }
    pub fn clear_beam_model(&mut self) -> RoboticsResult<()> {
        status(unsafe { sys::pfgpu_pf_beam_clear(self.h) })
    }
    /// try_update_with_scan under the beam model
    pub fn try_update_with_beam_scan(&mut self, ranges: &[f64], angle_min: f64, angle_increment: f64) -> RoboticsResult<()> {
        status(unsafe { sys::pfgpu_pf_update_beam(self.h, ranges.as_ptr(), ranges.len(), angle_min, angle_increment) })?;
        self.refresh_cache()
    }
    /// try_step with a laser scan under the beam model
    pub fn try_step_beam_scan(&mut self, control: &PFControl, ranges: &[f64], angle_min: f64, angle_increment: f64) -> RoboticsResult<PFState> {
        let mut est = [0.0f64; 4];
        status(unsafe { sys::pfgpu_pf_step_beam(self.h, control.as_ptr(), ranges.as_ptr(), ranges.len(), angle_min, angle_increment,
                                                est.as_mut_ptr()) })?;
        self.refresh_cache()?;
        Ok(self.state_estimate)
    }
    /// the odometry motion model (DESIGN §3.14): alpha = ROS AMCL's odom_alpha1..4, each finite and >= 0 (0.2 each at creation)
    pub fn set_odometry_noise(&mut self, alpha: [f64; 4]) -> RoboticsResult<()> {
        status(unsafe { sys::pfgpu_pf_set_odom_noise(self.h, alpha.as_ptr()) })
    }
    pub fn odometry_noise(&self) -> RoboticsResult<[f64; 4]> {
        let mut a = [0.0f64; 4];
        status(unsafe { sys::pfgpu_pf_odom_noise(self.h, a.as_mut_ptr()) })?;
        Ok(a)
    }
    /// move every particle by the increment from odometry pose `prev` = (x, y, yaw) to `cur` instead of by a control over dt
    pub fn try_predict_with_odometry(&mut self, prev: [f64; 3], cur: [f64; 3]) -> RoboticsResult<()> {
        let o = [prev[0], prev[1], prev[2], cur[0], cur[1], cur[2]];
        status(unsafe { sys::pfgpu_pf_predict_odom(self.h, o.as_ptr()) })?;
        self.refresh_cache()
    }
    /// try_step with the odometry motion model
    pub fn try_step_odometry(&mut self, prev: [f64; 3], cur: [f64; 3], observations: &PFMeasurement) -> RoboticsResult<PFState> {
        let o = [prev[0], prev[1], prev[2], cur[0], cur[1], cur[2]];
        let flat: Vec<f64> = observations.iter().flat_map(|&(d, x, y)| [d, x, y]).collect();
        let mut est = [0.0f64; 4];
        status(unsafe { sys::pfgpu_pf_step_odom(self.h, o.as_ptr(), flat.as_ptr(), observations.len(), est.as_mut_ptr()) })?;
        self.refresh_cache()?;
        Ok(self.state_estimate)
    }
    /// try_step_scan (likelihood field) with the odometry motion model
    pub fn try_step_scan_odometry(&mut self, prev: [f64; 3], cur: [f64; 3], ranges: &[f64], angle_min: f64, angle_increment: f64)
                                  -> RoboticsResult<PFState> {
        let o = [prev[0], prev[1], prev[2], cur[0], cur[1], cur[2]];
        let mut est = [0.0f64; 4];
        status(unsafe { sys::pfgpu_pf_step_scan_odom(self.h, o.as_ptr(), ranges.as_ptr(), ranges.len(), angle_min, angle_increment,
                                                     est.as_mut_ptr()) })?;
        self.refresh_cache()?;
        Ok(self.state_estimate)
    }
    /// try_step_beam_scan (beam model) with the odometry motion model
    pub fn try_step_beam_scan_odometry(&mut self, prev: [f64; 3], cur: [f64; 3], ranges: &[f64], angle_min: f64, angle_increment: f64)
                                       -> RoboticsResult<PFState> {
        let o = [prev[0], prev[1], prev[2], cur[0], cur[1], cur[2]];
        let mut est = [0.0f64; 4];
        status(unsafe { sys::pfgpu_pf_step_beam_odom(self.h, o.as_ptr(), ranges.as_ptr(), ranges.len(), angle_min, angle_increment,
                                                     est.as_mut_ptr()) })?;
        self.refresh_cache()?;
        Ok(self.state_estimate)
    }
    /// expected ranges of poses (x, y, yaw) x n_beams in the beam map: out[p * n_beams + b]
    pub fn expected_scan(&mut self, poses: &[[f64; 3]], n_beams: usize, angle_min: f64, angle_increment: f64) -> RoboticsResult<Vec<f64>> {
        let mut out = vec![0.0f64; poses.len() * n_beams];
        status(unsafe { sys::pfgpu_pf_beam_raycast(self.h, poses.as_ptr() as *const f64, poses.len(), n_beams, angle_min, angle_increment,
                                                   out.as_mut_ptr()) })?;
        Ok(out)
    }
    pub fn try_predict_with_control(&mut self, control: &PFControl) -> RoboticsResult<()> {          // mcl.rs:209-257
        status(unsafe { sys::pfgpu_pf_predict(self.h, control.as_ptr()) })?;
        self.refresh_cache()
    }
    pub fn try_update_with_observations(&mut self, observations: &PFMeasurement) -> RoboticsResult<()> {   // mcl.rs:260-288
        let flat: Vec<f64> = observations.iter().flat_map(|&(d, x, y)| [d, x, y]).collect();
        status(unsafe { sys::pfgpu_pf_update(self.h, flat.as_ptr(), observations.len()) })?;
        self.refresh_cache()
    }
    pub fn try_step(&mut self, control: &PFControl, observations: &PFMeasurement) -> RoboticsResult<PFState> {   // mcl.rs:291-300
        let flat: Vec<f64> = observations.iter().flat_map(|&(d, x, y)| [d, x, y]).collect();
        let mut est = [0.0f64; 4];
        status(unsafe { sys::pfgpu_pf_step(self.h, control.as_ptr(), flat.as_ptr(), observations.len(), est.as_mut_ptr()) })?;
        self.refresh_cache()?;
        Ok(self.state_estimate)
    }
    pub fn estimate(&self) -> PFState { self.state_estimate }                                          // mcl.rs:302-304
    pub fn state_2d(&self) -> State2D { let e = self.state_estimate; State2D::new(e[0], e[1], e[2], e[3]) }
    pub fn particle_count(&self) -> usize {                                                            // mcl.rs:318-320
        let (mut nl, mut ng) = (0usize, 0usize);
        let _ = unsafe { sys::pfgpu_pf_count(self.h, &mut nl, &mut ng) };
        ng
    }
    pub fn get_particles(&mut self) -> &[Particle] {
        if self.dirty {
            let n = self.particle_count();
            let mut aos = vec![0.0f64; 5 * n];
            let _ = unsafe { sys::pfgpu_pf_download(self.h, aos.as_mut_ptr(), n) };
            self.particles = aos.chunks(5).map(|c| Particle { x: c[0], y: c[1], yaw: c[2], v: c[3], w: c[4] }).collect();
            self.dirty = false;
        }
        &self.particles
    }
    fn resample(&mut self) {                                                                           // resample_adaptive mcl.rs:322-365
        let mut did = 0;
        let _ = unsafe { sys::pfgpu_pf_resample(self.h, &mut did) };
        let _ = self.refresh_cache();
    }
    fn refresh_cache(&mut self) -> RoboticsResult<()> {                                                // mcl.rs:413-447
        let (mut est, mut cov) = ([0.0f64; 4], [0.0f64; 16]);
        status(unsafe { sys::pfgpu_pf_estimate(self.h, est.as_mut_ptr(), cov.as_mut_ptr()) })?;
        self.state_estimate = PFState::from_column_slice(&est);
        self.covariance_dyn = DMatrix::from_column_slice(4, 4, &cov);
        self.dirty = true;
        Ok(())
    }
}
impl Drop for MonteCarloLocalizer { fn drop(&mut self) { unsafe { sys::pfgpu_pf_destroy(self.h) } } }

impl StateEstimator for MonteCarloLocalizer {                                                          // mcl.rs:450-471 (errors are swallowed there too)
    type State = Vector4<f64>; type Measurement = PFMeasurement; type Control = Vector2<f64>;
    fn predict(&mut self, control: &Self::Control, _dt: f64) { let _ = self.try_predict_with_control(control); }
    fn update(&mut self, measurement: &Self::Measurement) { let _ = self.try_update_with_observations(measurement); self.resample(); }
    fn get_state(&self) -> &Self::State { &self.state_estimate }
    fn get_covariance(&self) -> Option<&DMatrix<f64>> { Some(&self.covariance_dyn) }
}
