//! ParticleFilterLocalizer over the GPU engine — mirrors crates/rust_robotics_localization/src/particle_filter.rs.
use nalgebra::{DMatrix, Matrix4, Vector2, Vector4};
use pfgpu_sys as sys;
use rust_robotics_core::{ControlInput, Obstacles, Point2D, RoboticsError, RoboticsResult, State2D, StateEstimator};
use std::cell::{Ref, RefCell};
use std::time::{SystemTime, UNIX_EPOCH};

pub type PFState = Vector4<f64>;
pub type PFControl = Vector2<f64>;
pub type PFMeasurement = Vec<(f64, f64, f64)>;

#[derive(Debug, Clone)]
pub struct Particle { pub x: f64, pub y: f64, pub yaw: f64, pub v: f64, pub w: f64 }   // pf.rs:26-32

#[derive(Debug, Clone)]
pub struct ParticleFilterConfig {                                                      // pf.rs:52-78
    pub n_particles: usize, pub resample_threshold: f64, pub range_noise: f64,
    pub velocity_noise: f64, pub yaw_rate_noise: f64, pub dt: f64,
}
impl Default for ParticleFilterConfig {
    fn default() -> Self {
        Self { n_particles: 100, resample_threshold: 0.5, range_noise: 0.2, velocity_noise: 2.0,
               yaw_rate_noise: 40.0_f64.to_radians(), dt: 0.1 }
    }
}
impl ParticleFilterConfig {
    fn to_c(&self) -> sys::pfgpu_pf_config {
        sys::pfgpu_pf_config { n_particles: self.n_particles as u64, resample_threshold: self.resample_threshold,
            range_noise: self.range_noise, velocity_noise: self.velocity_noise, yaw_rate_noise: self.yaw_rate_noise,
            dt: self.dt, mode: 0, _pad: 0, max_particles: self.n_particles as u64, kld_epsilon: 0.05, kld_z: 2.326 }
    }
    pub fn validate(&self) -> RoboticsResult<()> { status(unsafe { sys::pfgpu_pf_config_validate(&self.to_c()) }) }  // pf.rs:81-117
}

fn status(rc: i32) -> RoboticsResult<()> {
    if rc == 0 { return Ok(()); }
    let msg = unsafe { std::ffi::CStr::from_ptr(sys::pfgpu_strerror(rc)) }.to_string_lossy().into_owned();
    Err(RoboticsError::InvalidParameter(msg))            // rc > 0 (CUDA/NCCL) would map to an EstimationError variant
}

/// Seed for a new localizer.  The reference draws from the thread-local `rand::rng()` (pf.rs:177,258,443): independent
/// filters get independent noise, so the default here is entropy, not a constant; `try_new_seeded` pins it for tests.
fn entropy_seed() -> u64 {
    let t = SystemTime::now().duration_since(UNIX_EPOCH).map(|d| d.as_nanos() as u64).unwrap_or(0);
    let a = &t as *const u64 as u64;                       // stack address: differs between instances created in one tick
    (t ^ a.rotate_left(32)).wrapping_mul(0x9E37_79B9_7F4A_7C15)
}

pub struct ParticleFilterLocalizer {
    h: *mut sys::pfgpu_pf,
    config: ParticleFilterConfig,
    landmarks: Vec<Point2D>,                // stored, never read by the filter maths (pf.rs:124,218; SURVEY.md App. B.13)
    state_estimate: PFState,                // refreshed after every phase, like pf.rs:499-503
    covariance_dyn: DMatrix<f64>,
    // host mirror for get_particles(&self) -> &[Particle] (pf.rs:244): refreshed lazily behind interior mutability so the
    // reference's `&self` signature is kept
    particles: RefCell<Vec<Particle>>,
    dirty: RefCell<bool>,
}
unsafe impl Send for ParticleFilterLocalizer {}

impl ParticleFilterLocalizer {
    pub fn try_new(config: ParticleFilterConfig) -> RoboticsResult<Self> { Self::try_new_seeded(config, entropy_seed(), 0) }   // pf.rs:139-156
    /// explicit Philox seed and CUDA device (not in the reference: its RNG is not injectable)
    pub fn try_new_seeded(config: ParticleFilterConfig, seed: u64, device: i32) -> RoboticsResult<Self> {
        let mut h = std::ptr::null_mut();
        status(unsafe { sys::pfgpu_pf_create(&config.to_c(), seed, device, &mut h) })?;
        let mut s = Self { h, config, landmarks: Vec::new(), state_estimate: PFState::zeros(), covariance_dyn: DMatrix::zeros(4, 4),
                           particles: RefCell::new(Vec::new()), dirty: RefCell::new(true) };
        s.refresh_cache()?;
        Ok(s)
    }
    pub fn new(config: ParticleFilterConfig) -> Self { Self::try_new(config).expect("invalid particle filter configuration") }
    pub fn with_defaults() -> Self { Self::new(ParticleFilterConfig::default()) }                 // pf.rs:159
    pub fn with_initial_state(initial_state: PFState, config: ParticleFilterConfig) -> Self {     // pf.rs:164
        Self::try_with_initial_state(initial_state, config).expect("invalid particle filter initial state or configuration")
    }
    pub fn with_initial_state_2d(initial_state: State2D, config: ParticleFilterConfig) -> RoboticsResult<Self> {   // pf.rs:202
        Self::try_with_initial_state(initial_state.to_vector(), config)
    }
    pub fn set_landmarks(&mut self, landmarks: Vec<Point2D>) {                                    // pf.rs:210
        self.try_set_landmarks(landmarks).expect("particle filter landmarks must contain only finite values")
    }
    pub fn try_set_landmarks(&mut self, landmarks: Vec<Point2D>) -> RoboticsResult<()> {          // pf.rs:216
        if landmarks.iter().any(|p| !p.x.is_finite() || !p.y.is_finite()) {
            return Err(RoboticsError::InvalidParameter("particle filter landmarks must contain only finite values".to_string()));
        }
        self.landmarks = landmarks;
        Ok(())
    }
    pub fn set_landmarks_from_obstacles(&mut self, landmarks: &Obstacles) -> RoboticsResult<()> { self.try_set_landmarks(landmarks.points.clone()) }   // pf.rs:223
    pub fn get_landmarks(&self) -> &[Point2D] { &self.landmarks }                                  // pf.rs:239
    pub fn predict_with_control(&mut self, control: &PFControl) {                                 // pf.rs:249
        self.try_predict_with_control(control).expect("invalid particle filter prediction input")
    }
    pub fn update_with_observations(&mut self, observations: &PFMeasurement) {                    // pf.rs:304
        self.try_update_with_observations(observations).expect("invalid particle filter observations")
    }
    pub fn try_predict_input(&mut self, control: ControlInput) -> RoboticsResult<()> { self.try_predict_with_control(&control.to_vector()) }   // pf.rs:368
    pub fn try_with_initial_state(initial_state: PFState, config: ParticleFilterConfig) -> RoboticsResult<Self> {   // pf.rs:170-199
        let mut s = Self::try_new(config)?;
        status(unsafe { sys::pfgpu_pf_init_state(s.h, initial_state.as_ptr()) })?;
        s.refresh_cache()?;
        Ok(s)
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
    pub fn try_with_region(region: [f64; 4], config: ParticleFilterConfig) -> RoboticsResult<Self> {
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
    pub fn try_predict_with_control(&mut self, control: &PFControl) -> RoboticsResult<()> {      // pf.rs:255-301
        status(unsafe { sys::pfgpu_pf_predict(self.h, control.as_ptr()) })?;
        self.refresh_cache()
    }
    pub fn try_update_with_observations(&mut self, observations: &PFMeasurement) -> RoboticsResult<()> {   // pf.rs:310-334
        let flat: Vec<f64> = observations.iter().flat_map(|&(d, x, y)| [d, x, y]).collect();
        status(unsafe { sys::pfgpu_pf_update(self.h, flat.as_ptr(), observations.len()) })?;
        self.refresh_cache()
    }
    /// pf.rs:337-345.  The reference's signature returns nothing and cannot fail; a device failure here is a broken CUDA
    /// context, which is not recoverable, so it panics with the engine's message instead of being dropped.
    pub fn resample(&mut self) {
        let mut did = 0;
        status(unsafe { sys::pfgpu_pf_resample(self.h, &mut did) }).expect("particle filter resample failed on the device");
        self.refresh_cache().expect("particle filter estimate failed on the device");
    }
    pub fn try_step(&mut self, control: &PFControl, observations: &PFMeasurement) -> RoboticsResult<PFState> {   // pf.rs:488-497
        let flat: Vec<f64> = observations.iter().flat_map(|&(d, x, y)| [d, x, y]).collect();
        let mut est = [0.0f64; 4];
        status(unsafe { sys::pfgpu_pf_step(self.h, control.as_ptr(), flat.as_ptr(), observations.len(), est.as_mut_ptr()) })?;
        self.refresh_cache()?;
        Ok(self.state_estimate)
    }
    pub fn step(&mut self, control: &PFControl, observations: &PFMeasurement) -> PFState {
        self.try_step(control, observations).expect("invalid particle filter step input")
    }
    pub fn try_step_state(&mut self, control: ControlInput, observations: &PFMeasurement) -> RoboticsResult<State2D> {   // pf.rs:373-380
        self.try_step(&control.to_vector(), observations)?;
        Ok(self.state_2d())
    }
    pub fn estimate(&self) -> PFState { self.state_estimate }                                      // pf.rs:348
    pub fn state_2d(&self) -> State2D { let e = self.state_estimate; State2D::new(e[0], e[1], e[2], e[3]) }
    pub fn calc_covariance(&self) -> Matrix4<f64> { Matrix4::from_fn(|i, j| self.covariance_dyn[(i, j)]) }
    pub fn set_range_noise(&mut self, s: f64) -> RoboticsResult<()> { status(unsafe { sys::pfgpu_pf_set_range_noise(self.h, s) })?; self.config.range_noise = s; Ok(()) }
    /// pf.rs:244 with the reference's `&self`: the device state is downloaded once per phase, on demand.  The slice is
    /// handed out through `Ref::leak`-free borrowing: callers get a `Ref<[Particle]>`, which derefs to `&[Particle]` at
    /// every reference call site (`for p in pf.get_particles().iter()`, `.len()`, indexing).
    pub fn get_particles(&self) -> Ref<'_, [Particle]> {
        if *self.dirty.borrow() {
            let (mut n, mut ng) = (0usize, 0usize);
            status(unsafe { sys::pfgpu_pf_count(self.h, &mut n, &mut ng) }).expect("pfgpu_pf_count");
            let mut aos = vec![0.0f64; 5 * n];
            status(unsafe { sys::pfgpu_pf_download(self.h, aos.as_mut_ptr(), n) }).expect("pfgpu_pf_download");
            *self.particles.borrow_mut() = aos.chunks(5).map(|c| Particle { x: c[0], y: c[1], yaw: c[2], v: c[3], w: c[4] }).collect();
            *self.dirty.borrow_mut() = false;
        }
        Ref::map(self.particles.borrow(), |v| v.as_slice())
    }
    fn refresh_cache(&mut self) -> RoboticsResult<()> {
        let (mut est, mut cov) = ([0.0f64; 4], [0.0f64; 16]);
        status(unsafe { sys::pfgpu_pf_estimate(self.h, est.as_mut_ptr(), cov.as_mut_ptr()) })?;
        self.state_estimate = PFState::from_column_slice(&est);
        self.covariance_dyn = DMatrix::from_column_slice(4, 4, &cov);       // the ABI is column-major like nalgebra
        *self.dirty.borrow_mut() = true;
        Ok(())
    }
}
impl Drop for ParticleFilterLocalizer { fn drop(&mut self) { unsafe { sys::pfgpu_pf_destroy(self.h) } } }

impl StateEstimator for ParticleFilterLocalizer {                                                  // pf.rs:552-573
    type State = PFState; type Measurement = PFMeasurement; type Control = PFControl;
    fn predict(&mut self, control: &Self::Control, _dt: f64) { self.try_predict_with_control(control).expect("invalid particle filter prediction input") }
    fn update(&mut self, measurement: &Self::Measurement) { self.try_update_with_observations(measurement).expect("invalid particle filter observations"); self.resample(); }
    fn get_state(&self) -> &Self::State { &self.state_estimate }
    fn get_covariance(&self) -> Option<&DMatrix<f64>> { Some(&self.covariance_dyn) }
}
