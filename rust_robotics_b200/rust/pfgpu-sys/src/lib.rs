//! pfgpu-sys — raw `extern "C"` bindings to libpfgpu.so (include/pfgpu.h).
//!
//! NOT COMPILED IN THIS REPOSITORY'S CI: the build image has no Rust toolchain (SURVEY.md Appendix C).  The same ABI
//! is exercised by the C++ mirror (rust_robotics_b200/host/) and the Python mirror (rust_robotics_b200/api.py).
//! The reference's library crates are `#![forbid(unsafe_code)]` (crates/*/src/lib.rs:1), so the `extern` block lives
//! in this separate -sys crate; `rust_robotics_gpu` wraps it behind the reference's safe API.
#![allow(non_camel_case_types)]
use std::os::raw::{c_char, c_int, c_void};

#[repr(C)]
#[derive(Clone, Copy)]
pub struct pfgpu_pf_config {
    pub n_particles: u64,
    pub resample_threshold: f64,
    pub range_noise: f64,
    pub velocity_noise: f64,
    pub yaw_rate_noise: f64,
    pub dt: f64,
    pub mode: i32,
    pub _pad: i32,
    pub max_particles: u64,
    pub kld_epsilon: f64,
    pub kld_z: f64,
}
/// pfgpu_fs_moments: weight, mean and central second moments (m2: xx xy xyaw yy yyaw yawyaw) of one handle's pose deviations
/// from the centre `c`
#[repr(C)]
#[derive(Clone, Copy, Default)]
pub struct pfgpu_fs_pose_moments { pub w: f64, pub c: [f64; 3], pub mean: [f64; 3], pub m2: [f64; 6] }
/// per landmark: weight of the copies that passed cov00 < cov00_max, their mean, sum w (P + d d^T) in (c00, c01, c10, c11) order
#[repr(C)]
#[derive(Clone, Copy, Default)]
pub struct pfgpu_fs_lm_moments { pub w: f64, pub mean: [f64; 2], pub m2: [f64; 4] }
#[repr(C)]
#[derive(Clone, Copy)]
pub struct pfgpu_fs_config {
    pub dt: f64,
    pub max_range: f64,
    pub nth: f64,
    pub q00: f64,
    pub q11: f64,
    pub r00: f64,
    pub r11: f64,
    pub init_weight: f64,
}
#[repr(C)]
#[derive(Clone, Copy)]
pub struct pfgpu_fs_obs {
    pub d: f64,
    pub angle: f64,
    pub lm_id: u64,
}
/// the likelihood-field scan model's parameters (pfgpu_pf_lfield_set; ROS AMCL's defaults 0.2, 0.95, 0.05, 30, 60)
#[repr(C)]
#[derive(Clone, Copy)]
pub struct pfgpu_lfield_config {
    pub resolution: f64,
    pub sigma_hit: f64,
    pub z_hit: f64,
    pub z_rand: f64,
    pub max_range: f64,
    pub max_beams: u32,
    pub _pad: u32,
}
/// one cluster of the particle cloud (pfgpu_pf_hypotheses): mass, mean (x, y, circular-mean yaw, v), column-major covariance
#[repr(C)]
#[derive(Clone, Copy)]
pub struct pfgpu_pf_hypothesis {
    pub mass: f64,
    pub mean: [f64; 4],
    pub cov: [f64; 16],
    pub count: u64,
    pub bins: u64,
    pub label: u64,
}
/// the beam scan model's parameters (pfgpu_pf_beam_set; ROS AMCL's defaults 0.2, 0.95, 0.1, 0.05, 0.05, 0.1, 30, 60)
#[repr(C)]
#[derive(Clone, Copy)]
pub struct pfgpu_beam_config {
    pub resolution: f64,
    pub sigma_hit: f64,
    pub z_hit: f64,
    pub z_short: f64,
    pub z_max: f64,
    pub z_rand: f64,
    pub lambda_short: f64,
    pub max_range: f64,
    pub max_beams: u32,
    pub _pad: u32,
}
/// OccupancyGridConfig (pfgpu_ogm_create; the reference's defaults 0.5, 100, 100, 0, 0.85, -0.4, 5, -5)
#[repr(C)]
#[derive(Clone, Copy)]
pub struct pfgpu_ogm_config {
    pub resolution: f64,
    pub width: u64,
    pub height: u64,
    pub prior_log_odds: f64,
    pub occupied_log_odds: f64,
    pub free_log_odds: f64,
    pub max_log_odds: f64,
    pub min_log_odds: f64,
}
/// the last pfgpu_ogm_update_scans: cell updates, chunks, the most updates of one cell in one chunk, the chunk cap
#[repr(C)]
#[derive(Clone, Copy, Default)]
pub struct pfgpu_ogm_stats {
    pub events: u64,
    pub chunks: u64,
    pub longest_run: u64,
    pub event_cap: u64,
}
pub enum pfgpu_pf {}
pub enum pfgpu_fs {}
pub enum pfgpu_ogm {}
/// grid-based FastSLAM (pfgpu_gs_create; defaults 100 particles, nth 50, 0.95, 0.05, 30, 60 beams, R = 1)
#[repr(C)]
#[derive(Clone, Copy)]
pub struct pfgpu_gs_config {
    pub ogm: pfgpu_ogm_config,
    pub n_particles: u64,
    pub nth: f64,
    pub z_hit: f64,
    pub z_rand: f64,
    pub max_range: f64,
    pub max_beams: u32,
    pub search_radius: u32,
}
/// steps so far and the last step's N_eff, resampled flag, grids copied and fuse cell updates
#[repr(C)]
#[derive(Clone, Copy, Default)]
pub struct pfgpu_gs_stats {
    pub steps: u64,
    pub neff: f64,
    pub resampled: u64,
    pub copies: u64,
    pub events: u64,
}
pub enum pfgpu_gs {}
/// grid FastSLAM's scan-matched proposal (pfgpu_gs_default_proposal: off, +-0.1 m at 0.025 m, +-0.05 rad at 0.0125 rad, lattice k = 1
/// at 0.01 m and 0.005 rad, min_hits 10)
#[repr(C)]
#[derive(Clone, Copy, Default, Debug, PartialEq)]
pub struct pfgpu_gs_proposal {
    pub enabled: u32,
    pub half_width: u32,
    pub linear_range: f64,
    pub linear_step: f64,
    pub angular_range: f64,
    pub angular_step: f64,
    pub lattice_linear_step: f64,
    pub lattice_angular_step: f64,
    pub min_hits: u32,
    pub _pad: u32,
}
/// CorrelativeScanMatcherConfig (pfgpu_csm_match; the reference's defaults 1.0, 0.2, 0.1, 0.02, 0.05)
#[repr(C)]
#[derive(Clone, Copy)]
pub struct pfgpu_csm_config {
    pub linear_search_range: f64,
    pub angular_search_range: f64,
    pub linear_step: f64,
    pub angular_step: f64,
    pub grid_resolution: f64,
}
/// ScanMatchResult with converged as 0 / 1
#[repr(C)]
#[derive(Clone, Copy, Default)]
pub struct pfgpu_csm_result {
    pub x: f64,
    pub y: f64,
    pub yaw: f64,
    pub score: f64,
    pub converged: u32,
    pub _pad: u32,
}
pub enum pfgpu_csm {}

#[link(name = "pfgpu")]
extern "C" {
    pub fn pfgpu_strerror(status: c_int) -> *const c_char;
    pub fn pfgpu_last_error() -> *const c_char;
    pub fn pfgpu_pf_config_validate(cfg: *const pfgpu_pf_config) -> c_int;
    pub fn pfgpu_pf_create(cfg: *const pfgpu_pf_config, seed: u64, device: c_int, out: *mut *mut pfgpu_pf) -> c_int;
    pub fn pfgpu_pf_create_sharded(cfg: *const pfgpu_pf_config, seed: u64, device: c_int, nccl_unique_id: *const c_void,
                                   rank: c_int, world: c_int, out: *mut *mut pfgpu_pf) -> c_int;
    pub fn pfgpu_pf_destroy(h: *mut pfgpu_pf);
    pub fn pfgpu_pf_init_state(h: *mut pfgpu_pf, init: *const f64) -> c_int;
    pub fn pfgpu_pf_upload(h: *mut pfgpu_pf, aos5: *const f64, n: usize) -> c_int;
    pub fn pfgpu_pf_download(h: *mut pfgpu_pf, aos5: *mut f64, n: usize) -> c_int;
    pub fn pfgpu_pf_count(h: *mut pfgpu_pf, n_local: *mut usize, n_global: *mut usize) -> c_int;
    pub fn pfgpu_pf_predict(h: *mut pfgpu_pf, u: *const f64) -> c_int;
    pub fn pfgpu_pf_update(h: *mut pfgpu_pf, obs3: *const f64, k: usize) -> c_int;
    pub fn pfgpu_pf_resample(h: *mut pfgpu_pf, did_resample: *mut c_int) -> c_int;
    pub fn pfgpu_pf_step(h: *mut pfgpu_pf, u: *const f64, obs3: *const f64, k: usize, est: *mut f64) -> c_int;
    pub fn pfgpu_pf_estimate(h: *mut pfgpu_pf, est: *mut f64, cov16_colmajor: *mut f64) -> c_int;
    pub fn pfgpu_pf_set_range_noise(h: *mut pfgpu_pf, range_noise: f64) -> c_int;
    pub fn pfgpu_pf_recovery_enable(h: *mut pfgpu_pf, alpha_slow: f64, alpha_fast: f64, region: *const f64) -> c_int;
    pub fn pfgpu_pf_recovery_state(h: *mut pfgpu_pf, out3: *mut f64, injected_last: *mut u64) -> c_int;
    pub fn pfgpu_pf_init_region(h: *mut pfgpu_pf, region: *const f64) -> c_int;
    pub fn pfgpu_pf_lfield_set(h: *mut pfgpu_pf, mask: *const u8, width: usize, height: usize, cfg: *const pfgpu_lfield_config) -> c_int;
    pub fn pfgpu_pf_lfield_clear(h: *mut pfgpu_pf) -> c_int;
    pub fn pfgpu_pf_lfield_info(h: *mut pfgpu_pf, width: *mut usize, height: *mut usize, max_used_beams: *mut u64) -> c_int;
    pub fn pfgpu_pf_lfield_download(h: *mut pfgpu_pf, d: *mut f64, q: *mut f64, cells: usize) -> c_int;
    pub fn pfgpu_pf_update_scan(h: *mut pfgpu_pf, ranges: *const f64, n_ranges: usize, angle_min: f64, angle_inc: f64) -> c_int;
    pub fn pfgpu_pf_step_scan(h: *mut pfgpu_pf, u: *const f64, ranges: *const f64, n_ranges: usize, angle_min: f64, angle_inc: f64,
                              est: *mut f64) -> c_int;
    pub fn pfgpu_pf_hypotheses(h: *mut pfgpu_pf, xy_res: f64, yaw_bins: u32, out: *mut pfgpu_pf_hypothesis, cap: usize,
                               n_total: *mut usize, rank_of_slot: *mut u32) -> c_int;
    pub fn pfgpu_pf_beam_set(h: *mut pfgpu_pf, mask: *const u8, width: usize, height: usize, cfg: *const pfgpu_beam_config) -> c_int;
    pub fn pfgpu_pf_beam_clear(h: *mut pfgpu_pf) -> c_int;
    pub fn pfgpu_pf_beam_info(h: *mut pfgpu_pf, width: *mut usize, height: *mut usize, max_used_beams: *mut u64) -> c_int;
    pub fn pfgpu_pf_beam_download(h: *mut pfgpu_pf, clearance: *mut u8, cells: usize) -> c_int;
    pub fn pfgpu_pf_update_beam(h: *mut pfgpu_pf, ranges: *const f64, n_ranges: usize, angle_min: f64, angle_inc: f64) -> c_int;
    pub fn pfgpu_pf_step_beam(h: *mut pfgpu_pf, u: *const f64, ranges: *const f64, n_ranges: usize, angle_min: f64, angle_inc: f64,
                              est: *mut f64) -> c_int;
    pub fn pfgpu_pf_beam_raycast(h: *mut pfgpu_pf, poses3: *const f64, n: usize, n_beams: usize, angle_min: f64, angle_inc: f64,
                                 out: *mut f64) -> c_int;
    pub fn pfgpu_pf_set_odom_noise(h: *mut pfgpu_pf, alpha: *const f64) -> c_int;
    pub fn pfgpu_pf_odom_noise(h: *mut pfgpu_pf, alpha: *mut f64) -> c_int;
    pub fn pfgpu_pf_predict_odom(h: *mut pfgpu_pf, odom: *const f64) -> c_int;
    pub fn pfgpu_pf_step_odom(h: *mut pfgpu_pf, odom: *const f64, obs3: *const f64, k: usize, est: *mut f64) -> c_int;
    pub fn pfgpu_pf_step_scan_odom(h: *mut pfgpu_pf, odom: *const f64, ranges: *const f64, n_ranges: usize, angle_min: f64, angle_inc: f64,
                                   est: *mut f64) -> c_int;
    pub fn pfgpu_pf_step_beam_odom(h: *mut pfgpu_pf, odom: *const f64, ranges: *const f64, n_ranges: usize, angle_min: f64, angle_inc: f64,
                                   est: *mut f64) -> c_int;
    pub fn pfgpu_ogm_create(cfg: *const pfgpu_ogm_config, device: c_int, out: *mut *mut pfgpu_ogm) -> c_int;
    pub fn pfgpu_ogm_destroy(h: *mut pfgpu_ogm);
    pub fn pfgpu_ogm_update_scans(h: *mut pfgpu_ogm, poses3: *const f64, n_scans: usize, ranges: *const f64, n_ranges: usize,
                                  angle_min: f64, angle_inc: f64) -> c_int;
    pub fn pfgpu_ogm_set(h: *mut pfgpu_ogm, grid: *const f64, cells: usize) -> c_int;
    pub fn pfgpu_ogm_read(h: *mut pfgpu_ogm, first: usize, count: usize, out: *mut f64) -> c_int;
    pub fn pfgpu_ogm_obstacles(h: *mut pfgpu_ogm, threshold: f64, mask_out: *mut u8, cells: usize) -> c_int;
    pub fn pfgpu_ogm_info(h: *mut pfgpu_ogm, width: *mut usize, height: *mut usize, stats: *mut pfgpu_ogm_stats) -> c_int;
    pub fn pfgpu_pf_lfield_set_grid(h: *mut pfgpu_pf, grid: *const pfgpu_ogm, threshold: f64, cfg: *const pfgpu_lfield_config) -> c_int;
    pub fn pfgpu_pf_beam_set_grid(h: *mut pfgpu_pf, grid: *const pfgpu_ogm, threshold: f64, cfg: *const pfgpu_beam_config) -> c_int;
    pub fn pfgpu_gs_default_config(cfg: *mut pfgpu_gs_config);
    pub fn pfgpu_gs_create(cfg: *const pfgpu_gs_config, seed: u64, start_pose: *const f64, device: c_int, out: *mut *mut pfgpu_gs) -> c_int;
    pub fn pfgpu_gs_destroy(h: *mut pfgpu_gs);
    pub fn pfgpu_gs_set_odom_noise(h: *mut pfgpu_gs, alpha: *const f64) -> c_int;
    pub fn pfgpu_gs_odom_noise(h: *mut pfgpu_gs, alpha: *mut f64) -> c_int;
    pub fn pfgpu_gs_step(h: *mut pfgpu_gs, odom: *const f64, ranges: *const f64, n_ranges: usize, angle_min: f64, angle_inc: f64) -> c_int;
    pub fn pfgpu_gs_download(h: *mut pfgpu_gs, poses3: *mut f64, weights: *mut f64, n: usize) -> c_int;
    pub fn pfgpu_gs_best(h: *mut pfgpu_gs, slot: *mut usize, pose3: *mut f64) -> c_int;
    pub fn pfgpu_gs_grid_read(h: *mut pfgpu_gs, slot: usize, first: usize, count: usize, out: *mut f64) -> c_int;
    pub fn pfgpu_gs_grid_to_ogm(h: *mut pfgpu_gs, slot: usize, ogm: *mut pfgpu_ogm) -> c_int;
    pub fn pfgpu_gs_last_indices(h: *mut pfgpu_gs, idx: *mut u32, cap: usize, n: *mut usize) -> c_int;
    pub fn pfgpu_gs_info(h: *mut pfgpu_gs, width: *mut usize, height: *mut usize, n: *mut usize, max_used_beams: *mut u64,
                         stats: *mut pfgpu_gs_stats) -> c_int;
    pub fn pfgpu_gs_sync(h: *mut pfgpu_gs) -> c_int;
    pub fn pfgpu_gs_default_proposal(p: *mut pfgpu_gs_proposal);
    pub fn pfgpu_gs_set_proposal(h: *mut pfgpu_gs, p: *const pfgpu_gs_proposal) -> c_int;
    pub fn pfgpu_gs_get_proposal(h: *mut pfgpu_gs, p: *mut pfgpu_gs_proposal) -> c_int;
    pub fn pfgpu_gs_last_proposal(h: *mut pfgpu_gs, matched3: *mut f64, eta: *mut f64, took: *mut u8, n: usize) -> c_int;
    pub fn pfgpu_csm_create(device: c_int, out: *mut *mut pfgpu_csm) -> c_int;
    pub fn pfgpu_csm_destroy(h: *mut pfgpu_csm);
    pub fn pfgpu_csm_set_reference(h: *mut pfgpu_csm, x: *const f64, y: *const f64, n: usize) -> c_int;
    pub fn pfgpu_csm_set_reference_grid(h: *mut pfgpu_csm, grid: *const pfgpu_ogm, threshold: f64) -> c_int;
    pub fn pfgpu_csm_reference_size(h: *mut pfgpu_csm, n: *mut usize) -> c_int;
    pub fn pfgpu_csm_match(h: *mut pfgpu_csm, cfg: *const pfgpu_csm_config, poses3: *const f64, n_queries: usize, qx: *const f64,
                           qy: *const f64, offsets: *const u64, results: *mut pfgpu_csm_result) -> c_int;
    pub fn pfgpu_csm_table_info(h: *mut pfgpu_csm, resolution: f64, origin_x: *mut i64, origin_y: *mut i64, width: *mut u64,
                                height: *mut u64, radius: *mut i32) -> c_int;
    pub fn pfgpu_csm_table_read(h: *mut pfgpu_csm, first: usize, count: usize, out: *mut f64) -> c_int;
    pub fn pfgpu_fs_default_config(cfg: *mut pfgpu_fs_config);
    pub fn pfgpu_fs_create(cfg: *const pfgpu_fs_config, n_particles: usize, n_landmarks: usize, seed: u64, device: c_int,
                           out: *mut *mut pfgpu_fs) -> c_int;
    pub fn pfgpu_fs_destroy(h: *mut pfgpu_fs);
    pub fn pfgpu_fs_upload(h: *mut pfgpu_fs, pose_w: *const f64, lm: *const f64, n: usize) -> c_int;
    pub fn pfgpu_fs_download(h: *mut pfgpu_fs, pose_w: *mut f64, lm: *mut f64, n: usize) -> c_int;
    pub fn pfgpu_fs_step(h: *mut pfgpu_fs, u: *const f64, z: *const pfgpu_fs_obs, k: usize, did_resample: *mut c_int) -> c_int;
    pub fn pfgpu_fs_best(h: *mut pfgpu_fs, index_global: *mut usize, pose_w4: *mut f64) -> c_int;
    pub fn pfgpu_fs_get_observations(h: *mut pfgpu_fs, x_true: *const f64, landmarks_xy: *const f64, n_landmarks: usize, call: u32,
                                     out: *mut pfgpu_fs_obs, k: *mut usize) -> c_int;
    pub fn pfgpu_fs_last_gate(h: *mut pfgpu_fs, did_resample: *mut c_int) -> c_int;
    pub fn pfgpu_fs_set_variant(h: *mut pfgpu_fs, variant: c_int) -> c_int;
    // FastSLAM 2.0 with unknown data association (no reference counterpart in fastslam2; ekf_slam.rs:284-308's rule per particle)
    pub fn pfgpu_fs_step_unknown(h: *mut pfgpu_fs, u: *const f64, z2: *const f64, k: usize, gate_d2: f64, did_resample: *mut c_int) -> c_int;
    pub fn pfgpu_fs_assoc_counts(h: *mut pfgpu_fs, counts: *mut u64) -> c_int;
    // FastSLAM's odometry motion model (no reference counterpart; DESIGN §3.15)
    pub fn pfgpu_fs_set_odom_noise(h: *mut pfgpu_fs, alpha: *const f64) -> c_int;
    pub fn pfgpu_fs_odom_noise(h: *mut pfgpu_fs, alpha: *mut f64) -> c_int;
    pub fn pfgpu_fs_step_odom(h: *mut pfgpu_fs, odom: *const f64, z: *const pfgpu_fs_obs, k: usize, did_resample: *mut c_int) -> c_int;
    pub fn pfgpu_fs_step_unknown_odom(h: *mut pfgpu_fs, odom: *const f64, z2: *const f64, k: usize, gate_d2: f64,
                                      did_resample: *mut c_int) -> c_int;
    pub fn pfgpu_fs_last_neff(h: *mut pfgpu_fs, neff: *mut f64) -> c_int;
    pub fn pfgpu_fs_particle_landmarks(h: *mut pfgpu_fs, index_local: usize, lm6: *mut f64) -> c_int;
    pub fn pfgpu_fs_count(h: *mut pfgpu_fs, n_local: *mut usize, n_global: *mut usize, n_landmarks: *mut usize) -> c_int;
    pub fn pfgpu_fs_sync(h: *mut pfgpu_fs) -> c_int;
    // estimate (no reference counterpart): moments per handle, then a host-only merge over the ranks in rank order
    pub fn pfgpu_fs_moments(h: *mut pfgpu_fs, cov00_max: f64, pose: *mut pfgpu_fs_pose_moments, lm: *mut pfgpu_fs_lm_moments) -> c_int;
    pub fn pfgpu_fs_estimate_merge(pose: *const pfgpu_fs_pose_moments, lm: *const *const pfgpu_fs_lm_moments, world: c_int, n_landmarks: usize,
                                   pose_mean3: *mut f64, pose_cov9_colmajor: *mut f64, lm_mass: *mut f64, lm_mean2: *mut f64,
                                   lm_cov4: *mut f64) -> c_int;
    // path history (no reference counterpart): a ring of per-step poses and resample parents, DESIGN §3.6
    pub fn pfgpu_fs_history_enable(h: *mut pfgpu_fs, capacity: usize) -> c_int;
    pub fn pfgpu_fs_history_window(h: *mut pfgpu_fs, first_step: *mut u64, last_step: *mut u64) -> c_int;
    pub fn pfgpu_fs_path(h: *mut pfgpu_fs, index_global: usize, max_steps: usize, step: *mut u64, slot: *mut u32, pose3: *mut f64,
                         n: *mut usize) -> c_int;
    pub fn pfgpu_fs_path_moments(h: *mut pfgpu_fs, max_steps: usize, step: *mut u64, out: *mut pfgpu_fs_pose_moments, n: *mut usize) -> c_int;
    // landmark existence counters for unknown data association (no reference counterpart), DESIGN §3.7
    pub fn pfgpu_fs_existence_enable(h: *mut pfgpu_fs, range: f64) -> c_int;
    pub fn pfgpu_fs_existence_counts(h: *mut pfgpu_fs, first_local: usize, count: usize, out: *mut i32) -> c_int;
    pub fn pfgpu_fs_existence_removed(h: *mut pfgpu_fs, removed: *mut u64) -> c_int;
    pub fn pfgpu_pf_sync(h: *mut pfgpu_pf) -> c_int;
    // multi-GPU: one process per GPU; rank 0 makes the id, the host program broadcasts its 128 bytes, every rank creates
    // its shard with the GLOBAL particle count (INTEGRATION.md "Multi-GPU")
    pub fn pfgpu_device_count(count: *mut c_int) -> c_int;
    pub fn pfgpu_nccl_unique_id(out128: *mut c_void) -> c_int;
    pub fn pfgpu_fs_create_sharded(cfg: *const pfgpu_fs_config, n_particles_global: usize, n_landmarks: usize, seed: u64,
                                   device: c_int, nccl_unique_id: *const c_void, rank: c_int, world: c_int,
                                   out: *mut *mut pfgpu_fs) -> c_int;
    /// all ranks inside one process (devices may repeat)
    pub fn pfgpu_fs_create_sharded_local(cfg: *const pfgpu_fs_config, n_particles_global: usize, n_landmarks: usize, seed: u64,
                                         devices: *const c_int, world: c_int, out: *mut *mut pfgpu_fs) -> c_int;
    /// 0 = one GPU, 2 = sharded over peer memory (NVLink)
    pub fn pfgpu_fs_shard_mode(h: *mut pfgpu_fs, mode: *mut c_int) -> c_int;
}
