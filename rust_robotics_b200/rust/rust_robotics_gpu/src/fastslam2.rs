//! FastSLAM 2.0 over the GPU engine — mirrors crates/rust_robotics_slam/src/fastslam2.rs: the same device-resident particle set
//! as `fastslam1` with `pfgpu_fs_set_variant(h, 2)`, i.e. poses sampled from the observation-informed proposal (fs2.rs:173-239)
//! and `update_landmark_and_weight` (fs2.rs:242-280).  Types and helpers are fastslam1's (the reference defines identical
//! `Landmark` / `Particle` structs in both modules, fs2.rs:33-82).
use nalgebra::Vector2;
use pfgpu_sys as sys;

pub use crate::fastslam1::{get_best_particle, get_observations, odometry_noise, set_odometry_noise, Estimate, FastSlam, Landmark, Particle};

/// create_particles fs2.rs:418-422
pub fn create_particles(n_particles: usize, n_landmarks: usize) -> FastSlam {
    let p = crate::fastslam1::create_particles(n_particles, n_landmarks);
    let rc = unsafe { sys::pfgpu_fs_set_variant(p.raw(), 2) };
    assert_eq!(rc, 0, "pfgpu_fs_set_variant failed");
    p
}
/// fastslam2_update fs2.rs:376-383
pub fn fastslam2_update(particles: &mut FastSlam, u: Vector2<f64>, z: &[(f64, f64, usize)]) {
    crate::fastslam1::fastslam_update(particles, u, z)      // the handle carries the variant
}
/// FastSLAM 2.0 with UNKNOWN data association (not in fs2.rs): `z` holds (distance, angle) pairs without landmark ids, and every
/// particle associates each one with the landmark of its own map at the smallest Mahalanobis distance below the gate
/// M_DIST_TH^2 = 16 of ekf_slam.rs:19, or adds it in its lowest empty slot (DESIGN §3.5).  Slot l is then not the same landmark
/// in every particle: read a map from one particle (`get_best_particle`).
pub fn fastslam2_update_unknown(particles: &mut FastSlam, u: Vector2<f64>, z: &[(f64, f64)]) {
    let uu = [u[0], u[1]];
    let z2: Vec<f64> = z.iter().flat_map(|&(d, a)| [d, a]).collect();
    let rc = unsafe { sys::pfgpu_fs_step_unknown(particles.raw(), uu.as_ptr(), z2.as_ptr(), z.len(), 16.0, std::ptr::null_mut()) };
    assert_eq!(rc, 0, "pfgpu_fs_step_unknown failed");
}
/// fastslam2_update with the odometry motion model (DESIGN §3.15): the proposal fuses the first observation with the prior the
/// odometry increment from `prev` to `cur` induces
pub fn fastslam2_update_odometry(particles: &mut FastSlam, prev: [f64; 3], cur: [f64; 3], z: &[(f64, f64, usize)]) {
    crate::fastslam1::fastslam_update_odometry(particles, prev, cur, z)      // the handle carries the variant
}
/// fastslam2_update_unknown with the odometry motion model
pub fn fastslam2_update_unknown_odometry(particles: &mut FastSlam, prev: [f64; 3], cur: [f64; 3], z: &[(f64, f64)]) {
    let o = [prev[0], prev[1], prev[2], cur[0], cur[1], cur[2]];
    let z2: Vec<f64> = z.iter().flat_map(|&(d, a)| [d, a]).collect();
    let rc = unsafe { sys::pfgpu_fs_step_unknown_odom(particles.raw(), o.as_ptr(), z2.as_ptr(), z.len(), 16.0, std::ptr::null_mut()) };
    assert_eq!(rc, 0, "pfgpu_fs_step_unknown_odom failed");
}
/// (matched, born, dropped) observations of the last `fastslam2_update_unknown`, summed over the particles
pub fn assoc_counts(particles: &FastSlam) -> [u64; 3] {
    let mut c = [0u64; 3];
    let rc = unsafe { sys::pfgpu_fs_assoc_counts(particles.raw(), c.as_mut_ptr()) };
    assert_eq!(rc, 0, "pfgpu_fs_assoc_counts failed");
    c
}
/// Landmark existence counters (not in fs2.rs, DESIGN §3.7): from now on every `fastslam2_update_unknown` removes landmark copies
/// that lie within `range` of their particle's pose but keep going unobserved.  `range` > 0 (inf allowed) enables, 0 disables;
/// every counter starts at 1.  While enabled `fastslam2_update` (known ids) is refused.
pub fn enable_existence(particles: &mut FastSlam, range: f64) {
    let rc = unsafe { sys::pfgpu_fs_existence_enable(particles.raw(), range) };
    assert_eq!(rc, 0, "pfgpu_fs_existence_enable failed");
}
/// the counters of particles `first .. first + count`, `count` x m particle-major; 0 for an empty slot
pub fn existence_counts(particles: &FastSlam, first: usize, count: usize) -> Vec<i32> {
    let (mut nl, mut ng, mut m) = (0usize, 0usize, 0usize);
    let rc = unsafe { sys::pfgpu_fs_count(particles.raw(), &mut nl, &mut ng, &mut m) };
    assert_eq!(rc, 0, "pfgpu_fs_count failed");
    let mut out = vec![0i32; count * m];
    let rc = unsafe { sys::pfgpu_fs_existence_counts(particles.raw(), first, count, out.as_mut_ptr()) };
    assert_eq!(rc, 0, "pfgpu_fs_existence_counts failed");
    out
}
/// landmark copies removed by the last `fastslam2_update_unknown`
pub fn removed_count(particles: &FastSlam) -> u64 {
    let mut r = 0u64;
    let rc = unsafe { sys::pfgpu_fs_existence_removed(particles.raw(), &mut r) };
    assert_eq!(rc, 0, "pfgpu_fs_existence_removed failed");
    r
}
