//! FastSLAM 2.0 over the GPU engine — mirrors crates/rust_robotics_slam/src/fastslam2.rs: the same device-resident particle set
//! as `fastslam1` with `pfgpu_fs_set_variant(h, 2)`, i.e. poses sampled from the observation-informed proposal (fs2.rs:173-239)
//! and `update_landmark_and_weight` (fs2.rs:242-280).  Types and helpers are fastslam1's (the reference defines identical
//! `Landmark` / `Particle` structs in both modules, fs2.rs:33-82).
use nalgebra::Vector2;
use pfgpu_sys as sys;

pub use crate::fastslam1::{get_best_particle, get_observations, Estimate, FastSlam, Landmark, Particle};

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
