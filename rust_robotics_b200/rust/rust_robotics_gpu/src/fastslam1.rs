//! FastSLAM 1.0 over the GPU engine — mirrors crates/rust_robotics_slam/src/fastslam1.rs.
//! The reference's functions mutate a caller-owned `Vec<Particle>`; here the particles live on the device inside
//! `FastSlam` (SURVEY.md §8b) and `download()` materialises the reference's `Vec<Particle>` when a caller wants it.
use nalgebra::{Matrix2, Matrix3, Vector2, Vector3};
use pfgpu_sys as sys;

#[derive(Clone)]
pub struct Landmark { pub x: f64, pub y: f64, pub cov: Matrix2<f64> }                  // fs1.rs:27-31
#[derive(Clone)]
pub struct Particle { pub weight: f64, pub x: f64, pub y: f64, pub yaw: f64, pub landmarks: Vec<Landmark> }   // fs1.rs:45-51

/// FastSlam::estimate (no reference counterpart; include/pfgpu.h pfgpu_fs_moments): weighted pose mean (x, y, yaw) and covariance;
/// per landmark the weight mass of the copies with cov00 < cov00_max, their weighted mean and mixture covariance (NaN at mass 0)
pub struct Estimate { pub pose: Vector3<f64>, pub pose_cov: Matrix3<f64>, pub mass: Vec<f64>, pub mean: Vec<Vector2<f64>>, pub cov: Vec<Matrix2<f64>> }

pub struct FastSlam { h: *mut sys::pfgpu_fs, n: usize, m: usize, calls: u32 }
unsafe impl Send for FastSlam {}

/// create_particles fs1.rs:302-306.  NOTE for call sites: the reference returns `Vec<Particle>` and its free functions take
/// `&mut Vec<Particle>`; here the same function names take / return the engine handle `FastSlam` (SURVEY.md §8b: the
/// alternative, upload + download around every call, is PCIe-bound).  Code that indexes the Vec calls `.download()`.
pub fn create_particles(n_particles: usize, n_landmarks: usize) -> FastSlam {
    let t = std::time::SystemTime::now().duration_since(std::time::UNIX_EPOCH).map(|d| d.as_nanos() as u64).unwrap_or(0);
    create_particles_seeded(n_particles, n_landmarks, t.wrapping_mul(0x9E37_79B9_7F4A_7C15), 0)   // the reference is unseeded (fs1.rs:129,220)
}
pub fn create_particles_seeded(n_particles: usize, n_landmarks: usize, seed: u64, device: i32) -> FastSlam {
    let mut cfg = std::mem::MaybeUninit::<sys::pfgpu_fs_config>::uninit();
    unsafe { sys::pfgpu_fs_default_config(cfg.as_mut_ptr()) };
    let mut h = std::ptr::null_mut();
    let rc = unsafe { sys::pfgpu_fs_create(cfg.as_ptr(), n_particles, n_landmarks, seed, device, &mut h) };
    assert_eq!(rc, 0, "pfgpu_fs_create failed");
    FastSlam { h, n: n_particles, m: n_landmarks, calls: 0 }
}
/// get_observations fs1.rs:277-299 on the device (Philox stream OBS; the reference draws from rand::rng())
pub fn get_observations(particles: &mut FastSlam, x_true: &nalgebra::Vector3<f64>, landmarks: &[(f64, f64)]) -> Vec<(f64, f64, usize)> {
    let flat: Vec<f64> = landmarks.iter().flat_map(|&(x, y)| [x, y]).collect();
    let mut out = vec![sys::pfgpu_fs_obs { d: 0.0, angle: 0.0, lm_id: 0 }; landmarks.len().max(1)];
    let mut k = 0usize;
    let rc = unsafe { sys::pfgpu_fs_get_observations(particles.h, x_true.as_ptr(), flat.as_ptr(), landmarks.len(), particles.calls, out.as_mut_ptr(), &mut k) };
    assert_eq!(rc, 0, "pfgpu_fs_get_observations failed");
    particles.calls += 1;
    out[..k].iter().map(|o| (o.d, o.angle, o.lm_id as usize)).collect()
}
/// fastslam_update fs1.rs:237-266
pub fn fastslam_update(particles: &mut FastSlam, u: Vector2<f64>, z: &[(f64, f64, usize)]) {
    let obs: Vec<sys::pfgpu_fs_obs> = z.iter().map(|&(d, angle, id)| sys::pfgpu_fs_obs { d, angle, lm_id: id as u64 }).collect();
    let rc = unsafe { sys::pfgpu_fs_step(particles.h, u.as_ptr(), obs.as_ptr(), obs.len(), std::ptr::null_mut()) };
    assert_eq!(rc, 0, "pfgpu_fs_step failed");       // lm_id out of range panics in the reference too (Vec index, fs1.rs:141)
}
/// The odometry motion model (not in fs1.rs; DESIGN §3.15): alpha = ROS AMCL's odom_alpha1..4, each finite and >= 0 (0.2 each at
/// creation).  Panics on a refused value, as the other wrappers here do.
pub fn set_odometry_noise(particles: &mut FastSlam, alpha: [f64; 4]) {
    let rc = unsafe { sys::pfgpu_fs_set_odom_noise(particles.h, alpha.as_ptr()) };
    assert_eq!(rc, 0, "pfgpu_fs_set_odom_noise failed");
}
/// (alpha1, alpha2, alpha3, alpha4)
pub fn odometry_noise(particles: &FastSlam) -> [f64; 4] {
    let mut a = [0.0f64; 4];
    let rc = unsafe { sys::pfgpu_fs_odom_noise(particles.h, a.as_mut_ptr()) };
    assert_eq!(rc, 0, "pfgpu_fs_odom_noise failed");
    a
}
/// fastslam_update with the odometry motion model: every particle moves by the increment from odometry pose `prev` = (x, y, yaw)
/// to `cur` instead of by a control over dt
pub fn fastslam_update_odometry(particles: &mut FastSlam, prev: [f64; 3], cur: [f64; 3], z: &[(f64, f64, usize)]) {
    let o = [prev[0], prev[1], prev[2], cur[0], cur[1], cur[2]];
    let obs: Vec<sys::pfgpu_fs_obs> = z.iter().map(|&(d, angle, id)| sys::pfgpu_fs_obs { d, angle, lm_id: id as u64 }).collect();
    let rc = unsafe { sys::pfgpu_fs_step_odom(particles.h, o.as_ptr(), obs.as_ptr(), obs.len(), std::ptr::null_mut()) };
    assert_eq!(rc, 0, "pfgpu_fs_step_odom failed");
}
/// get_best_particle fs1.rs:269-274
pub fn get_best_particle(particles: &FastSlam) -> Particle {
    let (mut idx, mut pw) = (0usize, [0.0f64; 4]);
    unsafe { sys::pfgpu_fs_best(particles.h, &mut idx, pw.as_mut_ptr()) };
    let mut lm = vec![0.0f64; 6 * particles.m];
    unsafe { sys::pfgpu_fs_particle_landmarks(particles.h, idx, lm.as_mut_ptr()) };
    Particle { weight: pw[0], x: pw[1], y: pw[2], yaw: pw[3],
               landmarks: lm.chunks(6).map(|q| Landmark { x: q[0], y: q[1], cov: Matrix2::new(q[2], q[3], q[4], q[5]) }).collect() }
}
impl FastSlam {
    pub fn len(&self) -> usize { self.n }
    /// the posterior estimate over all particles (what render_gif_slam.rs:183-191 reads from the best particle, with its
    /// `cov[(0,0)] < 100` filter as `cov00_max = 100.0`); `landmarks = false`: pose only, empty landmark vectors
    pub fn estimate(&self, cov00_max: f64, landmarks: bool) -> Estimate {
        let mut pm = sys::pfgpu_fs_pose_moments::default();
        let m = if landmarks { self.m } else { 0 };
        let mut lm = vec![sys::pfgpu_fs_lm_moments::default(); m];
        let rc = unsafe { sys::pfgpu_fs_moments(self.h, cov00_max, &mut pm, if landmarks { lm.as_mut_ptr() } else { std::ptr::null_mut() }) };
        assert_eq!(rc, 0, "pfgpu_fs_moments failed");
        let (mut mean3, mut cov9) = ([0.0f64; 3], [0.0f64; 9]);
        let (mut mass, mut mean2, mut cov4) = (vec![0.0f64; m], vec![0.0f64; 2 * m], vec![0.0f64; 4 * m]);
        let one = [lm.as_ptr()];
        let rc = unsafe { sys::pfgpu_fs_estimate_merge(&pm, if landmarks { one.as_ptr() } else { std::ptr::null() }, 1, m, mean3.as_mut_ptr(),
                                                        cov9.as_mut_ptr(), mass.as_mut_ptr(), mean2.as_mut_ptr(), cov4.as_mut_ptr()) };
        assert_eq!(rc, 0, "pfgpu_fs_estimate_merge failed");
        Estimate { pose: Vector3::from_column_slice(&mean3), pose_cov: Matrix3::from_column_slice(&cov9), mass,
                   mean: mean2.chunks(2).map(|q| Vector2::new(q[0], q[1])).collect(),
                   cov: cov4.chunks(4).map(|q| Matrix2::new(q[0], q[1], q[2], q[3])).collect() }
    }
    /// keep the last `capacity` steps of every particle's path on the device (no reference counterpart, DESIGN §3.6); 0 disables
    pub fn enable_history(&mut self, capacity: usize) {
        let rc = unsafe { sys::pfgpu_fs_history_enable(self.h, capacity) };
        assert_eq!(rc, 0, "pfgpu_fs_history_enable failed");
    }
    /// the path of global slot `index`, oldest first: (step, slot at that step, pose x y yaw) — the poses that produced the
    /// particle's map; at most `max_steps` entries
    pub fn path(&self, index: usize, max_steps: usize) -> Vec<(u64, u32, Vector3<f64>)> {
        let (mut step, mut slot, mut pose) = (vec![0u64; max_steps], vec![0u32; max_steps], vec![0.0f64; 3 * max_steps]);
        let mut n = 0usize;
        let rc = unsafe { sys::pfgpu_fs_path(self.h, index, max_steps, step.as_mut_ptr(), slot.as_mut_ptr(), pose.as_mut_ptr(), &mut n) };
        assert_eq!(rc, 0, "pfgpu_fs_path failed");
        (0..n).map(|j| (step[j], slot[j], Vector3::new(pose[3 * j], pose[3 * j + 1], pose[3 * j + 2]))).collect()
    }
    pub(crate) fn raw(&self) -> *mut sys::pfgpu_fs { self.h }
    /// the reference's Vec<Particle>, materialised (checkpoint / API-compat)
    pub fn download(&self) -> Vec<Particle> {
        let (mut pw, mut lm) = (vec![0.0f64; 4 * self.n], vec![0.0f64; 6 * self.n * self.m]);
        unsafe { sys::pfgpu_fs_download(self.h, pw.as_mut_ptr(), lm.as_mut_ptr(), self.n) };
        (0..self.n).map(|i| Particle { weight: pw[4 * i], x: pw[4 * i + 1], y: pw[4 * i + 2], yaw: pw[4 * i + 3],
            landmarks: lm[6 * self.m * i..6 * self.m * (i + 1)].chunks(6)
                .map(|q| Landmark { x: q[0], y: q[1], cov: Matrix2::new(q[2], q[3], q[4], q[5]) }).collect() }).collect()
    }
}
impl Drop for FastSlam { fn drop(&mut self) { unsafe { sys::pfgpu_fs_destroy(self.h) } } }
