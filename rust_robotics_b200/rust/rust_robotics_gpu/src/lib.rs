//! rust_robotics_gpu — drop-in for the hot path of rust_robotics_localization / rust_robotics_slam.
//!
//! Same type and method names as the reference (crates/rust_robotics_localization/src/particle_filter.rs,
//! crates/rust_robotics_slam/src/fastslam1.rs and fastslam2.rs); every method body is ONE call into libpfgpu.so.  A downstream crate
//! switches by changing `use rust_robotics_localization::ParticleFilterLocalizer` to
//! `use rust_robotics_gpu::ParticleFilterLocalizer`.  Build: `cargo build -p rust_robotics_gpu` with libpfgpu.so built in-tree
//! (pfgpu-sys/build.rs finds it; PFGPU_LIB_DIR overrides).  NOT COMPILED IN THIS REPOSITORY (no Rust toolchain in the build image):
//! the identical C ABI is exercised by the C++ mirror (host/, run by tests) and the Python mirror (api.py).
pub mod correlative_scan_matching;
pub mod fastslam1;
pub mod fastslam2;
pub mod grid_fastslam;
pub mod monte_carlo_localization;
pub mod occupancy_grid_map;
pub mod particle_filter;
pub use correlative_scan_matching::{correlative_scan_match, CorrelativeScanMatcher, CorrelativeScanMatcherConfig, ScanMatchResult};
pub use grid_fastslam::{GridFastSlam, GridFastSlamConfig};
pub use monte_carlo_localization::{MonteCarloLocalizationConfig, MonteCarloLocalizer};
pub use occupancy_grid_map::{OccupancyGridConfig, OccupancyGridMap};
pub use particle_filter::{ParticleFilterConfig, ParticleFilterLocalizer};
