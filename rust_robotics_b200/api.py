"""Python mirror of the reference's public API for the hot path, over the C ABI (include/pfgpu.h).

Names and argument meanings follow the Rust reference so the parity tests read like its own tests:
  ParticleFilterConfig / ParticleFilterLocalizer   crates/rust_robotics_localization/src/particle_filter.rs:50-573
  MonteCarloLocalizationConfig / MonteCarloLocalizer   .../monte_carlo_localization.rs:50-471
  FastSlam1 (create_particles / fastslam_update / get_best_particle)   crates/rust_robotics_slam/src/fastslam1.rs:237-306
Errors: status < 0 -> InvalidParameter (RoboticsError::InvalidParameter, rust_robotics_core/src/error.rs:8-24);
status > 0 -> PfgpuError (CUDA/NCCL).  No CPU fallback exists.
"""
import collections
import ctypes as C
import math
import os

import numpy as np

_PKG = os.path.dirname(os.path.abspath(__file__))
_LIB = None

c_dp = C.POINTER(C.c_double)
c_u32p = C.POINTER(C.c_uint32)


class InvalidParameter(ValueError):
    """RoboticsError::InvalidParameter"""


class PfgpuError(RuntimeError):
    """CUDA / NCCL failure, or no device"""


class _PfCfg(C.Structure):
    _fields_ = [("n_particles", C.c_uint64), ("resample_threshold", C.c_double), ("range_noise", C.c_double),
                ("velocity_noise", C.c_double), ("yaw_rate_noise", C.c_double), ("dt", C.c_double),
                ("mode", C.c_int32), ("_pad", C.c_int32), ("max_particles", C.c_uint64),
                ("kld_epsilon", C.c_double), ("kld_z", C.c_double)]


class _FsCfg(C.Structure):
    _fields_ = [("dt", C.c_double), ("max_range", C.c_double), ("nth", C.c_double), ("q00", C.c_double),
                ("q11", C.c_double), ("r00", C.c_double), ("r11", C.c_double), ("init_weight", C.c_double)]


class _LfCfg(C.Structure):
    _fields_ = [("resolution", C.c_double), ("sigma_hit", C.c_double), ("z_hit", C.c_double), ("z_rand", C.c_double),
                ("max_range", C.c_double), ("max_beams", C.c_uint32), ("_pad", C.c_uint32)]


class _BmCfg(C.Structure):
    _fields_ = [("resolution", C.c_double), ("sigma_hit", C.c_double), ("z_hit", C.c_double), ("z_short", C.c_double),
                ("z_max", C.c_double), ("z_rand", C.c_double), ("lambda_short", C.c_double), ("max_range", C.c_double),
                ("max_beams", C.c_uint32), ("_pad", C.c_uint32)]


class _OgmCfg(C.Structure):
    _fields_ = [("resolution", C.c_double), ("width", C.c_uint64), ("height", C.c_uint64), ("prior_log_odds", C.c_double),
                ("occupied_log_odds", C.c_double), ("free_log_odds", C.c_double), ("max_log_odds", C.c_double),
                ("min_log_odds", C.c_double)]


class _OgmStats(C.Structure):
    _fields_ = [("events", C.c_uint64), ("chunks", C.c_uint64), ("longest_run", C.c_uint64), ("event_cap", C.c_uint64)]


class _GsCfg(C.Structure):
    _fields_ = [("ogm", _OgmCfg), ("n_particles", C.c_uint64), ("nth", C.c_double), ("z_hit", C.c_double), ("z_rand", C.c_double),
                ("max_range", C.c_double), ("max_beams", C.c_uint32), ("search_radius", C.c_uint32)]


class _GsStats(C.Structure):
    _fields_ = [("steps", C.c_uint64), ("neff", C.c_double), ("resampled", C.c_uint64), ("copies", C.c_uint64), ("events", C.c_uint64)]


class _GsProp(C.Structure):
    _fields_ = [("enabled", C.c_uint32), ("half_width", C.c_uint32), ("linear_range", C.c_double), ("linear_step", C.c_double),
                ("angular_range", C.c_double), ("angular_step", C.c_double), ("lattice_linear_step", C.c_double),
                ("lattice_angular_step", C.c_double), ("min_hits", C.c_uint32), ("_pad", C.c_uint32)]


class _CsmCfg(C.Structure):
    _fields_ = [("linear_search_range", C.c_double), ("angular_search_range", C.c_double), ("linear_step", C.c_double),
                ("angular_step", C.c_double), ("grid_resolution", C.c_double)]


class _CsmResult(C.Structure):
    _fields_ = [("x", C.c_double), ("y", C.c_double), ("yaw", C.c_double), ("score", C.c_double), ("converged", C.c_uint32),
                ("_pad", C.c_uint32)]


class _Hyp(C.Structure):
    _fields_ = [("mass", C.c_double), ("mean", C.c_double * 4), ("cov", C.c_double * 16), ("count", C.c_uint64),
                ("bins", C.c_uint64), ("label", C.c_uint64)]


class _FsObs(C.Structure):
    _fields_ = [("d", C.c_double), ("angle", C.c_double), ("lm_id", C.c_uint64)]


class Stats(C.Structure):
    _fields_ = [("kernel_launches", C.c_uint64), ("steps", C.c_uint64), ("resamples", C.c_uint64),
                ("serial_fallbacks", C.c_uint64), ("xsum_dirty_last", C.c_uint64),
                ("main_kernel_ms_sum", C.c_double), ("main_kernel_count", C.c_uint64), ("compactions", C.c_uint64),
                ("imported_particles", C.c_uint64)]


class _FsPoseMoments(C.Structure):
    _fields_ = [("w", C.c_double), ("c", C.c_double * 3), ("mean", C.c_double * 3), ("m2", C.c_double * 6)]


# FastSlam1.estimate(): pose (3,) mean of (x, y, yaw), pose_cov (3, 3); per landmark (None when not asked for) mass (m,),
# mean (m, 2), cov (m, 2, 2)
FsEstimate = collections.namedtuple("FsEstimate", ["pose", "pose_cov", "mass", "mean", "cov"])
# FastSlam1.path(): steps (L,) u64, slots (L,) u32 (global slot at each step), poses (L, 3); oldest first
FsPath = collections.namedtuple("FsPath", ["steps", "slots", "poses"])
# FastSlam1.path_estimate(): steps (L,), pose (L, 3) weighted mean of the lineage poses, pose_cov (L, 3, 3); oldest first
FsPathEstimate = collections.namedtuple("FsPathEstimate", ["steps", "pose", "pose_cov"])
# _PfBase.hypotheses(): one cluster of the particle cloud: weight (its mass), count, bins, label (smallest global slot), mean (4,) =
# (x, y, circular-mean yaw, v), cov (4, 4) over (x, y, wrapped yaw deviation, v)
PfHypothesis = collections.namedtuple("PfHypothesis", ["weight", "count", "bins", "label", "mean", "cov"])


EXPORTS = [
    "pfgpu_strerror", "pfgpu_last_error", "pfgpu_device_count",
    "pfgpu_pf_default_config", "pfgpu_pf_config_validate", "pfgpu_pf_create", "pfgpu_pf_create_sharded",
    "pfgpu_pf_destroy", "pfgpu_pf_init_state", "pfgpu_pf_upload", "pfgpu_pf_download", "pfgpu_pf_count",
    "pfgpu_pf_predict", "pfgpu_pf_update", "pfgpu_pf_resample", "pfgpu_pf_step", "pfgpu_pf_estimate",
    "pfgpu_pf_neff", "pfgpu_pf_set_range_noise", "pfgpu_pf_last_indices", "pfgpu_pf_sync",
    "pfgpu_fs_default_config", "pfgpu_fs_create", "pfgpu_fs_create_sharded", "pfgpu_fs_create_sharded_local", "pfgpu_fs_destroy",
    "pfgpu_fs_upload", "pfgpu_fs_download", "pfgpu_fs_seed_map", "pfgpu_fs_step", "pfgpu_fs_best", "pfgpu_fs_particle_landmarks",
    "pfgpu_fs_get_observations", "pfgpu_fs_last_indices", "pfgpu_fs_last_neff", "pfgpu_fs_last_gate", "pfgpu_fs_set_variant", "pfgpu_fs_count", "pfgpu_fs_sync",
    "pfgpu_nccl_unique_id", "pfgpu_pf_stats", "pfgpu_fs_stats", "pfgpu_pf_time_main_kernel",
    "pfgpu_fs_time_main_kernel", "pfgpu_pf_mark", "pfgpu_pf_elapsed_ms", "pfgpu_fs_mark", "pfgpu_fs_elapsed_ms",
    "pfgpu_pf_flush_l2", "pfgpu_fs_flush_l2", "pfgpu_fs_post_trace", "pfgpu_fs_post_shape", "pfgpu_fs_post_k1", "pfgpu_fs_shard_mode",
    "pfgpu_fs_moments", "pfgpu_fs_estimate_merge", "pfgpu_fs_step_unknown", "pfgpu_fs_assoc_counts",
    "pfgpu_fs_set_odom_noise", "pfgpu_fs_odom_noise", "pfgpu_fs_step_odom", "pfgpu_fs_step_unknown_odom",
    "pfgpu_fs_history_enable", "pfgpu_fs_history_window", "pfgpu_fs_path", "pfgpu_fs_path_moments",
    "pfgpu_fs_existence_enable", "pfgpu_fs_existence_counts", "pfgpu_fs_existence_removed",
    "pfgpu_pf_recovery_enable", "pfgpu_pf_recovery_state", "pfgpu_pf_init_region",
    "pfgpu_pf_lfield_set", "pfgpu_pf_lfield_clear", "pfgpu_pf_lfield_info", "pfgpu_pf_lfield_download", "pfgpu_pf_update_scan",
    "pfgpu_pf_step_scan", "pfgpu_pf_hypotheses",
    "pfgpu_pf_beam_set", "pfgpu_pf_beam_clear", "pfgpu_pf_beam_info", "pfgpu_pf_beam_download", "pfgpu_pf_update_beam",
    "pfgpu_pf_step_beam", "pfgpu_pf_beam_raycast",
    "pfgpu_pf_set_odom_noise", "pfgpu_pf_odom_noise", "pfgpu_pf_predict_odom", "pfgpu_pf_step_odom", "pfgpu_pf_step_scan_odom",
    "pfgpu_pf_step_beam_odom",
    "pfgpu_ogm_create", "pfgpu_ogm_destroy", "pfgpu_ogm_update_scans", "pfgpu_ogm_set", "pfgpu_ogm_read", "pfgpu_ogm_obstacles",
    "pfgpu_ogm_info", "pfgpu_pf_lfield_set_grid", "pfgpu_pf_beam_set_grid",
    "pfgpu_csm_create", "pfgpu_csm_destroy", "pfgpu_csm_set_reference", "pfgpu_csm_set_reference_grid", "pfgpu_csm_reference_size",
    "pfgpu_csm_match", "pfgpu_csm_table_info", "pfgpu_csm_table_read",
    "pfgpu_gs_default_config", "pfgpu_gs_create", "pfgpu_gs_destroy", "pfgpu_gs_set_odom_noise", "pfgpu_gs_odom_noise", "pfgpu_gs_step",
    "pfgpu_gs_download", "pfgpu_gs_best", "pfgpu_gs_grid_read", "pfgpu_gs_grid_to_ogm", "pfgpu_gs_last_indices", "pfgpu_gs_info",
    "pfgpu_gs_sync", "pfgpu_gs_default_proposal", "pfgpu_gs_set_proposal", "pfgpu_gs_get_proposal", "pfgpu_gs_last_proposal",
]


def library_path():
    return os.path.join(_PKG, "libpfgpu.so")


def load_library():
    """Load libpfgpu.so (never builds; never falls back).  Raises PfgpuError if it is missing."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = library_path()
    if not os.path.exists(path):
        raise PfgpuError(f"{path} not built: run `python -c 'import __graft_entry__ as g; g.build()'`")
    L = C.CDLL(path)
    vp = C.c_void_p
    L.pfgpu_strerror.restype = C.c_char_p
    L.pfgpu_last_error.restype = C.c_char_p
    L.pfgpu_device_count.argtypes = [C.POINTER(C.c_int)]
    L.pfgpu_pf_default_config.argtypes = [C.POINTER(_PfCfg), C.c_int]
    L.pfgpu_pf_config_validate.argtypes = [C.POINTER(_PfCfg)]
    L.pfgpu_pf_create.argtypes = [C.POINTER(_PfCfg), C.c_uint64, C.c_int, C.POINTER(vp)]
    L.pfgpu_pf_create_sharded.argtypes = [C.POINTER(_PfCfg), C.c_uint64, C.c_int, vp, C.c_int, C.c_int, C.POINTER(vp)]
    L.pfgpu_pf_destroy.argtypes = [vp]
    L.pfgpu_pf_destroy.restype = None
    L.pfgpu_pf_init_state.argtypes = [vp, c_dp]
    L.pfgpu_pf_upload.argtypes = [vp, c_dp, C.c_size_t]
    L.pfgpu_pf_download.argtypes = [vp, c_dp, C.c_size_t]
    L.pfgpu_pf_count.argtypes = [vp, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    L.pfgpu_pf_predict.argtypes = [vp, c_dp]
    L.pfgpu_pf_update.argtypes = [vp, c_dp, C.c_size_t]
    L.pfgpu_pf_resample.argtypes = [vp, C.POINTER(C.c_int)]
    L.pfgpu_pf_step.argtypes = [vp, c_dp, c_dp, C.c_size_t, c_dp]
    L.pfgpu_pf_estimate.argtypes = [vp, c_dp, c_dp]
    L.pfgpu_pf_neff.argtypes = [vp, c_dp]
    L.pfgpu_pf_set_range_noise.argtypes = [vp, C.c_double]
    L.pfgpu_pf_last_indices.argtypes = [vp, c_u32p, C.c_size_t, C.POINTER(C.c_size_t)]
    L.pfgpu_pf_sync.argtypes = [vp]
    L.pfgpu_pf_recovery_enable.argtypes = [vp, C.c_double, C.c_double, c_dp]
    L.pfgpu_pf_recovery_state.argtypes = [vp, c_dp, C.POINTER(C.c_uint64)]
    L.pfgpu_pf_init_region.argtypes = [vp, c_dp]
    L.pfgpu_pf_lfield_set.argtypes = [vp, C.POINTER(C.c_uint8), C.c_size_t, C.c_size_t, C.POINTER(_LfCfg)]
    L.pfgpu_pf_lfield_clear.argtypes = [vp]
    L.pfgpu_pf_lfield_info.argtypes = [vp, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.POINTER(C.c_uint64)]
    L.pfgpu_pf_lfield_download.argtypes = [vp, c_dp, c_dp, C.c_size_t]
    L.pfgpu_pf_update_scan.argtypes = [vp, c_dp, C.c_size_t, C.c_double, C.c_double]
    L.pfgpu_pf_step_scan.argtypes = [vp, c_dp, c_dp, C.c_size_t, C.c_double, C.c_double, c_dp]
    L.pfgpu_pf_hypotheses.argtypes = [vp, C.c_double, C.c_uint32, C.POINTER(_Hyp), C.c_size_t, C.POINTER(C.c_size_t), c_u32p]
    L.pfgpu_pf_beam_set.argtypes = [vp, C.POINTER(C.c_uint8), C.c_size_t, C.c_size_t, C.POINTER(_BmCfg)]
    L.pfgpu_pf_beam_clear.argtypes = [vp]
    L.pfgpu_pf_beam_info.argtypes = [vp, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.POINTER(C.c_uint64)]
    L.pfgpu_pf_beam_download.argtypes = [vp, C.POINTER(C.c_uint8), C.c_size_t]
    L.pfgpu_pf_update_beam.argtypes = [vp, c_dp, C.c_size_t, C.c_double, C.c_double]
    L.pfgpu_pf_step_beam.argtypes = [vp, c_dp, c_dp, C.c_size_t, C.c_double, C.c_double, c_dp]
    L.pfgpu_pf_beam_raycast.argtypes = [vp, c_dp, C.c_size_t, C.c_size_t, C.c_double, C.c_double, c_dp]
    L.pfgpu_pf_set_odom_noise.argtypes = [vp, c_dp]
    L.pfgpu_pf_odom_noise.argtypes = [vp, c_dp]
    L.pfgpu_pf_predict_odom.argtypes = [vp, c_dp]
    L.pfgpu_pf_step_odom.argtypes = [vp, c_dp, c_dp, C.c_size_t, c_dp]
    L.pfgpu_pf_step_scan_odom.argtypes = [vp, c_dp, c_dp, C.c_size_t, C.c_double, C.c_double, c_dp]
    L.pfgpu_pf_step_beam_odom.argtypes = [vp, c_dp, c_dp, C.c_size_t, C.c_double, C.c_double, c_dp]
    L.pfgpu_ogm_create.argtypes = [C.POINTER(_OgmCfg), C.c_int, C.POINTER(vp)]
    L.pfgpu_ogm_destroy.argtypes = [vp]
    L.pfgpu_ogm_destroy.restype = None
    L.pfgpu_ogm_update_scans.argtypes = [vp, c_dp, C.c_size_t, c_dp, C.c_size_t, C.c_double, C.c_double]
    L.pfgpu_ogm_set.argtypes = [vp, c_dp, C.c_size_t]
    L.pfgpu_ogm_read.argtypes = [vp, C.c_size_t, C.c_size_t, c_dp]
    L.pfgpu_ogm_obstacles.argtypes = [vp, C.c_double, C.POINTER(C.c_uint8), C.c_size_t]
    L.pfgpu_ogm_info.argtypes = [vp, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.POINTER(_OgmStats)]
    L.pfgpu_pf_lfield_set_grid.argtypes = [vp, vp, C.c_double, C.POINTER(_LfCfg)]
    L.pfgpu_pf_beam_set_grid.argtypes = [vp, vp, C.c_double, C.POINTER(_BmCfg)]
    L.pfgpu_csm_create.argtypes = [C.c_int, C.POINTER(vp)]
    L.pfgpu_csm_destroy.argtypes = [vp]
    L.pfgpu_csm_destroy.restype = None
    L.pfgpu_csm_set_reference.argtypes = [vp, c_dp, c_dp, C.c_size_t]
    L.pfgpu_csm_set_reference_grid.argtypes = [vp, vp, C.c_double]
    L.pfgpu_csm_reference_size.argtypes = [vp, C.POINTER(C.c_size_t)]
    L.pfgpu_csm_match.argtypes = [vp, C.POINTER(_CsmCfg), c_dp, C.c_size_t, c_dp, c_dp, C.POINTER(C.c_uint64), C.POINTER(_CsmResult)]
    L.pfgpu_csm_table_info.argtypes = [vp, C.c_double, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_uint64),
                                       C.POINTER(C.c_uint64), C.POINTER(C.c_int32)]
    L.pfgpu_csm_table_read.argtypes = [vp, C.c_size_t, C.c_size_t, c_dp]
    L.pfgpu_fs_default_config.argtypes = [C.POINTER(_FsCfg)]
    L.pfgpu_fs_create.argtypes = [C.POINTER(_FsCfg), C.c_size_t, C.c_size_t, C.c_uint64, C.c_int, C.POINTER(vp)]
    L.pfgpu_fs_create_sharded.argtypes = [C.POINTER(_FsCfg), C.c_size_t, C.c_size_t, C.c_uint64, C.c_int, vp, C.c_int,
                                          C.c_int, C.POINTER(vp)]
    L.pfgpu_fs_create_sharded_local.argtypes = [C.POINTER(_FsCfg), C.c_size_t, C.c_size_t, C.c_uint64, C.POINTER(C.c_int), C.c_int,
                                                C.POINTER(vp)]
    L.pfgpu_fs_destroy.argtypes = [vp]
    L.pfgpu_fs_destroy.restype = None
    L.pfgpu_fs_upload.argtypes = [vp, c_dp, c_dp, C.c_size_t]
    L.pfgpu_fs_download.argtypes = [vp, c_dp, c_dp, C.c_size_t]
    L.pfgpu_fs_seed_map.argtypes = [vp, c_dp, c_dp, C.c_size_t, C.c_double, C.c_double]
    L.pfgpu_fs_step.argtypes = [vp, c_dp, C.POINTER(_FsObs), C.c_size_t, C.POINTER(C.c_int)]
    L.pfgpu_fs_best.argtypes = [vp, C.POINTER(C.c_size_t), c_dp]
    L.pfgpu_fs_particle_landmarks.argtypes = [vp, C.c_size_t, c_dp]
    L.pfgpu_fs_last_indices.argtypes = [vp, c_u32p, C.c_size_t, C.POINTER(C.c_size_t)]
    L.pfgpu_fs_last_neff.argtypes = [vp, c_dp]
    L.pfgpu_fs_last_gate.argtypes = [vp, C.POINTER(C.c_int)]
    L.pfgpu_fs_set_variant.argtypes = [vp, C.c_int]
    L.pfgpu_fs_get_observations.argtypes = [vp, c_dp, c_dp, C.c_size_t, C.c_uint32, C.POINTER(_FsObs), C.POINTER(C.c_size_t)]
    L.pfgpu_fs_count.argtypes = [vp, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    L.pfgpu_fs_sync.argtypes = [vp]
    L.pfgpu_nccl_unique_id.argtypes = [vp]
    L.pfgpu_pf_stats.argtypes = [vp, C.POINTER(Stats)]
    L.pfgpu_fs_stats.argtypes = [vp, C.POINTER(Stats)]
    L.pfgpu_pf_time_main_kernel.argtypes = [vp, C.c_int]
    L.pfgpu_fs_time_main_kernel.argtypes = [vp, C.c_int]
    for k in ("pf", "fs"):
        getattr(L, f"pfgpu_{k}_mark").argtypes = [vp, C.c_int]
        getattr(L, f"pfgpu_{k}_elapsed_ms").argtypes = [vp, C.c_int, C.c_int, c_dp]
        getattr(L, f"pfgpu_{k}_flush_l2").argtypes = [vp]
    L.pfgpu_fs_post_trace.argtypes = [vp, C.POINTER(C.c_ulonglong)]
    L.pfgpu_fs_post_shape.argtypes = [vp, C.POINTER(C.c_uint), C.POINTER(C.c_uint), C.POINTER(C.c_uint), C.POINTER(C.c_int)]
    L.pfgpu_fs_post_k1.argtypes = [vp, C.POINTER(C.c_int)]
    L.pfgpu_fs_shard_mode.argtypes = [vp, C.POINTER(C.c_int)]
    L.pfgpu_fs_moments.argtypes = [vp, C.c_double, C.POINTER(_FsPoseMoments), c_dp]
    L.pfgpu_fs_estimate_merge.argtypes = [C.POINTER(_FsPoseMoments), C.POINTER(c_dp), C.c_int, C.c_size_t, c_dp, c_dp, c_dp, c_dp, c_dp]
    L.pfgpu_fs_step_unknown.argtypes = [vp, c_dp, c_dp, C.c_size_t, C.c_double, C.POINTER(C.c_int)]
    L.pfgpu_fs_assoc_counts.argtypes = [vp, C.POINTER(C.c_uint64)]
    L.pfgpu_fs_set_odom_noise.argtypes = [vp, c_dp]
    L.pfgpu_fs_odom_noise.argtypes = [vp, c_dp]
    L.pfgpu_fs_step_odom.argtypes = [vp, c_dp, C.POINTER(_FsObs), C.c_size_t, C.POINTER(C.c_int)]
    L.pfgpu_fs_step_unknown_odom.argtypes = [vp, c_dp, c_dp, C.c_size_t, C.c_double, C.POINTER(C.c_int)]
    L.pfgpu_fs_history_enable.argtypes = [vp, C.c_size_t]
    L.pfgpu_fs_history_window.argtypes = [vp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    L.pfgpu_fs_path.argtypes = [vp, C.c_size_t, C.c_size_t, C.POINTER(C.c_uint64), c_u32p, c_dp, C.POINTER(C.c_size_t)]
    L.pfgpu_fs_path_moments.argtypes = [vp, C.c_size_t, C.POINTER(C.c_uint64), C.POINTER(_FsPoseMoments), C.POINTER(C.c_size_t)]
    L.pfgpu_fs_existence_enable.argtypes = [vp, C.c_double]
    L.pfgpu_fs_existence_counts.argtypes = [vp, C.c_size_t, C.c_size_t, C.POINTER(C.c_int32)]
    L.pfgpu_fs_existence_removed.argtypes = [vp, C.POINTER(C.c_uint64)]
    L.pfgpu_gs_default_config.argtypes, L.pfgpu_gs_default_config.restype = [C.POINTER(_GsCfg)], None
    L.pfgpu_gs_create.argtypes = [C.POINTER(_GsCfg), C.c_uint64, c_dp, C.c_int, C.POINTER(vp)]
    L.pfgpu_gs_destroy.argtypes, L.pfgpu_gs_destroy.restype = [vp], None
    L.pfgpu_gs_set_odom_noise.argtypes = [vp, c_dp]
    L.pfgpu_gs_odom_noise.argtypes = [vp, c_dp]
    L.pfgpu_gs_step.argtypes = [vp, c_dp, c_dp, C.c_size_t, C.c_double, C.c_double]
    L.pfgpu_gs_download.argtypes = [vp, c_dp, c_dp, C.c_size_t]
    L.pfgpu_gs_best.argtypes = [vp, C.POINTER(C.c_size_t), c_dp]
    L.pfgpu_gs_grid_read.argtypes = [vp, C.c_size_t, C.c_size_t, C.c_size_t, c_dp]
    L.pfgpu_gs_grid_to_ogm.argtypes = [vp, C.c_size_t, vp]
    L.pfgpu_gs_last_indices.argtypes = [vp, c_u32p, C.c_size_t, C.POINTER(C.c_size_t)]
    L.pfgpu_gs_info.argtypes = [vp, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.POINTER(C.c_uint64),
                                C.POINTER(_GsStats)]
    L.pfgpu_gs_sync.argtypes = [vp]
    L.pfgpu_gs_default_proposal.argtypes, L.pfgpu_gs_default_proposal.restype = [C.POINTER(_GsProp)], None
    L.pfgpu_gs_set_proposal.argtypes = [vp, C.POINTER(_GsProp)]
    L.pfgpu_gs_get_proposal.argtypes = [vp, C.POINTER(_GsProp)]
    L.pfgpu_gs_last_proposal.argtypes = [vp, c_dp, c_dp, C.POINTER(C.c_uint8), C.c_size_t]
    L.pfgpu_test_div.argtypes = [C.c_ulonglong, C.c_uint64, C.POINTER(C.c_ulonglong), C.c_int]
    L.pfgpu_test_xsum.argtypes = [c_dp, C.c_size_t, c_dp, c_dp, C.POINTER(C.c_int), C.c_int]
    L.pfgpu_test_pf_tail.argtypes = [vp, c_dp, C.c_size_t, c_dp, C.POINTER(C.c_int)]
    _LIB = L
    return L


def _check(L, rc):
    if rc == 0:
        return
    msg = L.pfgpu_strerror(rc).decode()
    if rc < 0:
        raise InvalidParameter(msg)
    raise PfgpuError(f"{msg}: {L.pfgpu_last_error().decode()}")


def _f64(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64))


def _dp(a):
    return a.ctypes.data_as(c_dp)


def _obstacle_mask(obstacles):
    """(pointer, W, H) of obstacles[ix, iy] != 0 as a uint8 mask (the pointer keeps the mask alive)"""
    m = np.ascontiguousarray(np.asarray(obstacles) != 0, dtype=np.uint8)
    if m.ndim != 2:
        raise InvalidParameter("obstacles: a 2-D (W, H) mask")
    return m.ctypes.data_as(C.POINTER(C.c_uint8)), m.shape[0], m.shape[1]


# ------------------------------------------------------------------------------------------------
class ParticleFilterConfig:
    """pf.rs:50-78"""

    def __init__(self, n_particles=100, resample_threshold=0.5, range_noise=0.2, velocity_noise=2.0,
                 yaw_rate_noise=math.radians(40.0), dt=0.1):
        self.n_particles, self.resample_threshold, self.range_noise = n_particles, resample_threshold, range_noise
        self.velocity_noise, self.yaw_rate_noise, self.dt = velocity_noise, yaw_rate_noise, dt

    def _c(self):
        return _PfCfg(self.n_particles, self.resample_threshold, self.range_noise, self.velocity_noise,
                      self.yaw_rate_noise, self.dt, 0, 0, self.n_particles, 0.05, 2.326)

    def validate(self):
        L = load_library()
        _check(L, L.pfgpu_pf_config_validate(C.byref(self._c())))


class MonteCarloLocalizationConfig:
    """mcl.rs:50-74"""

    def __init__(self, min_particles=100, max_particles=5000, kld_epsilon=0.05, kld_z=2.326, range_noise=0.2,
                 velocity_noise=2.0, yaw_rate_noise=math.radians(40.0), dt=0.1):
        self.min_particles, self.max_particles, self.kld_epsilon, self.kld_z = min_particles, max_particles, kld_epsilon, kld_z
        self.range_noise, self.velocity_noise, self.yaw_rate_noise, self.dt = range_noise, velocity_noise, yaw_rate_noise, dt

    def _c(self):
        return _PfCfg(self.min_particles, 0.0, self.range_noise, self.velocity_noise, self.yaw_rate_noise, self.dt,
                      1, 0, self.max_particles, self.kld_epsilon, self.kld_z)

    def validate(self):
        L = load_library()
        _check(L, L.pfgpu_pf_config_validate(C.byref(self._c())))


class _PfBase:
    def __init__(self, ccfg, seed, device, shard=None):
        self.L = load_library()
        self.h = C.c_void_p()
        if shard is None:
            _check(self.L, self.L.pfgpu_pf_create(C.byref(ccfg), seed, device, C.byref(self.h)))
        else:
            uid, rank, world = shard
            buf = C.create_string_buffer(bytes(uid), 128)
            _check(self.L, self.L.pfgpu_pf_create_sharded(C.byref(ccfg), seed, device, buf, rank, world, C.byref(self.h)))

    def close(self):
        if getattr(self, "h", None) and self.h.value:
            self.L.pfgpu_pf_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- reference API --
    def try_predict_with_control(self, control):
        u = _f64(control)
        _check(self.L, self.L.pfgpu_pf_predict(self.h, _dp(u)))

    predict_with_control = try_predict_with_control

    def try_update_with_observations(self, observations):
        o = _f64(observations).reshape(-1, 3)
        _check(self.L, self.L.pfgpu_pf_update(self.h, _dp(o), o.shape[0]))

    update_with_observations = try_update_with_observations

    def resample(self):
        did = C.c_int()
        _check(self.L, self.L.pfgpu_pf_resample(self.h, C.byref(did)))
        return bool(did.value)

    def try_step(self, control, observations, want_estimate=True):
        u = control if isinstance(control, np.ndarray) and control.dtype == np.float64 else _f64(control)
        o = _f64(observations).reshape(-1, 3)
        est = np.empty(4)
        _check(self.L, self.L.pfgpu_pf_step(self.h, _dp(u), _dp(o), o.shape[0], _dp(est) if want_estimate else None))
        return est if want_estimate else None

    step = try_step

    # -- impl StateEstimator (traits.rs:31-52; pf.rs:552-573, mcl.rs:450-471) --
    def predict(self, control, dt=None):
        """`predict(&mut self, control, _dt)`: the dt argument is ignored, the filter steps with its configured dt (pf.rs:558-560)"""
        self.try_predict_with_control(control)

    def update(self, measurement):
        """`update(&mut self, measurement)` = update_with_observations + resample (pf.rs:562-565)"""
        self.try_update_with_observations(measurement)
        self.resample()

    def get_state(self):
        return self.estimate()

    def get_covariance(self):
        return self.calc_covariance()

    def estimate(self):
        est = np.empty(4)
        _check(self.L, self.L.pfgpu_pf_estimate(self.h, _dp(est), None))
        return est

    def calc_covariance(self):
        cov = np.empty(16)
        _check(self.L, self.L.pfgpu_pf_estimate(self.h, None, _dp(cov)))
        return cov.reshape(4, 4).T        # column-major -> [i, j]

    def state_2d(self):
        return tuple(self.estimate())

    def get_particles(self):
        n = self.particle_count(local=True)
        a = np.empty((n, 5))
        _check(self.L, self.L.pfgpu_pf_download(self.h, _dp(a), n))
        return a

    def set_particles(self, aos5):
        a = _f64(aos5)
        _check(self.L, self.L.pfgpu_pf_upload(self.h, _dp(a), a.shape[0]))

    def particle_count(self, local=False):
        nl, ng = C.c_size_t(), C.c_size_t()
        _check(self.L, self.L.pfgpu_pf_count(self.h, C.byref(nl), C.byref(ng)))
        return nl.value if local else ng.value

    def set_range_noise(self, s):
        _check(self.L, self.L.pfgpu_pf_set_range_noise(self.h, float(s)))

    # -- parity / bench hooks --
    def n_eff(self):
        v = C.c_double()
        _check(self.L, self.L.pfgpu_pf_neff(self.h, C.byref(v)))
        return v.value

    def last_indices(self):
        n = self.particle_count(local=True)
        idx = np.empty(n, dtype=np.uint32)
        cnt = C.c_size_t()
        _check(self.L, self.L.pfgpu_pf_last_indices(self.h, idx.ctypes.data_as(c_u32p), n, C.byref(cnt)))
        return idx[:cnt.value]

    def sync(self):
        _check(self.L, self.L.pfgpu_pf_sync(self.h))

    def stats(self):
        s = Stats()
        _check(self.L, self.L.pfgpu_pf_stats(self.h, C.byref(s)))
        return s

    def time_main_kernel(self, on=True):
        _check(self.L, self.L.pfgpu_pf_time_main_kernel(self.h, int(on)))

    def mark(self, slot):
        _check(self.L, self.L.pfgpu_pf_mark(self.h, slot))

    def elapsed_ms(self, a, b):
        v = C.c_double()
        _check(self.L, self.L.pfgpu_pf_elapsed_ms(self.h, a, b, C.byref(v)))
        return v.value

    def flush_l2(self):
        _check(self.L, self.L.pfgpu_pf_flush_l2(self.h))

    # -- augmented MCL (not in the reference, whose cloud only copies particles it has; DESIGN §3.8) --
    def enable_recovery(self, alpha_slow=0.001, alpha_fast=0.1, region=None):
        """Random-particle injection for global localisation and kidnapped-robot recovery (Probabilistic Robotics Table 8.3; ROS
        AMCL's recovery_alpha_slow / recovery_alpha_fast).  The filter tracks short- and long-term averages of the mean likelihood;
        when the short one falls below the long one, the first predict after a resample replaces each particle with probability
        p = max(0, 1 - w_fast / w_slow) by a pose drawn uniformly over region = (x0, x1, y0, y1).  alpha_slow = alpha_fast = 0
        disables.  Resets w_slow = w_fast = 0 (so do set_particles, init_state and init_region).  On a sharded engine every rank
        makes the same call."""
        reg = _f64(region) if region is not None else None
        if reg is not None and reg.size != 4:
            raise InvalidParameter("region = (x0, x1, y0, y1)")
        _check(self.L, self.L.pfgpu_pf_recovery_enable(self.h, float(alpha_slow), float(alpha_fast), _dp(reg) if reg is not None else None))

    def disable_recovery(self):
        self.enable_recovery(0.0, 0.0, None)

    def recovery_state(self):
        """(w_slow, w_fast, p, injected): the averages, the injection probability of the next armed predict, and the particles
        this handle's last predict injected.  Synchronises."""
        out, inj = np.empty(3), C.c_uint64()
        _check(self.L, self.L.pfgpu_pf_recovery_state(self.h, _dp(out), C.byref(inj)))
        return float(out[0]), float(out[1]), float(out[2]), int(inj.value)

    def init_region(self, region):
        """global initialisation: every particle uniform over region = (x0, x1, y0, y1), yaw uniform in [-pi, pi), v = 0, w = 1/n"""
        reg = _f64(region)
        if reg.size != 4:
            raise InvalidParameter("region = (x0, x1, y0, y1)")
        _check(self.L, self.L.pfgpu_pf_init_region(self.h, _dp(reg)))

    @classmethod
    def try_with_region(cls, region, config, **kw):
        """a filter that does not know where it is: init_region(region) instead of try_with_initial_state's +-1 m cloud"""
        f = cls(config, **kw)
        f.init_region(region)
        return f

    # -- what the two scan models share: fn is the model's C entry point --
    def _set_map(self, fn, source, cfg_type, resolution, *params, max_beams):
        """load a map from source = _obstacle_mask(...) or (grid handle, threshold) with the config (resolution, *params, max_beams)"""
        if not (max_beams >= 2 and max_beams < 2 ** 32):
            raise InvalidParameter("max_beams >= 2")
        cfg = cfg_type(float(resolution), *(float(v) for v in params), int(max_beams), 0)
        _check(self.L, fn(self.h, *source, C.byref(cfg)))

    def _update_scan(self, fn, ranges, angle_min, angle_increment):
        r = _f64(ranges).ravel()
        _check(self.L, fn(self.h, _dp(r), r.size, float(angle_min), float(angle_increment)))

    def _step_scan(self, fn, control, ranges, angle_min, angle_increment, want_estimate):
        u = control if isinstance(control, np.ndarray) and control.dtype == np.float64 else _f64(control)
        r = _f64(ranges).ravel()
        est = np.empty(4)
        _check(self.L, fn(self.h, _dp(u), _dp(r), r.size, float(angle_min), float(angle_increment), _dp(est) if want_estimate else None))
        return est if want_estimate else None

    # -- likelihood-field scan model (not in the reference, whose MCL only ranges to known landmarks; DESIGN §3.9) --
    def set_likelihood_field(self, obstacles, resolution, sigma_hit=0.2, z_hit=0.95, z_rand=0.05, max_range=30.0, max_beams=60):
        """Load an occupancy map for scan updates: obstacles[ix, iy] (W x H, nonzero = obstacle; obstacles_from_log_odds turns an
        OccupancyGridMap's log-odds into one), `resolution` metres per cell, world (0, 0) at the grid centre.  Builds the distance
        field and the per-cell likelihood q = z_hit * N(d; 0, sigma_hit) + z_rand / max_range on the device (ROS AMCL's
        likelihood_field with its defaults).  On a sharded engine every rank makes the same call."""
        self._set_map(self.L.pfgpu_pf_lfield_set, _obstacle_mask(obstacles), _LfCfg, resolution, sigma_hit, z_hit, z_rand, max_range,
                      max_beams=max_beams)

    def clear_likelihood_field(self):
        _check(self.L, self.L.pfgpu_pf_lfield_clear(self.h))

    def likelihood_field_info(self):
        """(W, H, L): the map's shape and the most beams a scan may use (0, 0, 0 without a map)"""
        W, H, L = C.c_size_t(), C.c_size_t(), C.c_uint64()
        _check(self.L, self.L.pfgpu_pf_lfield_info(self.h, C.byref(W), C.byref(H), C.byref(L)))
        return W.value, H.value, L.value

    def likelihood_field(self):
        """(D, q, L): the distance field in cells and the per-cell likelihood, both (W, H) f64, and the beam limit"""
        W, H, L = self.likelihood_field_info()
        if not W:
            raise InvalidParameter("no likelihood field loaded")
        D, q = np.empty((W, H)), np.empty((W, H))
        _check(self.L, self.L.pfgpu_pf_lfield_download(self.h, _dp(D), _dp(q), W * H))
        return D, q, L

    def try_update_with_scan(self, ranges, angle_min, angle_increment):
        """The measurement update from a laser scan (ranges[i] at angle_min + i * angle_increment from the heading; the
        convention of OccupancyGridMap::update_with_scan): every particle's weight becomes the likelihood field of the used beams"""
        self._update_scan(self.L.pfgpu_pf_update_scan, ranges, angle_min, angle_increment)

    update_with_scan = try_update_with_scan

    def try_step_scan(self, control, ranges, angle_min, angle_increment, want_estimate=True):
        """try_step with a laser scan in place of the landmark observations"""
        return self._step_scan(self.L.pfgpu_pf_step_scan, control, ranges, angle_min, angle_increment, want_estimate)

    step_scan = try_step_scan

    # -- beam scan model (not in the reference; Probabilistic Robotics Table 6.1, ROS AMCL's beam model; DESIGN §3.11) --
    def set_beam_model(self, obstacles, resolution, sigma_hit=0.2, z_hit=0.95, z_short=0.1, z_max=0.05, z_rand=0.05, lambda_short=0.1,
                       max_range=30.0, max_beams=60):
        """Load an occupancy map for beam-model scan updates (the likelihood field's conventions: obstacles[ix, iy], W x H, nonzero =
        obstacle, `resolution` metres per cell, world (0, 0) at the grid centre).  Every particle's expected range along every used
        beam is ray-cast in the map and compared with the measured one (ROS AMCL's beam model with its defaults).  Builds the
        clearance table on the device.  Separate from the likelihood field; on a sharded engine every rank makes the same call."""
        self._set_map(self.L.pfgpu_pf_beam_set, _obstacle_mask(obstacles), _BmCfg, resolution, sigma_hit, z_hit, z_short, z_max, z_rand,
                      lambda_short, max_range, max_beams=max_beams)

    def set_likelihood_field_from_grid(self, grid_map, threshold=0.5, sigma_hit=0.2, z_hit=0.95, z_rand=0.05, max_range=30.0,
                                       max_beams=60):
        """set_likelihood_field(grid_map.obstacles(threshold), grid_map.config.resolution, ...) without leaving the device: the
        OccupancyGridMap's obstacle mask is built on the device and the same table is loaded.  The grid is copied now: later
        updates of grid_map do not change the loaded field.  grid_map must live on this filter's device."""
        self._set_map(self.L.pfgpu_pf_lfield_set_grid, (grid_map.h, float(threshold)), _LfCfg, grid_map.config.resolution, sigma_hit, z_hit,
                      z_rand, max_range, max_beams=max_beams)

    def set_beam_model_from_grid(self, grid_map, threshold=0.5, sigma_hit=0.2, z_hit=0.95, z_short=0.1, z_max=0.05, z_rand=0.05,
                                 lambda_short=0.1, max_range=30.0, max_beams=60):
        """set_beam_model(grid_map.obstacles(threshold), grid_map.config.resolution, ...) without leaving the device (see
        set_likelihood_field_from_grid)"""
        self._set_map(self.L.pfgpu_pf_beam_set_grid, (grid_map.h, float(threshold)), _BmCfg, grid_map.config.resolution, sigma_hit, z_hit,
                      z_short, z_max, z_rand, lambda_short, max_range, max_beams=max_beams)

    def clear_beam_model(self):
        _check(self.L, self.L.pfgpu_pf_beam_clear(self.h))

    def beam_model_info(self):
        """(W, H, L): the beam map's shape and the most beams a scan may use (0, 0, 0 without one)"""
        W, H, L = C.c_size_t(), C.c_size_t(), C.c_uint64()
        _check(self.L, self.L.pfgpu_pf_beam_info(self.h, C.byref(W), C.byref(H), C.byref(L)))
        return W.value, H.value, L.value

    def beam_model(self):
        """the clearance table, (W, H) uint8: Chebyshev distance in cells to the nearest occupied or outside cell, capped at 255"""
        W, H, _ = self.beam_model_info()
        if not W:
            raise InvalidParameter("no beam model loaded")
        out = np.empty((W, H), dtype=np.uint8)
        _check(self.L, self.L.pfgpu_pf_beam_download(self.h, out.ctypes.data_as(C.POINTER(C.c_uint8)), W * H))
        return out

    def try_update_with_beam_scan(self, ranges, angle_min, angle_increment):
        """try_update_with_scan under the beam model"""
        self._update_scan(self.L.pfgpu_pf_update_beam, ranges, angle_min, angle_increment)

    update_with_beam_scan = try_update_with_beam_scan

    def try_step_beam_scan(self, control, ranges, angle_min, angle_increment, want_estimate=True):
        """try_step with a laser scan under the beam model"""
        return self._step_scan(self.L.pfgpu_pf_step_beam, control, ranges, angle_min, angle_increment, want_estimate)

    step_beam_scan = try_step_beam_scan

    def expected_scan(self, poses, n_beams, angle_min, angle_increment):
        """(n, n_beams) expected ranges of poses (n, 3) = (x, y, yaw) in the beam map, ray-cast on the device: beam b at
        (yaw + angle_min) + b * angle_increment; 0 from a pose in an obstacle or outside the grid, max_range when nothing is hit"""
        p = np.ascontiguousarray(_f64(poses).reshape(-1, 3))
        B = int(n_beams)
        if B < 0:
            raise InvalidParameter("n_beams >= 0")
        out = np.empty((p.shape[0], B))
        _check(self.L, self.L.pfgpu_pf_beam_raycast(self.h, _dp(p), p.shape[0], B, float(angle_min), float(angle_increment), _dp(out)))
        return out

    # -- pose hypotheses (not in the reference; ROS AMCL's pose hypotheses; DESIGN §3.10) --
    # -- odometry motion model (not in the reference, whose filters only have the velocity model; DESIGN §3.14) --
    def set_odometry_noise(self, alpha1=0.2, alpha2=0.2, alpha3=0.2, alpha4=0.2):
        """ROS AMCL's odom_alpha1..4 (diff-corrected): rotation noise from rotation, rotation noise from translation, translation
        noise from translation, translation noise from rotation.  Each finite and >= 0; a filter starts at 0.2 each."""
        a = _f64([alpha1, alpha2, alpha3, alpha4])
        _check(self.L, self.L.pfgpu_pf_set_odom_noise(self.h, _dp(a)))

    def odometry_noise(self):
        """(alpha1, alpha2, alpha3, alpha4)"""
        a = np.empty(4)
        _check(self.L, self.L.pfgpu_pf_odom_noise(self.h, _dp(a)))
        return tuple(float(v) for v in a)

    @staticmethod
    def _odom_pair(odom_prev, odom_cur):
        o = np.concatenate([_f64(odom_prev).ravel(), _f64(odom_cur).ravel()])
        if o.size != 6:
            raise InvalidParameter("odometry poses are (x, y, yaw)")
        return o

    def try_predict_with_odometry(self, odom_prev, odom_cur):
        """move every particle by the increment from odometry pose odom_prev = (x, y, yaw) to odom_cur (Probabilistic Robotics
        Table 5.6, include/pf_odom_math.h) instead of by a control over dt; v is left as it was"""
        o = self._odom_pair(odom_prev, odom_cur)
        _check(self.L, self.L.pfgpu_pf_predict_odom(self.h, _dp(o)))

    def try_step_odometry(self, odom_prev, odom_cur, observations, want_estimate=True):
        """try_step with the odometry motion model: predict_with_odometry, update with the landmark ranges, resample"""
        o = self._odom_pair(odom_prev, odom_cur)
        obs = _f64(observations).reshape(-1, 3)
        est = np.empty(4)
        _check(self.L, self.L.pfgpu_pf_step_odom(self.h, _dp(o), _dp(obs), obs.shape[0], _dp(est) if want_estimate else None))
        return est if want_estimate else None

    def try_step_scan_odometry(self, odom_prev, odom_cur, ranges, angle_min, angle_increment, want_estimate=True):
        """try_step_scan (likelihood field) with the odometry motion model"""
        return self._step_scan(self.L.pfgpu_pf_step_scan_odom, self._odom_pair(odom_prev, odom_cur), ranges, angle_min, angle_increment,
                               want_estimate)

    def try_step_beam_scan_odometry(self, odom_prev, odom_cur, ranges, angle_min, angle_increment, want_estimate=True):
        """try_step_beam_scan (beam model) with the odometry motion model"""
        return self._step_scan(self.L.pfgpu_pf_step_beam_odom, self._odom_pair(odom_prev, odom_cur), ranges, angle_min, angle_increment,
                               want_estimate)

    def hypotheses(self, max_count=16, xy_res=0.5, yaw_bins=24, labels=False):
        """The particle cloud clustered in a fixed histogram of xy_res x xy_res x (2 pi / yaw_bins) bins (26-connected, cyclic in yaw):
        ([PfHypothesis] of the max_count heaviest clusters, heaviest first, total number of clusters), and with labels=True also an
        int64 rank per local particle (-1: not a member: a non-finite pose or a weight not in (0, inf)).  The set estimate() describes;
        the same bits on every call.  Synchronises; on a sharded engine every rank makes the same call and gets the same clusters."""
        if not (max_count >= 0 and yaw_bins >= 0 and yaw_bins < 2 ** 32):
            raise InvalidParameter("max_count >= 0, 0 < yaw_bins <= 65536")
        out = (_Hyp * max(int(max_count), 1))()
        total = C.c_size_t()
        rk = np.empty(self.particle_count(local=True), dtype=np.uint32) if labels else None
        _check(self.L, self.L.pfgpu_pf_hypotheses(self.h, float(xy_res), int(yaw_bins), out, int(max_count), C.byref(total),
                                                  rk.ctypes.data_as(c_u32p) if labels else None))
        hs = [PfHypothesis(out[i].mass, int(out[i].count), int(out[i].bins), int(out[i].label), np.array(out[i].mean[:]),
                           np.array(out[i].cov[:]).reshape(4, 4).T) for i in range(min(int(max_count), total.value))]
        if not labels:
            return hs, total.value
        r = rk.astype(np.int64)
        r[rk == 0xFFFFFFFF] = -1
        return hs, total.value, r


def obstacles_from_log_odds(grid, threshold=0.5):
    """Obstacle mask of an occupancy grid of log-odds l (OccupancyGridMap's grid[ix][iy], rust_robotics_mapping/src/
    occupancy_grid_map.rs): is_occupied's rule 1 - 1 / (1 + exp(l)) > threshold (:136-159), on the host"""
    g = np.asarray(grid, dtype=np.float64)
    with np.errstate(over="ignore"):
        return (1.0 - 1.0 / (1.0 + np.exp(g))) > threshold


# ------------------------------------------------------------------------------------------------
class OccupancyGridConfig:
    """occupancy_grid_map.rs:6-41"""

    def __init__(self, resolution=0.5, width=100, height=100, prior_log_odds=0.0, occupied_log_odds=0.85, free_log_odds=-0.4,
                 max_log_odds=5.0, min_log_odds=-5.0):
        self.resolution, self.width, self.height = resolution, width, height
        self.prior_log_odds, self.occupied_log_odds, self.free_log_odds = prior_log_odds, occupied_log_odds, free_log_odds
        self.max_log_odds, self.min_log_odds = max_log_odds, min_log_odds

    def _c(self):
        if not (0 <= int(self.width) < 2 ** 64 and 0 <= int(self.height) < 2 ** 64):
            raise InvalidParameter("width, height: 1 .. 65536")
        return _OgmCfg(float(self.resolution), int(self.width), int(self.height), float(self.prior_log_odds), float(self.occupied_log_odds),
                       float(self.free_log_odds), float(self.max_log_odds), float(self.min_log_odds))


# OccupancyGridMap.stats(): the last update's cell updates, the chunks it ran in, the most updates one cell took in one chunk, and
# the events a chunk holds at most
OgmStats = collections.namedtuple("OgmStats", ["events", "chunks", "longest_run", "event_cap"])


class OccupancyGridMap:
    """occupancy_grid_map.rs:43-160 on the device (DESIGN §3.12): a W x H log-odds grid, grid[ix, iy], world (0, 0) at the grid centre.
    Scans are fused on the device with update_with_scan's sequential result bit for bit; the grid stays there until read."""

    def __init__(self, config=None, device=0):
        self.config = config or OccupancyGridConfig()
        self.L = load_library()
        self.h = C.c_void_p()
        self.device = device
        _check(self.L, self.L.pfgpu_ogm_create(C.byref(self.config._c()), device, C.byref(self.h)))
        self.W, self.H = int(self.config.width), int(self.config.height)

    @classmethod
    def new(cls, config, **kw):
        return cls(config, **kw)

    def close(self):
        if getattr(self, "h", None) and self.h.value:
            self.L.pfgpu_ogm_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- reference API --
    def update_with_scan(self, robot_x, robot_y, robot_yaw, scan_ranges, angle_min, angle_increment):
        """Fuse one scan: scan_ranges[i] at robot_yaw + angle_min + i * angle_increment from the pose (:69-131)"""
        self.update_with_scans([(robot_x, robot_y, robot_yaw)], [scan_ranges], angle_min, angle_increment)

    def get_probability(self, ix, iy):
        """1 - 1 / (1 + exp(l)) of cell (ix, iy) (:133-138)"""
        l = self._cell(ix, iy)
        try:
            e = math.exp(l)
        except OverflowError:
            e = math.inf
        return 1.0 - 1.0 / (1.0 + e)

    def world_to_grid(self, x, y):
        """(ix, iy), or None outside the grid (:140-153)"""
        ix = _sat_floor_i32(float(x) / float(self.config.resolution) + self.W / 2.0)
        iy = _sat_floor_i32(float(y) / float(self.config.resolution) + self.H / 2.0)
        return (ix, iy) if 0 <= ix < self.W and 0 <= iy < self.H else None

    def is_occupied(self, ix, iy, threshold):
        return self.get_probability(ix, iy) > threshold

    @property
    def grid(self):
        """the log-odds grid, (W, H) f64, downloaded"""
        out = np.empty((self.W, self.H))
        _check(self.L, self.L.pfgpu_ogm_read(self.h, 0, out.size, _dp(out)))
        return out

    # -- batched and device-side additions --
    def update_with_scans(self, poses, scan_ranges, angle_min, angle_increment):
        """Fuse S scans in order in one call: poses (S, 3) = (x, y, yaw), scan_ranges (S, B); the same bits as S update_with_scan calls"""
        p = np.ascontiguousarray(_f64(poses).reshape(-1, 3))
        r = _f64(scan_ranges)
        if p.shape[0] == 0:
            return
        r = np.ascontiguousarray(r.reshape(p.shape[0], -1))
        _check(self.L, self.L.pfgpu_ogm_update_scans(self.h, _dp(p), p.shape[0], _dp(r), r.shape[1], float(angle_min), float(angle_increment)))

    def set_grid(self, grid):
        """replace the log-odds grid: (W, H) values (any; they are not clamped)"""
        g = np.ascontiguousarray(_f64(grid))
        if g.shape != (self.W, self.H):
            raise InvalidParameter(f"grid: shape ({self.W}, {self.H})")
        _check(self.L, self.L.pfgpu_ogm_set(self.h, _dp(g), g.size))

    def obstacles(self, threshold=0.5):
        """is_occupied of every cell, computed on the device: (W, H) bool (obstacles_from_log_odds's rule with the contract exp)"""
        m = np.empty((self.W, self.H), dtype=np.uint8)
        _check(self.L, self.L.pfgpu_ogm_obstacles(self.h, float(threshold), m.ctypes.data_as(C.POINTER(C.c_uint8)), m.size))
        return m.view(bool)

    def stats(self):
        """OgmStats of the last update"""
        s = _OgmStats()
        _check(self.L, self.L.pfgpu_ogm_info(self.h, None, None, C.byref(s)))
        return OgmStats(s.events, s.chunks, s.longest_run, s.event_cap)

    def _cell(self, ix, iy):
        ix, iy = int(ix), int(iy)
        if not (0 <= ix < self.W and 0 <= iy < self.H):
            raise IndexError(f"cell ({ix}, {iy}) outside a {self.W} x {self.H} grid")
        out = np.empty(1)
        _check(self.L, self.L.pfgpu_ogm_read(self.h, ix * self.H + iy, 1, _dp(out)))
        return float(out[0])


# ------------------------------------------------------------------------------------------------
class GridFastSlamConfig:
    """Grid-based FastSLAM (DESIGN §3.16): every particle's grid (an OccupancyGridConfig), the particle count, the N_eff threshold
    (absolute; None = n_particles / 2) and the endpoint model (z_hit, z_rand, max_range, max_beams, search_radius R: the window is
    (2R + 1)^2 cells)"""

    def __init__(self, grid=None, n_particles=100, nth=None, z_hit=0.95, z_rand=0.05, max_range=30.0, max_beams=60, search_radius=1):
        self.grid = grid or OccupancyGridConfig()
        self.n_particles, self.nth = n_particles, nth
        self.z_hit, self.z_rand, self.max_range, self.max_beams, self.search_radius = z_hit, z_rand, max_range, max_beams, search_radius

    def _c(self):
        n = int(self.n_particles)
        if not (0 <= n < 2 ** 64 and 0 <= int(self.max_beams) < 2 ** 32 and 0 <= int(self.search_radius) < 2 ** 32):
            raise InvalidParameter("n_particles, max_beams, search_radius: out of range")
        nth = n / 2.0 if self.nth is None else float(self.nth)
        return _GsCfg(self.grid._c(), n, nth, float(self.z_hit), float(self.z_rand), float(self.max_range), int(self.max_beams),
                      int(self.search_radius))


class GridFastSlamProposal:
    """The scan-matched proposal of grid FastSLAM (GMapping's improved proposal, DESIGN §3.17): a correlative match of each particle's
    scan against its own grid in a window of +-linear_range (linear_step) and +-angular_range (angular_step) around the odometry
    move, then a lattice of (2 half_width + 1)^3 points at (lattice_linear_step, lattice_angular_step) around the winner; a match with
    fewer than min_hits beams on occupied cells falls back to the plain odometry move.  See include/pfgpu.h for the rule."""

    def __init__(self, linear_range=0.1, linear_step=0.025, angular_range=0.05, angular_step=0.0125, half_width=1,
                 lattice_linear_step=0.01, lattice_angular_step=0.005, min_hits=10):
        self.linear_range, self.linear_step, self.angular_range, self.angular_step = linear_range, linear_step, angular_range, angular_step
        self.half_width, self.lattice_linear_step, self.lattice_angular_step = half_width, lattice_linear_step, lattice_angular_step
        self.min_hits = min_hits

    def _c(self, enabled=True):
        if not (0 <= int(self.half_width) < 2 ** 32 and 0 <= int(self.min_hits) < 2 ** 32):
            raise InvalidParameter("half_width, min_hits: out of range")
        return _GsProp(int(enabled), int(self.half_width), float(self.linear_range), float(self.linear_step), float(self.angular_range),
                       float(self.angular_step), float(self.lattice_linear_step), float(self.lattice_angular_step), int(self.min_hits), 0)

    def as_dict(self):
        return dict(linear_range=self.linear_range, linear_step=self.linear_step, angular_range=self.angular_range,
                    angular_step=self.angular_step, half_width=self.half_width, lattice_linear_step=self.lattice_linear_step,
                    lattice_angular_step=self.lattice_angular_step, min_hits=self.min_hits)


# GridFastSlam.last_proposal(): per slot, the last step's match winner (N, 3) (NaN where no match ran), eta (N,) (NaN where no
# lattice ran) and took (N,) bool: whether the particle took the proposal rather than the fallback
GsProposal = collections.namedtuple("GsProposal", ["matched", "eta", "took"])


# GridFastSlam.stats(): steps so far, and the last step's N_eff, whether it resampled, the grids it copied (N - distinct ancestors)
# and the cell updates its fuse applied
GsStats = collections.namedtuple("GsStats", ["steps", "neff", "resampled", "copies", "events"])


class GridFastSlam:
    """FastSLAM with occupancy grids (Probabilistic Robotics Table 13.4) on the device: N particles, each a pose, a weight and its
    own log-odds grid laid out as OccupancyGridMap's.  A step moves every particle by two odometry poses, weighs it by the scan's
    endpoints against its own grid, normalises, fuses the scan into every grid and resamples when N_eff < nth; see include/pfgpu.h
    for the rule, which the device follows bit for bit."""

    def __init__(self, config=None, start_pose=(0.0, 0.0, 0.0), seed=0, device=0):
        self.config = config or GridFastSlamConfig()
        self.L = load_library()
        self.h = C.c_void_p()
        self.device = device
        _check(self.L, self.L.pfgpu_gs_create(C.byref(self.config._c()), int(seed), _dp(_f64(start_pose)), device, C.byref(self.h)))
        self.n = int(self.config.n_particles)
        self.W, self.H = int(self.config.grid.width), int(self.config.grid.height)

    def close(self):
        if getattr(self, "h", None) and self.h.value:
            self.L.pfgpu_gs_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_odometry_noise(self, alpha):
        """alpha = (alpha1 .. alpha4), each finite and >= 0 (AMCL's odom_alpha1..4; 0.2 each at the start)"""
        _check(self.L, self.L.pfgpu_gs_set_odom_noise(self.h, _dp(_f64(alpha))))

    def odometry_noise(self):
        a = np.empty(4)
        _check(self.L, self.L.pfgpu_gs_odom_noise(self.h, _dp(a)))
        return tuple(float(v) for v in a)

    def step(self, odom_prev, odom_cur, ranges, angle_min, angle_increment):
        """One step with the odometry poses (x, y, yaw) before and after it and the scan taken after it; enqueued, not waited for"""
        o = _f64(list(odom_prev) + list(odom_cur))
        if o.shape != (6,):
            raise InvalidParameter("odom_prev, odom_cur: (x, y, yaw) each")
        r = _f64(ranges).ravel()
        _check(self.L, self.L.pfgpu_gs_step(self.h, _dp(o), _dp(r), r.size, float(angle_min), float(angle_increment)))

    def particles(self):
        """(N, 3) poses"""
        p = np.empty((self.n, 3))
        _check(self.L, self.L.pfgpu_gs_download(self.h, _dp(p), None, self.n))
        return p

    def weights(self):
        w = np.empty(self.n)
        _check(self.L, self.L.pfgpu_gs_download(self.h, None, _dp(w), self.n))
        return w

    def best(self):
        """(slot, pose (3,)) of the largest weight, ties to the lowest slot"""
        s, p = C.c_size_t(), np.empty(3)
        _check(self.L, self.L.pfgpu_gs_best(self.h, C.byref(s), _dp(p)))
        return int(s.value), p

    def grid(self, slot):
        """slot's log-odds grid, (W, H) f64, downloaded"""
        out = np.empty((self.W, self.H))
        _check(self.L, self.L.pfgpu_gs_grid_read(self.h, int(slot), 0, out.size, _dp(out)))
        return out

    def copy_grid_to(self, slot, grid_map):
        """slot's grid into an OccupancyGridMap of the same config on the same device, without leaving the device"""
        _check(self.L, self.L.pfgpu_gs_grid_to_ogm(self.h, int(slot), grid_map.h))

    def last_indices(self):
        """ancestors of the last step's resample; empty when it did not resample"""
        idx = np.empty(self.n, dtype=np.uint32)
        k = C.c_size_t()
        _check(self.L, self.L.pfgpu_gs_last_indices(self.h, idx.ctypes.data_as(c_u32p), idx.size, C.byref(k)))
        return idx[:k.value].copy()

    def max_used_beams(self):
        """L: the most used beams a scan may have"""
        L = C.c_uint64()
        _check(self.L, self.L.pfgpu_gs_info(self.h, None, None, None, C.byref(L), None))
        return int(L.value)

    def stats(self):
        s = _GsStats()
        _check(self.L, self.L.pfgpu_gs_info(self.h, None, None, None, None, C.byref(s)))
        return GsStats(int(s.steps), float(s.neff), bool(s.resampled), int(s.copies), int(s.events))

    def set_proposal(self, proposal):
        """enable the scan-matched proposal with a GridFastSlamProposal, or disable it with None; applies from the next step"""
        c = GridFastSlamProposal()._c(False) if proposal is None else proposal._c(True)
        _check(self.L, self.L.pfgpu_gs_set_proposal(self.h, C.byref(c)))

    def proposal(self):
        """the GridFastSlamProposal in use, or None when the proposal is off"""
        c = _GsProp()
        _check(self.L, self.L.pfgpu_gs_get_proposal(self.h, C.byref(c)))
        if not c.enabled:
            return None
        return GridFastSlamProposal(c.linear_range, c.linear_step, c.angular_range, c.angular_step, int(c.half_width),
                                    c.lattice_linear_step, c.lattice_angular_step, int(c.min_hits))

    def last_proposal(self):
        """GsProposal of the last step (all NaN / False when it ran without the proposal)"""
        xh, eta, took = np.empty((self.n, 3)), np.empty(self.n), np.zeros(self.n, dtype=np.uint8)
        _check(self.L, self.L.pfgpu_gs_last_proposal(self.h, _dp(xh), _dp(eta), took.ctypes.data_as(C.POINTER(C.c_uint8)), self.n))
        return GsProposal(xh, eta, took.astype(bool))

    def sync(self):
        _check(self.L, self.L.pfgpu_gs_sync(self.h))


# ------------------------------------------------------------------------------------------------
class CorrelativeScanMatcherConfig:
    """correlative_scan_matching.rs:17-42"""

    def __init__(self, linear_search_range=1.0, angular_search_range=0.2, linear_step=0.1, angular_step=0.02, grid_resolution=0.05):
        self.linear_search_range, self.angular_search_range = linear_search_range, angular_search_range
        self.linear_step, self.angular_step, self.grid_resolution = linear_step, angular_step, grid_resolution

    def _c(self):
        return _CsmCfg(float(self.linear_search_range), float(self.angular_search_range), float(self.linear_step), float(self.angular_step),
                       float(self.grid_resolution))


# correlative_scan_matching.rs:44-52
ScanMatchResult = collections.namedtuple("ScanMatchResult", ["x", "y", "yaw", "score", "converged"])


class CorrelativeScanMatcher:
    """correlative_scan_match (correlative_scan_matching.rs:55-197) on the device (DESIGN §3.13): reference points held on one device,
    their lookup table built there for each resolution a match asks for, every candidate pose of the window scored there, the
    reference's result bit for bit.  One call matches one query or a batch of queries against the same reference."""

    def __init__(self, device=0):
        self.L = load_library()
        self.h = C.c_void_p()
        self.device = device
        _check(self.L, self.L.pfgpu_csm_create(int(device), C.byref(self.h)))

    def close(self):
        if getattr(self, "h", None) and self.h.value:
            self.L.pfgpu_csm_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_reference(self, reference_x, reference_y):
        """the reference scan (world points); copied to the device"""
        x, y = _f64(reference_x).ravel(), _f64(reference_y).ravel()
        if x.size != y.size:
            raise InvalidParameter("reference_x and reference_y differ in length")
        _check(self.L, self.L.pfgpu_csm_set_reference(self.h, _dp(x), _dp(y), x.size))

    def set_reference_from_grid(self, grid_map, threshold=0.5):
        """the centres of grid_map's obstacle cells at `threshold` (OccupancyGridMap.obstacles), built on the device; the grid is copied
        now, so later updates of grid_map do not change the matcher.  grid_map must live on this matcher's device."""
        _check(self.L, self.L.pfgpu_csm_set_reference_grid(self.h, grid_map.h, float(threshold)))

    @property
    def reference_size(self):
        n = C.c_size_t()
        _check(self.L, self.L.pfgpu_csm_reference_size(self.h, C.byref(n)))
        return int(n.value)

    def match(self, query_x, query_y, initial_pose, config=None):
        """One query: query_x, query_y (sequences of floats) and initial_pose (x, y, yaw) -> ScanMatchResult.  A batch: query_x and
        query_y lists of per-query sequences (any lengths) and initial_pose (Q, 3) -> a list of ScanMatchResult."""
        cfg = (config or CorrelativeScanMatcherConfig())._c()
        p = _f64(initial_pose)
        single = p.ndim == 1
        p = np.ascontiguousarray(p.reshape(-1, 3))
        qxs = [query_x] if single else list(query_x)
        qys = [query_y] if single else list(query_y)
        if len(qxs) != p.shape[0] or len(qys) != p.shape[0]:
            raise InvalidParameter("one point list per initial pose")
        xs, ys = [_f64(a).ravel() for a in qxs], [_f64(a).ravel() for a in qys]
        if any(a.size != b.size for a, b in zip(xs, ys)):
            raise InvalidParameter("query_x and query_y differ in length")
        off = np.zeros(len(xs) + 1, dtype=np.uint64)
        off[1:] = np.cumsum([a.size for a in xs])
        qx = np.ascontiguousarray(np.concatenate(xs) if xs else np.zeros(0))
        qy = np.ascontiguousarray(np.concatenate(ys) if ys else np.zeros(0))
        out = (_CsmResult * max(1, p.shape[0]))()
        _check(self.L, self.L.pfgpu_csm_match(self.h, C.byref(cfg), _dp(p), p.shape[0], _dp(qx), _dp(qy),
                                              off.ctypes.data_as(C.POINTER(C.c_uint64)), out))
        res = [ScanMatchResult(r.x, r.y, r.yaw, r.score, bool(r.converged)) for r in out[:p.shape[0]]]
        return res[0] if single else res

    def table_info(self, grid_resolution=0.05):
        """(origin_x, origin_y, width, height, R) of the lookup table for grid_resolution (built now if it is not the current one)"""
        ox, oy, W, H, R = C.c_int64(), C.c_int64(), C.c_uint64(), C.c_uint64(), C.c_int32()
        _check(self.L, self.L.pfgpu_csm_table_info(self.h, float(grid_resolution), C.byref(ox), C.byref(oy), C.byref(W), C.byref(H),
                                                   C.byref(R)))
        return int(ox.value), int(oy.value), int(W.value), int(H.value), int(R.value)

    def lookup_table(self, grid_resolution=0.05):
        """the lookup table for grid_resolution: (dense (width, height) f64 array, (origin_x, origin_y), R); cell (ix, iy) is
        table[ix - origin_x, iy - origin_y], and every cell outside reads 0.0 (build_lookup_table's HashMap, :129-159)"""
        ox, oy, W, H, R = self.table_info(grid_resolution)
        t = np.zeros((W, H))
        if t.size:
            _check(self.L, self.L.pfgpu_csm_table_read(self.h, 0, t.size, _dp(t)))
        return t, (ox, oy), R


def correlative_scan_match(reference_x, reference_y, query_x, query_y, initial_pose, config=None, device=0):
    """correlative_scan_matching.rs:55-120 with its signature: a one-shot matcher on `device`"""
    m = CorrelativeScanMatcher(device)
    try:
        m.set_reference(reference_x, reference_y)
        return m.match(query_x, query_y, tuple(initial_pose), config)
    finally:
        m.close()


def _sat_floor_i32(v):
    """Rust's `floor() as i32`: saturating, NaN -> 0"""
    if v != v:
        return 0
    if v >= 2147483647.0:
        return 2147483647
    if v <= -2147483648.0:
        return -2147483648
    return int(math.floor(v))


class ParticleFilterLocalizer(_PfBase):
    """pf.rs:121-573"""

    def __init__(self, config=None, seed=42, device=0, shard=None):
        self.config = config or ParticleFilterConfig()
        super().__init__(self.config._c(), seed, device, shard)

    @classmethod
    def try_new(cls, config, **kw):
        return cls(config, **kw)

    new = try_new

    @classmethod
    def with_defaults(cls, **kw):
        return cls(ParticleFilterConfig(), **kw)

    @classmethod
    def try_with_initial_state(cls, initial_state, config, **kw):
        f = cls(config, **kw)
        s = _f64(initial_state)
        _check(f.L, f.L.pfgpu_pf_init_state(f.h, _dp(s)))
        return f

    with_initial_state = try_with_initial_state
    with_initial_state_2d = try_with_initial_state


class MonteCarloLocalizer(_PfBase):
    """mcl.rs:133-471"""

    def __init__(self, config=None, seed=42, device=0, shard=None):
        self.config = config or MonteCarloLocalizationConfig()
        super().__init__(self.config._c(), seed, device, shard)

    @classmethod
    def try_new(cls, config, **kw):
        return cls(config, **kw)

    new = try_new

    @classmethod
    def try_with_initial_state(cls, initial_state, config, **kw):
        f = cls(config, **kw)
        s = _f64(initial_state)
        _check(f.L, f.L.pfgpu_pf_init_state(f.h, _dp(s)))
        return f

    with_initial_state = try_with_initial_state


# ------------------------------------------------------------------------------------------------
class FsConfig:
    """fs1.rs:13-23 module constants as fields"""

    def __init__(self, dt=0.1, max_range=20.0, nth=100.0 / 1.5, q00=0.3, q11=0.0305, r00=0.5, r11=0.0305,
                 init_weight=1.0 / 100.0):
        self.dt, self.max_range, self.nth, self.q00, self.q11 = dt, max_range, nth, q00, q11
        self.r00, self.r11, self.init_weight = r00, r11, init_weight

    def _c(self):
        return _FsCfg(self.dt, self.max_range, self.nth, self.q00, self.q11, self.r00, self.r11, self.init_weight)


class FastSlam1:
    """Engine form of fs1.rs's free functions over a caller-owned Vec<Particle> (SURVEY.md §8b):
    create_particles -> __init__; fastslam_update -> fastslam_update/step; get_best_particle -> get_best_particle."""

    def __init__(self, n_particles, n_landmarks, config=None, seed=42, device=0, shard=None):
        self.L = load_library()
        self.config = config or FsConfig()
        self.h = C.c_void_p()
        cc = self.config._c()
        if shard is None:
            _check(self.L, self.L.pfgpu_fs_create(C.byref(cc), n_particles, n_landmarks, seed, device, C.byref(self.h)))
        else:
            uid, rank, world = shard
            buf = C.create_string_buffer(bytes(uid), 128)
            _check(self.L, self.L.pfgpu_fs_create_sharded(C.byref(cc), n_particles, n_landmarks, seed, device, buf,
                                                          rank, world, C.byref(self.h)))
        nl, ng, m = C.c_size_t(), C.c_size_t(), C.c_size_t()
        _check(self.L, self.L.pfgpu_fs_count(self.h, C.byref(nl), C.byref(ng), C.byref(m)))
        self.n_local, self.n_global, self.m = nl.value, ng.value, m.value
        if self.VARIANT != 1:
            _check(self.L, self.L.pfgpu_fs_set_variant(self.h, self.VARIANT))

    VARIANT = 1                      # which reference module the step mirrors: fastslam1 (FastSlam2 below: fastslam2)
    create_particles = classmethod(lambda cls, n, m, **kw: cls(n, m, **kw))

    @classmethod
    def create_sharded_local(cls, n_particles_global, n_landmarks, devices, config=None, seed=42):
        """All ranks of the sharded engine inside this process (pfgpu_fs_create_sharded_local): one FastSlam1 per entry of
        `devices` (entries may repeat).  Drive them with step_all()."""
        L = load_library()
        config = config or FsConfig()
        cc = config._c()
        world = len(devices)
        devs = (C.c_int * world)(*devices)
        hs = (C.c_void_p * world)()
        _check(L, L.pfgpu_fs_create_sharded_local(C.byref(cc), n_particles_global, n_landmarks, seed, devs, world, hs))
        out = []
        for r in range(world):
            g = cls.__new__(cls)
            g.L, g.config, g.h = L, config, C.c_void_p(hs[r])
            nl, ng, m = C.c_size_t(), C.c_size_t(), C.c_size_t()
            _check(L, L.pfgpu_fs_count(g.h, C.byref(nl), C.byref(ng), C.byref(m)))
            g.n_local, g.n_global, g.m = nl.value, ng.value, m.value
            if cls.VARIANT != 1:
                _check(L, L.pfgpu_fs_set_variant(g.h, cls.VARIANT))
            out.append(g)
        return out

    @staticmethod
    def step_all(ranks, u, z):
        """one fastslam_update on every in-process rank: enqueue everywhere first, then synchronise; returns did_resample"""
        for g in ranks:
            g.fastslam_update(u, z, want_flag=False)
        for g in ranks:
            g.sync()
        return ranks[0].did_resample()

    def did_resample(self):
        """whether the last step resampled (synchronises)"""
        return self.last_gate()

    def last_gate(self):
        idx = C.c_size_t()
        _check(self.L, self.L.pfgpu_fs_best(self.h, C.byref(idx), None))      # synchronises the stream
        g = C.c_int()
        _check(self.L, self.L.pfgpu_fs_last_gate(self.h, C.byref(g)))
        return bool(g.value)

    def close(self):
        if getattr(self, "h", None) and self.h.value:
            self.L.pfgpu_fs_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _obs(z):
        arr = (_FsObs * max(len(z), 1))()
        for i, (d, a, l) in enumerate(z):
            arr[i].d, arr[i].angle, arr[i].lm_id = float(d), float(a), int(l)
        return arr

    def fastslam_update(self, u, z, want_flag=True, obs_array=None):
        """fs1.rs:237-266.  Returns whether the step resampled (None when want_flag is False: no host sync)."""
        uu = _f64(u)
        arr = obs_array if obs_array is not None else self._obs(z)
        k = len(z)
        did = C.c_int()
        _check(self.L, self.L.pfgpu_fs_step(self.h, _dp(uu), arr, k, C.byref(did) if want_flag else None))
        return bool(did.value) if want_flag else None

    step = fastslam_update

    # -- odometry motion model (not in fs1.rs / fs2.rs, whose steps take a velocity command; DESIGN §3.15) --
    def set_odometry_noise(self, alpha1=0.2, alpha2=0.2, alpha3=0.2, alpha4=0.2):
        """ROS AMCL's odom_alpha1..4 (diff-corrected), as ParticleFilterLocalizer.set_odometry_noise: each finite and >= 0; a handle
        starts at 0.2 each.  On a sharded engine every rank makes the same call."""
        a = _f64([alpha1, alpha2, alpha3, alpha4])
        _check(self.L, self.L.pfgpu_fs_set_odom_noise(self.h, _dp(a)))

    def odometry_noise(self):
        """(alpha1, alpha2, alpha3, alpha4)"""
        a = np.empty(4)
        _check(self.L, self.L.pfgpu_fs_odom_noise(self.h, _dp(a)))
        return tuple(float(v) for v in a)

    def fastslam_update_odometry(self, odom_prev, odom_cur, z, want_flag=True):
        """fastslam_update with the odometry motion model: every particle moves by the increment from odometry pose odom_prev =
        (x, y, yaw) to odom_cur (include/fs_odom_math.h) instead of by a control over dt.  Returns whether the step resampled
        (None when want_flag is False: no host sync)."""
        o = _PfBase._odom_pair(odom_prev, odom_cur)
        did = C.c_int()
        _check(self.L, self.L.pfgpu_fs_step_odom(self.h, _dp(o), self._obs(z), len(z), C.byref(did) if want_flag else None))
        return bool(did.value) if want_flag else None

    @staticmethod
    def step_all_odometry(ranks, odom_prev, odom_cur, z):
        """one fastslam_update_odometry on every in-process rank: enqueue everywhere first, then synchronise; returns did_resample"""
        for g in ranks:
            g.fastslam_update_odometry(odom_prev, odom_cur, z, want_flag=False)
        for g in ranks:
            g.sync()
        return ranks[0].did_resample()

    def get_observations(self, x_true, landmarks_xy, call):
        """fs1.rs:277-299 on the device (Philox stream OBS keyed by the handle's seed, `call` and the landmark id)"""
        xt, lm = _f64(x_true), _f64(landmarks_xy)
        n = lm.size // 2
        out = (_FsObs * max(n, 1))()
        k = C.c_size_t()
        _check(self.L, self.L.pfgpu_fs_get_observations(self.h, _dp(xt), _dp(lm), n, call, out, C.byref(k)))
        return [(out[i].d, out[i].angle, int(out[i].lm_id)) for i in range(k.value)]

    def get_best_particle(self):
        idx = C.c_size_t()
        pw = np.empty(4)
        _check(self.L, self.L.pfgpu_fs_best(self.h, C.byref(idx), _dp(pw)))
        return idx.value, pw

    def particle_landmarks(self, i):
        out = np.empty((self.m, 6))
        _check(self.L, self.L.pfgpu_fs_particle_landmarks(self.h, i, _dp(out)))
        return out

    def set_state(self, pose_w, lm=None):
        p = _f64(pose_w)
        l = _f64(lm) if lm is not None else None
        _check(self.L, self.L.pfgpu_fs_upload(self.h, _dp(p), _dp(l) if l is not None else None, p.shape[0]))

    def seed_map(self, pose3, landmarks_xy, sigma=1.0, cov0=10.0):
        """initialised map (EKF branch live from step 0); see include/pfgpu.h pfgpu_fs_seed_map"""
        p, l = _f64(pose3), _f64(landmarks_xy)
        _check(self.L, self.L.pfgpu_fs_seed_map(self.h, _dp(p), _dp(l), l.size // 2, float(sigma), float(cov0)))

    def state(self, landmarks=True):
        p = np.empty((self.n_local, 4))
        l = np.empty((self.n_local, self.m, 6)) if landmarks else None
        _check(self.L, self.L.pfgpu_fs_download(self.h, _dp(p), _dp(l) if landmarks else None, self.n_local))
        return p, l

    def last_indices(self):
        idx = np.empty(self.n_local, dtype=np.uint32)
        cnt = C.c_size_t()
        _check(self.L, self.L.pfgpu_fs_last_indices(self.h, idx.ctypes.data_as(c_u32p), self.n_local, C.byref(cnt)))
        return idx[:cnt.value]

    def last_neff(self):
        v = C.c_double()
        _check(self.L, self.L.pfgpu_fs_last_neff(self.h, C.byref(v)))
        return v.value

    def sync(self):
        _check(self.L, self.L.pfgpu_fs_sync(self.h))

    def stats(self):
        s = Stats()
        _check(self.L, self.L.pfgpu_fs_stats(self.h, C.byref(s)))
        return s

    def shard_mode(self):
        """0 = one GPU, 2 = sharded over peer memory (NVLink)."""
        m = C.c_int()
        _check(self.L, self.L.pfgpu_fs_shard_mode(self.h, C.byref(m)))
        return m.value

    def post_shape(self):
        """(tiles, threads, values per thread, "shared" or "global"): the fused post-step kernel's shape, and where its weight
        tiles live (global memory for particle counts whose tile does not fit in shared memory)."""
        t, nt, k, gl = C.c_uint(), C.c_uint(), C.c_uint(), C.c_int()
        _check(self.L, self.L.pfgpu_fs_post_shape(self.h, C.byref(t), C.byref(nt), C.byref(k), C.byref(gl)))
        return t.value, nt.value, k.value, "global" if gl.value else "shared"

    def post_k1(self):
        """True when the post-step kernel runs its instantiation for one value and at most one local slot per thread (config 3
        on one GPU; PFGPU_POST_K1=0 at creation forces the generic kernel)."""
        k1 = C.c_int()
        _check(self.L, self.L.pfgpu_fs_post_k1(self.h, C.byref(k1)))
        return bool(k1.value)

    # -- estimate (no reference counterpart: fs1.rs's callers read the best particle's map, keeping landmarks with cov00 < 100) --
    def moments(self, cov00_max=100.0, landmarks=True):
        """pfgpu_fs_moments: (pose moments, (m, 7) landmark moments or None) of the particles this handle owns"""
        pose = _FsPoseMoments()
        lm = np.empty((self.m, 7)) if landmarks else None
        _check(self.L, self.L.pfgpu_fs_moments(self.h, float(cov00_max), C.byref(pose), _dp(lm) if lm is not None else None))
        return pose, lm

    @staticmethod
    def merge_moments(moments):
        """pfgpu_fs_estimate_merge over [(pose moments, landmark moments or None)] in rank order -> FsEstimate"""
        L = load_library()
        world = len(moments)
        poses = (_FsPoseMoments * world)(*[p for p, _ in moments])
        lms = [l for _, l in moments]
        with_lm = lms[0] is not None
        m = lms[0].shape[0] if with_lm else 0
        mean, cov = np.empty(3), np.empty(9)
        mass, lmean, lcov = (np.empty(m), np.empty((m, 2)), np.empty((m, 2, 2))) if with_lm else (None, None, None)
        ptrs = (c_dp * world)(*[_dp(l) for l in lms]) if with_lm else None
        _check(L, L.pfgpu_fs_estimate_merge(poses, ptrs, world, m, _dp(mean), _dp(cov), *(_dp(a) if a is not None else None for a in (mass, lmean, lcov))))
        return FsEstimate(mean, cov.reshape(3, 3).T, mass, lmean, lcov)

    def estimate(self, cov00_max=100.0, landmarks=True):
        """Weighted posterior estimate (DESIGN §3.4): FsEstimate(pose (3,), pose_cov (3, 3), mass (m,), mean (m, 2), cov (m, 2, 2));
        the landmark fields are None with landmarks=False.  Only landmark copies with cov00 < cov00_max count (the examples'
        filter; inf takes every copy).  After fastslam2_update_unknown steps slot l is not the same landmark in every particle, so
        the landmark fields mix landmarks: read the best particle's map (get_best_particle + particle_landmarks).  Synchronises."""
        return self.merge_moments([self.moments(cov00_max, landmarks)])

    @staticmethod
    def estimate_all(ranks, cov00_max=100.0, landmarks=True):
        """estimate() of an in-process sharded engine (create_sharded_local): synchronises every rank, then collects their moments
        and merges them in rank order"""
        for g in ranks:
            g.sync()
        return FastSlam1.merge_moments([g.moments(cov00_max, landmarks) for g in ranks])

    # -- path history (no reference counterpart: fs1.rs's particles keep no past poses; DESIGN §3.6) --
    def enable_history(self, capacity):
        """Keep the last `capacity` steps of every particle's path on the device (28 bytes per particle and step); 0 disables.
        Starts a new window at the current poses.  On a sharded engine every rank makes the same call."""
        _check(self.L, self.L.pfgpu_fs_history_enable(self.h, int(capacity)))

    def history_window(self):
        """(first, last): the steps of the oldest and the newest entry held"""
        a, b = C.c_uint64(), C.c_uint64()
        _check(self.L, self.L.pfgpu_fs_history_window(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def _max_steps(self, max_steps):
        if max_steps is not None:
            return int(max_steps)
        first, last = self.history_window()
        return last - first + 1

    def path(self, index=None, max_steps=None):
        """FsPath of global slot `index` (default: the best particle), oldest first: the poses of its lineage, which are the poses
        that produced its map.  At most max_steps entries (default: the whole window).  Synchronises."""
        if index is None:
            index = self.get_best_particle()[0]
        cap = self._max_steps(max_steps)
        steps, slots, poses = np.empty(max(cap, 1), dtype=np.uint64), np.empty(max(cap, 1), dtype=np.uint32), np.empty((max(cap, 1), 3))
        n = C.c_size_t()
        _check(self.L, self.L.pfgpu_fs_path(self.h, int(index), cap, steps.ctypes.data_as(C.POINTER(C.c_uint64)),
                                            slots.ctypes.data_as(c_u32p), _dp(poses), C.byref(n)))
        return FsPath(steps[:n.value], slots[:n.value], poses[:n.value])

    def path_moments(self, max_steps=None):
        """pfgpu_fs_path_moments: (steps, [pose moments per step]) of the particles this handle owns, oldest first"""
        cap = self._max_steps(max_steps)
        steps = np.empty(max(cap, 1), dtype=np.uint64)
        out = (_FsPoseMoments * max(cap, 1))()
        n = C.c_size_t()
        _check(self.L, self.L.pfgpu_fs_path_moments(self.h, cap, steps.ctypes.data_as(C.POINTER(C.c_uint64)), out, C.byref(n)))
        return steps[:n.value], [out[j] for j in range(n.value)]

    @staticmethod
    def merge_path_moments(per_rank):
        """[(steps, moments)] in rank order -> FsPathEstimate: every step merged with pfgpu_fs_estimate_merge (pose only)"""
        steps = per_rank[0][0]
        assert all(np.array_equal(s, steps) for s, _ in per_rank), "ranks hold different history windows"
        L = load_library()
        world = len(per_rank)
        pose, cov = np.empty((len(steps), 3)), np.empty((len(steps), 3, 3))
        for j in range(len(steps)):
            poses = (_FsPoseMoments * world)(*[m[j] for _, m in per_rank])
            mean, c9 = np.empty(3), np.empty(9)
            _check(L, L.pfgpu_fs_estimate_merge(poses, None, world, 0, _dp(mean), _dp(c9), None, None, None))
            pose[j], cov[j] = mean, c9.reshape(3, 3).T
        return FsPathEstimate(steps, pose, cov)

    def path_estimate(self, max_steps=None):
        """Genealogy smoother (DESIGN §3.6): at every step of the window, the weighted mean and covariance of the current particles'
        lineage poses under their current weights; FsPathEstimate, oldest first.  Synchronises."""
        return self.merge_path_moments([self.path_moments(max_steps)])

    @staticmethod
    def path_estimate_all(ranks, max_steps=None):
        """path_estimate() of an in-process sharded engine: synchronises every rank, then merges their moments step by step"""
        for g in ranks:
            g.sync()
        return FastSlam1.merge_path_moments([g.path_moments(max_steps) for g in ranks])

    def time_main_kernel(self, on=True):
        _check(self.L, self.L.pfgpu_fs_time_main_kernel(self.h, int(on)))

    def mark(self, slot):
        _check(self.L, self.L.pfgpu_fs_mark(self.h, slot))

    def elapsed_ms(self, a, b):
        v = C.c_double()
        _check(self.L, self.L.pfgpu_fs_elapsed_ms(self.h, a, b, C.byref(v)))
        return v.value

    def flush_l2(self):
        _check(self.L, self.L.pfgpu_fs_flush_l2(self.h))


class FastSlam2(FastSlam1):
    """rust_robotics_slam::fastslam2 (crates/rust_robotics_slam/src/fastslam2.rs): create_particles :418-422, fastslam2_update
    :376-383, get_best_particle :385-390, get_observations :418-421 over the same device-resident particle set as FastSlam1; the
    step samples every pose from the observation-informed proposal (:173-239) and runs update_landmark_and_weight (:242-280)."""
    VARIANT = 2

    def fastslam2_update(self, u, z, **kw):
        return self.fastslam_update(u, z, **kw)

    def fastslam2_update_odometry(self, odom_prev, odom_cur, z, **kw):
        """fastslam2_update with the odometry motion model: the proposal fuses the first observation with the prior the odometry
        increment induces (include/fs_odom_math.h)"""
        return self.fastslam_update_odometry(odom_prev, odom_cur, z, **kw)

    # -- unknown data association (not in fs2.rs; the rule of ekf_slam.rs:284-308 per particle, DESIGN §3.5) --
    def fastslam2_update_unknown(self, u, z, gate_d2=16.0, want_flag=True):
        """One step from observations WITHOUT landmark ids: z = k (d, angle) pairs.  Every particle associates each observation with
        the landmark of its own map at the smallest Mahalanobis distance below gate_d2, or adds a landmark in its lowest empty slot
        (an observation is dropped when the map is full).  Returns whether the step resampled (None when want_flag is False: no
        host sync).  Slot l is then NOT the same landmark in every particle: read a map from one particle (get_best_particle and
        particle_landmarks), not from estimate()."""
        uu = _f64(u)
        zz = _f64(z).reshape(-1, 2) if len(z) else np.zeros((0, 2))
        did = C.c_int()
        _check(self.L, self.L.pfgpu_fs_step_unknown(self.h, _dp(uu), _dp(zz) if zz.size else None, zz.shape[0], float(gate_d2),
                                                    C.byref(did) if want_flag else None))
        return bool(did.value) if want_flag else None

    def fastslam2_update_unknown_odometry(self, odom_prev, odom_cur, z, gate_d2=16.0, want_flag=True):
        """fastslam2_update_unknown with the odometry motion model (see fastslam2_update_odometry)"""
        o = _PfBase._odom_pair(odom_prev, odom_cur)
        zz = _f64(z).reshape(-1, 2) if len(z) else np.zeros((0, 2))
        did = C.c_int()
        _check(self.L, self.L.pfgpu_fs_step_unknown_odom(self.h, _dp(o), _dp(zz) if zz.size else None, zz.shape[0], float(gate_d2),
                                                         C.byref(did) if want_flag else None))
        return bool(did.value) if want_flag else None

    @staticmethod
    def step_all_unknown_odometry(ranks, odom_prev, odom_cur, z, gate_d2=16.0):
        """one fastslam2_update_unknown_odometry on every in-process rank: enqueue everywhere, then synchronise"""
        for g in ranks:
            g.fastslam2_update_unknown_odometry(odom_prev, odom_cur, z, gate_d2, want_flag=False)
        for g in ranks:
            g.sync()
        return ranks[0].did_resample()

    @staticmethod
    def step_all_unknown(ranks, u, z, gate_d2=16.0):
        """one fastslam2_update_unknown on every in-process rank (create_sharded_local): enqueue everywhere, then synchronise"""
        for g in ranks:
            g.fastslam2_update_unknown(u, z, gate_d2, want_flag=False)
        for g in ranks:
            g.sync()
        return ranks[0].did_resample()

    def assoc_counts(self):
        """(matched, born, dropped) observations of the last unknown-association step over this handle's particles (synchronises)"""
        c = (C.c_uint64 * 3)()
        _check(self.L, self.L.pfgpu_fs_assoc_counts(self.h, c))
        return tuple(int(v) for v in c)

    # -- landmark existence counters (not in fs2.rs, which takes ids and never removes a landmark; DESIGN §3.7) --
    def enable_existence(self, range=None):
        """Track an existence counter per landmark copy in fastslam2_update_unknown: +1 per match, 1 at a birth, -1 when the copy
        lies within `range` of the sampled pose and no observation went to it; below 0 the copy is removed and its slot is empty
        again.  range=None: config.max_range; inf allowed; 0 disables.  Every counter starts at 1 (also after set_state and
        seed_map).  While enabled known-id steps are refused.  On a sharded engine every rank makes the same call."""
        r = self.config.max_range if range is None else float(range)
        _check(self.L, self.L.pfgpu_fs_existence_enable(self.h, r))

    def existence_counts(self, first=0, count=None):
        """(count, m) int32: the counters of local slots first .. first + count - 1 (default: all), 0 for an empty slot.  Synchronises."""
        if count is None:
            count = self.n_local - first
        out = np.zeros((count, self.m), dtype=np.int32)
        _check(self.L, self.L.pfgpu_fs_existence_counts(self.h, int(first), int(count), out.ctypes.data_as(C.POINTER(C.c_int32))))
        return out

    def removed_count(self):
        """landmark copies removed by the last fastslam2_update_unknown over this handle's particles (0 when disabled); synchronises"""
        v = C.c_uint64()
        _check(self.L, self.L.pfgpu_fs_existence_removed(self.h, C.byref(v)))
        return int(v.value)
