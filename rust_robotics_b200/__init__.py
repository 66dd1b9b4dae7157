"""rust_robotics_b200 — H100-native particle-filter / FastSLAM 1.0 engine behind the rust_robotics API.

The product is the CUDA library (csrc/ -> libpfgpu.so, C ABI in include/pfgpu.h).  `api` mirrors the
reference's public types (ParticleFilterLocalizer, MonteCarloLocalizer, fastslam1) over that ABI with
ctypes.  There is no CPU fallback: constructing any filter without a CUDA device raises.
"""
from .api import (CorrelativeScanMatcher, CorrelativeScanMatcherConfig, FastSlam1, FastSlam2, FsConfig, InvalidParameter,  # noqa: F401
                  GridFastSlam, GridFastSlamConfig, GridFastSlamProposal, GsProposal, GsStats, MonteCarloLocalizationConfig, MonteCarloLocalizer,
                  OccupancyGridConfig, OccupancyGridMap, OgmStats, ParticleFilterConfig, ParticleFilterLocalizer, PfgpuError, PfHypothesis,
                  ScanMatchResult, correlative_scan_match, load_library, obstacles_from_log_odds)
