// correlative_scan_matching.hpp — C++ host-side mirror of the reference's correlative scan matcher over the C ABI (include/pfgpu.h,
// DESIGN §3.13), with the SAME type names, function name and argument meaning as
// crates/rust_robotics_slam/src/correlative_scan_matching.rs, plus a CorrelativeScanMatcher that keeps the reference (and its lookup
// table) on the device between calls and matches batches.  Header-only; link against libpfgpu.so.  No CPU fallback.
#pragma once
#include <cstdint>
#include <tuple>
#include <vector>
#include "occupancy_grid_map.hpp"  // OccupancyGridMap::handle(), RoboticsError, check

namespace rust_robotics_b200 {

struct CorrelativeScanMatcherConfig {                                    // correlative_scan_matching.rs:17-42
    double linear_search_range = 1.0, angular_search_range = 0.2, linear_step = 0.1, angular_step = 0.02, grid_resolution = 0.05;
    pfgpu_csm_config to_c() const { return pfgpu_csm_config{linear_search_range, angular_search_range, linear_step, angular_step, grid_resolution}; }
};

struct ScanMatchResult {                                                 // correlative_scan_matching.rs:44-52
    double x = 0.0, y = 0.0, yaw = 0.0, score = 0.0;
    bool converged = false;
};

class CorrelativeScanMatcher {
    pfgpu_csm* h_ = nullptr;
    static ScanMatchResult from_c(const pfgpu_csm_result& r) { return ScanMatchResult{r.x, r.y, r.yaw, r.score, r.converged != 0}; }
public:
    explicit CorrelativeScanMatcher(int device = 0) { check(pfgpu_csm_create(device, &h_), "correlative scan matcher"); }
    CorrelativeScanMatcher(const CorrelativeScanMatcher&) = delete;
    CorrelativeScanMatcher& operator=(const CorrelativeScanMatcher&) = delete;
    ~CorrelativeScanMatcher() { pfgpu_csm_destroy(h_); }

    void set_reference(const std::vector<double>& reference_x, const std::vector<double>& reference_y) {
        if (reference_x.size() != reference_y.size()) throw RoboticsError(RoboticsError::InvalidParameter, "reference_x / reference_y sizes");
        check(pfgpu_csm_set_reference(h_, reference_x.data(), reference_y.data(), reference_x.size()), "set_reference");
    }
    // the centres of the grid's obstacle cells at `threshold`, built on the device; the grid is copied now
    void set_reference_from_grid(const OccupancyGridMap& grid, double threshold = 0.5) {
        check(pfgpu_csm_set_reference_grid(h_, grid.handle(), threshold), "set_reference_from_grid");
    }
    ScanMatchResult match(const std::vector<double>& query_x, const std::vector<double>& query_y, std::tuple<double, double, double> initial_pose,
                          const CorrelativeScanMatcherConfig& config = {}) {
        if (query_x.size() != query_y.size()) throw RoboticsError(RoboticsError::InvalidParameter, "query_x / query_y sizes");
        const double pose[3] = {std::get<0>(initial_pose), std::get<1>(initial_pose), std::get<2>(initial_pose)};
        const uint64_t off[2] = {0, query_x.size()};
        const pfgpu_csm_config c = config.to_c();
        pfgpu_csm_result r{};
        check(pfgpu_csm_match(h_, &c, pose, 1, query_x.data(), query_y.data(), off, &r), "match");
        return from_c(r);
    }
    // Q queries: poses3 Q x (x, y, yaw); query q's points are qx[k], qy[k] for offsets[q] <= k < offsets[q + 1]
    std::vector<ScanMatchResult> match_batch(const std::vector<double>& poses3, const std::vector<double>& qx, const std::vector<double>& qy,
                                             const std::vector<uint64_t>& offsets, const CorrelativeScanMatcherConfig& config = {}) {
        const size_t Q = poses3.size() / 3;
        if (poses3.size() != 3 * Q || offsets.size() != Q + 1 || qx.size() != qy.size() || (Q && offsets[Q] != qx.size()))
            throw RoboticsError(RoboticsError::InvalidParameter, "match_batch: poses3 Q x 3, offsets Q + 1, offsets[Q] points");
        const pfgpu_csm_config c = config.to_c();
        std::vector<pfgpu_csm_result> r(Q);
        check(pfgpu_csm_match(h_, &c, poses3.data(), Q, qx.data(), qy.data(), offsets.data(), r.data()), "match_batch");
        std::vector<ScanMatchResult> out;
        for (const auto& x : r) out.push_back(from_c(x));
        return out;
    }
};

// correlative_scan_matching.rs:55-120 with its signature: a one-shot matcher on device 0
inline ScanMatchResult correlative_scan_match(const std::vector<double>& reference_x, const std::vector<double>& reference_y,
                                              const std::vector<double>& query_x, const std::vector<double>& query_y,
                                              std::tuple<double, double, double> initial_pose, const CorrelativeScanMatcherConfig& config) {
    CorrelativeScanMatcher m(0);
    m.set_reference(reference_x, reference_y);
    return m.match(query_x, query_y, initial_pose, config);
}

}  // namespace rust_robotics_b200
