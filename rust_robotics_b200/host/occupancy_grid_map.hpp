// occupancy_grid_map.hpp — C++ host-side mirror of the reference's OccupancyGridMap over the C ABI (include/pfgpu.h, DESIGN §3.12),
// with the SAME type names, method names and argument meaning as crates/rust_robotics_mapping/src/occupancy_grid_map.rs.  The grid
// lives on the device; `grid()` downloads it.  Header-only; link against libpfgpu.so.  No CPU fallback.
#pragma once
#include <cmath>
#include <cstdint>
#include <optional>
#include <utility>
#include <vector>
#include "particle_filter.hpp"    // RoboticsError, check

namespace rust_robotics_b200 {

struct OccupancyGridConfig {                                             // occupancy_grid_map.rs:6-41
    double resolution = 0.5;
    size_t width = 100, height = 100;
    double prior_log_odds = 0.0, occupied_log_odds = 0.85, free_log_odds = -0.4, max_log_odds = 5.0, min_log_odds = -5.0;
    pfgpu_ogm_config to_c() const {
        pfgpu_ogm_config c{};
        c.resolution = resolution; c.width = width; c.height = height; c.prior_log_odds = prior_log_odds;
        c.occupied_log_odds = occupied_log_odds; c.free_log_odds = free_log_odds; c.max_log_odds = max_log_odds; c.min_log_odds = min_log_odds;
        return c;
    }
};

class OccupancyGridMap {                                                 // occupancy_grid_map.rs:43-160
    pfgpu_ogm* h_ = nullptr;
public:
    OccupancyGridConfig config;
    explicit OccupancyGridMap(OccupancyGridConfig c, int device = 0) : config(c) {
        const pfgpu_ogm_config cc = c.to_c();
        check(pfgpu_ogm_create(&cc, device, &h_), "occupancy grid");
    }
    OccupancyGridMap(const OccupancyGridMap&) = delete;
    OccupancyGridMap& operator=(const OccupancyGridMap&) = delete;
    ~OccupancyGridMap() { pfgpu_ogm_destroy(h_); }
    const pfgpu_ogm* handle() const { return h_; }

    void update_with_scan(double robot_x, double robot_y, double robot_yaw, const std::vector<double>& scan_ranges, double angle_min,
                          double angle_increment) {
        const double pose[3] = {robot_x, robot_y, robot_yaw};
        check(pfgpu_ogm_update_scans(h_, pose, 1, scan_ranges.data(), scan_ranges.size(), angle_min, angle_increment), "update_with_scan");
    }
    // S scans in order: poses3 S x (x, y, yaw), ranges S x B row-major
    void update_with_scans(const std::vector<double>& poses3, const std::vector<double>& ranges, size_t n_ranges, double angle_min,
                           double angle_increment) {
        const size_t S = poses3.size() / 3;
        if (poses3.size() != 3 * S || ranges.size() != S * n_ranges)
            throw RoboticsError(RoboticsError::InvalidParameter, "update_with_scans: poses3 S x 3, ranges S x n_ranges");
        check(pfgpu_ogm_update_scans(h_, poses3.data(), S, ranges.data(), n_ranges, angle_min, angle_increment), "update_with_scans");
    }
    double get_probability(size_t ix, size_t iy) const {
        double l = 0.0;
        check(pfgpu_ogm_read(h_, ix * config.height + iy, 1, &l), "get_probability");
        return 1.0 - 1.0 / (1.0 + std::exp(l));
    }
    std::optional<std::pair<size_t, size_t>> world_to_grid(double x, double y) const {
        const int64_t ix = sat(std::floor(x / config.resolution + (double)config.width / 2.0));
        const int64_t iy = sat(std::floor(y / config.resolution + (double)config.height / 2.0));
        if (ix >= 0 && ix < (int64_t)config.width && iy >= 0 && iy < (int64_t)config.height) return std::make_pair((size_t)ix, (size_t)iy);
        return std::nullopt;
    }
    bool is_occupied(size_t ix, size_t iy, double threshold) const { return get_probability(ix, iy) > threshold; }
    // grid[ix * height + iy]
    std::vector<double> grid() const {
        std::vector<double> g(config.width * config.height);
        check(pfgpu_ogm_read(h_, 0, g.size(), g.data()), "grid");
        return g;
    }
    std::vector<uint8_t> obstacles(double threshold = 0.5) const {
        std::vector<uint8_t> m(config.width * config.height);
        check(pfgpu_ogm_obstacles(h_, threshold, m.data(), m.size()), "obstacles");
        return m;
    }
    pfgpu_ogm_stats stats() const {
        pfgpu_ogm_stats s{};
        check(pfgpu_ogm_info(h_, nullptr, nullptr, &s), "stats");
        return s;
    }
private:
    static int64_t sat(double v) {                                       // Rust's `as i32`
        if (v != v) return 0;
        if (v >= 2147483647.0) return 2147483647;
        if (v <= -2147483648.0) return -2147483648LL;
        return (int64_t)v;
    }
};

}  // namespace rust_robotics_b200
