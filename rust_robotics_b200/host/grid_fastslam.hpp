// grid_fastslam.hpp — C++ host-side mirror of grid-based FastSLAM over the C ABI (include/pfgpu.h pfgpu_gs_*, DESIGN §3.16), with
// the Python mirror's names (GridFastSlam).  The particles and their grids live on the device.  Header-only; link against
// libpfgpu.so.  No CPU fallback.
#pragma once
#include <array>
#include <utility>
#include <vector>
#include "occupancy_grid_map.hpp"

namespace rust_robotics_b200 {

struct GridFastSlamConfig {
    OccupancyGridConfig grid;
    size_t n_particles = 100;
    double nth = 50.0;              // resample when N_eff < nth
    double z_hit = 0.95, z_rand = 0.05, max_range = 30.0;
    uint32_t max_beams = 60, search_radius = 1;
    pfgpu_gs_config to_c() const {
        pfgpu_gs_config c{};
        c.ogm = grid.to_c(); c.n_particles = n_particles; c.nth = nth; c.z_hit = z_hit; c.z_rand = z_rand; c.max_range = max_range;
        c.max_beams = max_beams; c.search_radius = search_radius;
        return c;
    }
};

// the scan-matched proposal's parameters (pfgpu_gs_proposal without `enabled`), the defaults of pfgpu_gs_default_proposal
struct GridFastSlamProposal {
    double linear_range = 0.1, linear_step = 0.025, angular_range = 0.05, angular_step = 0.0125;
    uint32_t half_width = 1;
    double lattice_linear_step = 0.01, lattice_angular_step = 0.005;
    uint32_t min_hits = 10;
    pfgpu_gs_proposal to_c() const {
        pfgpu_gs_proposal c{};
        c.half_width = half_width; c.linear_range = linear_range; c.linear_step = linear_step; c.angular_range = angular_range;
        c.angular_step = angular_step; c.lattice_linear_step = lattice_linear_step; c.lattice_angular_step = lattice_angular_step;
        c.min_hits = min_hits;
        return c;
    }
};

class GridFastSlam {
    pfgpu_gs* h_ = nullptr;
public:
    GridFastSlamConfig config;
    GridFastSlam(GridFastSlamConfig c, const std::array<double, 3>& start_pose, uint64_t seed = 0, int device = 0) : config(c) {
        const pfgpu_gs_config cc = c.to_c();
        check(pfgpu_gs_create(&cc, seed, start_pose.data(), device, &h_), "grid FastSLAM");
    }
    GridFastSlam(const GridFastSlam&) = delete;
    GridFastSlam& operator=(const GridFastSlam&) = delete;
    ~GridFastSlam() { pfgpu_gs_destroy(h_); }

    void set_odometry_noise(const std::array<double, 4>& alpha) { check(pfgpu_gs_set_odom_noise(h_, alpha.data()), "set_odometry_noise"); }
    std::array<double, 4> odometry_noise() const {
        std::array<double, 4> a{};
        check(pfgpu_gs_odom_noise(h_, a.data()), "odometry_noise");
        return a;
    }
    // one step: the odometry poses (x, y, yaw) before and after it and the scan taken after it; enqueued, not waited for
    void step(const std::array<double, 3>& odom_prev, const std::array<double, 3>& odom_cur, const std::vector<double>& ranges,
              double angle_min, double angle_increment) {
        const double o[6] = {odom_prev[0], odom_prev[1], odom_prev[2], odom_cur[0], odom_cur[1], odom_cur[2]};
        check(pfgpu_gs_step(h_, o, ranges.data(), ranges.size(), angle_min, angle_increment), "step");
    }
    // n x (x, y, yaw)
    std::vector<double> particles() const {
        std::vector<double> p(3 * config.n_particles);
        check(pfgpu_gs_download(h_, p.data(), nullptr, config.n_particles), "particles");
        return p;
    }
    std::vector<double> weights() const {
        std::vector<double> w(config.n_particles);
        check(pfgpu_gs_download(h_, nullptr, w.data(), config.n_particles), "weights");
        return w;
    }
    // (slot, pose) of the largest weight, ties to the lowest slot
    std::pair<size_t, std::array<double, 3>> best() const {
        size_t s = 0;
        std::array<double, 3> p{};
        check(pfgpu_gs_best(h_, &s, p.data()), "best");
        return {s, p};
    }
    // slot's grid[ix * height + iy]
    std::vector<double> grid(size_t slot) const {
        std::vector<double> g(config.grid.width * config.grid.height);
        check(pfgpu_gs_grid_read(h_, slot, 0, g.size(), g.data()), "grid");
        return g;
    }
    // slot's grid into an OccupancyGridMap of the same config on the same device, without leaving the device
    void copy_grid_to(size_t slot, OccupancyGridMap& m) { check(pfgpu_gs_grid_to_ogm(h_, slot, const_cast<pfgpu_ogm*>(m.handle())), "copy_grid_to"); }
    std::vector<uint32_t> last_indices() const {
        std::vector<uint32_t> idx(config.n_particles);
        size_t n = 0;
        check(pfgpu_gs_last_indices(h_, idx.data(), idx.size(), &n), "last_indices");
        idx.resize(n);
        return idx;
    }
    pfgpu_gs_stats stats() const {
        pfgpu_gs_stats s{};
        check(pfgpu_gs_info(h_, nullptr, nullptr, nullptr, nullptr, &s), "stats");
        return s;
    }
    // the scan-matched proposal (DESIGN §3.17): enabled with a config, disabled with nullptr; applies from the next step
    void set_proposal(const GridFastSlamProposal* p) {
        pfgpu_gs_proposal c{};
        pfgpu_gs_default_proposal(&c);
        if (p) { c = p->to_c(); c.enabled = 1; }
        check(pfgpu_gs_set_proposal(h_, &c), "set_proposal");
    }
    pfgpu_gs_proposal proposal() const {
        pfgpu_gs_proposal c{};
        check(pfgpu_gs_get_proposal(h_, &c), "proposal");
        return c;
    }
    // the last step's per-slot match winners (n x 3), eta and whether each particle took the proposal
    struct Proposal { std::vector<double> matched, eta; std::vector<uint8_t> took; };
    Proposal last_proposal() const {
        Proposal r{std::vector<double>(3 * config.n_particles), std::vector<double>(config.n_particles), std::vector<uint8_t>(config.n_particles)};
        check(pfgpu_gs_last_proposal(h_, r.matched.data(), r.eta.data(), r.took.data(), config.n_particles), "last_proposal");
        return r;
    }
    void sync() { check(pfgpu_gs_sync(h_), "sync"); }
};

}  // namespace rust_robotics_b200
