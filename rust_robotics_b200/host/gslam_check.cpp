// gslam_check.cpp — drives grid-based FastSLAM through the C++ mirror (grid_fastslam.hpp): 16 particles on a 12 m x 8 m grid at
// 10 cm, six steps of a 90-beam scan with odometry, then (one line each) the poses and weights as hex floats, the last step's
// ancestors, its stats (resampled, copies, events) and the best particle's grid; finally that grid handed to an OccupancyGridMap.
// tests/test_gpu_gslam.py builds it, links libpfgpu.so and compares what it prints with the CPU oracle.
#include <cmath>
#include <cstdio>
#include <exception>
#include "grid_fastslam.hpp"

using namespace rust_robotics_b200;

int main() {
    try {
        GridFastSlamConfig c;
        c.grid.resolution = 0.1; c.grid.width = 120; c.grid.height = 80;
        c.n_particles = 16; c.nth = 12.0;
        GridFastSlam f(c, {0.2, -0.1, 0.3}, 11, 0);
        std::vector<double> ranges(90);
        for (size_t i = 0; i < ranges.size(); ++i) ranges[i] = 0.5 + 0.1 * (double)((i * 7) % 50);
        ranges[5] = INFINITY;
        for (int t = 0; t < 6; ++t) f.step({0.1 * t, 0.0, 0.02 * t}, {0.1 * t + 0.1, 0.01, 0.02 * t + 0.02}, ranges, -M_PI, 2.0 * M_PI / 90.0);
        for (double v : f.particles()) std::printf("%a ", v);
        std::printf("\n");
        for (double v : f.weights()) std::printf("%a ", v);
        std::printf("\n");
        for (uint32_t v : f.last_indices()) std::printf("%u ", v);
        std::printf("\n");
        const pfgpu_gs_stats s = f.stats();
        std::printf("%llu %llu %llu\n", (unsigned long long)s.resampled, (unsigned long long)s.copies, (unsigned long long)s.events);
        const auto b = f.best();
        for (double v : f.grid(b.first)) std::printf("%a ", v);
        std::printf("\n");
        OccupancyGridMap m(c.grid, 0);
        f.copy_grid_to(b.first, m);
        std::printf("%d\n", m.grid() == f.grid(b.first) ? 1 : 0);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "gslam_check: %s\n", e.what());
        return 1;
    }
    return 0;
}
