// ogm_check.cpp — drives occupancy grid mapping through the C++ mirror (occupancy_grid_map.hpp): a 12 m x 8 m grid at 10 cm, four
// 90-beam scans, then the grid (hex floats on one line) and the number of obstacle cells at 0.5; finally the grid handed to an MCL
// filter's beam model.  tests/test_gpu_ogm.py builds it, links libpfgpu.so and compares what it prints with the CPU oracle.
#include <cmath>
#include <cstdio>
#include <exception>
#include "occupancy_grid_map.hpp"

using namespace rust_robotics_b200;

int main() {
    try {
        OccupancyGridConfig c;
        c.resolution = 0.1; c.width = 120; c.height = 80;
        OccupancyGridMap m(c, 0);
        std::vector<double> ranges(90);
        for (size_t i = 0; i < ranges.size(); ++i) ranges[i] = 0.5 + 0.1 * (double)((i * 7) % 50);
        ranges[5] = INFINITY;
        for (int s = 0; s < 4; ++s) m.update_with_scan(0.5 * s - 1.0, 0.2 * s, 0.3 * s, ranges, -M_PI, 2.0 * M_PI / 90.0);
        for (double v : m.grid()) std::printf("%a ", v);
        std::printf("\n");
        size_t occ = 0;
        for (uint8_t b : m.obstacles(0.5)) occ += b;
        std::printf("%zu\n", occ);
        MonteCarloLocalizationConfig mc;
        mc.min_particles = mc.max_particles = 1024;
        MonteCarloLocalizer f(mc, 3, 0);
        f.set_beam_model_from_grid(m.handle(), 0.5, MonteCarloLocalizer::beam_defaults(c.resolution));
    } catch (const std::exception& e) {
        std::fprintf(stderr, "ogm_check: %s\n", e.what());
        return 1;
    }
    return 0;
}
