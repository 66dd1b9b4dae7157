// beam_check.cpp — drives the beam scan model through the C++ mirror (particle_filter.hpp): an MCL filter with a 20 m x 20 m walled
// room at 10 cm loaded as a beam map, started from a region, a few beam steps and one beam update, printing the estimate after each,
// then the expected ranges of two poses.  tests/test_gpu_beam.py builds it, links libpfgpu.so and compares what it prints with the
// Python mirror on the same seed and inputs.
#include <array>
#include <cmath>
#include <cstdio>
#include <exception>
#include "particle_filter.hpp"

using namespace rust_robotics_b200;

int main() {
    try {
        MonteCarloLocalizationConfig c;
        c.min_particles = c.max_particles = 4096; c.velocity_noise = 0.2; c.yaw_rate_noise = 0.1;
        MonteCarloLocalizer f(c, 13, 0);
        const size_t W = 200, H = 200;
        std::vector<uint8_t> mask(W * H, 0);
        for (size_t i = 0; i < W; ++i)
            for (size_t j = 0; j < H; ++j)
                mask[i * H + j] = (i < 2 || j < 2 || i >= W - 2 || j >= H - 2 || (i >= 120 && i < 124 && j < 130)) ? 1 : 0;
        pfgpu_beam_config bc = MonteCarloLocalizer::beam_defaults(0.1);
        bc.max_range = 12.0;
        f.set_beam_model(mask, W, H, bc);
        f.init_region({-9.0, 9.0, -9.0, 9.0});
        for (int t = 0; t < 8; ++t) {
            std::vector<double> ranges(90);
            for (size_t i = 0; i < ranges.size(); ++i) ranges[i] = 2.0 + 0.05 * (double)((i * 7 + (size_t)t) % 40);
            ranges[(size_t)t] = INFINITY;
            const PFState e = f.try_step_beam_scan({1.0, 0.1}, ranges, -M_PI, 2.0 * M_PI / 90.0);
            std::printf("%a %a %a\n", e[0], e[1], e[2]);
        }
        f.try_update_with_beam_scan(std::vector<double>(90, 3.0), -M_PI, 2.0 * M_PI / 90.0);
        const PFState e = f.estimate();
        std::printf("%a %a %a\n", e[0], e[1], e[2]);
        const std::vector<std::array<double, 3>> poses = {{0.5, -1.0, 0.3}, {3.0, 3.0, -2.0}};
        for (double r : f.expected_scan(poses, 5, -1.0, 0.5)) std::printf("%a\n", r);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "beam_check: %s\n", e.what());
        return 1;
    }
    return 0;
}
