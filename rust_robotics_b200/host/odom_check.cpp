// odom_check.cpp — drives the odometry motion model through the C++ mirror (particle_filter.hpp): a PF with landmark steps and an MCL
// filter with a 20 m x 20 m walled room at 10 cm as a beam map, each moved by odometry pairs (a turn in place, a stop, a reverse),
// printing the estimate after each step.  tests/test_gpu_odom.py builds it, links libpfgpu.so and compares what it prints with the
// Python mirror on the same seed and inputs.
#include <array>
#include <cmath>
#include <cstdio>
#include <exception>
#include "particle_filter.hpp"

using namespace rust_robotics_b200;

int main() {
    try {
        const std::array<std::array<double, 3>, 7> odom = {{{0.0, 0.0, 0.0}, {0.1, 0.0, 0.01}, {0.1, 0.0, 0.4}, {0.1, 0.0, 0.4},
                                                           {0.05, -0.02, 0.41}, {0.15, 0.02, 0.42}, {0.25, 0.06, 0.43}}};
        ParticleFilterConfig pc;
        pc.n_particles = 4096;
        ParticleFilterLocalizer p(pc, 7, 0);
        p.set_odometry_noise({0.1, 0.05, 0.1, 0.05});
        const PFMeasurement z = {{5.0, 3.0, 4.0}, {4.0, -2.0, 3.5}, {6.5, 1.0, -6.0}};
        for (size_t t = 0; t + 1 < odom.size(); ++t) {
            const PFState e = p.try_step_odometry(odom[t], odom[t + 1], z);
            std::printf("%a %a %a\n", e[0], e[1], e[2]);
        }
        const auto a = p.odometry_noise();
        std::printf("%a %a %a %a\n", a[0], a[1], a[2], a[3]);
        MonteCarloLocalizationConfig c;
        c.min_particles = c.max_particles = 4096;
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
        for (size_t t = 0; t + 1 < odom.size(); ++t) {
            std::vector<double> ranges(90);
            for (size_t i = 0; i < ranges.size(); ++i) ranges[i] = 2.0 + 0.05 * (double)((i * 7 + t) % 40);
            const PFState e = f.try_step_beam_scan_odometry(odom[t], odom[t + 1], ranges, -M_PI, 2.0 * M_PI / 90.0);
            std::printf("%a %a %a\n", e[0], e[1], e[2]);
        }
        f.try_predict_with_odometry(odom[0], odom[1]);
        const PFState e = f.estimate();
        std::printf("%a %a %a\n", e[0], e[1], e[2]);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "odom_check: %s\n", e.what());
        return 1;
    }
    return 0;
}
