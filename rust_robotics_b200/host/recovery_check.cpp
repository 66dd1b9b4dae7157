// recovery_check.cpp — drives augmented MCL through the C++ mirror (particle_filter.hpp): an MCL filter started from a region, a
// few steps from observations that fit, then ones that fit nowhere (every likelihood underflows: a kidnap), printing (w_slow, w_fast, p,
// injected) and the estimate after each.  tests/test_gpu_recovery.py builds it, links libpfgpu.so and compares what it prints with
// the Python mirror on the same seed and inputs.
#include <cstdio>
#include <exception>
#include "particle_filter.hpp"

using namespace rust_robotics_b200;

int main() {
    try {
        MonteCarloLocalizationConfig c;
        c.min_particles = c.max_particles = 4096; c.range_noise = 0.5; c.velocity_noise = 0.1; c.yaw_rate_noise = 0.05;
        MonteCarloLocalizer f(c, 11, 0);
        f.enable_recovery(0.1, 0.6, {-10.0, 10.0, -10.0, 10.0});
        f.init_region({-10.0, 10.0, -10.0, 10.0});
        const double lms[4][2] = {{10.0, 0.0}, {0.0, 10.0}, {-10.0, 0.0}, {0.0, -10.0}};
        for (int t = 0; t < 10; ++t) {
            PFMeasurement z;
            for (auto& l : lms) {
                const double dx = 2.0 + 0.1 * t - l[0], dy = -1.0 - l[1];
                z.emplace_back(t >= 5 ? 1.0e4 : __builtin_sqrt(dx * dx + dy * dy), l[0], l[1]);
            }
            const PFState e = f.try_step({1.0, 0.0}, z);
            const auto s = f.recovery_state();
            std::printf("%a %a %a %llu %a %a\n", s.w_slow, s.w_fast, s.p, (unsigned long long)s.injected, e[0], e[1]);
        }
    } catch (const std::exception& e) {
        std::fprintf(stderr, "recovery_check: %s\n", e.what());
        return 1;
    }
    return 0;
}
