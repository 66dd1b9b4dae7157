// cluster_check.cpp — drives the pose hypotheses through the C++ mirror (particle_filter.hpp): an MCL filter started from a region,
// a few landmark steps, then the five heaviest hypotheses and the first 64 per-slot ranks (-1 for a non-member), one number per
// line.  tests/test_gpu_hypotheses.py builds it, links libpfgpu.so and compares what it prints with the Python mirror on the same
// seed and inputs.
#include <cstdio>
#include <exception>
#include "particle_filter.hpp"

using namespace rust_robotics_b200;

int main() {
    try {
        MonteCarloLocalizationConfig c;
        c.min_particles = c.max_particles = 4096; c.velocity_noise = 0.2; c.yaw_rate_noise = 0.1;
        MonteCarloLocalizer f(c, 13, 0);
        f.init_region({-9.0, 9.0, -9.0, 9.0});
        const PFMeasurement z = {{5.0, 1.0, 1.0}, {4.0, -2.0, 0.5}, {6.0, 3.0, -3.0}};
        for (int t = 0; t < 4; ++t) f.try_step({1.0, 0.1}, z);
        size_t total = 0;
        std::vector<uint32_t> rank;
        const std::vector<pfgpu_pf_hypothesis> hs = f.hypotheses(5, 0.5, 24, &total, &rank);
        std::printf("%a\n", (double)total);
        for (const pfgpu_pf_hypothesis& h : hs) {
            std::printf("%a\n", h.mass);
            for (double m : h.mean) std::printf("%a\n", m);
            for (double v : h.cov) std::printf("%a\n", v);
            std::printf("%a\n%a\n%a\n", (double)h.count, (double)h.bins, (double)h.label);
        }
        for (size_t i = 0; i < 64 && i < rank.size(); ++i) std::printf("%a\n", rank[i] == UINT32_MAX ? -1.0 : (double)rank[i]);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "cluster_check: %s\n", e.what());
        return 1;
    }
    return 0;
}
