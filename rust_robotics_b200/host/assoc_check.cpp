// assoc_check.cpp — drives fastslam2::FastSlam::update_unknown of the C++ mirror (fastslam1.hpp): a fresh map, a few steps with
// observations that carry no landmark id, then the counts and the best particle.  tests/test_gpu_assoc.py builds it, links
// libpfgpu.so and compares what it prints with the Python mirror's fastslam2_update_unknown on the same seed and inputs.
#include <cstdio>
#include <exception>
#include "fastslam1.hpp"

using namespace rust_robotics_b200;

int main() {
    try {
        fastslam2::FastSlam fs(1000, 6, 42, 0);
        const std::vector<std::pair<double, double>> z = {{5.0, 0.1}, {7.0, -0.4}, {5.1, 0.12}};
        for (int t = 0; t < 4; ++t) {
            const bool did = fastslam2::fastslam2_update_unknown(fs, {1.0, 0.1}, z);
            const auto c = fs.assoc_counts();
            std::printf("%d %llu %llu %llu\n", did ? 1 : 0, (unsigned long long)c[0], (unsigned long long)c[1], (unsigned long long)c[2]);
        }
        const fastslam1::Particle p = fastslam2::get_best_particle(fs);
        std::printf("%.17g\n%.17g\n%.17g\n%.17g\n", p.weight, p.x, p.y, p.yaw);
        for (const auto& l : p.landmarks) std::printf("%.17g\n%.17g\n%.17g\n", l.x, l.y, l.cov[0]);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "assoc_check: %s\n", e.what());
        return 1;
    }
    return 0;
}
