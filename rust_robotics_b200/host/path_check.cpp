// path_check.cpp — drives FastSlam::best_path() of the C++ mirror (fastslam1.hpp): history enabled, a few fastslam_update steps,
// then the best particle's path.  tests/test_gpu_path.py builds it, links libpfgpu.so and compares what it prints with the
// Python mirror's path() on the same seed and inputs.
#include <cstdio>
#include <exception>
#include "fastslam1.hpp"

using namespace rust_robotics_b200;

int main() {
    try {
        fastslam1::FastSlam fs(1000, 4, 42, 0);
        fs.enable_history(100);
        const std::vector<fastslam1::Observation> z = {{5.0, 0.1, 0}, {7.0, -0.4, 2}};
        for (int t = 0; t < 5; ++t) fastslam1::fastslam_update(fs, {1.0, 0.1}, z);
        for (const auto& e : fs.best_path(100))
            std::printf("%llu\n%u\n%.17g\n%.17g\n%.17g\n", (unsigned long long)e.step, e.slot, e.x, e.y, e.yaw);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "path_check: %s\n", e.what());
        return 1;
    }
    return 0;
}
