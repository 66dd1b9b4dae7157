// existence_check.cpp — drives the landmark existence counters of the C++ mirror (fastslam1.hpp): a fresh map with counters
// enabled, a few unknown-association steps, the removals of each, then the best particle's counters.  tests/test_gpu_existence.py
// builds it, links libpfgpu.so and compares what it prints with the Python mirror on the same seed and inputs.
#include <cstdio>
#include <exception>
#include "fastslam1.hpp"

using namespace rust_robotics_b200;

int main() {
    try {
        fastslam2::FastSlam fs(1000, 6, 42, 0);
        fs.enable_existence(6.0);
        for (int t = 0; t < 6; ++t) {
            const std::vector<std::pair<double, double>> z = t % 3 != 2 ? std::vector<std::pair<double, double>>{{5.0, 0.1}, {7.0, -0.4}}
                                                                        : std::vector<std::pair<double, double>>{{3.0, 1.2}};
            const bool did = fastslam2::fastslam2_update_unknown(fs, {1.0, 0.1}, z);
            std::printf("%d %llu\n", did ? 1 : 0, (unsigned long long)fs.removed_count());
        }
        for (int32_t v : fs.existence_counts(fs.best_index(), 1)) std::printf("%d\n", v);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "existence_check: %s\n", e.what());
        return 1;
    }
    return 0;
}
