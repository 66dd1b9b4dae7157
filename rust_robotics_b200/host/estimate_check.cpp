// estimate_check.cpp — drives FastSlam::estimate() of the C++ mirror (fastslam1.hpp): a few fastslam_update steps, then the
// estimate with every landmark copy counted (cov00_max = inf) and with the default filter.  tests/test_gpu_estimate.py builds it,
// links libpfgpu.so and compares what it prints with the Python mirror's estimate() on the same seed and inputs.
#include <cmath>
#include <cstdio>
#include <exception>
#include "fastslam1.hpp"

using namespace rust_robotics_b200;

static void print(const fastslam1::Estimate& e) {
    for (double v : e.pose) std::printf("%.17g\n", v);
    for (double v : e.pose_cov) std::printf("%.17g\n", v);
    for (size_t l = 0; l < e.mass.size(); ++l) {
        std::printf("%.17g\n%.17g\n%.17g\n", e.mass[l], e.mean[l][0], e.mean[l][1]);
        for (double v : e.cov[l]) std::printf("%.17g\n", v);
    }
}

int main() {
    try {
        fastslam1::FastSlam fs(1000, 4, 42, 0);
        const std::vector<fastslam1::Observation> z = {{5.0, 0.1, 0}, {7.0, -0.4, 2}};
        for (int t = 0; t < 3; ++t) fastslam1::fastslam_update(fs, {1.0, 0.1}, z);
        print(fs.estimate(INFINITY));
        print(fs.estimate());
        print(fs.estimate(100.0, false));
    } catch (const std::exception& e) {
        std::fprintf(stderr, "estimate_check: %s\n", e.what());
        return 1;
    }
    return 0;
}
