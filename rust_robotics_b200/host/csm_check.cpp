// csm_check.cpp — drives correlative scan matching through the C++ mirror (correlative_scan_matching.hpp): the reference's seven
// fixture points, one shifted query through correlative_scan_match, then a batch of two queries (the second one empty) on a
// CorrelativeScanMatcher; each result as x y yaw score (hex floats) and converged on a line.  tests/test_gpu_csm.py builds it, links
// libpfgpu.so and compares what it prints with the CPU oracle.
#include <cstdio>
#include <exception>
#include "correlative_scan_matching.hpp"

using namespace rust_robotics_b200;

static void print(const ScanMatchResult& r) { std::printf("%a %a %a %a %d\n", r.x, r.y, r.yaw, r.score, r.converged ? 1 : 0); }

int main() {
    try {
        const std::vector<double> fx = {0.0, 1.0, 2.0, 0.0, 0.0, 1.0, 1.5}, fy = {0.0, 0.0, 0.0, 1.0, 2.0, 1.0, 2.0};
        std::vector<double> qx, qy;
        for (size_t i = 0; i < fx.size(); ++i) { qx.push_back(fx[i] + 0.1); qy.push_back(fy[i] - 0.05); }
        CorrelativeScanMatcherConfig c;
        c.linear_search_range = 0.3; c.angular_search_range = 0.1; c.linear_step = 0.05; c.angular_step = 0.02; c.grid_resolution = 0.05;
        print(correlative_scan_match(fx, fy, qx, qy, {0.0, 0.0, 0.0}, c));
        CorrelativeScanMatcher m(0);
        m.set_reference(fx, fy);
        for (const auto& r : m.match_batch({0.2, -0.1, 0.05, 0.5, 0.5, 7.0}, fx, fy, {0, fx.size(), fx.size()}, c)) print(r);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "csm_check: %s\n", e.what());
        return 1;
    }
    return 0;
}
