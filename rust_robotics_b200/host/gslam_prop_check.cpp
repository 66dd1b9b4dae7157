// gslam_prop_check.cpp — drives grid FastSLAM's scan-matched proposal through the C++ mirror (grid_fastslam.hpp): 16 particles on a
// 12 m x 8 m grid at 10 cm with the default proposal and min_hits 2, six steps of a 90-beam scan with odometry, then (one line each)
// the poses and weights as hex floats, the last step's took flags and eta as hex floats, and whether the handle reports the
// proposal enabled.  tests/test_gpu_gslam_proposal.py builds it, links libpfgpu.so and compares what it prints with the CPU oracle.
#include <cmath>
#include <cstdio>
#include <exception>
#include "grid_fastslam.hpp"

using namespace rust_robotics_b200;

int main() {
    try {
        GridFastSlamConfig c;
        c.grid.resolution = 0.1; c.grid.width = 120; c.grid.height = 80;
        c.n_particles = 16; c.nth = 12.0;
        GridFastSlam f(c, {0.2, -0.1, 0.3}, 11, 0);
        GridFastSlamProposal p;
        p.min_hits = 2;
        f.set_proposal(&p);
        std::vector<double> ranges(90);
        for (size_t i = 0; i < ranges.size(); ++i) ranges[i] = 0.5 + 0.1 * (double)((i * 7) % 50);
        ranges[5] = INFINITY;
        for (int t = 0; t < 6; ++t) f.step({0.1 * t, 0.0, 0.02 * t}, {0.1 * t + 0.1, 0.01, 0.02 * t + 0.02}, ranges, -M_PI, 2.0 * M_PI / 90.0);
        for (double v : f.particles()) std::printf("%a ", v);
        std::printf("\n");
        for (double v : f.weights()) std::printf("%a ", v);
        std::printf("\n");
        const GridFastSlam::Proposal lp = f.last_proposal();
        for (uint8_t v : lp.took) std::printf("%u ", (unsigned)v);
        std::printf("\n");
        for (double v : lp.eta) std::printf("%a ", v);
        std::printf("\n");
        std::printf("%u\n", f.proposal().enabled);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "gslam_prop_check: %s\n", e.what());
        return 1;
    }
    return 0;
}
