// fs_odom_check.cpp — drives FastSLAM's odometry motion model through the C++ mirror (fastslam1.hpp): FastSLAM 1.0 and 2.0 with
// known ids and FastSLAM 2.0 with unknown association, each moved by odometry pairs (a drive, a stop, a turn in place, a reverse),
// printing the best particle's weight and pose after each step.  tests/test_gpu_fs_odom.py builds it, links libpfgpu.so and compares
// what it prints with the Python mirror on the same seed and inputs.
#include <array>
#include <cmath>
#include <cstdio>
#include <exception>
#include "fastslam1.hpp"

using namespace rust_robotics_b200;

int main() {
    try {
        const std::array<std::array<double, 3>, 6> odom = {{{0.0, 0.0, 0.0}, {0.1, 0.0, 0.01}, {0.1, 0.0, 0.01}, {0.1, 0.0, 0.4},
                                                           {0.05, -0.02, 0.41}, {0.15, 0.02, 0.42}}};
        const std::vector<fastslam1::Observation> z = {{5.0, 0.6, 0}, {4.2, -0.5, 1}, {6.5, 2.0, 2}};
        const std::vector<std::pair<double, double>> z2 = {{5.0, 0.6}, {4.2, -0.5}, {6.5, 2.0}};
        pfgpu_fs_config c; pfgpu_fs_default_config(&c);
        c.nth = 1024 / 1.5;
        fastslam1::FastSlam f1(1024, 4, 7, 0, &c);
        fastslam2::FastSlam f2(1024, 4, 7, 0, &c);
        fastslam2::FastSlam fu(1024, 8, 7, 0, &c);
        f1.set_odometry_noise({0.1, 0.05, 0.1, 0.05});
        const auto a = f1.odometry_noise();
        std::printf("%a %a %a %a\n", a[0], a[1], a[2], a[3]);
        for (size_t t = 0; t + 1 < odom.size(); ++t) {
            fastslam1::fastslam_update_odometry(f1, odom[t], odom[t + 1], z);
            f2.step_odometry(odom[t], odom[t + 1], z);
            fu.update_unknown_odometry(odom[t], odom[t + 1], z2);
            for (const fastslam1::FastSlam* f : {static_cast<const fastslam1::FastSlam*>(&f1), static_cast<const fastslam1::FastSlam*>(&f2),
                                                 static_cast<const fastslam1::FastSlam*>(&fu)}) {
                const fastslam1::Particle p = f->best();
                std::printf("%a %a %a %a\n", p.weight, p.x, p.y, p.yaw);
            }
        }
    } catch (const std::exception& e) {
        std::fprintf(stderr, "fs_odom_check: %s\n", e.what());
        return 1;
    }
    return 0;
}
