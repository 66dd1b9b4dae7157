// fastslam1.hpp — C++ host-side mirror of crates/rust_robotics_slam/src/fastslam1.rs (fs1.rs) over include/pfgpu.h.
// The reference is a set of free functions over a caller-owned Vec<Particle>; the GPU form keeps the particles on the
// device inside an engine object (SURVEY.md §8b) and offers the same four entry points under the same names.
#pragma once
#include <array>
#include <tuple>
#include <utility>
#include <vector>
#include "pfgpu.h"
#include "particle_filter.hpp"

namespace rust_robotics_b200 { namespace fastslam1 {

struct Landmark { double x, y; std::array<double, 4> cov; };              // fs1.rs:27-31 (cov row-major c00 c01 c10 c11)
struct Particle { double weight, x, y, yaw; std::vector<Landmark> landmarks; };   // fs1.rs:45-51
using Observation = std::tuple<double, double, size_t>;                   // (distance, angle, landmark_id) fs1.rs:240
// weighted posterior estimate (no reference counterpart; include/pfgpu.h pfgpu_fs_moments): pose mean (x, y, yaw) and covariance
// (column-major), per landmark the weight mass of the copies with cov00 < cov00_max, their mean and mixture covariance
struct Estimate {
    std::array<double, 3> pose; std::array<double, 9> pose_cov;
    std::vector<double> mass; std::vector<std::array<double, 2>> mean; std::vector<std::array<double, 4>> cov;
};
// one step of a particle's path (include/pfgpu.h pfgpu_fs_path): step number, the lineage's global slot then, its pose
struct PathEntry { uint64_t step; uint32_t slot; double x, y, yaw; };

class FastSlam {
    pfgpu_fs* h_ = nullptr;
    size_t n_ = 0, m_ = 0;
public:
    FastSlam(size_t n_particles, size_t n_landmarks, uint64_t seed = 42, int device = 0, const pfgpu_fs_config* cfg = nullptr) {
        pfgpu_fs_config c; pfgpu_fs_default_config(&c); if (cfg) c = *cfg;
        check(pfgpu_fs_create(&c, n_particles, n_landmarks, seed, device, &h_), "create_particles");
        n_ = n_particles; m_ = n_landmarks;
    }
    FastSlam(const FastSlam&) = delete;
    FastSlam& operator=(const FastSlam&) = delete;
    ~FastSlam() { pfgpu_fs_destroy(h_); }
    // fastslam_update fs1.rs:237-266
    bool step(const std::array<double, 2>& u, const std::vector<Observation>& z) {
        std::vector<pfgpu_fs_obs> o(z.size());
        for (size_t i = 0; i < z.size(); ++i) { o[i].d = std::get<0>(z[i]); o[i].angle = std::get<1>(z[i]); o[i].lm_id = std::get<2>(z[i]); }
        int did = 0;
        check(pfgpu_fs_step(h_, u.data(), o.data(), o.size(), &did), "fastslam_update");
        return did != 0;
    }
    // the odometry motion model (no reference counterpart; DESIGN §3.15): ROS AMCL's odom_alpha1..4, each finite and >= 0 (0.2 each
    // at creation)
    void set_odometry_noise(const std::array<double, 4>& alpha) { check(pfgpu_fs_set_odom_noise(h_, alpha.data()), "set_odometry_noise"); }
    std::array<double, 4> odometry_noise() const {
        std::array<double, 4> a{};
        check(pfgpu_fs_odom_noise(h_, a.data()), "odometry_noise");
        return a;
    }
    // step with the odometry motion model: every particle moves by the increment from odometry pose prev = (x, y, yaw) to cur
    bool step_odometry(const std::array<double, 3>& prev, const std::array<double, 3>& cur, const std::vector<Observation>& z) {
        std::vector<pfgpu_fs_obs> o(z.size());
        for (size_t i = 0; i < z.size(); ++i) { o[i].d = std::get<0>(z[i]); o[i].angle = std::get<1>(z[i]); o[i].lm_id = std::get<2>(z[i]); }
        const std::array<double, 6> od = { prev[0], prev[1], prev[2], cur[0], cur[1], cur[2] };
        int did = 0;
        check(pfgpu_fs_step_odom(h_, od.data(), o.data(), o.size(), &did), "fastslam_update_odometry");
        return did != 0;
    }
    // get_best_particle fs1.rs:269-274 (pose + weight + that particle's landmarks, what render_gif_slam.rs:183-191 reads)
    Particle best() const {
        size_t idx = 0; double pw[4];
        check(pfgpu_fs_best(h_, &idx, pw), "get_best_particle");
        Particle p{pw[0], pw[1], pw[2], pw[3], {}};
        std::vector<double> lm(6 * m_);
        check(pfgpu_fs_particle_landmarks(h_, idx, lm.data()), "landmarks");
        for (size_t l = 0; l < m_; ++l) p.landmarks.push_back({lm[6 * l], lm[6 * l + 1], {lm[6 * l + 2], lm[6 * l + 3], lm[6 * l + 4], lm[6 * l + 5]}});
        return p;
    }
    // Vec<Particle> view (checkpoint / API-compat tests)
    std::vector<Particle> download() const {
        std::vector<double> pw(4 * n_), lm(6 * n_ * m_);
        check(pfgpu_fs_download(h_, pw.data(), lm.data(), n_), "download");
        std::vector<Particle> out(n_);
        for (size_t i = 0; i < n_; ++i) {
            out[i] = {pw[4 * i], pw[4 * i + 1], pw[4 * i + 2], pw[4 * i + 3], {}};
            for (size_t l = 0; l < m_; ++l) { const double* q = &lm[(i * m_ + l) * 6]; out[i].landmarks.push_back({q[0], q[1], {q[2], q[3], q[4], q[5]}}); }
        }
        return out;
    }
    // pfgpu_fs_moments + pfgpu_fs_estimate_merge on this (one-GPU) engine; landmarks = false: pose only
    Estimate estimate(double cov00_max = 100.0, bool landmarks = true) const {
        pfgpu_fs_pose_moments pm;
        std::vector<pfgpu_fs_lm_moments> lm(landmarks ? m_ : 0);
        check(pfgpu_fs_moments(h_, cov00_max, &pm, landmarks ? lm.data() : nullptr), "estimate");
        Estimate e;
        const size_t m = lm.size();
        e.mass.resize(m); e.mean.resize(m); e.cov.resize(m);
        const pfgpu_fs_lm_moments* one = lm.data();
        check(pfgpu_fs_estimate_merge(&pm, landmarks ? &one : nullptr, 1, m, e.pose.data(), e.pose_cov.data(), e.mass.data(),
                                      m ? e.mean[0].data() : nullptr, m ? e.cov[0].data() : nullptr), "estimate");
        return e;
    }
    // path history (no reference counterpart; include/pfgpu.h pfgpu_fs_history_enable): keep the last `capacity` steps of every
    // particle's path on the device; 0 disables
    void enable_history(size_t capacity) { check(pfgpu_fs_history_enable(h_, capacity), "enable_history"); }
    // the path of global slot `index` (the poses of its lineage), oldest first, at most max_steps entries
    std::vector<PathEntry> path(size_t index, size_t max_steps) const {
        std::vector<uint64_t> step(max_steps); std::vector<uint32_t> slot(max_steps); std::vector<double> pose(3 * max_steps);
        size_t n = 0;
        check(pfgpu_fs_path(h_, index, max_steps, step.data(), slot.data(), pose.data(), &n), "path");
        std::vector<PathEntry> out(n);
        for (size_t j = 0; j < n; ++j) out[j] = {step[j], slot[j], pose[3 * j], pose[3 * j + 1], pose[3 * j + 2]};
        return out;
    }
    // the path of the best particle (get_best_particle's index)
    std::vector<PathEntry> best_path(size_t max_steps) const {
        size_t idx = 0;
        check(pfgpu_fs_best(h_, &idx, nullptr), "get_best_particle");
        return path(idx, max_steps);
    }
    size_t len() const { return n_; }
    // 1 = fastslam1::fastslam_update, 2 = fastslam2::fastslam2_update (crates/rust_robotics_slam/src/fastslam2.rs:376-383)
    void set_variant(int variant) { check(pfgpu_fs_set_variant(h_, variant), "set_variant"); }
protected:
    pfgpu_fs* handle() const { return h_; }
};

// the reference's free-function names
inline FastSlam create_particles(size_t n_particles, size_t n_landmarks) = delete;   // engines are not copyable: construct FastSlam directly
inline bool fastslam_update(FastSlam& particles, const std::array<double, 2>& u, const std::vector<Observation>& z) { return particles.step(u, z); }
inline Particle get_best_particle(const FastSlam& particles) { return particles.best(); }
inline bool fastslam_update_odometry(FastSlam& particles, const std::array<double, 3>& prev, const std::array<double, 3>& cur,
                                     const std::vector<Observation>& z) { return particles.step_odometry(prev, cur, z); }

}  // namespace fastslam1

// crates/rust_robotics_slam/src/fastslam2.rs: the same engine object with the proposal-sampling step
namespace fastslam2 {
using fastslam1::Landmark; using fastslam1::Particle; using fastslam1::Observation; using fastslam1::get_best_particle;
struct FastSlam : fastslam1::FastSlam {
    FastSlam(size_t n_particles, size_t n_landmarks, uint64_t seed = 42, int device = 0, const pfgpu_fs_config* cfg = nullptr)
        : fastslam1::FastSlam(n_particles, n_landmarks, seed, device, cfg) { set_variant(2); }
    // observations WITHOUT landmark ids, (distance, angle): every particle associates them with its own map (pfgpu_fs_step_unknown)
    bool update_unknown(const std::array<double, 2>& u, const std::vector<std::pair<double, double>>& z, double gate_d2 = 16.0) {
        std::vector<double> z2(2 * z.size());
        for (size_t i = 0; i < z.size(); ++i) { z2[2 * i] = z[i].first; z2[2 * i + 1] = z[i].second; }
        int did = 0;
        check(pfgpu_fs_step_unknown(handle(), u.data(), z2.data(), z.size(), gate_d2, &did), "fastslam2_update_unknown");
        return did != 0;
    }
    // update_unknown with the odometry motion model (DESIGN §3.15)
    bool update_unknown_odometry(const std::array<double, 3>& prev, const std::array<double, 3>& cur,
                                 const std::vector<std::pair<double, double>>& z, double gate_d2 = 16.0) {
        std::vector<double> z2(2 * z.size());
        for (size_t i = 0; i < z.size(); ++i) { z2[2 * i] = z[i].first; z2[2 * i + 1] = z[i].second; }
        const std::array<double, 6> od = { prev[0], prev[1], prev[2], cur[0], cur[1], cur[2] };
        int did = 0;
        check(pfgpu_fs_step_unknown_odom(handle(), od.data(), z2.data(), z.size(), gate_d2, &did), "fastslam2_update_unknown_odometry");
        return did != 0;
    }
    // (matched, born, dropped) observations of the last update_unknown over all particles
    std::array<uint64_t, 3> assoc_counts() const {
        std::array<uint64_t, 3> c{};
        check(pfgpu_fs_assoc_counts(handle(), c.data()), "assoc_counts");
        return c;
    }
    // landmark existence counters (DESIGN §3.7): range > 0 (inf allowed) enables, 0 disables; every counter starts at 1
    void enable_existence(double range) { check(pfgpu_fs_existence_enable(handle(), range), "enable_existence"); }
    // the counters of particles first .. first + count - 1, count x m particle-major; 0 for an empty slot
    std::vector<int32_t> existence_counts(size_t first, size_t count) const {
        size_t nl = 0, ng = 0, m = 0;
        check(pfgpu_fs_count(handle(), &nl, &ng, &m), "count");
        std::vector<int32_t> out(count * m);
        check(pfgpu_fs_existence_counts(handle(), first, count, out.data()), "existence_counts");
        return out;
    }
    // landmark copies removed by the last update_unknown
    uint64_t removed_count() const {
        uint64_t r = 0;
        check(pfgpu_fs_existence_removed(handle(), &r), "removed_count");
        return r;
    }
    size_t best_index() const {
        size_t idx = 0;
        check(pfgpu_fs_best(handle(), &idx, nullptr), "get_best_particle");
        return idx;
    }
};
inline bool fastslam2_update(FastSlam& particles, const std::array<double, 2>& u, const std::vector<Observation>& z) { return particles.step(u, z); }
inline bool fastslam2_update_unknown(FastSlam& particles, const std::array<double, 2>& u, const std::vector<std::pair<double, double>>& z) {
    return particles.update_unknown(u, z);
}
}  // namespace fastslam2
}  // namespace rust_robotics_b200
