// particle_filter.hpp — C++ host-side mirror of the reference's ParticleFilterLocalizer / MonteCarloLocalizer over
// the C ABI (include/pfgpu.h).  The reference is compiled code (Rust) and this image has no Rust toolchain, so the
// host side above the ABI is written in C++ with the SAME type names, method names, argument meaning and error
// behaviour as crates/rust_robotics_localization/src/particle_filter.rs (pf.rs) and monte_carlo_localization.rs
// (mcl.rs).  Header-only; link against libpfgpu.so.  No CPU fallback: constructors throw when no CUDA device exists.
#pragma once
#include <array>
#include <stdexcept>
#include <string>
#include <tuple>
#include <vector>
#include "pfgpu.h"

namespace rust_robotics_b200 {

// crates/rust_robotics_core/src/error.rs:8-24 — this path only ever produces InvalidParameter
struct RoboticsError : std::runtime_error {
    enum Kind { InvalidParameter, Runtime } kind;
    RoboticsError(Kind k, const std::string& m) : std::runtime_error(m), kind(k) {}
};
inline void check(int status, const char* what) {
    if (status == PFGPU_OK) return;
    std::string msg = std::string(what) + ": " + pfgpu_strerror(status);
    if (status > 0) msg += std::string(" (") + pfgpu_last_error() + ")";
    throw RoboticsError(status < 0 ? RoboticsError::InvalidParameter : RoboticsError::Runtime, msg);
}

using PFState = std::array<double, 4>;                                   // Vector4<f64> pf.rs:16
using PFControl = std::array<double, 2>;                                 // Vector2<f64> pf.rs:19
using PFMeasurement = std::vector<std::tuple<double, double, double>>;   // (distance, landmark_x, landmark_y) pf.rs:22
struct Particle { double x, y, yaw, v, w; };                             // pf.rs:26-32

struct ParticleFilterConfig {                                            // pf.rs:52-78
    size_t n_particles = 100;
    double resample_threshold = 0.5, range_noise = 0.2, velocity_noise = 2.0;
    double yaw_rate_noise = 40.0 * 3.14159265358979323846 / 180.0, dt = 0.1;
    pfgpu_pf_config to_c() const { pfgpu_pf_config c{}; c.n_particles = n_particles; c.resample_threshold = resample_threshold;
        c.range_noise = range_noise; c.velocity_noise = velocity_noise; c.yaw_rate_noise = yaw_rate_noise; c.dt = dt; c.mode = 0;
        c.max_particles = n_particles; c.kld_epsilon = 0.05; c.kld_z = 2.326; return c; }
    void validate() const { auto c = to_c(); check(pfgpu_pf_config_validate(&c), "particle filter configuration"); }   // pf.rs:81-117
};

struct MonteCarloLocalizationConfig {                                    // mcl.rs:50-74
    size_t min_particles = 100, max_particles = 5000;
    double kld_epsilon = 0.05, kld_z = 2.326, range_noise = 0.2, velocity_noise = 2.0;
    double yaw_rate_noise = 40.0 * 3.14159265358979323846 / 180.0, dt = 0.1;
    pfgpu_pf_config to_c() const { pfgpu_pf_config c{}; c.n_particles = min_particles; c.range_noise = range_noise;
        c.velocity_noise = velocity_noise; c.yaw_rate_noise = yaw_rate_noise; c.dt = dt; c.mode = 1; c.max_particles = max_particles;
        c.kld_epsilon = kld_epsilon; c.kld_z = kld_z; return c; }
    void validate() const { auto c = to_c(); check(pfgpu_pf_config_validate(&c), "MCL configuration"); }               // mcl.rs:87-130
};

namespace detail {
class PfHandle {
protected:
    pfgpu_pf* h_ = nullptr;
    mutable std::vector<Particle> mirror_;     // get_particles() returns a reference in the reference API: lazily refreshed host mirror
    mutable bool dirty_ = true;
    PfHandle(const pfgpu_pf_config& c, uint64_t seed, int device) { check(pfgpu_pf_create(&c, seed, device, &h_), "create"); }
public:
    PfHandle(const PfHandle&) = delete;
    PfHandle& operator=(const PfHandle&) = delete;
    ~PfHandle() { pfgpu_pf_destroy(h_); }
    static std::vector<double> flat(const PFMeasurement& z) {
        std::vector<double> o; o.reserve(3 * z.size());
        for (auto& t : z) { o.push_back(std::get<0>(t)); o.push_back(std::get<1>(t)); o.push_back(std::get<2>(t)); }
        return o;
    }
    void try_predict_with_control(const PFControl& u) { check(pfgpu_pf_predict(h_, u.data()), "predict"); dirty_ = true; }        // pf.rs:255
    void try_update_with_observations(const PFMeasurement& z) { auto f = flat(z); check(pfgpu_pf_update(h_, f.data(), z.size()), "update"); dirty_ = true; }  // pf.rs:310
    void resample() { int did = 0; check(pfgpu_pf_resample(h_, &did), "resample"); dirty_ = true; }                               // pf.rs:337
    PFState try_step(const PFControl& u, const PFMeasurement& z) {                                                               // pf.rs:488
        auto f = flat(z); PFState est{}; check(pfgpu_pf_step(h_, u.data(), f.data(), z.size(), est.data()), "step"); dirty_ = true; return est; }
    PFState step(const PFControl& u, const PFMeasurement& z) { return try_step(u, z); }
    PFState estimate() const { PFState e{}; check(pfgpu_pf_estimate(h_, e.data(), nullptr), "estimate"); return e; }            // pf.rs:348
    std::array<double, 16> calc_covariance() const { std::array<double, 16> c{}; check(pfgpu_pf_estimate(h_, nullptr, c.data()), "covariance"); return c; }  // column-major, pf.rs:363
    size_t particle_count() const { size_t nl = 0, ng = 0; check(pfgpu_pf_count(h_, &nl, &ng), "count"); return ng; }            // mcl.rs:318
    const std::vector<Particle>& get_particles() const {                                                                         // pf.rs:244
        if (dirty_) { size_t nl = 0, ng = 0; check(pfgpu_pf_count(h_, &nl, &ng), "count"); mirror_.resize(nl);
            check(pfgpu_pf_download(h_, reinterpret_cast<double*>(mirror_.data()), nl), "download"); dirty_ = false; }
        return mirror_;
    }
    void init_state(const PFState& s) { check(pfgpu_pf_init_state(h_, s.data()), "initial state"); dirty_ = true; }
    // augmented MCL (not in the reference; DESIGN §3.8): region = (x0, x1, y0, y1); alpha_slow = alpha_fast = 0 disables
    using Region = std::array<double, 4>;
    struct RecoveryState { double w_slow, w_fast, p; uint64_t injected; };
    void enable_recovery(double alpha_slow, double alpha_fast, const Region& region) {
        check(pfgpu_pf_recovery_enable(h_, alpha_slow, alpha_fast, region.data()), "recovery");
    }
    void disable_recovery() { check(pfgpu_pf_recovery_enable(h_, 0.0, 0.0, nullptr), "recovery"); }
    RecoveryState recovery_state() const {
        double w[3] = {0.0, 0.0, 0.0}; uint64_t inj = 0;
        check(pfgpu_pf_recovery_state(h_, w, &inj), "recovery state");
        return {w[0], w[1], w[2], inj};
    }
    void init_region(const Region& region) { check(pfgpu_pf_init_region(h_, region.data()), "initial region"); dirty_ = true; }
    // likelihood-field scan model (not in the reference; DESIGN §3.9): mask[ix * height + iy], nonzero = obstacle
    static pfgpu_lfield_config lfield_defaults(double resolution) {                   // ROS AMCL's likelihood_field defaults
        pfgpu_lfield_config c{};
        c.resolution = resolution; c.sigma_hit = 0.2; c.z_hit = 0.95; c.z_rand = 0.05; c.max_range = 30.0; c.max_beams = 60;
        return c;
    }
    void set_likelihood_field(const std::vector<uint8_t>& mask, size_t width, size_t height, const pfgpu_lfield_config& c) {
        if (mask.size() != width * height) throw RoboticsError(RoboticsError::InvalidParameter, "likelihood field: mask size != width * height");
        check(pfgpu_pf_lfield_set(h_, mask.data(), width, height, &c), "likelihood field");
    }
    void clear_likelihood_field() { check(pfgpu_pf_lfield_clear(h_), "likelihood field"); }
    void try_update_with_scan(const std::vector<double>& ranges, double angle_min, double angle_increment) {
        check(pfgpu_pf_update_scan(h_, ranges.data(), ranges.size(), angle_min, angle_increment), "scan update"); dirty_ = true;
    }
    PFState try_step_scan(const PFControl& u, const std::vector<double>& ranges, double angle_min, double angle_increment) {
        PFState est{};
        check(pfgpu_pf_step_scan(h_, u.data(), ranges.data(), ranges.size(), angle_min, angle_increment, est.data()), "scan step");
        dirty_ = true;
        return est;
    }
    // beam scan model (not in the reference; DESIGN §3.11): the likelihood field's map conventions, a map of its own
    static pfgpu_beam_config beam_defaults(double resolution) {                       // ROS AMCL's beam-model defaults
        pfgpu_beam_config c{};
        c.resolution = resolution; c.sigma_hit = 0.2; c.z_hit = 0.95; c.z_short = 0.1; c.z_max = 0.05; c.z_rand = 0.05;
        c.lambda_short = 0.1; c.max_range = 30.0; c.max_beams = 60;
        return c;
    }
    void set_beam_model(const std::vector<uint8_t>& mask, size_t width, size_t height, const pfgpu_beam_config& c) {
        if (mask.size() != width * height) throw RoboticsError(RoboticsError::InvalidParameter, "beam model: mask size != width * height");
        check(pfgpu_pf_beam_set(h_, mask.data(), width, height, &c), "beam model");
    }
    // the obstacle mask of an occupancy grid on this handle's device (OccupancyGridMap::handle(), occupancy_grid_map.hpp), built
    // there at `threshold`: the same table as the host-mask calls; the grid is copied now
    void set_beam_model_from_grid(const pfgpu_ogm* grid, double threshold, const pfgpu_beam_config& c) {
        check(pfgpu_pf_beam_set_grid(h_, grid, threshold, &c), "beam model from grid");
    }
    void set_likelihood_field_from_grid(const pfgpu_ogm* grid, double threshold, const pfgpu_lfield_config& c) {
        check(pfgpu_pf_lfield_set_grid(h_, grid, threshold, &c), "likelihood field from grid");
    }
    void clear_beam_model() { check(pfgpu_pf_beam_clear(h_), "beam model"); }
    void try_update_with_beam_scan(const std::vector<double>& ranges, double angle_min, double angle_increment) {
        check(pfgpu_pf_update_beam(h_, ranges.data(), ranges.size(), angle_min, angle_increment), "beam scan update"); dirty_ = true;
    }
    PFState try_step_beam_scan(const PFControl& u, const std::vector<double>& ranges, double angle_min, double angle_increment) {
        PFState est{};
        check(pfgpu_pf_step_beam(h_, u.data(), ranges.data(), ranges.size(), angle_min, angle_increment, est.data()), "beam scan step");
        dirty_ = true;
        return est;
    }
    // the odometry motion model (DESIGN §3.14): alpha = AMCL's odom_alpha1..4; each motion is the previous then the current
    // odometry pose (x, y, yaw)
    using OdomPose = std::array<double, 3>;
    static std::array<double, 6> odom_pair(const OdomPose& prev, const OdomPose& cur) {
        return {prev[0], prev[1], prev[2], cur[0], cur[1], cur[2]};
    }
    void set_odometry_noise(const std::array<double, 4>& alpha) { check(pfgpu_pf_set_odom_noise(h_, alpha.data()), "odometry noise"); }
    std::array<double, 4> odometry_noise() const { std::array<double, 4> a{}; check(pfgpu_pf_odom_noise(h_, a.data()), "odometry noise"); return a; }
    void try_predict_with_odometry(const OdomPose& prev, const OdomPose& cur) {
        const auto o = odom_pair(prev, cur); check(pfgpu_pf_predict_odom(h_, o.data()), "odometry predict"); dirty_ = true;
    }
    PFState try_step_odometry(const OdomPose& prev, const OdomPose& cur, const PFMeasurement& z) {
        const auto o = odom_pair(prev, cur); auto f = flat(z); PFState est{};
        check(pfgpu_pf_step_odom(h_, o.data(), f.data(), z.size(), est.data()), "odometry step"); dirty_ = true; return est;
    }
    PFState try_step_scan_odometry(const OdomPose& prev, const OdomPose& cur, const std::vector<double>& ranges, double angle_min,
                                   double angle_increment) {
        const auto o = odom_pair(prev, cur); PFState est{};
        check(pfgpu_pf_step_scan_odom(h_, o.data(), ranges.data(), ranges.size(), angle_min, angle_increment, est.data()), "odometry scan step");
        dirty_ = true;
        return est;
    }
    PFState try_step_beam_scan_odometry(const OdomPose& prev, const OdomPose& cur, const std::vector<double>& ranges, double angle_min,
                                        double angle_increment) {
        const auto o = odom_pair(prev, cur); PFState est{};
        check(pfgpu_pf_step_beam_odom(h_, o.data(), ranges.data(), ranges.size(), angle_min, angle_increment, est.data()),
              "odometry beam scan step");
        dirty_ = true;
        return est;
    }
    // expected ranges of poses (x, y, yaw) x n_beams in the beam map: out[p * n_beams + b]
    std::vector<double> expected_scan(const std::vector<std::array<double, 3>>& poses, size_t n_beams, double angle_min,
                                      double angle_increment) {
        std::vector<double> p, out(poses.size() * n_beams);
        for (const auto& q : poses) p.insert(p.end(), q.begin(), q.end());
        check(pfgpu_pf_beam_raycast(h_, p.data(), poses.size(), n_beams, angle_min, angle_increment, out.data()), "expected scan");
        return out;
    }
    // pose hypotheses (not in the reference; ROS AMCL's pose hypotheses; DESIGN §3.10): the max_count heaviest clusters of the
    // cloud in xy_res x xy_res x (2 pi / yaw_bins) bins, heaviest first; *total = the number of clusters; rank_of_slot (when given)
    // = each local particle's cluster rank, UINT32_MAX for a non-member
    std::vector<pfgpu_pf_hypothesis> hypotheses(size_t max_count = 16, double xy_res = 0.5, uint32_t yaw_bins = 24, size_t* total = nullptr,
                                                std::vector<uint32_t>* rank_of_slot = nullptr) const {
        std::vector<pfgpu_pf_hypothesis> out(max_count);
        size_t n = 0, nl = 0, ng = 0;
        if (rank_of_slot) { check(pfgpu_pf_count(h_, &nl, &ng), "count"); rank_of_slot->resize(nl); }
        check(pfgpu_pf_hypotheses(h_, xy_res, yaw_bins, out.data(), max_count, &n, rank_of_slot ? rank_of_slot->data() : nullptr),
              "hypotheses");
        out.resize(n < max_count ? n : max_count);
        if (total) *total = n;
        return out;
    }
};
}  // namespace detail

class ParticleFilterLocalizer : public detail::PfHandle {                // pf.rs:121-573
public:
    explicit ParticleFilterLocalizer(const ParticleFilterConfig& c = {}, uint64_t seed = 42, int device = 0) : PfHandle(c.to_c(), seed, device) {}
    static ParticleFilterLocalizer try_with_initial_state(const PFState& s, const ParticleFilterConfig& c, uint64_t seed = 42, int device = 0) = delete;
    void with_initial_state(const PFState& s) { init_state(s); }                                                               // pf.rs:164-199
    void set_range_noise(double s) { check(pfgpu_pf_set_range_noise(h_, s), "range_noise"); }                                   // pf.rs:228
    // StateEstimator (traits.rs:31-52; pf.rs:552-573): update = update_with_observations + resample
    void predict(const PFControl& u, double /*dt ignored, pf.rs:557*/) { try_predict_with_control(u); }
    void update(const PFMeasurement& z) { try_update_with_observations(z); resample(); }
    PFState get_state() const { return estimate(); }
};

class MonteCarloLocalizer : public detail::PfHandle {                    // mcl.rs:133-471
public:
    explicit MonteCarloLocalizer(const MonteCarloLocalizationConfig& c = {}, uint64_t seed = 42, int device = 0) : PfHandle(c.to_c(), seed, device) {}
    void with_initial_state(const PFState& s) { init_state(s); }                                                               // mcl.rs:167-206
    void predict(const PFControl& u, double) { try_predict_with_control(u); }                                                   // mcl.rs:455
    void update(const PFMeasurement& z) { try_update_with_observations(z); resample(); }                                        // mcl.rs:459-462
};

}  // namespace rust_robotics_b200
