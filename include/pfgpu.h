/*
 * pfgpu.h — C ABI of the H100-native particle-filter / FastSLAM 1.0 engine (libpfgpu.so).
 *
 * This is the drop-in boundary.  The reference (rsasaki0109/rust_robotics) has no FFI of its own: its
 * boundary is the public Rust API of rust_robotics_localization::{ParticleFilterLocalizer,
 * MonteCarloLocalizer} and rust_robotics_slam::fastslam1.  A Rust shim (rust_robotics_b200/rust/, shown in
 * INTEGRATION.md) keeps those type and method names and forwards each method body to ONE entry point below;
 * the C++ mirror (rust_robotics_b200/host/ headers) and the Python mirror (rust_robotics_b200/api.py) do the same.
 * Each entry point cites the reference item it replaces ("pf.rs" = crates/rust_robotics_localization/src/
 * particle_filter.rs, "mcl.rs" = .../monte_carlo_localization.rs, "fs1.rs" = crates/rust_robotics_slam/src/
 * fastslam1.rs).
 *
 * Conventions
 *   - plain pointers and sizes only; all floating point is IEEE f64; matrices are column-major (nalgebra).
 *   - every call returns a status: 0 ok; <0 invalid parameter (maps to RoboticsError::InvalidParameter,
 *     crates/rust_robotics_core/src/error.rs:8-24); >0 CUDA / NCCL runtime failure.
 *   - one handle = one CUDA device + one stream; a handle is Send, not Sync (the reference API is &mut self).
 *   - there is NO CPU fallback: without a usable CUDA device create() fails with PFGPU_ERR_NO_DEVICE.
 *   - random draws follow the Philox contract of include/pf_contract_math.h (the reference is unseeded).
 */
#ifndef PFGPU_H
#define PFGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PFGPU_OK                 0
#define PFGPU_ERR_INVALID      (-1)   /* RoboticsError::InvalidParameter                       */
#define PFGPU_ERR_UNSUPPORTED  (-2)   /* valid in the reference, not built here (KLD-adaptive MCL on more than one GPU, ...) */
#define PFGPU_ERR_NO_DEVICE     1000  /* no CUDA device / extension cannot run: fail loudly      */
#define PFGPU_ERR_CUDA          1001
#define PFGPU_ERR_NCCL          1002

const char* pfgpu_strerror(int status);
/* last CUDA/NCCL error text of the calling thread (empty if none) */
const char* pfgpu_last_error(void);
int pfgpu_device_count(int* count);

/* ============================== ParticleFilterLocalizer / MonteCarloLocalizer ======================= */

/* ParticleFilterConfig (pf.rs:52-65) and MonteCarloLocalizationConfig (mcl.rs:50-59) */
typedef struct {
    uint64_t n_particles;        /* pf: n_particles (100); mcl: min_particles (100)        */
    double   resample_threshold; /* pf only (0.5)                                          */
    double   range_noise;        /* 0.2                                                    */
    double   velocity_noise;     /* 2.0                                                    */
    double   yaw_rate_noise;     /* 40 deg                                                 */
    double   dt;                 /* 0.1                                                    */
    int32_t  mode;               /* 0 = ParticleFilterLocalizer, 1 = MonteCarloLocalizer   */
    int32_t  _pad;
    uint64_t max_particles;      /* mcl only (5000); > n_particles: KLD-adaptive particle count (mcl.rs:322-365) */
    double   kld_epsilon;        /* mcl only (0.05)                                        */
    double   kld_z;              /* mcl only (2.326)                                       */
} pfgpu_pf_config;

typedef struct pfgpu_pf pfgpu_pf;

void pfgpu_pf_default_config(pfgpu_pf_config* cfg, int mode);      /* Default impls pf.rs:67-78, mcl.rs:61-74 */
int  pfgpu_pf_config_validate(const pfgpu_pf_config* cfg);         /* validate(): pf.rs:81-117, mcl.rs:87-130 */

/* try_new (pf.rs:139-156, mcl.rs:150-164): n particles at the origin, w = 1/n */
int  pfgpu_pf_create(const pfgpu_pf_config* cfg, uint64_t seed, int device, pfgpu_pf** out);
/* Sharded over `world` GPUs, one process per GPU (SURVEY.md §8e).  `nccl_unique_id` = the 128 bytes of an
 * ncclUniqueId produced by pfgpu_nccl_unique_id() on rank 0 and broadcast by the host program.  cfg->n_particles
 * is the GLOBAL particle count and must divide evenly. */
int  pfgpu_pf_create_sharded(const pfgpu_pf_config* cfg, uint64_t seed, int device,
                             const void* nccl_unique_id, int rank, int world, pfgpu_pf** out);
void pfgpu_pf_destroy(pfgpu_pf*);
/* try_with_initial_state (pf.rs:170-199, mcl.rs:176-206): init + uniform jitter, on device */
int  pfgpu_pf_init_state(pfgpu_pf*, const double init[4]);
/* get_particles() (pf.rs:244-246) / checkpoint: AoS (x, y, yaw, v, w), local shard */
int  pfgpu_pf_upload(pfgpu_pf*, const double* aos5, size_t n);
int  pfgpu_pf_download(pfgpu_pf*, double* aos5, size_t n);
int  pfgpu_pf_count(pfgpu_pf*, size_t* n_local, size_t* n_global);          /* particle_count() mcl.rs:318-320 */
int  pfgpu_pf_predict(pfgpu_pf*, const double u[2]);                         /* try_predict_with_control pf.rs:255-301, mcl.rs:209-257 */
int  pfgpu_pf_update(pfgpu_pf*, const double* obs3, size_t k);               /* try_update_with_observations pf.rs:310-334, mcl.rs:260-288; obs3 = k x (d, lx, ly) */
int  pfgpu_pf_resample(pfgpu_pf*, int* did_resample);                        /* resample() pf.rs:337-345; resample_adaptive mcl.rs:322-365 */
/* try_step (pf.rs:488-497, mcl.rs:291-300).  est (nullable): if non-NULL the call synchronises and returns
 * estimate(); if NULL the step is only enqueued on the handle's stream. */
int  pfgpu_pf_step(pfgpu_pf*, const double u[2], const double* obs3, size_t k, double est[4]);
int  pfgpu_pf_estimate(pfgpu_pf*, double est[4], double cov16_colmajor[16]); /* estimate()/calc_covariance() pf.rs:348-365 */
int  pfgpu_pf_neff(pfgpu_pf*, double* neff);                                 /* calc_n_eff pf.rs:416-423 */
int  pfgpu_pf_set_range_noise(pfgpu_pf*, double range_noise);                /* pf.rs:228-236 */
/* parity hook: ancestry of the last step's resample (global indices); *n = 0 when the last step did not resample */
int  pfgpu_pf_last_indices(pfgpu_pf*, uint32_t* idx, size_t cap, size_t* n);
int  pfgpu_pf_sync(pfgpu_pf*);
/* Global localisation and kidnapped-robot recovery: augmented MCL (not in the reference, whose cloud can only copy particles it
 * already has; Probabilistic Robotics Table 8.3, ROS AMCL's recovery_alpha_slow / recovery_alpha_fast; DESIGN §3.8).  Recovery
 * state: w_slow, w_fast (f64, both 0 at the start), 0 < alpha_slow < alpha_fast <= 1, and a box region = (x0, x1, y0, y1), finite,
 * x0 < x1, y0 < y1.
 *   filter     every time the engine computes S = sum w_raw (every pfgpu_pf_update and pfgpu_pf_step, on every path), with N the
 *              global particle count those weights belong to (before a KLD resample changes it): w_avg = S / N,
 *              w_slow = w_slow + alpha_slow * (w_avg - w_slow), w_fast = w_fast + alpha_fast * (w_avg - w_fast), in this order.  S NaN
 *              or +-inf: skipped.  S = 0 (every likelihood underflowed) is not skipped.  Then p = max(0, 1 - w_fast / w_slow), and
 *              p = 0 when w_slow <= 0 or the quotient is not finite.
 *   injection  the first predict (pfgpu_pf_predict, or the predict half of pfgpu_pf_step) after a resample stage (pfgpu_pf_step or
 *              pfgpu_pf_resample) that resampled, with no update in between, first replaces each slot independently with
 *              probability p: with the 53-bit uniforms (a0, a1) of Philox stream PF_INJECT_A and (b0, b1) of PF_INJECT_B, keyed by the
 *              predict's call index and the global slot, the slot is replaced when a0 < p, by x = x0 + a1 (x1 - x0),
 *              y = y0 + b0 (y1 - y0), yaw = b1 * 2 pi - pi, v = 0; its weight (1/N after the resample) stays.  Then every slot is
 *              predicted.  A PF step whose N_eff gate stays closed injects nothing in the next predict; nor does a second predict.
 *              The estimate and the particles a step returns are the resampled set before injection (no uniform sample enters the
 *              pose mean).  KLD-adaptive MCL: the slots of the new count.  Sharded: every rank holds the global S and the same p.
 * pfgpu_pf_recovery_enable: alpha_slow = alpha_fast = 0 disables (region may be NULL); anything else outside the rules above:
 *   PFGPU_ERR_INVALID.  Enabling (again), pfgpu_pf_upload, pfgpu_pf_init_state and pfgpu_pf_init_region reset w_slow = w_fast = 0
 *   and disarm the injection.  Disabled (the default) nothing changes.  While enabled every predict adds one memset and every S one
 *   single-thread launch; no host synchronisation.  On a sharded engine every rank makes the same calls.
 * pfgpu_pf_recovery_state: out3 = (w_slow, w_fast, p) and the slots the last predict injected on this handle (both nullable);
 *   synchronises.
 * pfgpu_pf_init_region: every particle uniform over the region (x, y fractions from stream REGION_A, the yaw fraction from
 *   REGION_B[0], call 0, the formulas above), v = 0, w = 1/N; KLD-adaptive MCL restarts at min_particles.  Works with recovery on or
 *   off. */
int  pfgpu_pf_recovery_enable(pfgpu_pf*, double alpha_slow, double alpha_fast, const double region[4]);
int  pfgpu_pf_recovery_state(pfgpu_pf*, double out3[3], uint64_t* injected_last);
int  pfgpu_pf_init_region(pfgpu_pf*, const double region[4]);
/* Localisation in an occupancy grid from a laser scan: the likelihood-field measurement model (not in the reference, whose MCL
 * only ranges to known landmarks; Probabilistic Robotics Table 6.3, ROS AMCL's likelihood_field; DESIGN §3.9).
 *   map        mask[ix * H + iy], W x H bytes, nonzero = obstacle; 1 <= W, H <= 65536, W * H <= 2^28.  World (0, 0) is the grid
 *              centre: ix = floor(x / res + W / 2.0) as i32 (Rust's saturating cast: NaN -> 0), likewise iy with H; inside when
 *              0 <= ix < W and 0 <= iy < H (world_to_grid, rust_robotics_mapping/src/occupancy_grid_map.rs:144-153).
 *   table      D = the Euclidean distance field in cells (compute_udf, distance_map.rs:15-100: INF = 1e20, dt_1d over every ix, then
 *              every iy, then sqrt; dt_1d's final loop reads the line's input, see DESIGN §3.9); per cell t = D * res,
 *              g = coeff * exp(-(t * t) / (2 * (sigma_hit * sigma_hit))) with coeff = 1 / sqrt(2 pi * (sigma_hit * sigma_hit)),
 *              q = z_hit * g + q_out, q_out = z_rand / max_range.  An endpoint outside the grid scores q_out.
 *   beams      ranges r_0 .. r_{B-1}: candidates i = 0, s, 2s, .. < B with s = max(1, (B - 1) / (max_beams - 1)) (integer
 *              division); a candidate is used unless r <= 0, r is not finite or r >= max_range.  a_i = i as f64 * angle_inc.
 *   weight     per particle, over the used beams in ascending i: angle = (yaw + angle_min) + a_i, ex = x + r cos(angle),
 *              ey = y + r sin(angle), w = w * q(ex, ey) from w = 1; w overwrites w_raw (no used beam: w = 1).  The rest of the
 *              update (normalisation, recovery filter) and of the step (gate, resample, estimate) is the landmark path's.
 *   bound      L = the largest count <= 4096 for which q_out^(L+1) >= DBL_MIN and q_max^(L+1) <= DBL_MAX (powers by repeated f64
 *              multiplication; q_max = z_hit * coeff + q_out); so every w_raw is a positive normal number.  A scan with more than L
 *              used beams is PFGPU_ERR_INVALID, and so is a map with L < 1.
 * pfgpu_pf_lfield_set: res, sigma_hit, z_rand, max_range positive and finite, z_hit >= 0 and finite, max_beams >= 2, else
 *   PFGPU_ERR_INVALID.  Replaces any map; builds the table on the device and synchronises.  On a sharded engine every rank makes the
 *   same call and holds its own table.  pfgpu_pf_lfield_clear frees it.  Setting or clearing the map does not touch the particles.
 * pfgpu_pf_lfield_info: W, H and L of the loaded map (all 0 without one).  pfgpu_pf_lfield_download: D and q (both nullable),
 *   cells = W * H entries each, f64, ix * H + iy.
 * pfgpu_pf_update_scan / pfgpu_pf_step_scan: pfgpu_pf_update / pfgpu_pf_step with the scan model; they may be mixed freely with the
 *   landmark calls.  No map loaded, angle_min or angle_inc not finite, ranges NULL with B > 0, or more than L used beams:
 *   PFGPU_ERR_INVALID. */
typedef struct {
    double   resolution;         /* metres per cell                                         */
    double   sigma_hit;          /* 0.2  (AMCL laser_sigma_hit)                             */
    double   z_hit;              /* 0.95 (AMCL laser_z_hit)                                 */
    double   z_rand;             /* 0.05 (AMCL laser_z_rand)                                */
    double   max_range;          /* 30   (AMCL laser_max_range)                             */
    uint32_t max_beams;          /* 60   (AMCL laser_max_beams)                             */
    uint32_t _pad;
} pfgpu_lfield_config;
int  pfgpu_pf_lfield_set(pfgpu_pf*, const uint8_t* mask, size_t width, size_t height, const pfgpu_lfield_config* cfg);
int  pfgpu_pf_lfield_clear(pfgpu_pf*);
int  pfgpu_pf_lfield_info(pfgpu_pf*, size_t* width, size_t* height, uint64_t* max_used_beams);
int  pfgpu_pf_lfield_download(pfgpu_pf*, double* D, double* q, size_t cells);
int  pfgpu_pf_update_scan(pfgpu_pf*, const double* ranges, size_t n_ranges, double angle_min, double angle_inc);
int  pfgpu_pf_step_scan(pfgpu_pf*, const double u[2], const double* ranges, size_t n_ranges, double angle_min, double angle_inc,
                        double est[4]);
/* Pose hypotheses: the particle cloud clustered in a fixed (x, y, yaw) histogram, each cluster's weight, mean and covariance (not in
 * the reference; ROS AMCL's pose hypotheses; DESIGN §3.10).  A query: no step computes anything differently or launches more.
 *   set        the particles and weights pfgpu_pf_estimate describes and pfgpu_pf_download returns (after a step, before any
 *              injection); KLD-adaptive MCL: the current generation; sharded: the global set in rank order (global slot indices).
 *   member     x, y, yaw and v finite and 0 < w < inf.  Other particles belong to no cluster.
 *   bin        r = xy_res, K = yaw_bins, T = PFC_TWO_PI (2 pi rounded to f64): kx = floor(x / r) and ky = floor(y / r) as i32 (Rust's
 *              saturating cast), theta = yaw - T * floor(yaw / T) (two rounded operations, no fused multiply-add),
 *              kt = floor(theta / (T / K)) clamped to [0, K - 1].  Single IEEE operations: the same bins in CUDA, C and Python.
 *   adjacency  two occupied bins (holding a member) with |dkx| <= 1, |dky| <= 1 and dkt in {-1, 0, 1} mod K: 26-connectivity, cyclic
 *              in yaw, not in x / y; neighbour keys beyond the i32 range do not exist.
 *   cluster    a connected component of occupied bins and the members in them: mass M = sum w, count, bins, label = the smallest
 *              global slot among its members, mean x, y, v = sum w (x, y, v) / M and yaw = atan2(sum w sin yaw, sum w cos yaw) (the
 *              contract math; 0 when both sums are 0), cov = sum (w / M) d d^T with d = (x - mean x, y - mean y, wrap(yaw - mean yaw),
 *              v - mean v), wrap(a) = a - T * floor((a + pi) / T) into [-pi, pi), column-major like pfgpu_pf_estimate's.
 *   order      mass descending, ties by ascending label.
 *   bits       the same particle set gives the same bits on every call, and a sharded engine gives on every rank the bits a single
 *              GPU holding the same global set gives (every rank clusters the gathered set).  No floating-point atomics.
 * pfgpu_pf_hypotheses: out = the first min(cap, total) clusters in that order; *n_total (nullable) = the number of clusters;
 *   rank_of_slot (nullable, n_local entries) = each local slot's cluster rank, UINT32_MAX for a non-member.  xy_res not positive and
 *   finite, yaw_bins 0 or above 65536, or cap > 0 with out NULL: PFGPU_ERR_INVALID; more than 2^31 - 1 particles:
 *   PFGPU_ERR_UNSUPPORTED.  No member: zero clusters.  Synchronises;
 *   collective on a sharded engine.  The workspace is allocated on the first call (DESIGN §3.10 gives its size); when that fails the
 *   call returns PFGPU_ERR_CUDA and the handle stays usable.  The captured step graph is kept. */
typedef struct {
    double   mass;
    double   mean[4];      /* x, y, circular-mean yaw in (-pi, pi], v */
    double   cov[16];      /* column-major, over (x, y, wrapped yaw deviation, v) */
    uint64_t count, bins, label;
} pfgpu_pf_hypothesis;
int  pfgpu_pf_hypotheses(pfgpu_pf*, double xy_res, uint32_t yaw_bins, pfgpu_pf_hypothesis* out, size_t cap, size_t* n_total,
                         uint32_t* rank_of_slot);
/* The beam measurement model: every particle's expected range along every used beam is ray-cast in the occupancy grid and compared
 * with the measured one (not in the reference; Probabilistic Robotics Table 6.1, ROS AMCL's laser_model_type beam; DESIGN §3.11).
 *   map        the likelihood field's conventions unchanged (mask[ix * H + iy], limits, world_to_grid with the saturating cast).  The
 *              beam map is separate state: a handle may hold both maps, and each step uses the model its entry point names.
 *   clearance  per cell, the Chebyshev (L-infinity) distance in cells to the nearest cell that is occupied or outside the grid, capped
 *              at 255 (0 = occupied); built on the device at set time.
 *   ray        pose (x, y, yaw), beam i: angle = (yaw + angle_min) + a_i, a_i = i as f64 * angle_inc; c0 = world_to_grid(x, y),
 *              c1 = world_to_grid(x + max_range * cos(angle), y + max_range * sin(angle)) (one sincos).  The cells are those of
 *              bresenham_line(c0, c1) (rust_robotics_mapping/src/occupancy_grid_map.rs:164-193, both ends included).  The first cell
 *              occupied or outside the grid stops the ray: r_hat = res * sqrt((f64)(dx * dx + dy * dy)), (dx, dy) its integer offset
 *              from c0, the sum of squares in int64.  No such cell up to and including c1: r_hat = max_range.  c0 occupied or outside:
 *              r_hat = 0.  max_range / res <= 2^20 keeps every integer product exact.
 *   beams      candidates i = 0, s, 2s, .. < B, s = max(1, (B - 1) / (max_beams - 1)); NaN or r <= 0: unused; r >= max_range (+inf
 *              included) is a max reading, used only when z_max > 0 and then scored with r = max_range.
 *   factor     per used beam, z = r - r_hat, coeff = 1 / sqrt(2 pi * (sigma_hit * sigma_hit)), in this order:
 *                q = (z_hit * coeff) * exp(-(z * z) / (2 * (sigma_hit * sigma_hit)))
 *                if z < 0:  q = q + (z_short * lambda_short) * exp(-(lambda_short * r))      (AMCL's short term, unnormalised)
 *                q = q + (max reading ? z_max : z_rand / max_range)
 *              w = w * q over the used beams in ascending i from w = 1; w overwrites w_raw.  The rest of the update and of the step is
 *              the landmark path's.
 *   bound      the likelihood field's rule with q_lo = z_rand / max_range (min(that, z_max) when z_max > 0) and
 *              q_hi = z_hit * coeff + z_short * lambda_short + max(z_rand / max_range, z_max).  More than L used beams:
 *              PFGPU_ERR_INVALID, so every w_raw is a positive normal number.
 * pfgpu_pf_beam_set: res, sigma_hit, z_rand, max_range, lambda_short positive and finite; z_hit, z_short, z_max >= 0 and finite;
 *   max_beams >= 2; max_range / res <= 2^20; L >= 1; else PFGPU_ERR_INVALID.  Replaces any beam map, builds the clearance on the
 *   device and synchronises.  On a sharded engine every rank makes the same call.  pfgpu_pf_beam_clear frees it.
 * pfgpu_pf_beam_info: W, H and L (all 0 without a beam map).  pfgpu_pf_beam_download: the clearance bytes, cells = W * H.
 * pfgpu_pf_update_beam / pfgpu_pf_step_beam: pfgpu_pf_update_scan / pfgpu_pf_step_scan with the beam model and the same refusals.
 * pfgpu_pf_beam_raycast: r_hat of n poses (x, y, yaw) x B beams at angle_min + b * angle_inc into out[p * B + b]; needs a beam map. */
typedef struct {
    double   resolution;         /* metres per cell                                         */
    double   sigma_hit;          /* 0.2  (AMCL laser_sigma_hit)                             */
    double   z_hit;              /* 0.95 (AMCL laser_z_hit)                                 */
    double   z_short;            /* 0.1  (AMCL laser_z_short)                               */
    double   z_max;              /* 0.05 (AMCL laser_z_max)                                 */
    double   z_rand;             /* 0.05 (AMCL laser_z_rand)                                */
    double   lambda_short;       /* 0.1  (AMCL laser_lambda_short)                          */
    double   max_range;          /* 30   (AMCL laser_max_range)                             */
    uint32_t max_beams;          /* 60   (AMCL laser_max_beams)                             */
    uint32_t _pad;
} pfgpu_beam_config;
int  pfgpu_pf_beam_set(pfgpu_pf*, const uint8_t* mask, size_t width, size_t height, const pfgpu_beam_config* cfg);
int  pfgpu_pf_beam_clear(pfgpu_pf*);
int  pfgpu_pf_beam_info(pfgpu_pf*, size_t* width, size_t* height, uint64_t* max_used_beams);
int  pfgpu_pf_beam_download(pfgpu_pf*, uint8_t* clearance, size_t cells);
int  pfgpu_pf_update_beam(pfgpu_pf*, const double* ranges, size_t n_ranges, double angle_min, double angle_inc);
int  pfgpu_pf_step_beam(pfgpu_pf*, const double u[2], const double* ranges, size_t n_ranges, double angle_min, double angle_inc,
                        double est[4]);
int  pfgpu_pf_beam_raycast(pfgpu_pf*, const double* poses3, size_t n, size_t n_beams, double angle_min, double angle_inc, double* out);
/* The odometry motion model: the predict moves every particle by the increment between two wheel-odometry poses instead of by a
 * control (v, yaw_rate) over dt (not in the reference, whose filters only have the velocity model pf.rs:279-296; Probabilistic
 * Robotics Table 5.6, ROS AMCL's odom_model_type diff-corrected with odom_alpha1..4; DESIGN §3.14).  The rule, its evaluation order
 * and its draws are include/pf_odom_math.h's: odom = (x, y, yaw) of the previous odometry pose, then (x, y, yaw) of the current one.
 * Noise grows with the motion: two equal poses move no particle.  The particle's v is left as it was.
 * pfgpu_pf_set_odom_noise: alpha = (alpha1 .. alpha4), each finite and >= 0, else PFGPU_ERR_INVALID; a handle starts at 0.2 each.
 *   pfgpu_pf_odom_noise returns them.
 * pfgpu_pf_predict_odom / pfgpu_pf_step_odom / pfgpu_pf_step_scan_odom / pfgpu_pf_step_beam_odom: pfgpu_pf_predict / pfgpu_pf_step /
 *   pfgpu_pf_step_scan / pfgpu_pf_step_beam with this motion in place of u, on every path those take (the call index, the recovery
 *   injection before the move, KLD-adaptive MCL, sharding), with the same launches; they mix freely with the velocity calls.  A
 *   component of odom that is not finite: PFGPU_ERR_INVALID, as a non-finite u is. */
int  pfgpu_pf_set_odom_noise(pfgpu_pf*, const double alpha[4]);
int  pfgpu_pf_odom_noise(pfgpu_pf*, double alpha[4]);
int  pfgpu_pf_predict_odom(pfgpu_pf*, const double odom[6]);
int  pfgpu_pf_step_odom(pfgpu_pf*, const double odom[6], const double* obs3, size_t k, double est[4]);
int  pfgpu_pf_step_scan_odom(pfgpu_pf*, const double odom[6], const double* ranges, size_t n_ranges, double angle_min, double angle_inc,
                             double est[4]);
int  pfgpu_pf_step_beam_odom(pfgpu_pf*, const double odom[6], const double* ranges, size_t n_ranges, double angle_min, double angle_inc,
                             double est[4]);

/* ===================================== Occupancy grid mapping ======================================= */

/* OccupancyGridMap (rust_robotics_mapping/src/occupancy_grid_map.rs) on the device: laser scans fused into a log-odds grid with the
 * reference's sequential result bit for bit, and its obstacle mask handed to the PF / MCL scan models without a host round trip
 * (DESIGN §3.12).
 *   grid       grid[ix * H + iy], f64 log-odds, initialised to prior_log_odds; world (0, 0) at the grid centre.  world_to_grid(x, y) =
 *              (floor(x / res + W as f64 / 2.0), floor(y / res + H as f64 / 2.0)) with Rust's saturating `as i32` (NaN -> 0), None
 *              when outside.
 *   one scan   pose (x, y, yaw), ranges r_0 .. r_{B-1}, exactly update_with_scan (:78-130):
 *              origin = world_to_grid(x, y); None: the whole scan is a no-op.  Beam i with r <= 0 or r not finite: skipped.  Else
 *              angle = (yaw + angle_min) + i as f64 * angle_inc, end = (x + r * cos(angle), y + r * sin(angle)) (one sincos);
 *              end_cell = world_to_grid(end) when inside, else BOTH coordinates round(end / res + W / 2) as i32 (round half away
 *              from zero, saturating) clamped to [0, W - 1] (resp. H).  The cells of bresenham_line(origin, end_cell) (:164-193)
 *              except the last get l = clamp(l + free_log_odds); the last gets l = clamp(l + occupied_log_odds) only when end was
 *              inside.  clamp(l) = l < min ? min : (l > max ? max : l) (Rust's f64::clamp; NaN stays NaN).
 *   batch      S poses x B ranges with one (angle_min, angle_inc): S single-scan updates in order.  The grid equals that bit for bit
 *              whatever the batch size and the internal chunking, on every call.  No floating-point atomics.
 *   obstacle   cell is an obstacle when 1.0 - 1.0 / (1.0 + exp(l)) > threshold (is_occupied, :136-159, with the contract exp).
 * pfgpu_ogm_create: 1 <= W, H <= 65536, W * H <= 2^28, resolution positive and finite, every log-odds field finite and
 *   min_log_odds <= max_log_odds (the prior may lie outside [min, max]); else PFGPU_ERR_INVALID.  The event workspace
 *   (DESIGN §3.12) is allocated by the first update.
 * pfgpu_ogm_update_scans: poses3 S x (x, y, yaw), ranges S x B row-major; S = 0 or B = 0 is a no-op.  Synchronises.
 * pfgpu_ogm_set: uploads cells = W * H log-odds (any values).  pfgpu_ogm_read: count cells from `first` into out.
 * pfgpu_ogm_obstacles: mask_out[c] = 1 for an obstacle cell, else 0, cells = W * H; threshold must be finite.
 * pfgpu_ogm_info: W, H and the last update's stats (all nullable).
 * pfgpu_pf_lfield_set_grid / pfgpu_pf_beam_set_grid: pfgpu_pf_lfield_set / pfgpu_pf_beam_set with the obstacle mask of `grid` at
 *   `threshold`, built on the device: the same tables, the same refusals.  The grid is copied at set time; later updates of it do not
 *   change the loaded model.  cfg->resolution must equal the grid's, and the grid must live on the handle's device; else
 *   PFGPU_ERR_INVALID.  On a sharded engine every rank passes a grid of the same cells on its own device. */
typedef struct {
    double   resolution;         /* 0.5  metres per cell                                   */
    uint64_t width, height;      /* 100, 100                                               */
    double   prior_log_odds;     /* 0                                                      */
    double   occupied_log_odds;  /* 0.85                                                   */
    double   free_log_odds;      /* -0.4                                                   */
    double   max_log_odds;       /* 5                                                      */
    double   min_log_odds;       /* -5                                                     */
} pfgpu_ogm_config;
typedef struct {
    uint64_t events;             /* cell updates of the last pfgpu_ogm_update_scans       */
    uint64_t chunks;             /* pieces it ran in (a chunk holds at most the event cap) */
    uint64_t longest_run;        /* the most updates one cell took in one chunk           */
    uint64_t event_cap;          /* events per chunk at most                              */
} pfgpu_ogm_stats;
typedef struct pfgpu_ogm pfgpu_ogm;
int  pfgpu_ogm_create(const pfgpu_ogm_config* cfg, int device, pfgpu_ogm** out);
void pfgpu_ogm_destroy(pfgpu_ogm*);
int  pfgpu_ogm_update_scans(pfgpu_ogm*, const double* poses3, size_t n_scans, const double* ranges, size_t n_ranges, double angle_min,
                            double angle_inc);
int  pfgpu_ogm_set(pfgpu_ogm*, const double* grid, size_t cells);
int  pfgpu_ogm_read(pfgpu_ogm*, size_t first, size_t count, double* out);
int  pfgpu_ogm_obstacles(pfgpu_ogm*, double threshold, uint8_t* mask_out, size_t cells);
int  pfgpu_ogm_info(pfgpu_ogm*, size_t* width, size_t* height, pfgpu_ogm_stats* stats);
int  pfgpu_pf_lfield_set_grid(pfgpu_pf*, const pfgpu_ogm* grid, double threshold, const pfgpu_lfield_config* cfg);
int  pfgpu_pf_beam_set_grid(pfgpu_pf*, const pfgpu_ogm* grid, double threshold, const pfgpu_beam_config* cfg);

/* ====================================== Correlative scan matching ===================================== */

/* correlative_scan_match (rust_robotics_slam/src/correlative_scan_matching.rs:55-197, Olson's brute-force correlative matcher) on
 * the device, the reference's result bit for bit (DESIGN §3.13).  A handle holds reference points on one device; the lookup table
 * for a resolution is built from them on first use and rebuilt when the resolution changes, so any config works on any reference.
 *   invalid    an empty reference or query, linear_step <= 0, angular_step <= 0 or grid_resolution <= 0 (:63-78): the result is
 *              (x, y, yaw) of the initial pose, yaw NOT normalised, score 0.0, converged 0.
 *   offsets    n = round(range / step) as i32 (round half away from zero, Rust's saturating cast); the offsets are i as f64 * step for
 *              i = -n ..= n (:122-127), none for n < 0.  No linear or no angular offset: (x, y, normalize_angle(yaw)), score -1.0,
 *              converged 0 (:84-90).
 *   table      sigma = res, R = ceil(3.0 * sigma / res) as i32 (R = 4 where 3 * res / res rounds above 3, as for res = 0.025, 0.05,
 *              0.1, 0.2; R = 3 for 0.01, 0.02, 0.25, 0.5, 1.0), inv = 0.5 / (sigma * sigma).  Each reference point (x, y) has centre
 *              cell (round(x / res), round(y / res)) as i32; every cell (ix, iy) of its (2R+1)^2 window gets
 *              w = exp((-d2) * inv), d2 = (gx - x) * (gx - x) + (gy - y) * (gy - y), gx = ix as f64 * res, gy = iy as f64 * res,
 *              unless w < 1e-6; a cell keeps the maximum of its weights, and a cell no point reached reads 0.0 (:129-159).
 *   score      for a candidate (cx, cy, cyaw) with cyaw = normalize_angle(yaw + dyaw), cx = x + dx, cy = y + dy and
 *              (c, s) = (cos cyaw, sin cyaw): per query point (px, py) in order, wx = ((c * px) - (s * py)) + cx,
 *              wy = ((s * px) + (c * py)) + cy, cell (round(wx / res), round(wy / res)) as i32; score = 0.0 + v_0 + v_1 + ...,
 *              one sequential sum (:161-180).
 *   winner     candidates in the loop order dx, then dy, then dyaw (:93-117), penalty = (dx * dx + dy * dy) + dyaw * dyaw; the
 *              loop keeps a candidate when score > best or (score == best and penalty < best penalty).  Every score is >= 0 > -1,
 *              so that loop's answer is the lexicographic optimum: the largest score, then the smallest penalty, then the earliest
 *              candidate.  The device reduces by exactly that total order, so no block or reduction order can change the result.
 *              The result is (cx, cy, cyaw, score) of the winner, converged = score > 0.0.
 *   normalize_angle is fs1.rs's loop (`-= 2.0 * PI` while > PI, `+= 2.0 * PI` while < -PI), capped at 2^22 turns (DESIGN §8
 *   deviation 2); cos, sin and exp are the contract's (pf_contract_math.h).
 * Refusals (DESIGN §8 deviation 16): a non-finite reference point, query point, pose or config field, or a reference cell with
 *   |round(x / res)| or |round(y / res)| above 2^30 (the reference's i32 window arithmetic would overflow): PFGPU_ERR_INVALID.  A table
 *   wider than PFGPU_CSM_TABLE_CAP cells, a resolution outside [2^-500, 2^500], n_linear > 2^15, n_angular > 2^22, more than
 *   2^34 candidates per query, or one query whose cell indices for one yaw exceed the workspace (8 (2 n_linear + 1) points bytes
 *   above 2^28): PFGPU_ERR_UNSUPPORTED, and the handle stays usable.  The table is built only for a call in which some query has
 *   candidates.
 * pfgpu_csm_set_reference: n points (n = 0 allowed: every match is then invalid), copied to the device.
 * pfgpu_csm_set_reference_grid: the cell centres of `grid`'s obstacle cells at `threshold` (pfgpu_ogm_obstacles' rule), in the
 *   grid's cell order: x = ((ix + 0.5) - W / 2.0) * res, y = ((iy + 0.5) - H / 2.0) * res (each an f64 operation in that order),
 *   built on the device without a host round trip.  The grid must live on the matcher's device and threshold be finite, else
 *   PFGPU_ERR_INVALID.  The points are copied now: later updates of the grid do not change the matcher until it is set again.
 * pfgpu_csm_match: Q queries against the reference under one config; query q has the initial pose poses3[3q .. 3q + 2] and the
 *   points qx[k], qy[k] for offsets[q] <= k < offsets[q + 1] (offsets[0] = 0, non-decreasing).  Each query's result is what
 *   correlative_scan_match returns for it alone; an invalid query gets the invalid result and the others are still matched.
 *   Synchronises.
 * pfgpu_csm_table_info: builds (or keeps) the table for `resolution` and reports its extent: cell (ix, iy) with
 *   origin_x <= ix < origin_x + width (likewise y) is at ix * height + iy relative to the origin, and every cell outside reads 0.0;
 *   the extent is the reference cells' bounding box grown by R.  No reference point: width = height = 0.  All outputs nullable.
 * pfgpu_csm_table_read: count f64 cells of the current table from `first`. */
#define PFGPU_CSM_TABLE_CAP ((uint64_t)1 << 26)
typedef struct {
    double linear_search_range;  /* 1.0   metres                                           */
    double angular_search_range; /* 0.2   radians                                          */
    double linear_step;          /* 0.1                                                    */
    double angular_step;         /* 0.02                                                   */
    double grid_resolution;      /* 0.05  metres per lookup cell                           */
} pfgpu_csm_config;
typedef struct {
    double   x, y, yaw, score;
    uint32_t converged, _pad;
} pfgpu_csm_result;
typedef struct pfgpu_csm pfgpu_csm;
int  pfgpu_csm_create(int device, pfgpu_csm** out);
void pfgpu_csm_destroy(pfgpu_csm*);
int  pfgpu_csm_set_reference(pfgpu_csm*, const double* x, const double* y, size_t n);
int  pfgpu_csm_set_reference_grid(pfgpu_csm*, const pfgpu_ogm* grid, double threshold);
int  pfgpu_csm_reference_size(pfgpu_csm*, size_t* n);
int  pfgpu_csm_match(pfgpu_csm*, const pfgpu_csm_config* cfg, const double* poses3, size_t n_queries, const double* qx, const double* qy,
                     const uint64_t* offsets, pfgpu_csm_result* results);
int  pfgpu_csm_table_info(pfgpu_csm*, double resolution, int64_t* origin_x, int64_t* origin_y, uint64_t* width, uint64_t* height,
                          int32_t* radius);
int  pfgpu_csm_table_read(pfgpu_csm*, size_t first, size_t count, double* out);

/* ====================================== Grid-based FastSLAM ========================================= */

/* Laser SLAM: a Rao-Blackwellised particle filter with one occupancy grid per particle (not in the reference; "FastSLAM with
 * occupancy grids", Probabilistic Robotics Table 13.4, the filter GMapping is built on; DESIGN §3.16).  A handle holds N particles on
 * one GPU, each a pose (x, y, yaw), a weight w and its own grid, laid out and configured exactly as pfgpu_ogm's (cell ix * H + iy,
 * world (0, 0) at the centre, world_to_grid with the saturating cast).  Every particle starts at the start pose with w = 1/N, its
 * grid at prior_log_odds.
 * pfgpu_gs_step(odom, ranges r_0 .. r_{B-1}, angle_min, angle_inc), in this order:
 *   move       every particle: m = pf_odom_increment(odom, alpha) once per call, then fs_odom_move (include/fs_odom_math.h: pf_odom_move,
 *              yaw = normalize(yaw)) with (za, zb) = the pair of Philox block (seed, PFC_STREAM_FS_PREDICT, call, slot) and zc = the first
 *              normal of block (seed, PFC_STREAM_FS_ODOM, call, slot); call = the handle's step counter (0 for the first step).  The
 *              alphas start at 0.2 each (pfgpu_gs_set_odom_noise: pfgpu_pf_set_odom_noise's rule).
 *   weigh      every particle against its own grid as it was before this step's scan (an endpoint, "map matching", model).  Used
 *              beams are the likelihood field's: candidates i = 0, s, 2s, .. < B with s = max(1, (B - 1) / (max_beams - 1)); a
 *              candidate is used unless r <= 0, r is not finite or r >= max_range.  Per used beam, in ascending i:
 *              angle = (yaw + angle_min) + i as f64 * angle_inc (one sincos), c = world_to_grid(x + r cos, y + r sin) (saturating,
 *              inside or not); l* = the maximum log-odds over the cells of the (2R + 1)^2 window around c that lie inside the grid (a
 *              NaN cell is skipped; no window cell inside, or every one NaN: q = q_out); else q = z_hit * p + q_out with
 *              p = 1.0 - 1.0 / (1.0 + exp(l*)) (is_occupied's probability, contract exp), q_out = z_rand / max_range.
 *              w_raw = 1 * q_0 * q_1 * .. over the used beams, w = w * w_raw (weights accumulate between resamples).
 *   normalise  fs1.rs:186-203: S = the sequential sum of w, w = w / S when S > 0; N_eff = 1 / (the sequential sum of w * w), 0 when
 *              that sum is 0.  The gate opens when N_eff < nth (absolute, like fs1.rs's NTH).
 *   fuse       every particle's scan at its moved pose into its own grid: exactly update_with_scan (the pfgpu_ogm rule above, every
 *              beam, unchanged).
 *   resample   when the gate opened, fs1.rs:206-234: normalise again (as above), cum = the sequential CDF, r_0 = u * (1/N - 0) + 0
 *              with u = pfc_u01_52 of the first u64 of block (seed, PFC_STREAM_FS_RESAMPLE, k, 0), k = the resamples so far; slot t
 *              takes ancestor j (the loop `while r > cum[j + 1] && j < N - 1: j += 1`, r += 1/N per slot): j's pose and a copy of
 *              j's fused grid; every weight becomes 1/N.
 *   bound      L = the likelihood field's rule with q_lo = q_out and q_hi = z_hit + q_out: the largest count <= 4096 with
 *              q_out^(L+1) >= DBL_MIN and q_hi^(L+1) <= DBL_MAX.  A scan with more than L used beams is PFGPU_ERR_INVALID, so
 *              DBL_MIN <= w_raw <= DBL_MAX.  Why S > 0 always holds: after a normalisation the weights sum to 1 within rounding, so the
 *              largest is at least about 1/N; that particle's w * w_raw is then at least DBL_MIN / N, a positive (possibly subnormal)
 *              number for any N below 2^52, and S is at least that term.  Likewise S stays finite: every w <= 1 and w_raw <= DBL_MAX.
 *   buffers    a resample copies N - (distinct ancestors) grids: the fuse runs once per parent (children share its pose, so they
 *              share its fused grid), the lowest slot among a parent's children keeps the parent's buffer, and every further child's
 *              grid is copied into the buffer of a parent without children.  Memory: N grids and a slot -> buffer table, not 2N.
 *   bits       poses, weights, ancestry and every grid equal the sequential statement above bit for bit.  No floating-point atomics.
 * pfgpu_gs_create: the ogm fields as pfgpu_ogm_create's; n_particles >= 1 and < 2^32; nth not NaN; z_hit >= 0 and finite; z_rand and
 *   max_range positive and finite; max_beams >= 2; 0 <= search_radius <= 8; L >= 1; start_pose finite; else PFGPU_ERR_INVALID.  N
 *   grids that do not fit in the device's free memory: PFGPU_ERR_UNSUPPORTED; an allocation that fails: PFGPU_ERR_CUDA.  Nothing is
 *   leaked on any refusal.
 * pfgpu_gs_step: enqueues only, no host synchronisation.  A non-finite odom component, angle_min or angle_inc, ranges NULL with B > 0,
 *   or more than L used beams: PFGPU_ERR_INVALID, and nothing changes (the step counter included).
 * pfgpu_gs_download: poses3 (n x 3) and weights (n), both nullable; n must be N.  pfgpu_gs_best: the largest weight, ties to the
 *   lowest slot.  pfgpu_gs_grid_read: count cells of slot's grid from `first`.  pfgpu_gs_grid_to_ogm: slot's grid into `ogm`, device
 *   to device; ogm must have the same config (every field) and live on the same device, else PFGPU_ERR_INVALID.
 * pfgpu_gs_last_indices: the ancestors of the last step's resample; *n = 0 when it did not resample.
 * pfgpu_gs_info: W, H, N, L and the last step's stats (all nullable).  Every query synchronises. */
typedef struct {
    pfgpu_ogm_config ogm;        /* the grid of every particle                             */
    uint64_t n_particles;        /* 100                                                    */
    double   nth;                /* 50: resample when N_eff < nth                          */
    double   z_hit;              /* 0.95                                                   */
    double   z_rand;             /* 0.05                                                   */
    double   max_range;          /* 30                                                     */
    uint32_t max_beams;          /* 60                                                     */
    uint32_t search_radius;      /* 1: R, the window is (2R + 1)^2 cells                  */
} pfgpu_gs_config;
typedef struct {
    uint64_t steps;              /* steps so far                                           */
    double   neff;               /* N_eff of the last step                                */
    uint64_t resampled;          /* 1 when the last step resampled                        */
    uint64_t copies;             /* grids the last step copied: N - distinct ancestors    */
    uint64_t events;             /* cell updates the last step's fuse applied: each parent's scan once when it resampled, else every particle's */
} pfgpu_gs_stats;
typedef struct pfgpu_gs pfgpu_gs;
void pfgpu_gs_default_config(pfgpu_gs_config* cfg);
int  pfgpu_gs_create(const pfgpu_gs_config* cfg, uint64_t seed, const double start_pose[3], int device, pfgpu_gs** out);
void pfgpu_gs_destroy(pfgpu_gs*);
int  pfgpu_gs_set_odom_noise(pfgpu_gs*, const double alpha[4]);
int  pfgpu_gs_odom_noise(pfgpu_gs*, double alpha[4]);
int  pfgpu_gs_step(pfgpu_gs*, const double odom[6], const double* ranges, size_t n_ranges, double angle_min, double angle_inc);
int  pfgpu_gs_download(pfgpu_gs*, double* poses3, double* weights, size_t n);
int  pfgpu_gs_best(pfgpu_gs*, size_t* slot, double pose3[3]);
int  pfgpu_gs_grid_read(pfgpu_gs*, size_t slot, size_t first, size_t count, double* out);
int  pfgpu_gs_grid_to_ogm(pfgpu_gs*, size_t slot, pfgpu_ogm* ogm);
int  pfgpu_gs_last_indices(pfgpu_gs*, uint32_t* idx, size_t cap, size_t* n);
int  pfgpu_gs_info(pfgpu_gs*, size_t* width, size_t* height, size_t* n, uint64_t* max_used_beams, pfgpu_gs_stats* stats);
int  pfgpu_gs_sync(pfgpu_gs*);

/* The scan-matched proposal (GMapping's improved proposal: Grisetti, Stachniss and Burgard, IEEE T-RO 23(1), 2007; DESIGN §3.17;
 * arithmetic in include/gs_prop_math.h).  Off by default; while it is off a step is exactly the rule above.  When it is on, the
 * move and weigh of pfgpu_gs_step become the following for every particle; normalise, gate, fuse and resample stay as they are,
 * the fuse at the pose chosen here.  m = pf_odom_increment(odom, alpha), p = the particle's pose before the step.
 *   0 fallback  the move and weigh above for this particle, unchanged (fs_odom_move with the FS_PREDICT pair and the FS_ODOM normal,
 *               w = w * w_raw(x')).  Taken when m stands still (every sigma 0, fs2_odom_case's STILL), when the prior covariance
 *               has no inverse, when the match is uninformative (2) or when eta is not a normal number (4).
 *   1 prior     (mu, Sigma) = fs_odom_prior(m, p): mu the noise-free move, Sigma with its eps = 1e-8 floor; A = fs2_inv33(Sigma).
 *   2 match     a brute-force correlative window around mu with CSM's conventions (pfgpu_csm_match): n_l = round(linear_range /
 *               linear_step), n_a = round(angular_range / angular_step); candidates (mu_x + a ls, mu_y + b ls, normalize(mu_yaw +
 *               e as)) with a as f64 times the step, |a|, |b| <= n_l, |e| <= n_a, loop index ((a + n_l) NL + b + n_l) NA + e + n_a
 *               (a outermost, e fastest; NL = 2 n_l + 1, NA = 2 n_a + 1).  A candidate's score is w_raw at its pose (the weigh's
 *               used beams, arithmetic and beam order); its penalty (dx dx + dy dy) + dyaw dyaw of its offsets.  The winner x^:
 *               the larger score, then the smaller penalty, then the earlier loop index.  h(x^) = the used beams whose window
 *               holds a cell inside the grid with l* > 0; h(x^) < min_hits is the uninformative match (e.g. every grid of the
 *               first step, at prior 0).
 *   3 lattice   K = (2k + 1)^3 points x_j = (x^_x + a kl, x^_y + b kl, normalize(x^_yaw + e ka)), offsets o_j = (a kl, b kl, e ka),
 *               |a|, |b|, |e| <= k, in the match's loop order.  L_j = w_raw(x_j); d_j = x_j - mu (yaw difference normalised);
 *               pi_j = exp(-0.5 * d_j^T A d_j) (contract exp; the quadratic form as gs_prop_quad orders it); tau_j = L_j pi_j.
 *               Sequential sums in lattice order: T = sum tau_j, m_o = (sum tau_j o_j) / T, C = (sum tau_j (o_j - m_o)(o_j -
 *               m_o)^T) / T + eps I.
 *   4 sample    the pose is FastSLAM 2.0's sample of N(x^ + m_o (yaw normalised), C): fs2_propose_pose's Cholesky factor (with its
 *               diagonal fallback), mean + L (n0, n1, n2) and set_pose's wrap; (n0, n1) = the FS_PREDICT pair, n2 = the first
 *               normal of block (seed, PFC_STREAM_FS2_POSE3, call, slot) (the draws of DESIGN §3.15).  eta = c T with
 *               c = kl kl ka / sqrt((2 pi)^3 det Sigma_0) (gs_prop_norm), Sigma_0 the prior covariance at yaw + rot1 = 0: V =
 *               blockdiag(R(yaw + rot1), 1) V_0 makes det Sigma the same for every particle in exact arithmetic, so c is one number
 *               per step, computed on the host.  eta is a Riemann estimate of the integral of p(z | m, x) p(x | p, u) over x, the
 *               quantity a fallback particle's w_raw(x') estimates with one sample, so the two kinds weigh against each other.
 *               w = w * eta.
 *   bound       every factor a weight is multiplied by stays in [DBL_MIN, DBL_MAX], so §3.16's argument for S > 0 and finite
 *               carries over.  w_raw is there by L.  eta: pi_j <= 1 and L_j <= q_hi^k (q_hi = z_hit + q_out), so eta <= c K q_hi^k;
 *               a non-still step where c K q_hi^k (evaluated as c K, then times q_hi once per used beam) is not <= DBL_MAX is
 *               PFGPU_ERR_INVALID with nothing changed (it needs q_hi > 1 and many beams; never at the defaults); eta below
 *               DBL_MIN (or 0, or NaN) takes the fallback.
 * pfgpu_gs_set_proposal: the ranges finite and >= 0, the four steps finite and > 0, enabled 0 or 1, else PFGPU_ERR_INVALID; a
 *   half_width above 3, more than 2048 match candidates or more than 1024 match yaws: PFGPU_ERR_UNSUPPORTED.  A refusal changes
 *   nothing.  It applies from the next step.
 * pfgpu_gs_last_proposal: per slot, of the last step: x^ (NaN when no match ran), eta (NaN when no lattice ran) and took (1 when
 *   the particle took the proposal, 0 for the fallback); all NaN / 0 when the last step ran without the proposal.  All nullable;
 *   n must be N.  Synchronises. */
typedef struct {
    uint32_t enabled;               /* 0                                                       */
    uint32_t half_width;            /* 1: the lattice's k, at most 3                          */
    double   linear_range;          /* 0.1 m: the match window                                */
    double   linear_step;           /* 0.025 m                                                 */
    double   angular_range;         /* 0.05 rad                                                */
    double   angular_step;          /* 0.0125 rad                                              */
    double   lattice_linear_step;   /* 0.01 m: kl (GMapping's sample step)                     */
    double   lattice_angular_step;  /* 0.005 rad: ka                                           */
    uint32_t min_hits;              /* 10: the fewest hits of an informative match             */
    uint32_t _pad;
} pfgpu_gs_proposal;
void pfgpu_gs_default_proposal(pfgpu_gs_proposal* p);
int  pfgpu_gs_set_proposal(pfgpu_gs*, const pfgpu_gs_proposal* p);
int  pfgpu_gs_get_proposal(pfgpu_gs*, pfgpu_gs_proposal* p);
int  pfgpu_gs_last_proposal(pfgpu_gs*, double* matched3, double* eta, uint8_t* took, size_t n);

/* ============================================ FastSLAM 1.0 ========================================== */

/* Module constants of fs1.rs:13-23 as fields; pfgpu_fs_default_config() fills in the reference values. */
typedef struct {
    double dt;           /* DT = 0.1                 */
    double max_range;    /* MAX_RANGE = 20 (only get_observations uses it) */
    double nth;          /* NTH = 100/1.5            */
    double q00, q11;     /* Q_SIM = diag(0.3, 0.0305) */
    double r00, r11;     /* R_SIM = diag(0.5, 0.0305) */
    double init_weight;  /* 1/N_PARTICLE = 0.01 (fs1.rs:56) */
} pfgpu_fs_config;

/* (distance, angle, landmark_id): the tuple of fs1.rs:240 */
typedef struct { double d, angle; uint64_t lm_id; } pfgpu_fs_obs;

typedef struct pfgpu_fs pfgpu_fs;

void pfgpu_fs_default_config(pfgpu_fs_config* cfg);
/* create_particles(n, m) fs1.rs:302-306.  0 <= n_landmarks <= 65536 (this and both sharded create calls); more returns
 * PFGPU_ERR_UNSUPPORTED with a message in pfgpu_last_error.  n_particles < 2^28 (per GPU when sharded); beyond that the limit
 * is device memory (about 104 * n_landmarks + 140 bytes per particle), and an allocation that fails returns PFGPU_ERR_CUDA. */
int  pfgpu_fs_create(const pfgpu_fs_config* cfg, size_t n_particles, size_t n_landmarks, uint64_t seed,
                     int device, pfgpu_fs** out);
/* Sharded over `world` (<= 8) GPUs of one NVLink domain, one process per GPU; collective over all ranks (same arguments
 * everywhere; n_particles_global / world must be a multiple of 64).  NCCL is used once, here, to exchange the cudaIpc handles of
 * the per-rank arenas.  The step itself runs over peer memory: every rank's EKF kernel pushes its 8 bytes per particle of
 * unnormalised weight into every rank's copy, every rank's post kernel evaluates the exact sums / CDF / resample indices
 * of ALL particles, and ancestors that live on another rank are read through NVLink when (and only when) one of their
 * landmarks is next observed — no NCCL call, no host synchronisation and no map copy per step.  Every rank must issue the
 * same sequence of pfgpu_fs_step calls; a rank that stops surfaces as PFGPU_ERR_CUDA at the others' next synchronising
 * call (spins time out; no hang). */
int  pfgpu_fs_create_sharded(const pfgpu_fs_config* cfg, size_t n_particles_global, size_t n_landmarks,
                             uint64_t seed, int device, const void* nccl_unique_id, int rank, int world,
                             pfgpu_fs** out);
/* The same sharded engine with all `world` ranks inside ONE process (no NCCL): out[r] runs on devices[r]; devices may
 * repeat (several ranks on one GPU — what the single-GPU parity tests use to exercise every cross-rank path).  One host
 * thread drives the ranks: issue each step to every handle with did_resample == NULL before synchronising any of them. */
int  pfgpu_fs_create_sharded_local(const pfgpu_fs_config* cfg, size_t n_particles_global, size_t n_landmarks,
                                   uint64_t seed, const int* devices, int world, pfgpu_fs** out);
void pfgpu_fs_destroy(pfgpu_fs*);
/* Vec<Particle> <-> device (fs1.rs:44-51).  pose_w: n x (weight, x, y, yaw); lm (nullable): n x m x
 * (x, y, c00, c01, c10, c11), particle-major AoS exactly like the reference's memory order. */
int  pfgpu_fs_upload(pfgpu_fs*, const double* pose_w, const double* lm, size_t n);
int  pfgpu_fs_download(pfgpu_fs*, double* pose_w, double* lm, size_t n);
/* Benchmark / test convenience (not in the reference): start from an INITIALISED map so that the EKF branch
 * fs1.rs:151-182 is live from step 0 (a fresh create_particles never reaches it: SURVEY.md App. B.3).
 * Every particle gets pose (x, y, yaw), weight 1/n, and for every landmark l: position = landmarks_xy[l] +
 * sigma * N(0,1)^2 (Philox stream INIT_A, index = particle*m + l), cov = cov0 * I (fs2.rs:254 convention). */
int  pfgpu_fs_seed_map(pfgpu_fs*, const double pose3[3], const double* landmarks_xy, size_t m, double sigma, double cov0);
/* fastslam_update fs1.rs:237-266.  did_resample (nullable): non-NULL synchronises. */
int  pfgpu_fs_step(pfgpu_fs*, const double u[2], const pfgpu_fs_obs* z, size_t k, int* did_resample);
/* get_observations fs1.rs:277-299, the simulator next to the filter, on the device: landmarks within cfg.max_range of x_true
 * (x, y, yaw), in landmark order; range / bearing noise N(0,1) * sqrt(R) from Philox stream PFC_STREAM_OBS keyed by (seed of the
 * handle, call, landmark id).  out has room for n_landmarks tuples; *k receives their number. */
int  pfgpu_fs_get_observations(pfgpu_fs*, const double x_true[3], const double* landmarks_xy, size_t n_landmarks, uint32_t call,
                               pfgpu_fs_obs* out, size_t* k);
/* get_best_particle fs1.rs:269-274 (last maximum wins); pose_w4 = (weight, x, y, yaw) */
int  pfgpu_fs_best(pfgpu_fs*, size_t* index_global, double pose_w4[4]);
/* landmarks of one particle (what render_gif_slam.rs:183-191 reads): lm6 = m x 6 */
int  pfgpu_fs_particle_landmarks(pfgpu_fs*, size_t index_local, double* lm6);
int  pfgpu_fs_last_indices(pfgpu_fs*, uint32_t* idx, size_t cap, size_t* n);  /* *n = 0 when the last step did not resample */
int  pfgpu_fs_last_neff(pfgpu_fs*, double* neff);
int  pfgpu_fs_last_gate(pfgpu_fs*, int* did_resample);     /* whether the last step resampled (fs1.rs:263); synchronises */
/* Which update pfgpu_fs_step runs: 1 = fastslam1::fastslam_update (fs1.rs:237-266, the default), 2 = fastslam2::fastslam2_update
 * (crates/rust_robotics_slam/src/fastslam2.rs:376-383 -> :330-374): the same particle set, normalisation, N_eff gate and
 * resampler; the pose of every particle is sampled from the proposal that fuses the motion prior (MOTION_COV, fs2.rs:31) with
 * the step's first observation (compute_proposal :173-216, sample_pose :219-239; three N(0,1) per particle), and
 * update_landmark_and_weight (:242-280) replaces update_landmark (landmark test `cov00 < 100`, birth with cov = 10 I, weight
 * factor 1e-10 when det S <= 0).  A step without observations is the motion model with two draws (:347-356).  May be changed
 * between steps; every rank of a sharded engine must make the same call. */
int  pfgpu_fs_set_variant(pfgpu_fs*, int variant);
/* FastSLAM 2.0 with UNKNOWN data association (not in the reference's fastslam2; its rule is ekf_slam.rs:284-308's, applied per
 * particle; DESIGN §3.5).  z2 = k (d, angle) pairs without landmark ids, k unbounded.  Per particle: the landmark of z2[0] for the
 * proposal is the association at the noise-free motion prediction; then, observation by observation at the sampled pose against
 * the map as the earlier observations left it, A = the initialised slot (cov00 < 100) with the smallest squared Mahalanobis
 * distance y^T S^-1 y (first minimum in slot order; det S == 0 skips the slot), accepted when below gate_d2 (16 = ekf_slam.rs:19's
 * M_DIST_TH^2).  Matched: update_landmark_and_weight on it; otherwise a birth in the lowest empty slot (!(cov00 < 100)); no
 * empty slot: the observation is dropped.  Normalise, gate and resample as pfgpu_fs_step.  k = 0 is pfgpu_fs_step with k = 0.
 * Variant 1: PFGPU_ERR_UNSUPPORTED.  Non-finite u / z2, or gate_d2 not > 0 (+inf allowed): PFGPU_ERR_INVALID.  May be interleaved
 * with pfgpu_fs_step; every rank of a sharded engine makes the same calls. */
int  pfgpu_fs_step_unknown(pfgpu_fs*, const double u[2], const double* z2, size_t k, double gate_d2, int* did_resample);
/* (matched, born, dropped) observation counts of the last pfgpu_fs_step_unknown, summed over this handle's particles; synchronises */
int  pfgpu_fs_assoc_counts(pfgpu_fs*, uint64_t counts[3]);
/* The odometry motion model for FastSLAM (not in the reference, whose fastslam1 / fastslam2 only have the velocity model
 * fs1.rs:123-137, fs2.rs:95-120; DESIGN §3.15): every particle moves by the increment between two wheel-odometry poses instead of
 * by a control over dt.  odom = (x, y, yaw) of the previous odometry pose, then of the current one.  The rule, its evaluation order
 * and its draws are include/fs_odom_math.h's: include/pf_odom_math.h's increment and move (yaw wrapped), and for FastSLAM 2.0 with
 * observations the proposal of the first observation fused with the prior the increment induces (covariance floored by 1e-8 on
 * the diagonal).  Standing still (odom' == odom) moves no particle; weights and maps still update from the observations.  Two rules
 * of FastSLAM 2.0 differ from its velocity proposal: a particle whose increment has no noise (every sigma 0) takes the noise-free
 * move without a draw; a particle with nothing to fuse (the first observation's landmark not initialised, cov00 >= 100, or with
 * unknown association no slot matched) takes FastSLAM 1.0's odometry move, not a sample of the linearised prior.
 * pfgpu_fs_set_odom_noise: alpha = (alpha1 .. alpha4) as pfgpu_pf_set_odom_noise, each finite and >= 0, else PFGPU_ERR_INVALID; a
 *   handle starts at 0.2 each.  pfgpu_fs_odom_noise returns them.  Every rank of a sharded engine makes the same calls.
 * pfgpu_fs_step_odom / pfgpu_fs_step_unknown_odom: pfgpu_fs_step / pfgpu_fs_step_unknown with this motion in place of u, with the
 *   same refusals (a non-finite component of odom: PFGPU_ERR_INVALID, as a non-finite u is; known ids while existence counters are
 *   on, unknown association on FastSLAM 1.0: PFGPU_ERR_UNSUPPORTED); k = 0 without existence counters is pfgpu_fs_step_odom with
 *   k = 0.  They mix freely with the velocity steps on one handle. */
int  pfgpu_fs_set_odom_noise(pfgpu_fs*, const double alpha[4]);
int  pfgpu_fs_odom_noise(pfgpu_fs*, double alpha[4]);
int  pfgpu_fs_step_odom(pfgpu_fs*, const double odom[6], const pfgpu_fs_obs* z, size_t k, int* did_resample);
int  pfgpu_fs_step_unknown_odom(pfgpu_fs*, const double odom[6], const double* z2, size_t k, double gate_d2, int* did_resample);
int  pfgpu_fs_count(pfgpu_fs*, size_t* n_local, size_t* n_global, size_t* n_landmarks);
/* Estimate (not in the reference, whose callers read the best particle's map, keeping landmarks with cov00 < 100).  With W the sum
 * of the stored weights (never assumed to be 1):
 *   pose      weighted mean and 3x3 covariance of (x, y, yaw); yaw deviations are wrapped differences from a centre c, the mean
 *             yaw is wrapped to [-pi, pi].  c = the current pose of the last particle (global index n - 1), read from the state at
 *             every call (after upload / seed_map too), so it is always a member of the cloud.
 *   landmark  over the particles whose copy passes cov00 < cov00_max: mass = (sum of their weights) / W, mean = weighted mean of
 *             the copies' (x, y), cov = sum w (P + (mu - mean)(mu - mean)^T) / sum w in (c00, c01, c10, c11) order.
 * mass 0: mean and cov are NaN.  W <= 0 or not finite: everything NaN, every mass 0 (a status of 0: the state has no mean).
 * Two steps, so that a sharded engine needs no cross-rank synchronisation inside the library:
 * pfgpu_fs_moments: moments of the particles this handle owns (one GPU: all of them) of the deviations from the centre c, which
 *   every rank reads bit for bit (through the peer mapping when sharded): total weight, weighted mean, and central second
 *   moments m2 = sum w (d - mean)(d - mean)^T.  lm (nullable: pose only) receives n_landmarks entries.  Synchronises and returns through host memory.  Valid
 *   where pfgpu_fs_download is: on a sharded engine no rank may step until every rank's call has returned.  cov00_max = INFINITY
 *   takes every copy; NaN is invalid. */
typedef struct { double w; double c[3]; double mean[3]; double m2[6]; } pfgpu_fs_pose_moments; /* m2: xx xy xyaw yy yyaw yawyaw */
typedef struct { double w; double mean[2]; double m2[4]; } pfgpu_fs_lm_moments;               /* m2 = sum w (P + d d^T), lm6 order */
int  pfgpu_fs_moments(pfgpu_fs*, double cov00_max, pfgpu_fs_pose_moments* pose, pfgpu_fs_lm_moments* lm);
/* Host only: merge `world` ranks' moments in rank order and finalise.  lm: [world] pointers to n_landmarks entries each, or NULL
 * (pose only).  Every output is nullable; pose_cov9_colmajor is column-major (nalgebra Matrix3), lm_mean2 n_landmarks x 2,
 * lm_cov4 n_landmarks x 4 (c00, c01, c10, c11).  Ranks merge with the pairwise (Chan) update; moments about different centres
 * are invalid. */
int  pfgpu_fs_estimate_merge(const pfgpu_fs_pose_moments* pose, const pfgpu_fs_lm_moments* const* lm, int world, size_t n_landmarks,
                             double pose_mean3[3], double pose_cov9_colmajor[9], double* lm_mass, double* lm_mean2, double* lm_cov4);
/* Path history (not in the reference, whose particles keep no past poses; DESIGN §3.6).  A FastSLAM particle is a path hypothesis;
 * the engine can keep the last `capacity` steps of every particle's path on the device:
 *   window   entry s is written after step s (s counts every pfgpu_fs_step / pfgpu_fs_step_unknown since create, k = 0 included).
 *            It holds, per slot i, the pose (x, y, yaw) after the step (after the resample's clone) and a parent a_s(i): the global
 *            ancestor of slot i when step s resampled, i itself otherwise.  Enabling writes a root entry (the current poses, every
 *            parent the slot itself) at the current step count; so do pfgpu_fs_upload and pfgpu_fs_seed_map while history is enabled,
 *            which restart the window.  A full ring drops its oldest entry; the oldest entry held is always a root.
 *   path     of global slot g: slot_S = g at the newest entry S, slot_{s-1} = a_s(slot_s); pose_s[slot_s] at every entry.  Equal to
 *            the list of past poses each particle would carry if it were cloned with the particle at every resample.
 *   moments  genealogy smoother: at every entry s, pfgpu_fs_moments' definition (DESIGN §3.4) over the lineage poses of the current
 *            particles with their CURRENT weights, about the centre c_s = the step-s pose on the lineage of global slot n - 1.
 *            Sharded: each rank returns its own particles' moments; merge entry by entry with pfgpu_fs_estimate_merge (lm = NULL).
 * pfgpu_fs_history_enable: capacity entries (capacity * ld * 28 bytes per rank, ld = local particles rounded up to 64); 0
 *   disables and frees.  Re-enabling starts a new window.  Collective on a sharded engine, with the same capacity on every rank.  A
 *   ring that does not fit in device memory: PFGPU_ERR_CUDA, and history stays as it was.  While enabled every step adds one
 *   kernel launch and no host synchronisation.
 * pfgpu_fs_history_window: the steps of the oldest and the newest entry held.
 * pfgpu_fs_path: the newest min(max_steps, window length) entries of slot index_global's path, oldest first: step numbers, slot ids
 *   and poses (pose3: 3 per entry); *n = entries written.  step / slot / pose3 are nullable, each holds max_steps entries.
 * pfgpu_fs_path_moments: the same entries' moments, oldest first, into out (max_steps entries).
 * Both queries synchronise and are valid where pfgpu_fs_download is (on a sharded engine no rank may step until every rank's call
 * has returned).  History disabled, an index out of range or max_steps == 0: PFGPU_ERR_INVALID. */
int  pfgpu_fs_history_enable(pfgpu_fs*, size_t capacity);
int  pfgpu_fs_history_window(pfgpu_fs*, uint64_t* first_step, uint64_t* last_step);
int  pfgpu_fs_path(pfgpu_fs*, size_t index_global, size_t max_steps, uint64_t* step, uint32_t* slot, double* pose3, size_t* n);
int  pfgpu_fs_path_moments(pfgpu_fs*, size_t max_steps, uint64_t* step, pfgpu_fs_pose_moments* out, size_t* n);
/* Landmark existence counters for unknown data association (not in the reference, which takes ids and never removes a landmark;
 * the counter of FastSLAM with unknown correspondences, Probabilistic Robotics Table 13.3; DESIGN §3.7).  While enabled every slot
 * of every particle carries an integer tau, cloned with the particle on resample.  In each pfgpu_fs_step_unknown, per particle:
 * a match sets tau += 1, a birth tau = 1, a drop changes nothing; then every initialised slot (cov00 < 100) that no observation of
 * the step matched or bore and that lies within `range` of the sampled pose (sqrt(dx^2 + dy^2) <= range) gets tau -= 1, and a
 * slot whose tau falls below 0 is removed: reset to the fresh landmark (0, 0, 1000 I), i.e. empty.  k = 0 steps run the same
 * pass after the motion step.  Weights never depend on tau.
 * pfgpu_fs_existence_enable: range > 0 (+inf allowed) enables and sets every tau to 1 (so do re-enabling, pfgpu_fs_upload and
 *   pfgpu_fs_seed_map while enabled); 0 disables and frees; NaN or negative: PFGPU_ERR_INVALID.  8 * m * ld bytes per rank.
 *   Collective on a sharded engine.  While enabled pfgpu_fs_step (known ids) returns PFGPU_ERR_UNSUPPORTED.  Disabled (the default)
 *   nothing changes.
 * pfgpu_fs_existence_counts: tau of local slots first_local .. first_local + count - 1, count x m particle-major; 0 for an empty
 *   slot.  Synchronises; valid where pfgpu_fs_download is.  Counters disabled: PFGPU_ERR_INVALID.
 * pfgpu_fs_existence_removed: copies removed by the last pfgpu_fs_step_unknown over this handle's particles (0 when disabled);
 *   synchronises. */
int  pfgpu_fs_existence_enable(pfgpu_fs*, double range);
int  pfgpu_fs_existence_counts(pfgpu_fs*, size_t first_local, size_t count, int32_t* out);
int  pfgpu_fs_existence_removed(pfgpu_fs*, uint64_t* removed);
int  pfgpu_fs_sync(pfgpu_fs*);

/* ============================================ plumbing ============================================== */
int  pfgpu_nccl_unique_id(void* out128);     /* ncclGetUniqueId; 128 bytes */

/* Counters for benches / tests.  kernel_launches = kernels of this library launched by the handle;
 * serial_fallbacks = times an exact-sum pipeline fell back to its single-thread path (should be 0).  PF / MCL with the fused
 * step (one launch after predict + likelihood): the separate kernels' count + the fused launch's serial walks + its refused
 * certificates, and xsum_dirty_last comes from whichever of the two ran the most recent exact sum. */
typedef struct {
    uint64_t kernel_launches;
    uint64_t steps;
    uint64_t resamples;
    uint64_t serial_fallbacks;
    uint64_t xsum_dirty_last;    /* dirty elements in the most recent exact scan */
    double   main_kernel_ms_sum; /* sum of CUDA-event times of the dominant kernel when timing is on */
    uint64_t main_kernel_count;
    uint64_t compactions;        /* sharded FastSLAM: guest-column compactions so far */
    uint64_t imported_particles; /* sharded FastSLAM: particles whose map came from another rank so far */
} pfgpu_stats;
int  pfgpu_pf_stats(pfgpu_pf*, pfgpu_stats*);
int  pfgpu_fs_stats(pfgpu_fs*, pfgpu_stats*);
/* debug (PFGPU_POST_TRACE=1): accumulated per-phase times [ns] of the fused post-step kernel; out32[31] = launches,
   out32[11] = resamples that ran the exact S2 and CDF sums instead of the certified CDF (counted with or without the trace) */
int  pfgpu_fs_post_trace(pfgpu_fs*, unsigned long long* out32);
/* shape of the fused post-step kernel: tiles (one co-resident CTA each) x threads x values per thread, and whether the tiles
   live in shared memory (*global_tile = 0) or, for particle counts whose tile does not fit on chip, in global memory (1) */
int  pfgpu_fs_post_shape(pfgpu_fs*, unsigned* tiles, unsigned* threads, unsigned* values_per_thread, int* global_tile);
/* *k1 = 1 when the post-step kernel runs its instantiation for one value and at most one local slot per thread (512 threads,
   shared-memory tiles; config 3 on one GPU), 0 when it runs the generic one (always, with PFGPU_POST_K1=0) */
int  pfgpu_fs_post_k1(pfgpu_fs*, int* k1);
/* how the coupled part of the step runs: 0 = one GPU, 2 = sharded over peer memory (NVLink loads / stores inside the kernels;
   no NCCL call and no host sync per step) */
int  pfgpu_fs_shard_mode(pfgpu_fs*, int* mode);
int  pfgpu_pf_time_main_kernel(pfgpu_pf*, int on);
int  pfgpu_fs_time_main_kernel(pfgpu_fs*, int on);
/* CUDA events on the handle's own stream (bench.py times steps with these): mark(slot 0..16383) records an
 * event; elapsed(a, b) synchronises on slot b and returns the device time between the two marks. */
int  pfgpu_pf_mark(pfgpu_pf*, int slot);
int  pfgpu_pf_elapsed_ms(pfgpu_pf*, int slot_a, int slot_b, double* ms);
int  pfgpu_fs_mark(pfgpu_fs*, int slot);
int  pfgpu_fs_elapsed_ms(pfgpu_fs*, int slot_a, int slot_b, double* ms);
/* Evict the L2 cache between timed steps: overwrites a scratch buffer larger than L2 on the handle's stream. */
int  pfgpu_pf_flush_l2(pfgpu_pf*);
int  pfgpu_fs_flush_l2(pfgpu_fs*);

#ifdef __cplusplus
}
#endif
#endif /* PFGPU_H */
