/*
 * include/artp.h -- C ABI of the CUDA-native art_planner hot path (libartp.so).
 *
 * Drop-in boundary (SURVEY.md section 8b): everything the reference's OMPL plugins for this path need,
 * as plain C: pointers + sizes, no C++/torch types, no exceptions across the boundary. Every entry point
 * returns 0 on success or a negative ARTP_E_* code; artp_last_error() gives the message.
 * There is NO CPU fallback: if no CUDA device / kernel image is usable the calls fail with ARTP_E_CUDA.
 *
 * Reference interfaces each entry point replaces (paths relative to the reference tree):
 *   artp_create / artp_destroy      art_planner::StateValidityChecker ctor (validity_checker.cpp:9-16) ->
 *                                   ValidityCheckerBody/Feet ctors -> HeightMapBoxChecker ctor
 *                                   (height_map_box_checker.cpp:11-26); parameters from art_planner::Params
 *                                   (include/art_planner/params.h:14-123)
 *   artp_set_map                    StateValidityChecker::setMap + updateHeightField (validity_checker.cpp:20-31)
 *                                   -> HeightMapBoxChecker::setHeightField (height_map_box_checker.cpp:38-54);
 *                                   installed at Planner::setMap (art_planner/src/planner.cpp:135-163)
 *   artp_check_poses[_device]       ompl::base::StateValidityChecker::isValid, i.e.
 *                                   art_planner::StateValidityChecker::isValid (validity_checker.cpp:39-45)
 *   artp_check_motions[_device]     ompl::base::MotionValidator::checkMotion as the reference uses it: OMPL's
 *                                   DiscreteMotionValidator over isValid (call sites prm_motion_cost.cpp:652,
 *                                   lazy_prm_star_min_update.cpp:725) and the in-tree interpolation loop
 *                                   PRMMotionCost::addValidMilestone (prm_motion_cost.cpp:341-372)
 *   artp_check_edge_interiors[_device]  that same addValidMilestone loop with its exact semantics: per-edge
 *                                   interior-state counts, no endpoint check, stop at the first invalid state
 *   artp_set_sampler, artp_sample_states[_device], artp_sample_valid[_device], artp_sampler_uniforms
 *                                   ompl::base::StateSampler::sampleUniform -> SE3FromSE2Sampler::sampleUniform
 *                                   (src/sampler.cpp:82-131, positions :40-77) and the rejection loops around it
 *                                   (prm_motion_cost.cpp:171-194, lazy_prm_star_min_update.cpp:549-556)
 *   artp_find_valid_near[_device], artp_ball_offsets
 *                                   StartState::sampleGoal (src/start.cpp:7-41, called from Planner::setStartAndGoal,
 *                                   planner.cpp:167-189) and GoalStateRegion::sampleGoal (src/goal.cpp:11-41, called by
 *                                   OMPL inside ss_->solve): the centre, then up to n_iter uniformInBall offsets in x / y,
 *                                   each through isValid, first valid wins
 *   artp_pose_from_2d               the goal's projection in Planner::plan (planner.cpp:223-237): grid_map isInside, then
 *                                   Map::get3DPoseFrom2D (src/map/map.cpp:77-90) + setSO3FromRPY (utils.h:101-115)
 *   artp_estimate_normals           art_planner::estimateNormals (src/utils.cpp:213-324; processors::Basic, basic.cpp:47)
 *   artp_compute_sample_cdf         computeCumulativeProbabilityDistribution
 *                                   (src/map/processors/probability_distribution.cpp:20-46)
 *   artp_compact_valid_device, artp_pack_valid_bits_device, artp_compact_bits_device
 *                                   no reference counterpart: the multi-GPU verdict exchange (SURVEY 8e)
 *   artp_path_length_cost[_device]  ompl::base::OptimizationObjective::motionCost ->
 *                                   PathLengthObjective::motionCost (objectives/path_length_objective.cpp:26-70)
 *   artp_set_cost_weights, artp_update_features, artp_motion_cost[_device]
 *                                   the MotionCostFunc batch functor (objectives/motion_cost_objective.h:22-23)
 *                                   = ROS service cost_query (art_planner_ros/src/planner_ros.cpp:283-308,
 *                                   art_planner_motion_cost/scripts/cost_query_server.py:145-169,
 *                                   predictor/predictor.py:28-44, predictor/cost_query.py:39-69)
 *   artp_combine_cost               MotionCostObjective::getCost / isFeasible (motion_cost_objective.h:54-66)
 *   artp_motion_cost_split[_device] ompl::base::OptimizationObjective::motionCost -> MotionCostObjective::motionCost
 *                                   (objectives/motion_cost_objective.cpp:36-95), the objective planner_ros.cpp:313-317
 *                                   installs; callers: path.cost(obj) in Planner::getSolutionPath (planner.cpp:281-283),
 *                                   opt_->motionCost (lazy_prm_star_min_update.cpp:436)
 */
#ifndef ARTP_H
#define ARTP_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ARTP_OK            0
#define ARTP_E_INVALID    -1   /* bad argument */
#define ARTP_E_NOMAP      -2   /* no map set (hasMap() == false) */
#define ARTP_E_CUDA       -3   /* CUDA runtime error / no device */
#define ARTP_E_LIMIT      -4   /* box/map combination exceeds a compiled limit */
#define ARTP_E_NOWEIGHTS  -5   /* motion-cost network weights / features not set */
#define ARTP_E_WINDOW     -6   /* a box reached outside the handle's map window (artp_set_map_window) */

/* art_planner::Params fields the hot path reads (include/art_planner/params.h). Doubles as in the reference. */
typedef struct artp_params {
  double torso_length, torso_width, torso_height;   /* params.h:92-94   */
  double torso_off_x, torso_off_y, torso_off_z;     /* params.h:96-100  */
  double feet_off_x, feet_off_y, feet_off_z;        /* params.h:106-110 */
  double reach_x, reach_y, reach_z;                 /* params.h:112-116 */
  int    unknown_space_untraversable;               /* params.h:26      */
  int    use_directional_cost;                      /* params.h:73      */
  double max_lon_vel, max_lat_vel, max_ang_vel;     /* params.h:74-76   */
  float  cost_w_energy, cost_w_time, cost_w_risk;   /* params.h:57-61   */
  float  risk_threshold;                            /* params.h:55      */
  int    device;                                    /* CUDA device ordinal for this handle */
} artp_params;

typedef struct artp_handle artp_handle;

typedef struct artp_stats {
  uint64_t poses_checked;      /* pose checks executed since creation */
  uint64_t poses_deferred;     /* deferred items summed over the calls whose stats were read (one read per call) */
  uint64_t kernel_launches;    /* kernels launched by this handle since creation */
  uint32_t last_deferred;      /* deferred count of the most recent check call */
  uint32_t last_launches;      /* kernels launched by the most recent call */
  uint32_t last_queued_boxes;  /* boxes the classify stage queued for the later stages in the most recent call's last round */
  uint32_t last_queued_warp_stage;   /* ... of which in the big-tile queue (torso boxes, reach boxes of unusual size) */
  uint32_t last_queued_reach_stage;  /* ... of which in the one-warp-per-box reach queue (zones with mergeable planes or not reduced by the tables) */
  uint32_t last_reach_plane_stage;   /* ... of which in the 8-lane-group reach queue (merge-free zones, with or without -inf) */
} artp_stats;

int  artp_create(const artp_params* params, artp_handle** out);
void artp_destroy(artp_handle* h);
const char* artp_last_error(const artp_handle* h);   /* h may be NULL: last creation error */

/* Layers are HOST pointers in grid_map layout: column-major rows x cols floats, (i,j) at data[i + j*rows];
 * lengths = rows*res, cols*res; centre (cx, cy). Heights must be finite or -inf. */
int artp_set_map(artp_handle* h, const float* elevation, const float* elevation_masked,
                 int rows, int cols, double res, double cx, double cy);
int artp_has_map(const artp_handle* h);
/* Spatial shard of a map (multi-GPU, SURVEY 8e): the handle receives only rows [row0, row0 + nrows) of the rows x cols
 * layers (HOST pointers to nrows x cols column-major matrices; row0 a multiple of 4) -- its slab plus a halo of at least
 * the largest box half-diagonal + box offsets -- while rows, res, cx, cy describe the FULL map. Geometry (ODE sample
 * spacing L / (N - 1), vertex coordinates, grid_map isInside) is that of the full map, so verdicts are bit-identical to a
 * handle holding everything; device memory and the range / plane tables shrink to the window. A pose whose boxes reach
 * outside the window is reported invalid and raises ARTP_E_WINDOW (sticky, like ARTP_E_LIMIT): route every sample to
 * the shard that holds it. The sampler, normal estimation and the cost network need the whole map (ARTP_E_INVALID). */
int artp_set_map_window(artp_handle* h, const float* elevation, const float* elevation_masked, int rows, int cols,
                        double res, double cx, double cy, int row0, int nrows);

/* n SE(3) states, 7 doubles each (x y z qx qy qz qw) -> valid[n] (0/1). HOST buffers; H2D/D2H inside. */
int artp_check_poses(artp_handle* h, const double* states, size_t n, uint8_t* valid);
/* Same with DEVICE buffers on `stream` (a cudaStream_t cast to void*, may be NULL); asynchronous. */
int artp_check_poses_device(artp_handle* h, const double* d_states, size_t n, uint8_t* d_valid, void* stream);

/* Pinned host memory for the adapter's batch buffers (states in, verdicts out): pages from cudaHostAlloc reach the device
 * at PCIe line rate, which memory pinned after the fact does not (profiles/pcie_probe.cu). NULL on failure. */
void* artp_host_alloc(size_t bytes);
void  artp_host_free(void* p);

/* float32 states (n x 7 floats): the caller applies the double -> float cast Pose3FromSE3 (utils.h:25-38) performs
 * first; results are identical to the double entry points at half the host<->device traffic. */
int artp_check_poses_f32(artp_handle* h, const float* states, size_t n, uint8_t* valid);
int artp_check_poses_f32_device(artp_handle* h, const float* d_states, size_t n, uint8_t* d_valid, void* stream);

/* Edge validity: valid(s2) && valid(interp(s1,s2,j/(n_steps+1))) for j = 1..n_steps (n_steps >= 0). */
int artp_check_motions(artp_handle* h, const double* s1, const double* s2, size_t n, int n_steps, uint8_t* valid);
int artp_check_motions_device(artp_handle* h, const double* d_s1, const double* d_s2, size_t n, int n_steps,
                              uint8_t* d_valid, void* stream);

/* ompl::base::DiscreteMotionValidator::checkMotion(s1, s2[, lastValid]) (OMPL 1.4.2; the reference's default motion
 * validator, call sites prm_motion_cost.cpp:652, lazy_prm_star_min_update.cpp:725) with PER-EDGE segment counts:
 * edge e is valid iff interpolate(s1, s2, j / nd[e]) is valid for j = 1 .. nd[e]-1 and s2 is valid. nd[e] =
 * SE3StateSpace::validSegmentCount(s1, s2); nd == NULL: computed by artp_valid_segment_count from *sp (the space
 * parameters Planner::setMap installs, planner.cpp:146-156). last_valid_t (nullable) receives lastValid.second: the
 * parameter of the last valid state before the first invalid one in OMPL's order ((j-1)/nd, or (nd-1)/nd when only s2
 * is invalid; 1.0 for valid edges) -- the caller obtains lastValid.first by interpolating at that parameter. */
typedef struct artp_se3_space {
  double low[3], high[3];                  /* RealVectorBounds of the SE3 space (planner.cpp:148-156) */
  double longest_valid_segment_fraction;   /* OMPL default 0.01 (the reference never changes it); <= 0 means 0.01 */
} artp_se3_space;
int artp_valid_segment_count(const artp_se3_space* sp, const double* s1, const double* s2, size_t n, int32_t* nd);
int artp_check_motions_segments(artp_handle* h, const double* s1, const double* s2, size_t n, const int32_t* nd,
                                const artp_se3_space* sp, uint8_t* valid, double* last_valid_t);

/* PRMMotionCost::addValidMilestone's connection test (prm_motion_cost.cpp:341-372), batched over the n candidate
 * edges of new milestones: edge e has n_interp[e] interior states at t = step * (1.0 / (n_interp[e] + 1)),
 * step = 1..n_interp[e] (endpoints are NOT checked there), and the reference loop stops at the first invalid one.
 * valid_prefix[e] = number of leading valid interior states; the connection is valid iff it equals n_interp[e], and
 * the caller inserts the first valid_prefix[e] states as intermediate milestones exactly like :356-366.
 * n_interp == NULL: computed per edge as (unsigned)(lateralDistance(s1, s2) / max_lateral) like :341-343
 * (the reference's max_lateral is 0.5). Total interior states must be < 2^32. */
int artp_check_edge_interiors(artp_handle* h, const double* s1, const double* s2, size_t n, const int32_t* n_interp,
                              double max_lateral, int32_t* valid_prefix);
/* DEVICE buffers: d_item_off = n + 1 exclusive prefix sums (uint32) of the per-edge interior-state counts,
 * total_items = d_item_off[n], d_item_valid = scratch of total_items bytes that receives the per-state flags. */
int artp_check_edge_interiors_device(artp_handle* h, const double* d_s1, const double* d_s2, size_t n,
                                     const uint32_t* d_item_off, size_t total_items, uint8_t* d_item_valid,
                                     int32_t* d_valid_prefix, void* stream);

/* ---- SE3FromSE2Sampler::sampleUniform (art_planner/src/sampler.cpp:40-131) on the device ------------------------
 * SURVEY 8(f) rank 2: candidates are generated where they are checked, so the rejection loops
 * (prm_motion_cost.cpp:171-194, lazy_prm_star_min_update.cpp:549-556) need no host->device pose stream.
 * One candidate consumes six uniform01 variates in the order the reference draws them:
 *   sample_from_distribution:  u0 = samp_col, u1 = samp_row (:56-57), u2 -> uniformReal(-1,1) (:103),
 *                              u3,u4,u5 -> RNG::eulerRPY roll, pitch, yaw (:114)
 *   otherwise:                 u0 -> x, u1 -> y in [low, high]; a position outside the map is a rejected candidate
 *                              (NaN state, rowcol -1, never valid) where the reference loop (:46-50) draws again.
 * The variates are either caller-provided (u != NULL) or produced by the documented counter-based stream
 * Philox4x32-10(key = seed, counter = (sample index, block 0..2, "ARTP")), see artp_sampler_uniforms(). */
typedef struct artp_sampler_params {
  double max_roll_pert, max_pitch_pert;   /* params.h:79-80, radians */
  int    sample_from_distribution;        /* params.h:81 */
  double low[2], high[2];                 /* SE3 position bounds x,y (planner.cpp:148-160); uniform mode only */
} artp_sampler_params;

/* Per-cell layers the sampler reads, HOST pointers in grid_map layout (like artp_set_map, which must come first and
 * provides "elevation" and the geometry): normal_x/y/z, plane_fit_std_dev (Map::getNormal / getPlaneFitStdDev,
 * map.h:94-116), "cum_prob" and column 0 of "cum_prob_rowwise_hack" (probability_distribution.cpp:20-46; may be NULL
 * when !sample_from_distribution). The four normal / plane-fit pointers may all be NULL after artp_estimate_normals.
 * CDF rows must be non-decreasing or all NaN (else ARTP_E_INVALID).
 * artp_set_map invalidates the sampler layers. */
/* art_planner::estimateNormals (art_planner/src/utils.cpp:213-324; called from processors::Basic, basic.cpp:47, with
 * estimation_radius = (torso.length + torso.width) * 0.25) for the elevation layer of the current map, on the device.
 * The four layers stay on the device as the sampler's normal / plane-fit layers (then artp_set_sampler may be called
 * with the four pointers NULL) and are copied to the non-NULL HOST outputs (grid_map layout). Bit-identical to the
 * reference's float arithmetic (the elevation layer's -0 is stored as +0, see artp_set_map). */
int artp_estimate_normals(artp_handle* h, double estimation_radius, float* normal_x, float* normal_y, float* normal_z,
                          float* plane_fit_std_dev);
/* computeCumulativeProbabilityDistribution (src/map/processors/probability_distribution.cpp:20-46) on the device:
 * "sample_probability" (HOST, grid_map layout) -> "cum_prob" and column 0 of "cum_prob_rowwise_hack", kept on the device
 * as the sampler's CDF layers (artp_set_sampler may then get NULL for both) and copied to the non-NULL HOST outputs.
 * Sums run left to right per row; rows without mass become NaN rows exactly like the reference's 0/0. */
int artp_compute_sample_cdf(artp_handle* h, const float* sample_probability, float* cum_prob, float* cum_prob_rowwise);
int artp_set_sampler(artp_handle* h, const artp_sampler_params* sp, const float* normal_x, const float* normal_y,
                     const float* normal_z, const float* plane_fit_std_dev, const float* cum_prob,
                     const float* cum_prob_rowwise);
/* The variates of samples first_sample .. first_sample+n-1 under `seed`: u[n][6] (host). */
int artp_sampler_uniforms(artp_handle* h, uint64_t seed, uint64_t first_sample, size_t n, double* u);
/* n candidates -> states[n][7] (x y z qx qy qz qw), rowcol[n][2] (sampled cell; nullable). u == NULL: Philox stream. */
int artp_sample_states(artp_handle* h, const double* u, uint64_t seed, uint64_t first_sample, size_t n, double* states,
                       int32_t* rowcol);
int artp_sample_states_device(artp_handle* h, const double* d_u, uint64_t seed, uint64_t first_sample, size_t n,
                              double* d_states, int32_t* d_rowcol, void* stream);
/* Fused sample -> isValid -> ordered compaction: draws candidates first_sample .. first_sample+n_draw-1 of the Philox
 * stream and writes the valid ones, in draw order, to states (at most `capacity`); *n_valid / *d_count = number of
 * valid candidates (> capacity: output truncated). */
int artp_sample_valid(artp_handle* h, uint64_t seed, uint64_t first_sample, size_t n_draw, double* states,
                      size_t capacity, size_t* n_valid);
int artp_sample_valid_device(artp_handle* h, uint64_t seed, uint64_t first_sample, size_t n_draw, double* d_states_out,
                             size_t capacity, uint32_t* d_count, void* stream);

/* ---- StartState / GoalStateRegion::sampleGoal (src/start.cpp:7-41, src/goal.cpp:11-41) on the device ---------------
 * n independent searches. For query q, candidate 0 is centres[q] unchanged; candidate k = 1..n_iter is centres[q] with
 * x += off[q][k-1][0], y += off[q][k-1][1] (double adds; z and the quaternion stay). states_out[q] = the first candidate, in
 * the order 0, 1, .., n_iter, that isValid accepts, and index[q] = its k. When none is valid, states_out[q] = candidate
 * n_iter (the last drawn one: what the reference's caller is left holding, since its `state = nullptr` only clears a
 * local) and index[q] = -1. All n * (n_iter + 1) candidates are checked in one pass.
 * Offsets: offsets != NULL gives them (n x n_iter x 2 doubles); NULL draws them from the counter-based stream
 *   Philox4x32-10(key = seed, counter = (draw lo, draw hi, q, "ARTB")), draw = first_draw + k - 1,
 *   u0, u1 = the two doubles of that block taken as in artp_sampler_uniforms, off = radius[q] * sqrt(u1) * (cos 2 pi u0,
 *   sin 2 pi u0).
 * That is the distribution of OMPL's RNG::uniformInBall(radius) in 2-D (uniform direction, radius r * u^(1/2)) but not its
 * stream, which is a serial mt19937: feed OMPL's own offsets to reproduce a reference run exactly. The reference draws k
 * offsets when it returns candidate k, n_iter when none is valid, none when the centre is valid.
 * radius: n doubles, finite and >= 0 (host form: else ARTP_E_INVALID; the device form does not read them back to check).
 * n < 2^32 and n * (n_iter + 1) < 2^32, else ARTP_E_INVALID. On a map window a candidate whose boxes leave the window is
 * invalid and the call raises ARTP_E_WINDOW, as every check does. */
int artp_find_valid_near(artp_handle* h, const double* centres, size_t n, const double* radius, uint32_t n_iter,
                         const double* offsets, uint64_t seed, uint64_t first_draw, double* states_out, int32_t* index);
int artp_find_valid_near_device(artp_handle* h, const double* d_centres, size_t n, const double* d_radius, uint32_t n_iter,
                                const double* d_offsets, uint64_t seed, uint64_t first_draw, double* d_states_out,
                                int32_t* d_index, void* stream);
/* The stream's offsets (n x n_iter x 2 doubles, host) that artp_find_valid_near draws with offsets == NULL. */
int artp_ball_offsets(artp_handle* h, uint64_t seed, uint64_t first_draw, size_t n, uint32_t n_iter, const double* radius,
                      double* offsets);
/* The goal projection of Planner::plan (planner.cpp:223-237): for a state whose (x, y) lies on the map (grid_map isInside
 * and getIndexFromPosition), z = the cell's "elevation", roll = -atan2(nb.y, nb.z), pitch = atan2(nb.x, nb.z) with
 * nb = AngleAxisd(yaw, UnitZ)^-1 * the cell's normal, yaw = getYawFromSO3 (double atan2 returned as float), and the
 * quaternion from setSO3FromRPY; x and y are not moved. Other states are copied unchanged with inside[i] = 0 (nullable).
 * HOST buffers. Needs the normal layers of the current map (artp_estimate_normals, or artp_set_sampler with host layers),
 * else ARTP_E_INVALID; ARTP_E_INVALID on a map window. The bounds clip before it (enforceBounds) stays with OMPL. */
int artp_pose_from_2d(artp_handle* h, const double* states_in, size_t n, double* states_out, uint8_t* inside);

/* PathLengthObjective::motionCost for n edges -> cost[n] (double). */
int artp_path_length_cost(artp_handle* h, const double* s1, const double* s2, size_t n, double* cost);
int artp_path_length_cost_device(artp_handle* h, const double* d_s1, const double* d_s2, size_t n,
                                 double* d_cost, void* stream);

/* Ordered compaction of a validity mask into indices (for the multi-GPU index all-gather):
 * d_indices[k] = base + i for the k-th i with d_valid[i] != 0; *d_count = number written. Device buffers. */
int artp_compact_valid_device(artp_handle* h, const uint8_t* d_valid, size_t n, int64_t base,
                              int64_t* d_indices, uint32_t* d_count, void* stream);
/* Multi-GPU exchange format: the mask bit-packed (item i = bit i&31 of word i>>5; (n+31)/32 words, tail bits 0) --
 * 125 KB per 10^6 poses on the wire instead of 8 MB of padded indices -- and the ordered compaction of such a
 * (gathered) bit mask, which every rank runs on the all-gathered words to obtain the global valid-index list. */
int artp_pack_valid_bits_device(artp_handle* h, const uint8_t* d_valid, size_t n, uint32_t* d_bits, void* stream);
/* A shard's step of the multi-GPU path in one call: isValid of its n samples (d_valid, bytes) and the bit-packed mask
 * (d_bits, (n+31)/32 words) that goes on the wire. */
int artp_check_poses_bits_device(artp_handle* h, const double* d_states, size_t n, uint8_t* d_valid, uint32_t* d_bits, void* stream);
/* Ordered compaction into 32-bit indices (base + i): the per-shard valid-sample list; a consumer that needs the global
 * list reads the per-rank counts + segments. */
int artp_compact_valid_u32_device(artp_handle* h, const uint8_t* d_valid, size_t n, uint32_t base, uint32_t* d_indices,
                                  uint32_t* d_count, void* stream);
int artp_compact_bits_device(artp_handle* h, const uint32_t* d_bits, size_t n, int64_t base, int64_t* d_indices,
                             uint32_t* d_count, void* stream);

int artp_get_stats(artp_handle* h, artp_stats* out);

/* Threads and streams. A handle is safe to share between threads (the reference's checkers are called from the planning
 * thread, the ROS callback threads and the cleaner thread, SURVEY 8b): every entry point holds the handle's lock for its
 * whole duration, host-buffer calls including their staging copies. The *_device entry points are asynchronous on the
 * caller's stream; calls issued on DIFFERENT streams are ordered against each other on the device (each waits for the
 * previous user of the handle's scratch buffers), so they are safe but do not overlap -- use one handle per stream for
 * concurrency.
 *
 * Errors detected on the device: if the plane-grouping stage cannot hold a zone in its shared-memory store (sized at
 * artp_set_map from the box diagonals; cannot happen for boxes that passed artp_set_map unless the test hook below is
 * used) the affected pose / edge is reported INVALID (fail closed) and a sticky error is raised: host-buffer calls return
 * ARTP_E_LIMIT from the call that caused it; after asynchronous *_device calls, synchronise the stream and call
 * artp_poll_error (returns ARTP_E_LIMIT once, then clears). artp_get_stats reports it too. */
int artp_poll_error(artp_handle* h);
/* Test hook: cap the plane store at max_triangles (0 = no cap) from the next artp_set_map on. */
int artp_debug_set_group_capacity(artp_handle* h, int max_triangles);
/* Test hook: *n = length of the one-warp-per-box reach queue of the most recent check call's last round; its first
 * min(*n, cap) records (80 bytes each, artp_kernels.cuh BoxRec) are copied to the HOST buffer recs. Synchronises the device. */
int artp_debug_get_reach_queue(artp_handle* h, void* recs, size_t cap, size_t* n);

/* Environment switch (a test hook, never needed in production):
 *   ARTP_NO_GROUPS=1        (read at artp_set_map) every undecided reach box takes the one-warp-per-box queue instead of the
 *                           8-lane-group kernel -- same verdicts (tests/test_pose_gpu.py runs both)
 * artp_set_timing(h, 1) makes the host-buffer calls copy their states before the kernels start and run the kernels in
 * order on one stream (the per-stage events need one stream), so that, as for the *_device calls, the events cover the
 * call's whole last round of up to 2^20 states: leave it off when measuring end-to-end throughput. */

/* Kernel timing for roofline reporting: when enabled, CUDA events are recorded on the launch stream around the three
 * stages of every check call; artp_get_last_timing waits for the last call's kernels and returns
 * ms3[0..2] = classify (thread/item), box stages (warp stage + reach-box stages), plane-grouping block stage, in ms. */
int artp_set_timing(artp_handle* h, int enable);
int artp_get_last_timing(artp_handle* h, float* ms3);
/* Per-stage form: ms5 = classify, big-tile queue (torso boxes), reach-box queue (warp per box), reach-box queue (8-lane
 * groups), plane grouping. */
int artp_get_last_stage_timing(artp_handle* h, float* ms5);

/* Test hook: 0 = normal (classify -> warp stage -> grouping stage for deferred boxes),
 *            1 = send every in-map box through the exact block-level grouping kernel. */
int artp_set_mode(artp_handle* h, int mode);

/* ---- processors::Basic::setMaskedElevationAndTraversability (art_planner/src/map/processors/basic.cpp:42-106) ------
 * The producer of `elevation_masked` on the device: traversability threshold (+ "observed" masking), hole closing,
 * drop / wall masks, safety-margin erosion, small-patch removal -- grey-scale morphology with OpenCV's circular
 * structuring element (art_planner/src/utils.cpp:106-209) as exact min / max filters -- then
 * elevation_masked = traversable ? elevation : -inf. Inputs are the INPAINTED layers (basic.cpp:44-45: TELEA inpainting
 * is a sequential fast-marching method and stays with the caller); HOST pointers, grid_map layout; `observed` may be NULL
 * when !unknown_space_untraversable. Outputs: elevation_masked and (nullable) "traversability_thresholded". */
typedef struct artp_basic_params {
  float  traversability_thres;                        /* params.h:23 */
  int    unknown_space_untraversable;                 /* params.h:26 */
  double foothold_margin, foothold_margin_max_hole_size, foothold_margin_max_drop,
         foothold_margin_max_drop_search_radius, foothold_margin_min_step, foothold_size;   /* params.h:28-35 */
} artp_basic_params;
int artp_process_basic(artp_handle* h, const float* elevation, const float* traversability, const float* observed, int rows,
                       int cols, double res, const artp_basic_params* bp, float* elevation_masked, float* traversability_thresholded);
/* Test hook: the size x size structuring element of getCircularKernel(size) (utils.cpp:106-111) as 0/1 bytes; returns its
 * edge length (3 for size <= 0: OpenCV's default box). */
int artp_debug_circular_kernel(int size, uint8_t* out);

/* ---- the sampler's distribution (Planner::setUpMapProcessors, planner.cpp:39-58) ----------------------------------
 * The chain the reference builds with sample_from_distribution, and re-applies from PRMMotionCostMaintainer::sampleGraph
 * every recompute_density_after_n_samples vertices (prm_motion_cost.cpp:190-193), on the device:
 *   artp_set_sample_filter           Basic::setTraversabilityFilter (basic.cpp:110-125): dilateAndErode of
 *                                    "traversability_thresholded" by (int)(sqrt(reach.x^2 + reach.y^2) / res), then erode by
 *                                    (int)(min((torso.length - reach.x) / 2, (torso.width - reach.y) / 2) / res) cells
 *                                    (geometry from artp_params); the result and the "observed" layer stay on the device.
 *   artp_update_sample_distribution  computeInverseSampleDensity (sample_density.cpp:12-43: histogram of the vertices'
 *                                    (x, y), Gaussian blur, max - n), applyBaseSampleDistribution (x the filter, when one is
 *                                    set), applyMaxUnknownProbability (probability_distribution.cpp:50-91) and the CDF of
 *                                    artp_compute_sample_cdf, which stays resident: re-arm the sampler with
 *                                    artp_set_sampler(h, sp, ..., NULL, NULL) afterwards.
 * Every layer is bit-identical to oracle/sample_distribution_oracle.py; the blur is within 2e-6 x max(layer) of
 * cv::GaussianBlur (DESIGN.md 4.4). A stateless call: with no vertex on the map the density is the uniform 1 (the
 * reference would keep its previous layer). artp_set_map drops the filter and observed layers; a map window is
 * ARTP_E_INVALID. */
typedef struct artp_sample_distribution_params {
  int    use_inverse_vertex_density;      /* params.h:82 */
  double density_blur_radius;             /* planner.cpp:48: (torso.length + torso.width) * 0.25; > 0 */
  int    use_max_prob_unknown_samples;    /* params.h:83 */
  double max_prob_unknown_samples;        /* params.h:84; in [0, 1] */
} artp_sample_distribution_params;
/* HOST grid_map layers of the current map's rows x cols. NULL = the layer the last artp_process_basic on this handle
 * received (observed) / produced (traversability_thresholded), when it ran on a map of the same size (else
 * ARTP_E_INVALID for traversability_thresholded; no observed layer for observed). traversability_sample_filter: nullable
 * HOST out. Structuring elements above 64 cells: ARTP_E_LIMIT. */
int artp_set_sample_filter(artp_handle* h, const float* traversability_thresholded, const float* observed,
                           float* traversability_sample_filter);
/* vertex_states: the roadmap's vertices, n x 7 doubles (only x, y read; order irrelevant; off-map or NaN positions are
 * not counted). Blur kernel (int)(6 r / res) (+1 if even) above 1023 cells: ARTP_E_LIMIT. The cap without an observed
 * layer, or bad parameters: ARTP_E_INVALID. sample_probability, cum_prob (rows x cols) and cum_prob_rowwise (rows):
 * nullable HOST outs. The _device form reads DEVICE vertex states and runs asynchronously on `stream`. */
int artp_update_sample_distribution(artp_handle* h, const artp_sample_distribution_params* dp,
                                    const double* vertex_states, size_t n, float* sample_probability,
                                    float* cum_prob, float* cum_prob_rowwise);
int artp_update_sample_distribution_device(artp_handle* h, const artp_sample_distribution_params* dp,
                                           const double* d_vertex_states, size_t n, void* stream);
/* Test hook: getGaussianKernel(ksize, sigma, CV_32F) as the blur uses it (odd ksize <= 1023, sigma > 0); returns ksize. */
int artp_debug_gaussian_kernel(int ksize, double sigma, float* out);

/* ---- PRM roadmap on the device (PRMMotionCost, art_planner/src/planners/prm_motion_cost.cpp) ----------------------
 * The handle owns an append-only roadmap: vertex states (7 doubles) with a kind byte each, and undirected edges (u, v),
 * both in the order PRMMotionCost::addValidMilestone (:325-390) inserts them into its Boost graph, so vertex i here is
 * vertex i of g_. Every milestone is added on the device with three kernels and no host synchronisation:
 *   neighbours  KStarStrategy (OMPL 1.4.2 ConnectionStrategy.h): k = ceil((e + e/6) ln V), V = num_vertices(g_) with the
 *               new milestone counted (LazyPRM::milestoneCount), over the vertices already in the roadmap, exact
 *               (GNAT nearestK is exact) in ascending SE3StateSpace::distance (R3 Euclidean + acos(|q1.q2|), 0 above
 *               1 - 1e-9); exact ties go to the lower vertex index (GNAT leaves them unspecified). Per neighbour
 *               n_interp = (unsigned)(lateralDistance / 0.5) interior states at step * (1.0 / (n_interp + 1)).
 *   check       every interior state through the validity pipeline's per-pose routine.
 *   commit      :335-387: the valid prefix of each connection becomes a chain of interpolated vertices and edges, the
 *               final edge only when the whole connection is valid, a direct edge when n_interp == 0.
 * Edges are priced and searched in place by the query calls below.
 * The map must be the whole map (a map window is ARTP_E_INVALID). A milestone that would overflow the store's capacity
 * is not added and the call returns ARTP_E_LIMIT (the roadmap keeps every earlier milestone). */
#define ARTP_ROADMAP_MILESTONE     1   /* a milestone (sampled, or added with artp_roadmap_add_milestones) */
#define ARTP_ROADMAP_INTERPOLATED  2   /* an interior state of a connection (prm_motion_cost.cpp:358-365) */
#define ARTP_ROADMAP_QUERY         4   /* with MILESTONE: added by artp_roadmap_add_milestones (start / goal, startM_ / goalM_) */
typedef struct artp_roadmap_params {
  size_t   max_n_vertices;                     /* params.h:51, 10000 */
  size_t   max_n_edges;                        /* params.h:52, 50000 */
  size_t   recompute_density_after_n_samples;  /* params.h:53, 1000; 0 = never */
  uint64_t max_draws;                          /* sampler draws the call may use: replaces max_sample_time (:177-184) */
} artp_roadmap_params;
/* PRMMotionCost::clear (:236-247): empties the roadmap and sizes its store for vertex_capacity vertices and
 * edge_capacity edges (> 0 and < 2^31; ARTP_E_INVALID otherwise). The store outlives artp_set_map. */
int artp_roadmap_clear(artp_handle* h, size_t vertex_capacity, size_t edge_capacity);
/* addValidMilestone for the n HOST states, in order (baseSolve's start and goal milestones, :451-479). Kind
 * MILESTONE | QUERY: these count in the sampling density like startM_ / goalM_ (LazyPRM::getPlannerData). No roadmap
 * (artp_roadmap_clear never called): ARTP_E_INVALID. */
int artp_roadmap_add_milestones(artp_handle* h, const double* states, size_t n);
/* PRMMotionCostMaintainer::sampleGraph's loop (:171-194): while V < max_n_vertices and E < max_n_edges (checked before
 * each milestone), the next valid draw of the sampler (artp_set_sampler; Philox draws first_sample, first_sample + 1, ...)
 * becomes a milestone; after it, when V / recompute_density_after_n_samples exceeds the number of recomputes so far
 * (once per milestone), the distribution is recomputed as artp_update_sample_distribution(h, dp, ...) over the vertices
 * LazyPRM::getPlannerData returns -- QUERY milestones and the endpoints of edges; an isolated milestone is not counted --
 * and the sampler is re-armed on it; sampling goes on at the draw after the last milestone. dp NULL: no recompute.
 * The loop also ends when max_draws draws are used. *draws_used (nullable): draws consumed, up to and including the last
 * milestone's, or max_draws. Needs a map and an armed sampler (ARTP_E_NOMAP). */
int artp_roadmap_sample_graph(artp_handle* h, const artp_roadmap_params* rp, const artp_sample_distribution_params* dp,
                              uint64_t seed, uint64_t first_sample, uint64_t* draws_used);
/* The roadmap's tail to HOST buffers: vertices first_vertex .. V-1 (states: 7 doubles each, kinds: 1 byte each; both
 * nullable) and edges first_edge .. E-1 (edges: 2 uint32 each, nullable). *nv = V, *ne = E (nullable). A cursor past
 * the end: ARTP_E_INVALID. */
int artp_roadmap_get(artp_handle* h, size_t first_vertex, double* states, uint8_t* kinds, size_t first_edge,
                     uint32_t* edges, size_t* nv, size_t* ne);

/* ---- queries on the device roadmap (updateEdges :27-73, computeCostForVertexEdges :77-128, baseSolve :440-532,
 * constructSolution :536-673) ------------------------------------------------------------------------------------------
 * Every edge carries a double weight and a flag byte. A never-priced edge weighs 0.0 with no flag (ob::Cost(),
 * VALIDITY_UNKNOWN). The store stays append-only: an edge a query removes keeps its slot, with the REMOVED flag. */
#define ARTP_ROADMAP_EDGE_VALID    1   /* VALIDITY_TRUE: priced feasible by artp_roadmap_update_edges, or motion-checked */
#define ARTP_ROADMAP_EDGE_REMOVED  2   /* removed by constructSolution's failed motion check; not part of the graph */
/* updateEdges over the whole store: every edge (u, v) is priced by the loaded network from u towards v (row
 * [v.x v.y yaw(v) u.x u.y yaw(u)], artp_edge_matrix_from_states' arithmetic on the device); weight = getCost and the
 * VALID flag when the risk is within the threshold, else +inf and the flag untouched. Equal bit for bit to
 * artp_motion_cost_states on the copied-out edges. No weights or features: ARTP_E_NOWEIGHTS; no roadmap: ARTP_E_INVALID. */
int artp_roadmap_update_edges(artp_handle* h);
#define ARTP_SOLVE_SOLVED            1
#define ARTP_SOLVE_NOT_CONNECTED     2   /* start and goal in different components (baseSolve returns TIMEOUT) */
#define ARTP_SOLVE_NO_FEASIBLE_PATH  3   /* connected, but not over edges of finite weight ("Could not find solution path") */
#define ARTP_SOLVE_INVALID_START     4
#define ARTP_SOLVE_INVALID_GOAL      5
typedef struct artp_roadmap_solve_info {
  int32_t  status;                     /* ARTP_SOLVE_* */
  uint32_t searches;                   /* constructSolution calls (shortest-path searches) */
  uint32_t sweeps;                     /* relaxation sweeps of all searches */
  uint32_t edges_checked;              /* edges motion-checked */
  uint32_t edges_removed;              /* edges removed (failed motion checks) */
  uint32_t start_vertex, goal_vertex;  /* their vertex indices */
  uint32_t* path_vertices;             /* in: nullable HOST buffer of path_capacity entries; the path's vertex indices */
} artp_roadmap_solve_info;
/* One query, Planner::plan's clearQuery + PRMMotionCost::baseSolve. start, goal: 7 HOST doubles each. A state outside
 * space's bounds or failing the pose check: status INVALID_START / INVALID_GOAL, the roadmap unchanged. Otherwise the
 * earlier QUERY vertices lose their QUERY bit, start and goal are added like artp_roadmap_add_milestones, and the edges
 * at the start, then at the goal, are priced from the query vertex towards its neighbour, validity untouched (an edge
 * joining the two ends with the goal's direction; the edges between the interpolated vertices of their connections stay
 * at 0.0). Then, on the device, until a path stands or start and goal are disconnected: distances from the start over
 * the live edges of finite weight (d[v] = min fl(d[u] + w): what Dijkstra with a zero heuristic computes); the path is
 * the optimal one with the fewest edges, the lowest predecessor index on ties (Boost leaves ties to its heap); its edges
 * without the VALID flag are motion-checked from the start-side to the goal-side vertex as artp_check_motions_segments
 * does (nd from *space), the passing ones become VALID, the first failing one from the goal's side is REMOVED.
 * path_states: nullable HOST buffer of path_capacity x 7 doubles, start to goal. *n_path: its length; above
 * path_capacity nothing is written and the call returns ARTP_E_LIMIT. *cost: the sum of the path's weights from the
 * start, left to right. info: nullable. A vertex capacity above what the search holds on chip (77 440): ARTP_E_LIMIT.
 * ARTP_E_NOWEIGHTS / ARTP_E_INVALID / ARTP_E_NOMAP as artp_roadmap_update_edges and artp_roadmap_add_milestones. */
int artp_roadmap_solve(artp_handle* h, const double* start, const double* goal, const artp_se3_space* space,
                       double* path_states, size_t path_capacity, size_t* n_path, double* cost,
                       artp_roadmap_solve_info* info);
/* The weights (doubles) and flags (bytes) of the edges first_edge .. E-1 to HOST buffers (both nullable), like
 * artp_roadmap_get. *n_live (nullable): edges without the REMOVED flag in the whole store. */
int artp_roadmap_get_edge_costs(artp_handle* h, size_t first_edge, double* cost, uint8_t* flags, size_t* n_live);

/* ---- the solution path simplified on the device (Planner::getSolutionPath(true), planner.cpp:266-298) -------------
 * OMPL 1.4.2's PathSimplifier::simplifyMax as the simplifier SimpleSetup::simplifySolution builds from the space
 * information (objective PathLengthOptimizationObjective: cost = SE3StateSpace::distance, combined by +, a < b better; no
 * goal region, so no findBetterGoal), then getSolutionPath's check and cost comparison. Restated in
 * oracle/path_simplify_oracle.py, which is the definition; the rules:
 *   schedule        fewer than 3 states: unchanged. Else reduceVertices; collapseCloseVertices; reduceVertices again
 *                   while the previous call changed the path, at most 5 more times; shortcutPath while the previous call
 *                   changed the path, at most 5 times; smoothBSpline(path, 3, length / 100); checkAndRepair's check.
 *                   Every call of these takes a maxSteps and maxEmptySteps of its entry state count.
 *   reduceVertices  checkMotion(front, back) first (success: the two states). Else attempts p1 = uniformInt(0, maxN),
 *                   p2 = uniformInt(max(p1 - range, 0), min(maxN, p1 + range)), range = 1 + floor(0.5 + count * 0.33);
 *                   |p1 - p2| < 2: p2 = p1 + 2 if p1 < maxN - 1, else p1 - 2 if p1 > 1, else no attempt; a passing
 *                   checkMotion(states[p1], states[p2]) erases the states between and resets the empty-step count.
 *   collapseCloseVertices  each step the pair (i, j >= i + 2) of least SE3 distance (first in (i, j) order on ties) not
 *                   marked: checkMotion passes -> the states between are erased; fails -> the pair is marked for good (the
 *                   mark belongs to the two states, not their positions).
 *   shortcutPath    points p0 = uniformReal(0, L), p1 = uniformReal(max(0, p0 - 0.33 L), min(p0 + 0.33 L, L)) along the
 *                   cumulative distances, each snapped to the next / previous waypoint within L * 0.005, else interpolated
 *                   on its segment; same or adjacent segments or waypoints: no attempt (OMPL 1.4.2's three tests and the
 *                   three of later releases, without which 1.4.2 erases a reversed range); checkMotion(s0, s1), then the shortcut is kept
 *                   unless the cost along the path (partial first segment, whole segments, partial last segment, left to
 *                   right) is strictly lower than distance(s0, s1); the four edits of OMPL 1.4.2's shortcutPath.
 *   smoothBSpline   up to 3 steps of: subdivide (the midpoint after every state but the last), then for every even i in
 *                   [2, n - 1): if isValid(states[i-1]), m = mid(mid(states[i-1], states[i]), mid(states[i], states[i+1]));
 *                   checkMotion(states[i-1], m) and then checkMotion(m, states[i+1]) pass and distance(states[i], m) >
 *                   length / 100 (fixed before the first step) -> states[i] = m. A step that replaces nothing ends it.
 *   check           checkAndRepair's check (both end states valid, then every motion in order) without its repair
 *                   sampling, then PathGeometric::check (first state valid, every motion in order). Either failing
 *                   returns the original path (OMPL would try to repair first).
 *   comparison      PathGeometric::cost of both paths under `objective` (left-to-right sum of motion costs from 0.0); the
 *                   original is returned only when its cost is strictly lower.
 *   checkMotion     DiscreteMotionValidator: interpolate(s1, s2, j / nd), j = 1 .. nd - 1, then s2, nd from *space as
 *                   artp_check_motions_segments computes it; isValid is the pose check.
 * Randomness: attempt i of the c-th simplifier call of the schedule (from 0, one per call of the five functions above)
 * takes the two doubles of Philox4x32-10(key = seed, counter = (i, c, 0, "ARTS")), formed as artp_sampler_uniforms forms
 * them; uniformInt(a, b) = a + min(floor(u * (b - a + 1)), b - a), uniformReal(a, b) = a + u * (b - a). This is not
 * OMPL's mt19937 stream: same rules, other draws.
 * The path stays on the device for the whole call; the host reads its control block once per batch of rounds. */
#define ARTP_OBJ_LEARNED       0   /* MotionCostObjective (planner_ros.cpp:313-317): artp_motion_cost_split's cost at the
                                      call's max_query_edge_length (params.h:54, 0.5; > 0), +inf above the risk threshold;
                                      needs weights and features. The argument is read for this objective only. */
#define ARTP_OBJ_PATH_LENGTH   1   /* getObjective (planner.cpp:27-35): PathLengthObjective at weight 1.0
                                      (artp_path_length_cost) */
#define ARTP_OBJ_NONE          2   /* no comparison: the simplified path whenever it passes the check (simplifyMax) */
#define ARTP_SIMPLIFY_MAX_STATES 4096   /* input states at most (ARTP_E_LIMIT above) */
typedef struct artp_simplify_info {
  uint32_t n_in, n_simplified, n_out;   /* states in, after the simplifier, returned */
  uint32_t reduce_edits;                /* reduceVertices erasures (front-back success included) */
  uint32_t collapse_edits;              /* collapseCloseVertices erasures */
  uint32_t shortcut_edits;              /* shortcutPath edits kept */
  uint32_t bspline_edits;               /* smoothBSpline replacements */
  uint32_t motion_checks, state_checks; /* checkMotion and isValid calls of the restated schedule and check */
  uint32_t rounds;                      /* device rounds (gather, pose check, apply) that checked states */
  uint32_t discarded;                   /* speculative attempts checked in a round after the attempt it applied */
  int32_t  check_passed;                /* the simplified path passed both checks */
  int32_t  returned_simplified;         /* 1: the output is the simplified path, 0: the original */
  double   cost_original, cost_simplified;   /* under `objective`; NaN when the check failed (not compared) */
} artp_simplify_info;
/* path: n HOST states (7 doubles each, finite), start to goal. max_query_edge_length: the learned objective's piece
 * length (MotionCostObjective's, params.h:54), read for ARTP_OBJ_LEARNED only. out: HOST buffer of capacity states; *n_out (nullable) =
 * the returned path's length; above capacity nothing is written and the call returns ARTP_E_LIMIT. info: nullable.
 * n == 0, a non-finite state, a bad space or objective, or a map window: ARTP_E_INVALID; no map: ARTP_E_NOMAP;
 * n > ARTP_SIMPLIFY_MAX_STATES, or one motion of more than 1024 states: ARTP_E_LIMIT (the state pool, 512 n + 64 states,
 * holds the worst case of the schedule); ARTP_OBJ_LEARNED without weights or features: ARTP_E_NOWEIGHTS (before any work). */
int artp_simplify_path(artp_handle* h, const double* path, size_t n, const artp_se3_space* space, int objective,
                       double max_query_edge_length, uint64_t seed, double* out, size_t capacity, size_t* n_out,
                       artp_simplify_info* info);
/* TEST HOOK, not part of the planner interface (like the other artp_debug_* entry points): dist[i] = SE3StateSpace::distance(a[i], b[i]) and interp[i] = interpolate(a[i], b[i], t[i]) (HOST buffers)
 * with the device arithmetic artp_simplify_path uses. Its decisions turn on exact ties (evenly spaced states give equal
 * distances) that CUDA's acos / sin and libm's may break differently, so a restatement compared with it bit for bit
 * takes these two functions from here. */
int artp_debug_se3_ops(artp_handle* h, const double* a, const double* b, const double* t, size_t n, double* dist,
                       double* interp);

/* ---- inpaintMatrix (art_planner/src/utils.cpp:13-63) --------------------------------------------------------------
 * The rows x cols column-major layer: its finite min / max, the NaN mask (+-inf cells are not masked), convertTo(CV_8U,
 * 255/(max-min), -min*255/(max-min)) with the fused multiply-add, cv::inpaint(radius 3, INPAINT_TELEA) on the cols x rows
 * image, back to float (* (max-min)/255, + min) and column / row 0 copied from column / row 1. Bit for bit with
 * oracle/inpaint_oracle.py (DESIGN.md section 4.6, which lists its one known divergence from cv2 4.13). rows, cols >= 2, rows * cols < 2^31; a layer without a
 * finite cell is ARTP_E_INVALID. _device: device buffers, on `stream` (a cudaStream_t cast to void*, may be NULL); one
 * host sync reads the finite count, the rest is asynchronous. */
int artp_inpaint_layer(artp_handle* h, const float* layer, int rows, int cols, float* out);
int artp_inpaint_layer_device(artp_handle* h, const float* d_layer, int rows, int cols, float* d_out, void* stream);

/* ---- the cost server's map preparation (cost_query_server.py, _elvMapProcess) -------------------------------------
 * What the learned cost's trunk is fed by the reference: the server prepares the RAW elevation itself, not
 * processors::Basic's output. All float32, round to nearest, no contraction (DESIGN.md section 4.7):
 *   1. E = layer[::-1, ::-1], rows x cols: E[r][c] = layer(rows-1-r, cols-1-c) (the trunk's input orientation).
 *   2. no cell NaN or +-inf: E itself (not quantised).
 *   3. otherwise mn / mx = min / max of the finite cells, d = mx - mn, q = trunc(((E - mn) * 255) / d) on the finite
 *      cells (the max cell may land at 254; mx == mn gives 0 / 0 -> byte 0, so the map is mn everywhere),
 *      mask = ~isfinite(E), masked cells 0 (both zeros are numpy's NaN -> uint8 on x86-64);
 *   4. cv::inpaint(q, mask, 3, INPAINT_TELEA) in E's orientation (artp_inpaint_layer's march);
 *   5. ((float)u * d) / 255 + mn on every cell, known cells too; no row / column 0 copies.
 * Refused with ARTP_E_INVALID before any work: a +-inf cell and a layer without a finite cell (the server's result is
 * NaN), and a range whose d * 255 overflows float (the server casts infinite quotients to 8 bits, undefined in numpy). rows, cols >= 2 and rows * cols < 2^31.
 * artp_cost_map_layer returns the prepared map P in grid_map layout (E'[r][c] = P(rows-1-r, cols-1-c)), so
 * artp_set_map(P as elevation) + artp_update_features feeds the trunk what the server fed it. _device: device buffers on
 * `stream` (may be NULL); one host sync reads the layer's range and flags, the rest is asynchronous. */
int artp_cost_map_layer(artp_handle* h, const float* raw, int rows, int cols, float* out);
int artp_cost_map_layer_device(artp_handle* h, const float* d_raw, int rows, int cols, float* d_out, void* stream);
/* The preparation above, then CostPredictor.updateFeatures on it: the trunk's features and the head's geometry (res,
 * cx, cy, rows * res x cols * res) as artp_update_features sets them from a map, but no installed map is needed or
 * changed. Without weights: ARTP_E_NOWEIGHTS. A refused call (any code before the trunk runs, the preparation's refusals
 * included) keeps the previous features. _device: d_raw on `stream`; the call returns when the features are made. */
int artp_update_features_raw(artp_handle* h, const float* raw, int rows, int cols, double res, double cx, double cy);
int artp_update_features_raw_device(artp_handle* h, const float* d_raw, int rows, int cols, double res, double cx,
                                    double cy, void* stream);

/* ---- the planner: Planner::setMap and Planner::plan + getSolutionPath for prm_motion_cost (planner.cpp:135-298) ----
 * The shipped replan (PlannerRos::updateMapAndPlanFromCurrentRobotPose, planner.name prm_motion_cost,
 * simplify_solution true) as two calls whose stages hand data to each other in device memory: no layer, state or path
 * goes through host memory between them. The host reads only control words: the finite range of the raw elevation, the
 * compact-code scales of the two uploaded layers, the loops' control blocks (sampleGraph, solve, simplify), the endpoints'
 * bounds verdict with their (x, y) (they size the roadmap's interior-state buffer), the learned cost's piece total and
 * per-edge costs, and at the end the returned path and the info record.
 *
 * artp_planner_set_map   Planner::setMap (:135-163) and Map::setMap's new-map chain (setUpMapProcessors, :39-58):
 *   observed           addKnownCells (basic.cpp:25-38): 1 where elevation and traversability (Map::setMap's basic layers,
 *                      map.cpp:16) are finite -- grid_map's isValid, which is not in the reference tree (unpinned
 *                      restatement). A NULL traversability is checkTraversability's 1.0 layer (basic.cpp:13-21).
 *   SE(3) bounds       x: cx -+ rows * res (the FULL length, not half of it), y: cy -+ cols * res, z:
 *                      (double)minCoeffOfFinites(raw elevation) - reach_z / 2 .. (double)maxCoeffOfFinites(..) + reach_z / 2,
 *                      from the RAW layer, before any processing; -0 is taken as +0. Min and max are order-free: exact.
 *                      A layer with no finite cell: ARTP_E_INVALID (grid_map's result there is not pinned).
 *   Basic              artp_process_basic on the INPAINTED layers (inpaintMatrix's output, which also quantises finite
 *                      cells to 8 bits; artp_planner_set_map_raw makes them on the device), then the map upload of the
 *                      inpainted elevation and elevation_masked straight from device memory (artp_set_map's rules).
 *   the chain          artp_estimate_normals ((torso.length + torso.width) * 0.25); with sample_from_distribution the
 *                      sample filter, the distribution without vertices and its CDF; the sampler armed with the bounds' x / y;
 *                      artp_update_features when weights are loaded; with cost_map_from_raw = 1 the trunk instead runs on
 *                      the cost server's preparation of the uploaded RAW elevation (artp_update_features_raw's features,
 *                      whose refusals are then checked with the others, before the installed map changes).
 *   generation         a map counter, +1 per installed map: it stands in for the grid_map timestamp that
 *                      PRMMotionCostMaintainer::sampleGraph compares (prm_motion_cost.cpp:146-153).
 * Layers are HOST pointers in grid_map layout (artp_set_map). Every check runs before the installed map changes, and a
 * refused map leaves the previous one installed. The checks are the arguments, the structuring elements' and the blur's
 * size limits (ARTP_E_LIMIT, as the chained calls) and the finite cell (found by the bounds' reduction). Only a CUDA error
 * after that leaves no planner map. info (nullable) receives the call's host synchronisations and bytes copied. artp_set_map / artp_set_map_window install a map the planner does not own: artp_plan then
 * answers NO_MAP.
 *
 * artp_plan   Planner::plan (:193-262) + getSolutionPath (:266-298), in the reference's order:
 *   1. no planner map: status NO_MAP (a map window: ARTP_E_INVALID); no weights or features: ARTP_E_NOWEIGHTS.
 *   2. clear_roadmap: PRMMotionCost::clear (the ROS node's ss_->clear(), planner_ros.cpp:359,373); the first plan of a
 *      handle creates the store (vertex_capacity, edge_capacity).
 *   3. sampleGraph + updateEdges (artp_roadmap_sample_graph, artp_roadmap_update_edges) ONLY when the map generation
 *      differs from the one the last sampleGraph saw. So clear_roadmap on an unchanged map plans on a roadmap that holds
 *      only start and goal: the reference's behaviour, reproduced on purpose.
 *   4. the goal: satisfiesBounds, else enforceBounds (:207-221), then the projection when (x, y) lies on the map (:223-237,
 *      artp_pose_from_2d). OMPL 1.4.2 is not in the tree; restated (unpinned): R3 passes when no coordinate has
 *      v - DBL_EPSILON > high or v + DBL_EPSILON < low, and enforceBounds clamps; SO3 passes when |norm - 1| < 1e-9
 *      (MAX_QUATERNION_NORM_ERROR), and enforceBounds acts when |x^2 + y^2 + z^2 + w^2 - 1| > DBL_EPSILON: the identity
 *      when the norm is below DBL_EPSILON, else each component divided by the norm. A failing test applies both
 *      components' enforceBounds. The start is neither clipped nor projected.
 *   5. setStartAndGoal (:167-189): the start search (start_radius) and the goal search (goal_radius), artp_find_valid_near.
 *   6. baseSolve on the device roadmap, as artp_roadmap_solve defines it, from the device endpoints.
 *   7. solved and simplify: artp_simplify_path under ARTP_OBJ_LEARNED at max_query_edge_length, from the device path.
 * Status (planner_status.h, planner.cpp:254-261): ARTP_SOLVE_NOT_CONNECTED and NO_FEASIBLE_PATH become NOT_SOLVED,
 * INVALID_START / INVALID_GOAL pass through. Unsolved: no path (*n_path = 0), as getSolutionPath throws.
 * Streams, all from `seed`: the sampler's "ARTP" stream (key seed) from draw info.first_sample; the start search's "ARTB"
 * stream (key seed) from info.start_draw and the goal search's (key ~seed) from info.goal_draw, each advanced like
 * StartState.sampleGoal's mirror (k draws for candidate k, n_iter when none is valid); the simplifier's key seed + c for the
 * handle's c-th simplify. A new seed restarts every position at 0. info reports the positions used, so the same replan
 * through the chained public calls gives the same result bit for bit.
 * path: HOST buffer of capacity states (nullable); a path above capacity: ARTP_E_LIMIT, nothing written. Bad parameters, a
 * non-finite start / goal or an n_iter of 2^32 - 1 (ARTP_E_INVALID), and the distribution's limits for sampleGraph's
 * recomputes (artp_update_sample_distribution's codes) are checked before any work. */
#define ARTP_PLANNER_UNKNOWN        0   /* art_planner::PlannerStatus (planner_status.h) */
#define ARTP_PLANNER_INVALID_START  1
#define ARTP_PLANNER_INVALID_GOAL   2
#define ARTP_PLANNER_NO_MAP         3
#define ARTP_PLANNER_NOT_SOLVED     4
#define ARTP_PLANNER_SOLVED         5
typedef struct artp_planner_params {
  double   start_radius, goal_radius;                 /* start_goal_search, params.h:38-40 */
  uint32_t n_iter;
  size_t   max_n_vertices, max_n_edges, recompute_density_after_n_samples;   /* prm_motion_cost, params.h:51-53 */
  double   max_query_edge_length;                     /* params.h:54; > 0 when simplify */
  uint64_t max_draws;                                 /* sampler draws per sampleGraph: replaces max_sample_time */
  size_t   vertex_capacity, edge_capacity;            /* the roadmap store (artp_roadmap_clear) */
  double   max_roll_pert, max_pitch_pert;             /* sampler, params.h:79-84 */
  int      sample_from_distribution, use_inverse_vertex_density, use_max_prob_unknown_samples;
  double   max_prob_unknown_samples;
  artp_basic_params basic;                            /* params.h:23-35 */
  int      simplify, clear_roadmap;                   /* simplify_solution; the ROS node's ss_->clear() */
  uint64_t seed;
  int      cost_map_from_raw;                         /* 0: features from the uploaded elevation; 1: from the raw one as
                                                         the cost server prepares it (artp_update_features_raw) */
} artp_planner_params;
typedef struct artp_plan_info {
  int32_t  status;                      /* ARTP_PLANNER_* */
  int32_t  sampled;                     /* sampleGraph and updateEdges ran (the map generation changed) */
  uint64_t first_sample, draws_used;    /* sampler draws used: first_sample .. first_sample + draws_used - 1 */
  uint64_t start_draw, goal_draw;       /* the first draws of the two searches */
  uint64_t simplify_seed;               /* artp_simplify_path's seed (when it ran) */
  uint64_t n_vertices, n_edges;         /* the roadmap after the plan */
  artp_roadmap_solve_info solve;        /* path_vertices: in, nullable */
  double   path_cost;                   /* artp_roadmap_solve's *cost of the solved path */
  artp_simplify_info simplify;          /* zero unless the simplifier ran */
  int32_t  goal_clipped, goal_inside;   /* enforceBounds applied; the projection applied */
  int32_t  start_index, goal_index;     /* the searches' candidate indices (-1: none valid) */
  double   goal_clipped_state[7], goal_projected[7], start_repaired[7], goal_repaired[7];
  float    ms_sample_graph, ms_update_edges, ms_endpoints, ms_solve, ms_simplify;   /* events on the call's stream */
  uint32_t host_syncs;                  /* host synchronisations of the call */
  uint64_t bytes_h2d, bytes_d2h;        /* bytes the call copied host -> device and device -> host */
} artp_plan_info;
typedef struct artp_planner_map_info {
  uint32_t host_syncs;                  /* host synchronisations of the call */
  uint64_t bytes_h2d, bytes_d2h;        /* bytes the call copied host -> device and device -> host */
} artp_planner_map_info;
int artp_planner_set_map(artp_handle* h, const artp_planner_params* pp, const float* elevation, const float* traversability,
                         const float* elevation_inpainted, const float* traversability_inpainted, int rows, int cols,
                         double res, double cx, double cy, artp_planner_map_info* info);
/* artp_planner_set_map with processors::Basic's two inpaintMatrix calls done on the device from the raw layers: only
 * elevation and traversability (NULL: checkTraversability's 1.0 layer, not inpainted) go up. It leaves the handle in the
 * state artp_planner_set_map leaves it in when given artp_inpaint_layer's outputs. A traversability layer without a
 * finite cell is ARTP_E_INVALID, checked before the installed map changes. */
int artp_planner_set_map_raw(artp_handle* h, const artp_planner_params* pp, const float* elevation,
                             const float* traversability, int rows, int cols, double res, double cx, double cy,
                             artp_planner_map_info* info);
/* The artp_se3_space artp_planner_set_map installed (ARTP_E_NOMAP before). */
int artp_planner_get_space(artp_handle* h, artp_se3_space* out);
int artp_plan(artp_handle* h, const artp_planner_params* pp, const double* start, const double* goal, double* path,
              size_t capacity, size_t* n_path, artp_plan_info* info);

/* ---- learned motion cost (MotionCostFunc, objectives/motion_cost_objective.h:22-23) ------------------------------
 * Weights: ONE flat fp32 blob in the layer order of the reference's `network` module: init_conv1..5, init_flatten,
 * tar0_conv1, out0_conv1, out1_conv1..3 -- each conv.weight [Cout][Cin][kh][kw] followed by its BatchNorm weight, bias,
 * running_mean, running_var -- then out2_conv1..3 as conv.weight followed by conv.bias. Two architectures share this
 * layout and differ only in their widths; the blob's length picks the one that runs:
 *   ARTP_COST_NET_LIGHT  network_light.py:9-63 (init 24/48 channels, out0 64->48, out1 48->24/24/36):
 *                        584 543 floats (583 767 parameters + BN buffers) = artp_cost_weights_size()
 *   ARTP_COST_NET_FULL   network.py:9-63 (init 32/64 channels, out0 80->64, out1 64->32/32/32):
 *                        1 036 771 floats (1 035 779 parameters + BN buffers)
 * artp_set_cost_weights takes either length (any other is ARTP_E_INVALID); a blob of the other architecture replaces
 * the loaded one, and artp_update_features must run again before the next cost query. */
#define ARTP_COST_NET_LIGHT 0
#define ARTP_COST_NET_FULL  1
size_t artp_cost_weights_size(void);
/* Blob length of `network` (ARTP_COST_NET_*), 0 for any other value. */
size_t artp_cost_weights_size_for(int network);
int artp_set_cost_weights(artp_handle* h, const float* blob, size_t n_floats);
/* The architecture of the loaded weights (ARTP_COST_NET_*); ARTP_E_NOWEIGHTS before any artp_set_cost_weights. */
int artp_get_cost_network(artp_handle* h, int* network);
/* CostPredictor.updateFeatures (predictor.py:28-36): run the CNN trunk over the `elevation` layer of the current map
 * (orientation as cost_query_server.py:74). Call after artp_set_map whenever the map changed.
 * The tensor-core path (the default artp_set_cnn_mode) stores the activations of init_conv1..5 as fp16 hi + lo pairs.
 * If one of them exceeds the fp16 range (|a| > 65504, e.g. raw elevations thousands of metres from the frame's origin
 * with weights calibrated near zero height), the call returns ARTP_E_LIMIT, artp_last_error() names the layer, and
 * the handle holds no features (cost queries return ARTP_E_NOWEIGHTS until an update succeeds). The CUDA-core path
 * (artp_set_cnn_mode bit 0) has fp32 range and never raises it. DESIGN.md section 4.3 gives the supported ranges. */
int artp_update_features(artp_handle* h);
/* GPUCostQueryServer.handle_cost_query_no_update (cost_query_server.py:120-141) = CostQuery.__call__: edges n x 6 floats
 * [target_x, target_y, target_yaw, start_x, start_y, start_yaw] in the map frame -> cost3 n x 3 floats
 * (energy, time, risk = 1 - p_success). HOST buffers. */
int artp_motion_cost(artp_handle* h, const float* edges, size_t n, float* cost3);
int artp_motion_cost_device(artp_handle* h, const float* d_edges, size_t n, float* d_cost3, void* stream);
/* PRMMotionCostMaintainer::updateEdges / computeCostForVertexEdges (prm_motion_cost.cpp:27-128) for n graph edges
 * (source vertex state s_start = v1, target vertex state s_target = v2): the [n x 6] float edge matrix
 * [tx, ty, tyaw, sx, sy, syaw] with getYawFromSO3 (utils.h:80-88) ... */
int artp_edge_matrix_from_states(const double* s_start, const double* s_target, size_t n, float* edges);
/* ... and the whole batch in one call: edge matrix -> cost query -> isFeasible / getCost per row. cost[i] = +inf for
 * infeasible (too risky) edges exactly like updateEdges (:56-59); cost3 (nullable): the raw (energy, time, risk) rows. */
int artp_motion_cost_states(artp_handle* h, const double* s_start, const double* s_target, size_t n, double* cost,
                            uint8_t* feasible, float* cost3);
/* MotionCostObjective::getCost / isFeasible (motion_cost_objective.h:54-66) on host arrays:
 * cost[i] = w_e*E + w_t*T + w_r*R, feasible[i] = R <= risk_threshold (weights / threshold from artp_params). */
int artp_combine_cost(artp_handle* h, const float* cost3, size_t n, double* cost, uint8_t* feasible);
/* MotionCostObjective::motionCost (motion_cost_objective.cpp:36-95) for n edges: split, query, sum. HOST buffers.
 * Edge e is split into n_interp + 1 pieces, n_interp = (unsigned)(lateralDistance(s1, s2) / max_query_edge_length)
 * (params.h:54: 0.5), at the knots s1, interpolate(s1, s2, j * (1.0 / (n_interp + 1))) for j = 1..n_interp, s2; each piece
 * is one edge-matrix row through the network. cost[e] = +inf when a piece's risk is above risk_threshold, else the
 * left-to-right double sum of getCost over the pieces. Needs artp_set_cost_weights + artp_update_features (else
 * ARTP_E_NOWEIGHTS); max_query_edge_length > 0; total pieces < 2^32 (else ARTP_E_INVALID). */
int artp_motion_cost_split(artp_handle* h, const double* s1, const double* s2, size_t n,
                           double max_query_edge_length, double* cost);
/* DEVICE buffers on `stream`: d_piece_off = n + 1 exclusive prefix sums of the per-edge piece counts (n_interp + 1),
 * total_pieces = d_piece_off[n]; d_rows (total_pieces x 6 floats) and d_cost3 (total_pieces x 3) are caller scratch
 * that receive the piece rows and their (energy, time, risk). */
int artp_motion_cost_split_device(artp_handle* h, const double* d_s1, const double* d_s2, size_t n,
                                  const uint32_t* d_piece_off, size_t total_pieces, float* d_rows, float* d_cost3,
                                  double* d_cost, void* stream);
/* Test hooks: feature map copy-out ([Hf][Wf][C] fp32, channels last, C = 48 light / 64 full: n_floats = Hf*Wf*C),
 * kernel selection (bit 0: CUDA-core fp32
 * reference for every layer instead of the tensor-core (wgmma) kernels; any other bit is ARTP_E_INVALID), trunk timings
 * ms3 = (3x3 stack, 15x15 layer, whole trunk) of the last artp_update_features. */
int artp_get_features(artp_handle* h, float* out, size_t n_floats, int* hf, int* wf);
int artp_set_cnn_mode(artp_handle* h, int mode);
int artp_get_cnn_timing(artp_handle* h, float* ms3);

/* Version string of the library / kernel image ("artp <ver> sm_90a"). */
const char* artp_version(void);

#ifdef __cplusplus
}
#endif
#endif
