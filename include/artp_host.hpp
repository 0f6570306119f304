// include/artp_host.hpp -- C++ host side of the CUDA-native art_planner hot path, above the C ABI (artp.h).
//
// Header-only mirror of the reference's plugin classes for this path -- same class and method names, argument meaning
// and error behaviour -- so that art_planner's planners and facade keep calling what they call today:
//   art_planner::StateValidityChecker   include/art_planner/validity_checker/validity_checker.h:21-39
//   ompl::base::MotionValidator         (OMPL DiscreteMotionValidator; call sites prm_motion_cost.cpp:652,
//                                        lazy_prm_star_min_update.cpp:725)
//   art_planner::PathLengthObjective    include/art_planner/objectives/path_length_objective.h, .cpp:26-70
//   art_planner::MotionCostObjective    include/art_planner/objectives/motion_cost_objective.h:19-78, .cpp:28-95
// OMPL / Eigen / grid_map are not available in this build image, so the classes are written against three tiny
// stand-ins (State = the seven doubles utils.h:25-38 reads from an SE3StateSpace::StateType, Map = two column-major
// float layers + geometry as grid_map stores them, EdgeMatrix = row-major float matrix). With -DARTP_WITH_OMPL the
// OMPL adapters at the bottom derive from the real ompl::base classes and forward to the same objects.
// There is no CPU fallback: construction throws std::runtime_error if the CUDA library cannot create a handle.
#pragma once

#include <cmath>
#include <cstdint>
#include <functional>
#include <limits>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "artp.h"

namespace artp_host {

// art_planner::Params, the fields this path reads, with the reference's nesting (params.h:14-123).
struct Params {
  struct {
    bool unknown_space_untraversable{true};
    struct {
      float max_query_edge_length{0.5f};
      float risk_threshold{0.1f};
      struct { float energy{0.0f}; float time{1.0f}; float risk{5.0f}; } cost_weights;
      unsigned int max_n_vertices{10000u};                    // params.h:51
      unsigned int max_n_edges{50000u};                       // params.h:52
      unsigned int recompute_density_after_n_samples{1000u};  // params.h:53
    } prm_motion_cost;
  } planner;
  struct {
    struct { bool use_directional_cost{false}; double max_lon_vel{0.5}; double max_lat_vel{0.1}; double max_ang_vel{0.5}; } custom_path_length;
  } objectives;
  struct {
    struct { double length{1.05}; double width{0.55}; double height{0.2}; struct { double x{0}, y{0}, z{0}; } offset; } torso;
    struct { struct { double x{0.362}, y{0.225}, z{-0.525}; } offset; struct { double x{0.25}, y{0.1}, z{0.15}; } reach; } feet;
  } robot;
  struct {
    double max_pitch_pert{10.0 / 180 * 3.14159265358979323846};   // params.h:79
    double max_roll_pert{3.33 / 180 * 3.14159265358979323846};    // params.h:80
    bool sample_from_distribution{true};                            // params.h:81
    bool use_inverse_vertex_density{false};                         // params.h:82
    bool use_max_prob_unknown_samples{false};                       // params.h:83
    double max_prob_unknown_samples{0.1};                           // params.h:84
  } sampler;
  int device{0};   // not in the reference: CUDA device ordinal
};
using ParamsConstPtr = std::shared_ptr<const Params>;

// The SE3StateSpace::StateType fields the reference reads (utils.h:25-38): position + quaternion, doubles.
struct State { double x{0}, y{0}, z{0}, qx{0}, qy{0}, qz{0}, qw{1}; };

// Stand-in for art_planner::Map / grid_map::GridMap: layers are column-major rows x cols (index (i,j) at i + j*rows).
struct Map {
  int rows{0}, cols{0};
  double resolution{0}, position_x{0}, position_y{0};
  std::vector<float> elevation, elevation_masked;
  // layers the sampler reads (Map::getNormal / getPlaneFitStdDev map.h:94-116, probability_distribution.cpp:20-46);
  // cum_prob_rowwise = column 0 of "cum_prob_rowwise_hack". Empty when no sampler is used.
  std::vector<float> normal_x, normal_y, normal_z, plane_fit_std_dev, cum_prob, cum_prob_rowwise;
  // the sampler's distribution (planner.cpp:39-58): inputs from processors::Basic, outputs of the device chain
  std::vector<float> traversability_thresholded, observed, traversability_sample_filter, sample_probability;
};

inline artp_params toArtp(const Params& p) {
  artp_params a{};
  a.torso_length = p.robot.torso.length; a.torso_width = p.robot.torso.width; a.torso_height = p.robot.torso.height;
  a.torso_off_x = p.robot.torso.offset.x; a.torso_off_y = p.robot.torso.offset.y; a.torso_off_z = p.robot.torso.offset.z;
  a.feet_off_x = p.robot.feet.offset.x; a.feet_off_y = p.robot.feet.offset.y; a.feet_off_z = p.robot.feet.offset.z;
  a.reach_x = p.robot.feet.reach.x; a.reach_y = p.robot.feet.reach.y; a.reach_z = p.robot.feet.reach.z;
  a.unknown_space_untraversable = p.planner.unknown_space_untraversable ? 1 : 0;
  a.use_directional_cost = p.objectives.custom_path_length.use_directional_cost ? 1 : 0;
  a.max_lon_vel = p.objectives.custom_path_length.max_lon_vel;
  a.max_lat_vel = p.objectives.custom_path_length.max_lat_vel;
  a.max_ang_vel = p.objectives.custom_path_length.max_ang_vel;
  a.cost_w_energy = p.planner.prm_motion_cost.cost_weights.energy;
  a.cost_w_time = p.planner.prm_motion_cost.cost_weights.time;
  a.cost_w_risk = p.planner.prm_motion_cost.cost_weights.risk;
  a.risk_threshold = p.planner.prm_motion_cost.risk_threshold;
  a.device = p.device;
  return a;
}

// The distribution parameters of the reference's Planner, with its density blur radius (planner.cpp:48).
inline artp_sample_distribution_params distributionParams(const Params& p) {
  artp_sample_distribution_params dp{};
  dp.use_inverse_vertex_density = p.sampler.use_inverse_vertex_density ? 1 : 0;
  dp.density_blur_radius = (p.robot.torso.length + p.robot.torso.width) * 0.25;
  dp.use_max_prob_unknown_samples = p.sampler.use_max_prob_unknown_samples ? 1 : 0;
  dp.max_prob_unknown_samples = p.sampler.max_prob_unknown_samples;
  return dp;
}

// Owns the artp_handle; shared by the plugin objects below (the reference shares its checker the same way,
// path_length_objective.cpp:20: checker_(si->getStateValidityChecker())).
class Handle {
 public:
  explicit Handle(const ParamsConstPtr& params) : params_(params) {
    const artp_params a = toArtp(*params);
    if (artp_create(&a, &h_) != ARTP_OK) throw std::runtime_error(std::string("artp_create: ") + artp_last_error(nullptr));
  }
  ~Handle() { artp_destroy(h_); }
  Handle(const Handle&) = delete;
  Handle& operator=(const Handle&) = delete;
  artp_handle* get() const { return h_; }
  const Params& params() const { return *params_; }
  void check(int rc, const char* what) const {
    if (rc != ARTP_OK) throw std::runtime_error(std::string(what) + ": " + artp_last_error(h_));
  }
 private:
  ParamsConstPtr params_;
  artp_handle* h_{nullptr};
};
using HandlePtr = std::shared_ptr<Handle>;

// art_planner::StateValidityChecker (validity_checker.cpp:9-45).
class StateValidityChecker {
 public:
  explicit StateValidityChecker(const ParamsConstPtr& params) : handle_(std::make_shared<Handle>(params)) {}
  explicit StateValidityChecker(const HandlePtr& handle) : handle_(handle) {}

  void setMap(const std::shared_ptr<Map>& map) { map_ = map; }                 // validity_checker.cpp:20-23

  void updateHeightField() {                                                    // validity_checker.cpp:27-31
    if (!map_) throw std::runtime_error("updateHeightField: no map");
    handle_->check(artp_set_map(handle_->get(), map_->elevation.data(), map_->elevation_masked.data(), map_->rows, map_->cols,
                                map_->resolution, map_->position_x, map_->position_y), "artp_set_map");
  }

  bool hasMap() const { return artp_has_map(handle_->get()) != 0; }             // validity_checker.cpp:33-35

  // art_planner::estimateNormals (utils.cpp:213-324) as processors::Basic calls it (basic.cpp:47), on the device; fills
  // the map's normal_x/y/z and plane_fit_std_dev layers and keeps them resident for SE3FromSE2Sampler.
  void estimateNormals() {
    if (!map_) throw std::runtime_error("estimateNormals: no map");
    const Params& p = handle_->params();
    const size_t ncell = static_cast<size_t>(map_->rows) * map_->cols;
    map_->normal_x.resize(ncell); map_->normal_y.resize(ncell); map_->normal_z.resize(ncell);
    map_->plane_fit_std_dev.resize(ncell);
    handle_->check(artp_estimate_normals(handle_->get(), (p.robot.torso.length + p.robot.torso.width) * 0.25,
                                         map_->normal_x.data(), map_->normal_y.data(), map_->normal_z.data(),
                                         map_->plane_fit_std_dev.data()), "artp_estimate_normals");
  }

  bool isValid(const State* state) const {                                      // validity_checker.cpp:39-45
    uint8_t v = 0;
    handle_->check(artp_check_poses(handle_->get(), &state->x, 1, &v), "artp_check_poses");
    return v != 0;
  }

  // Batch form for the rejection-sampling loops (prm_motion_cost.cpp:171-194, lazy_prm_star_min_update.cpp:549-556).
  // Pose3FromSE3 casts every field to float first (utils.h:25-38); doing that cast here halves the PCIe traffic and
  // gives identical flags.
  void isValidBatch(const std::vector<State>& states, std::vector<uint8_t>* valid) const {
    std::vector<float> buf(7 * states.size());
    for (size_t i = 0; i < states.size(); ++i) {
      const double* s = &states[i].x;
      for (int k = 0; k < 7; ++k) buf[7 * i + k] = static_cast<float>(s[k]);
    }
    valid->resize(states.size());
    handle_->check(artp_check_poses_f32(handle_->get(), buf.data(), states.size(), valid->data()), "artp_check_poses_f32");
  }

  // Why each state passes or fails isValid (artp_box_verdicts): one word per state, bit k set when box k fails (0 torso,
  // 1..4 the reach boxes), bit 8 + k when box k's centre is off the map (ARTP_BOX_*). (word & ARTP_BOX_FAIL_MASK) == 0
  // exactly where isValid is true. The lowest fail bit is the box where isValid stops.
  std::vector<uint16_t> boxVerdicts(const std::vector<State>& states) const {
    std::vector<uint16_t> why(states.size());
    if (states.empty()) return why;
    handle_->check(artp_box_verdicts(handle_->get(), &states[0].x, states.size(), why.data()), "artp_box_verdicts");
    return why;
  }

  // computeCumulativeProbabilityDistribution (probability_distribution.cpp:20-46) on the device: fills the map's cum_prob /
  // cum_prob_rowwise layers from `sample_probability` (rows x cols, column-major) and keeps them resident for the sampler.
  void computeSampleCdf(const std::vector<float>& sample_probability) {
    if (!map_) throw std::runtime_error("computeSampleCdf: no map");
    const size_t ncell = static_cast<size_t>(map_->rows) * map_->cols;
    if (sample_probability.size() != ncell) throw std::invalid_argument("computeSampleCdf: layer size mismatch");
    map_->cum_prob.resize(ncell);
    map_->cum_prob_rowwise.resize(map_->rows);
    handle_->check(artp_compute_sample_cdf(handle_->get(), sample_probability.data(), map_->cum_prob.data(),
                                           map_->cum_prob_rowwise.data()), "artp_compute_sample_cdf");
  }

  // Basic::setTraversabilityFilter (basic.cpp:110-125) on the device: fills the map's traversability_sample_filter from its
  // traversability_thresholded layer and keeps it, with the map's observed layer (empty: none), for updateSampleDistribution.
  void setSampleFilter() {
    if (!map_) throw std::runtime_error("setSampleFilter: no map");
    const size_t ncell = static_cast<size_t>(map_->rows) * map_->cols;
    if (map_->traversability_thresholded.size() != ncell || (!map_->observed.empty() && map_->observed.size() != ncell))
      throw std::invalid_argument("setSampleFilter: layer size mismatch");
    map_->traversability_sample_filter.resize(ncell);
    handle_->check(artp_set_sample_filter(handle_->get(), map_->traversability_thresholded.data(),
                                          map_->observed.empty() ? nullptr : map_->observed.data(),
                                          map_->traversability_sample_filter.data()), "artp_set_sample_filter");
  }

  // computeInverseSampleDensity -> applyBaseSampleDistribution -> applyMaxUnknownProbability ->
  // computeCumulativeProbabilityDistribution (planner.cpp:39-58) on the device for the roadmap's vertices, with the
  // sampler parameters and blur radius the reference's Planner uses; fills sample_probability / cum_prob /
  // cum_prob_rowwise and keeps the CDF resident (re-arm SE3FromSE2Sampler: updateDistribution does both).
  void updateSampleDistribution(const std::vector<State>& vertices) {
    if (!map_) throw std::runtime_error("updateSampleDistribution: no map");
    const artp_sample_distribution_params dp = distributionParams(handle_->params());
    const size_t ncell = static_cast<size_t>(map_->rows) * map_->cols;
    map_->sample_probability.resize(ncell);
    map_->cum_prob.resize(ncell);
    map_->cum_prob_rowwise.resize(map_->rows);
    handle_->check(artp_update_sample_distribution(handle_->get(), &dp, vertices.empty() ? nullptr : &vertices[0].x,
                                                   vertices.size(), map_->sample_probability.data(), map_->cum_prob.data(),
                                                   map_->cum_prob_rowwise.data()), "artp_update_sample_distribution");
  }

  // The rejection-sampling loop `do { sampleUniform(s) } while (!isValid(s))` (prm_motion_cost.cpp:171-194,
  // lazy_prm_star_min_update.cpp:549-556) in batches: draw `batch` candidates with the caller's sampler, check them in
  // one call, keep the valid ones in draw order; repeat until n_wanted states are collected or max_draws candidates
  // were drawn (the reference bounds the same loop by time). Returns the number of candidates drawn.
  template <class Sampler>   // void sampler(State* out)
  size_t sampleValidBatch(Sampler&& sampler, size_t n_wanted, size_t batch, size_t max_draws, std::vector<State>* out) const {
    out->clear();
    size_t drawn = 0;
    std::vector<State> cand;
    std::vector<uint8_t> valid;
    while (out->size() < n_wanted && drawn < max_draws) {
      const size_t m = std::min(batch, max_draws - drawn);
      cand.resize(m);
      for (size_t i = 0; i < m; ++i) sampler(&cand[i]);
      drawn += m;
      isValidBatch(cand, &valid);
      for (size_t i = 0; i < m && out->size() < n_wanted; ++i)
        if (valid[i]) out->push_back(cand[i]);
    }
    return drawn;
  }

  // StartState / GoalStateRegion::sampleGoal (start.cpp:7-41, goal.cpp:11-41) for a batch of queries in one device call
  // (artp_find_valid_near): per query the first valid of the centre and the centre moved in x / y by offsets 1..n_iter,
  // else the last candidate with index -1. offsets: n x n_iter x 2 doubles, or nullptr for the "ARTB" Philox stream.
  void findValidNearBatch(const std::vector<State>& centres, const std::vector<double>& radius, uint32_t n_iter,
                          const double* offsets, uint64_t seed, uint64_t first_draw, std::vector<State>* states,
                          std::vector<int32_t>* index) const {
    if (radius.size() != centres.size()) throw std::invalid_argument("findValidNearBatch: size mismatch");
    states->resize(centres.size());
    index->resize(centres.size());
    if (centres.empty()) return;
    handle_->check(artp_find_valid_near(handle_->get(), &centres[0].x, centres.size(), radius.data(), n_iter, offsets, seed,
                                        first_draw, &(*states)[0].x, index->data()), "artp_find_valid_near");
  }

  // The goal projection of Planner::plan (planner.cpp:223-237): states on the map get z and roll / pitch from the map
  // (Map::get3DPoseFrom2D, map.cpp:77-90), the others are copied with inside = 0. Needs the map's normals (estimateNormals).
  void poseFrom2D(const std::vector<State>& in, std::vector<State>* out, std::vector<uint8_t>* inside) const {
    out->resize(in.size());
    inside->resize(in.size());
    if (in.empty()) return;
    handle_->check(artp_pose_from_2d(handle_->get(), &in[0].x, in.size(), &(*out)[0].x, inside->data()), "artp_pose_from_2d");
  }

  // The valid-heading layer (artp_valid_heading_layer): per cell of the map (rows x cols, column-major), bit k is set iff a
  // goal at the cell's centre with yaw yaws[k] passes isValid once projected onto the map (1 to 32 yaws). Needs the map's
  // normals (estimateNormals).
  std::vector<uint32_t> validHeadingLayer(const std::vector<double>& yaws) const {
    if (!map_) throw std::runtime_error("validHeadingLayer: no map");
    std::vector<uint32_t> mask(static_cast<size_t>(map_->rows) * map_->cols);
    handle_->check(artp_valid_heading_layer(handle_->get(), yaws.data(), static_cast<int>(yaws.size()), mask.data()),
                   "artp_valid_heading_layer");
    return mask;
  }

  // The box-verdict layer (artp_box_verdict_layer): per cell of the map (rows x cols, column-major), the boxVerdicts word
  // of a goal at the cell's centre with yaw `yaw` once projected onto the map. Needs the map's normals (estimateNormals).
  std::vector<uint16_t> boxVerdictLayer(double yaw) const {
    if (!map_) throw std::runtime_error("boxVerdictLayer: no map");
    std::vector<uint16_t> words(static_cast<size_t>(map_->rows) * map_->cols);
    handle_->check(artp_box_verdict_layer(handle_->get(), yaw, words.data()), "artp_box_verdict_layer");
    return words;
  }

  const HandlePtr& handle() const { return handle_; }

 private:
  HandlePtr handle_;
  std::shared_ptr<Map> map_;
};
using StateValidityCheckerPtr = std::shared_ptr<StateValidityChecker>;

// art_planner::StartState (start.h, start.cpp:7-41): the start repaired by a disc search around it, in one device call.
// Offsets come from the "ARTB" Philox stream of `seed` (artp.h); the draw position advances by what the reference's loop
// consumes from its RNG: k draws when candidate k is returned, n_iter when none is valid, none for a valid centre.
// sampleGoal writes the repaired state (the last candidate when none is valid, like the reference) and returns its
// candidate index, -1 when none is valid.
class StartState {
 public:
  StartState(const StateValidityCheckerPtr& checker, uint64_t seed) : checker_(checker), seed_(seed) {}
  void setState(const State& state) { state_ = state; }
  void setThreshold(double threshold) { threshold_ = threshold; }
  void setMaxNumSamples(const unsigned int& num_samples) { max_num_samples_ = num_samples; }
  int sampleGoal(State* state) const {
    std::vector<State> out;
    std::vector<int32_t> index;
    checker_->findValidNearBatch({state_}, {threshold_}, max_num_samples_, nullptr, seed_, next_, &out, &index);
    *state = out[0];
    next_ += index[0] >= 0 ? static_cast<uint64_t>(index[0]) : max_num_samples_;
    return index[0];
  }
  uint64_t nextDraw() const { return next_; }
 private:
  StateValidityCheckerPtr checker_;
  uint64_t seed_;
  mutable uint64_t next_{0};
  State state_;
  double threshold_{0.0};
  unsigned int max_num_samples_{0};
};

// art_planner::GoalStateRegion (goal.h, goal.cpp:11-41): the same search; OMPL calls it from inside solve().
class GoalStateRegion : public StartState {
 public:
  using StartState::StartState;
};

// art_planner::SE3FromSE2Sampler (sampler.cpp:13-131): sampleUniform on the device, one candidate per Philox counter,
// and the rejection loop around it (prm_motion_cost.cpp:171-194) as one fused sample -> isValid -> compact call.
class SE3FromSE2Sampler {
 public:
  // bounds: SE3 position bounds x,y (planner.cpp:148-160); only read when !sample_from_distribution.
  SE3FromSE2Sampler(const StateValidityCheckerPtr& checker, const std::shared_ptr<Map>& map, uint64_t seed,
                    const double low[2], const double high[2])
      : checker_(checker), map_(map), seed_(seed) {
    const auto& h = checker_->handle();
    const Params& p = h->params();
    sp_.max_roll_pert = p.sampler.max_roll_pert; sp_.max_pitch_pert = p.sampler.max_pitch_pert;
    sp_.sample_from_distribution = p.sampler.sample_from_distribution ? 1 : 0;
    sp_.low[0] = low[0]; sp_.low[1] = low[1]; sp_.high[0] = high[0]; sp_.high[1] = high[1];
    h->check(artp_set_sampler(h->get(), &sp_, map->normal_x.data(), map->normal_y.data(), map->normal_z.data(),
                              map->plane_fit_std_dev.data(), map->cum_prob.empty() ? nullptr : map->cum_prob.data(),
                              map->cum_prob_rowwise.empty() ? nullptr : map->cum_prob_rowwise.data()), "artp_set_sampler");
  }
  // The reApplyPreprocessing step of PRMMotionCostMaintainer::sampleGraph (prm_motion_cost.cpp:190-193): the distribution
  // from the roadmap's vertices (StateValidityChecker::updateSampleDistribution), then the sampler re-armed on the
  // device-resident CDF.
  void updateDistribution(const std::vector<State>& vertices) {
    checker_->updateSampleDistribution(vertices);
    const auto& h = checker_->handle();
    h->check(artp_set_sampler(h->get(), &sp_, map_->normal_x.data(), map_->normal_y.data(), map_->normal_z.data(),
                              map_->plane_fit_std_dev.data(), nullptr, nullptr), "artp_set_sampler");
  }
  void sampleUniform(State* state) {                                             // sampler.cpp:82-131
    const auto& h = checker_->handle();
    do {   // uniform mode: a draw outside the map is a NaN candidate; samplePositionInMap (sampler.cpp:46-50) draws again
      h->check(artp_sample_states(h->get(), nullptr, seed_, next_, 1, &state->x, nullptr), "artp_sample_states");
      ++next_;
    } while (state->x != state->x);
  }
  // n states, none NaN: rejected (outside-map, uniform mode only) candidates are redrawn from the following counters of
  // the stream, like the reference's draw-again loop; the output keeps draw order.
  void sampleUniformBatch(size_t n, std::vector<State>* states) {
    states->clear();
    states->reserve(n);
    const auto& h = checker_->handle();
    std::vector<State> buf;
    while (states->size() < n) {
      const size_t m = n - states->size();
      buf.resize(m);
      h->check(artp_sample_states(h->get(), nullptr, seed_, next_, m, &buf[0].x, nullptr), "artp_sample_states");
      next_ += m;
      for (const State& s : buf) if (s.x == s.x) states->push_back(s);
    }
  }
  // Draws n_draw candidates, returns the valid ones in draw order (what n_draw iterations of
  // `do sampleUniform(s) while (!isValid(s))` would have accepted).
  void sampleValidBatch(size_t n_draw, std::vector<State>* valid) {
    valid->resize(n_draw);
    size_t n_valid = 0;
    const auto& h = checker_->handle();
    if (n_draw)
      h->check(artp_sample_valid(h->get(), seed_, next_, n_draw, &(*valid)[0].x, n_draw, &n_valid), "artp_sample_valid");
    next_ += n_draw;
    valid->resize(n_valid);
  }
  uint64_t nextIndex() const { return next_; }
  uint64_t seed() const { return seed_; }
  void skip(uint64_t n) { next_ += n; }   // draws another caller consumed from this stream (PRMRoadmap::sampleGraph)
 private:
  StateValidityCheckerPtr checker_;
  std::shared_ptr<Map> map_;
  artp_sampler_params sp_{};
  uint64_t seed_;
  uint64_t next_{0};
};

// PRMMotionCost's roadmap built on the device (prm_motion_cost.cpp:145-219, 236-247, 325-390; include/artp.h): the store
// keeps g_'s insertion order, so vertex i of vertices() is the i-th vertex the reference's addValidMilestone adds.
// updateEdges / solve / edgeCosts price, search and validate in place. With -DARTP_WITH_OMPL, PRMMotionCost::solve maps onto
// them as: sampleGraph (which ends in updateEdges, :209) -> sampleGraph(); updateEdges(), and baseSolve after
// Planner::plan's clearQuery -> solve(start, goal, space); the PathGeometric is built from the returned states.
class PRMRoadmap {
 public:
  explicit PRMRoadmap(const StateValidityCheckerPtr& checker, size_t vertex_capacity = 60000, size_t edge_capacity = 60000)
      : checker_(checker), vertex_capacity_(vertex_capacity), edge_capacity_(edge_capacity) { clear(); }
  void clear() {                                                                  // PRMMotionCost::clear (:236-247)
    const auto& h = checker_->handle();
    h->check(artp_roadmap_clear(h->get(), vertex_capacity_, edge_capacity_), "artp_roadmap_clear");
  }
  // addValidMilestone for each state in order: baseSolve's start / goal milestones (:451-479).
  void addValidMilestones(const std::vector<State>& states) {
    const auto& h = checker_->handle();
    h->check(artp_roadmap_add_milestones(h->get(), states.empty() ? nullptr : &states[0].x, states.size()),
             "artp_roadmap_add_milestones");
  }
  // PRMMotionCostMaintainer::sampleGraph's loop (:171-194) on `sampler`'s stream, continuing at its next draw; the caps
  // and the recompute interval from Params, the distribution re-applied as SE3FromSE2Sampler::updateDistribution does.
  // max_draws replaces max_sample_time. Returns the draws used (the sampler's stream moves past them).
  uint64_t sampleGraph(SE3FromSE2Sampler& sampler, uint64_t max_draws = 1ull << 26, bool distribution = true) {
    const auto& h = checker_->handle();
    const Params& p = h->params();
    const artp_roadmap_params rp{p.planner.prm_motion_cost.max_n_vertices, p.planner.prm_motion_cost.max_n_edges,
                                 p.planner.prm_motion_cost.recompute_density_after_n_samples, max_draws};
    const artp_sample_distribution_params dp = distributionParams(p);
    uint64_t used = 0;
    h->check(artp_roadmap_sample_graph(h->get(), &rp, distribution ? &dp : nullptr, sampler.seed(), sampler.nextIndex(), &used),
             "artp_roadmap_sample_graph");
    sampler.skip(used);
    return used;
  }
  // The vertices first .. V-1 (states and ARTP_ROADMAP_* kinds) and the edges first .. E-1 as (u, v) pairs.
  void vertices(size_t first, std::vector<State>* states, std::vector<uint8_t>* kinds) const {
    size_t nv = 0, ne = 0;
    counts(&nv, &ne);
    const size_t n = nv > first ? nv - first : 0;
    states->resize(n);
    kinds->resize(n);
    const auto& h = checker_->handle();
    h->check(artp_roadmap_get(h->get(), first, n ? &(*states)[0].x : nullptr, n ? kinds->data() : nullptr, 0, nullptr, nullptr,
                              nullptr), "artp_roadmap_get");
  }
  void edges(size_t first, std::vector<uint32_t>* uv) const {
    size_t nv = 0, ne = 0;
    counts(&nv, &ne);
    const size_t n = ne > first ? ne - first : 0;
    uv->resize(2 * n);
    const auto& h = checker_->handle();
    h->check(artp_roadmap_get(h->get(), 0, nullptr, nullptr, first, n ? uv->data() : nullptr, nullptr, nullptr), "artp_roadmap_get");
  }
  void counts(size_t* nv, size_t* ne) const {
    const auto& h = checker_->handle();
    h->check(artp_roadmap_get(h->get(), 0, nullptr, nullptr, 0, nullptr, nv, ne), "artp_roadmap_get");
  }
  // PRMMotionCostMaintainer::updateEdges (:27-73) over the whole store, on the device.
  void updateEdges() {
    const auto& h = checker_->handle();
    h->check(artp_roadmap_update_edges(h->get()), "artp_roadmap_update_edges");
  }
  // One query (clearQuery + PRMMotionCost::baseSolve) on the device. Returns info.status (ARTP_SOLVE_*); path and
  // path_vertices hold the solution from start to goal when it is ARTP_SOLVE_SOLVED, and are empty otherwise.
  struct Solution {
    std::vector<State> path;
    std::vector<uint32_t> path_vertices;
    double cost = 0.0;
    artp_roadmap_solve_info info{};
  };
  int solve(const State& start, const State& goal, const artp_se3_space& space, Solution* out, size_t path_capacity = 4096) {
    const auto& h = checker_->handle();
    out->path.resize(path_capacity);
    out->path_vertices.resize(path_capacity);
    out->info = artp_roadmap_solve_info{};
    out->info.path_vertices = out->path_vertices.data();
    size_t n = 0;
    h->check(artp_roadmap_solve(h->get(), &start.x, &goal.x, &space, &out->path[0].x, path_capacity, &n, &out->cost, &out->info),
             "artp_roadmap_solve");
    out->path.resize(n);
    out->path_vertices.resize(n);
    out->info.path_vertices = nullptr;
    return out->info.status;
  }
  // The weights and ARTP_ROADMAP_EDGE_* flags of the edges first .. E-1; returns the live edges of the whole store.
  size_t edgeCosts(size_t first, std::vector<double>* cost, std::vector<uint8_t>* flags) const {
    size_t nv = 0, ne = 0, live = 0;
    counts(&nv, &ne);
    const size_t n = ne > first ? ne - first : 0;
    cost->resize(n);
    flags->resize(n);
    const auto& h = checker_->handle();
    h->check(artp_roadmap_get_edge_costs(h->get(), first, n ? cost->data() : nullptr, n ? flags->data() : nullptr, &live),
             "artp_roadmap_get_edge_costs");
    return live;
  }
 private:
  StateValidityCheckerPtr checker_;
  size_t vertex_capacity_, edge_capacity_;
};

// Planner::getSolutionPath (planner.cpp:266-298) on the device (artp_simplify_path; the rules are in include/artp.h):
// OMPL 1.4.2's PathSimplifier::simplifyMax, the check of the simplified path and the strict cost comparison under the
// planner's objective -- LEARNED (MotionCostObjective, pieces of params().planner.prm_motion_cost.max_query_edge_length;
// needs weights and features) or PATH_LENGTH (getObjective's PathLengthObjective). The random stream is Philox under
// `seed`, not OMPL's mt19937. With -DARTP_WITH_OMPL, getSolutionPath(og::PathGeometric) builds the returned path.
class PathSimplifier {
 public:
  enum Objective { LEARNED = ARTP_OBJ_LEARNED, PATH_LENGTH = ARTP_OBJ_PATH_LENGTH };
  struct Result {
    std::vector<State> path;    // the returned path: the simplified one, or the original
    artp_simplify_info info{};  // state counts, edits per stage, checkMotion / isValid counts, check, both costs
  };
  PathSimplifier(const StateValidityCheckerPtr& checker, const artp_se3_space& space, Objective objective = LEARNED,
                 uint64_t seed = 0)
      : checker_(checker), space_(space), objective_(objective), seed_(seed) {}
  // getSolutionPath(simplify): without simplify the path comes back unchanged (info zeroed).
  Result getSolutionPath(const std::vector<State>& path, bool simplify = true) const {
    if (!simplify) return Result{path, artp_simplify_info{}};
    return run(path, objective_);
  }
  // simplifySolution + the check, without the cost comparison: the simplified path whenever it passes the check.
  Result simplifyMax(const std::vector<State>& path) const { return run(path, ARTP_OBJ_NONE); }
  void setSeed(uint64_t seed) { seed_ = seed; }
 private:
  Result run(const std::vector<State>& path, int objective) const {
    const auto& h = checker_->handle();
    Result r;
    r.path.resize(256 * path.size() + 64);   // the longest path the schedule can leave
    size_t n = 0;
    h->check(artp_simplify_path(h->get(), path.empty() ? nullptr : &path[0].x, path.size(), &space_, objective,
                                h->params().planner.prm_motion_cost.max_query_edge_length, seed_, &r.path[0].x, r.path.size(),
                                &n, &r.info), "artp_simplify_path");
    r.path.resize(n);
    return r;
  }
  StateValidityCheckerPtr checker_;
  artp_se3_space space_;
  Objective objective_;
  uint64_t seed_;
};

// art_planner::PlannerStatus (planner_status.h).
enum PlannerStatus { UNKNOWN = ARTP_PLANNER_UNKNOWN, INVALID_START = ARTP_PLANNER_INVALID_START,
                     INVALID_GOAL = ARTP_PLANNER_INVALID_GOAL, NO_MAP = ARTP_PLANNER_NO_MAP,
                     NOT_SOLVED = ARTP_PLANNER_NOT_SOLVED, SOLVED = ARTP_PLANNER_SOLVED };

// art_planner::inpaintMatrix (utils.cpp:13-63) on the device of `handle` (artp_inpaint_layer): the rows x cols
// column-major layer (NaN unknown) in, the inpainted layer out, bit for bit with OpenCV's chain (DESIGN.md section 4.6).
inline std::vector<float> inpaintMatrix(const Handle& handle, const std::vector<float>& layer, int rows, int cols) {
  if (layer.size() != (size_t)rows * (size_t)cols) throw std::runtime_error("inpaintMatrix: layer size is not rows * cols");
  std::vector<float> out(layer.size());
  handle.check(artp_inpaint_layer(handle.get(), layer.data(), rows, cols, out.data()), "artp_inpaint_layer");
  return out;
}

// The cost server's preparation of the RAW rows x cols column-major elevation layer (cost_query_server.py _elvMapProcess,
// artp_cost_map_layer): the layer whose network input is what the server feeds the trunk (DESIGN.md section 4.7).
inline std::vector<float> costServerMap(const Handle& handle, const std::vector<float>& layer, int rows, int cols) {
  if (layer.size() != (size_t)rows * (size_t)cols) throw std::runtime_error("costServerMap: layer size is not rows * cols");
  std::vector<float> out(layer.size());
  handle.check(artp_cost_map_layer(handle.get(), layer.data(), rows, cols, out.data()), "artp_cost_map_layer");
  return out;
}

// art_planner::Planner for planner.name prm_motion_cost (planner.cpp:135-298) on the device: setMap is
// artp_planner_set_map, plan is artp_plan (the simplification of getSolutionPath(true) runs inside it when
// parameters().simplify is set), and the stages hand data to each other in device memory. The parameters start from
// Params (caps, max_query_edge_length, sampler) and the shipped values of params.yaml for the rest; change them through
// parameters(). With -DARTP_WITH_OMPL, getSolutionPath(si) builds the returned og::PathGeometric.
class Planner {
 public:
  explicit Planner(const StateValidityCheckerPtr& checker) : checker_(checker) {
    const Params& p = checker->handle()->params();
    pp_.start_radius = 0.2; pp_.goal_radius = 0.5; pp_.n_iter = 1000;   // params.yaml:20-22
    pp_.max_n_vertices = p.planner.prm_motion_cost.max_n_vertices;
    pp_.max_n_edges = p.planner.prm_motion_cost.max_n_edges;
    pp_.recompute_density_after_n_samples = p.planner.prm_motion_cost.recompute_density_after_n_samples;
    pp_.max_query_edge_length = p.planner.prm_motion_cost.max_query_edge_length;
    pp_.max_draws = 1ull << 26;
    pp_.vertex_capacity = 2 * (size_t)pp_.max_n_vertices; pp_.edge_capacity = (size_t)pp_.max_n_edges + 10000;
    pp_.max_roll_pert = p.sampler.max_roll_pert; pp_.max_pitch_pert = p.sampler.max_pitch_pert;
    pp_.sample_from_distribution = p.sampler.sample_from_distribution;
    pp_.use_inverse_vertex_density = p.sampler.use_inverse_vertex_density;
    pp_.use_max_prob_unknown_samples = p.sampler.use_max_prob_unknown_samples;
    pp_.max_prob_unknown_samples = p.sampler.max_prob_unknown_samples;
    pp_.basic = artp_basic_params{0.15f, p.planner.unknown_space_untraversable ? 1 : 0, 0.3, 0.3, 0.3, 0.16, 0.3, 0.1};
    pp_.simplify = 1; pp_.clear_roadmap = 0; pp_.seed = 0;
    pp_.cost_map_from_raw = 0;   // 1: the trunk reads the cost server's preparation of the raw elevation
  }
  artp_planner_params& parameters() { return pp_; }

  // Planner::setMap: elevation / traversability are the RAW layers (NaN unknown; traversability may be empty), the
  // inpainted ones what inpaintMatrix returned for them (empty with an empty traversability). Geometry from `map`.
  void setMap(const Map& map, const std::vector<float>& elevation, const std::vector<float>& traversability,
              const std::vector<float>& elevation_inpainted, const std::vector<float>& traversability_inpainted) {
    const auto& h = checker_->handle();
    h->check(artp_planner_set_map(h->get(), &pp_, elevation.data(), traversability.empty() ? nullptr : traversability.data(),
                                  elevation_inpainted.data(),
                                  traversability_inpainted.empty() ? nullptr : traversability_inpainted.data(), map.rows,
                                  map.cols, map.resolution, map.position_x, map.position_y, &map_info_),
             "artp_planner_set_map");
  }
  // Planner::setMap from the RAW layers alone (artp_planner_set_map_raw): processors::Basic's two inpaintMatrix calls
  // (basic.cpp:42-45) run on the device; traversability may be empty. The handle ends in the state the overload above
  // leaves it in when given inpaintMatrix's outputs.
  void setMap(const Map& map, const std::vector<float>& elevation, const std::vector<float>& traversability) {
    const auto& h = checker_->handle();
    h->check(artp_planner_set_map_raw(h->get(), &pp_, elevation.data(), traversability.empty() ? nullptr : traversability.data(),
                                      map.rows, map.cols, map.resolution, map.position_x, map.position_y, &map_info_),
             "artp_planner_set_map_raw");
  }
  artp_se3_space space() const {
    artp_se3_space sp{};
    checker_->handle()->check(artp_planner_get_space(checker_->handle()->get(), &sp), "artp_planner_get_space");
    return sp;
  }
  PlannerStatus plan(const State& start, const State& goal) {
    const auto& h = checker_->handle();
    solved_ = false;                    // a failing call leaves no solution behind
    path_.assign(4 * pp_.vertex_capacity + 64, State{});
    size_t n = 0;
    info_ = artp_plan_info{};
    struct ClearOnThrow {
      std::vector<State>& p; bool armed = true;
      ~ClearOnThrow() { if (armed) p.clear(); }
    } guard{path_};
    h->check(artp_plan(h->get(), &pp_, &start.x, &goal.x, &path_[0].x, path_.size(), &n, &info_), "artp_plan");
    guard.armed = false;
    path_.resize(n);
    solved_ = info_.status == ARTP_PLANNER_SOLVED;
    return static_cast<PlannerStatus>(info_.status);
  }
  // The last plan's path (simplified when parameters().simplify is set); throws like planner.cpp:268-270.
  const std::vector<State>& getSolutionPath() const {
    if (!solved_) throw std::runtime_error("Requested failed solution path.");
    return path_;
  }
  const artp_plan_info& info() const { return info_; }
  const artp_planner_map_info& mapInfo() const { return map_info_; }   // the last setMap's syncs and bytes
 private:
  StateValidityCheckerPtr checker_;
  artp_planner_params pp_{};
  std::vector<State> path_;
  artp_plan_info info_{};
  artp_planner_map_info map_info_{};
  bool solved_{false};
};

// (unsigned)(lateralDistance(s1, s2) / length) (utils.h:52-61): the interior states of a roadmap connection
// (prm_motion_cost.cpp:341-343) and the split of a motion cost (motion_cost_objective.cpp:40-45).
inline unsigned lateralCount(const State& s1, const State& s2, double length) {
  const double dx = s2.x - s1.x, dy = s2.y - s1.y;
  return static_cast<unsigned>(std::sqrt(dx * dx + dy * dy) / length);
}

// ompl::base::MotionValidator as the reference uses it: discrete validation over isValid with nd segments.
class MotionValidator {
 public:
  MotionValidator(const StateValidityCheckerPtr& checker, int n_segments) : checker_(checker), nd_(n_segments) {}
  // valid(s2) && valid(interpolate(s1, s2, j/nd)) for j = 1..nd-1 (OMPL DiscreteMotionValidator::checkMotion)
  bool checkMotion(const State* s1, const State* s2) const {
    uint8_t v = 0;
    const auto& h = checker_->handle();
    h->check(artp_check_motions(h->get(), &s1->x, &s2->x, 1, nd_ - 1, &v), "artp_check_motions");
    return v != 0;
  }
  void checkMotionBatch(const std::vector<State>& s1, const std::vector<State>& s2, std::vector<uint8_t>* valid) const {
    if (s1.size() != s2.size()) throw std::invalid_argument("checkMotionBatch: size mismatch");
    valid->resize(s1.size());
    if (s1.empty()) return;
    const auto& h = checker_->handle();
    h->check(artp_check_motions(h->get(), &s1[0].x, &s2[0].x, s1.size(), nd_ - 1, valid->data()), "artp_check_motions");
  }
  // DiscreteMotionValidator::checkMotion(s1, s2, lastValid) with this validator's segment count: returns validity and,
  // for an invalid motion, lastValid.second = the parameter of the last valid state before the first invalid one in
  // OMPL's order (j = 1 .. nd-1, then s2); *last_valid (nullable) receives interpolate(s1, s2, that parameter).
  bool checkMotion(const State* s1, const State* s2, double* last_valid_t, State* last_valid) const {
    uint8_t v = 0;
    double t = 1.0;
    const int32_t nd = nd_;
    const auto& h = checker_->handle();
    h->check(artp_check_motions_segments(h->get(), &s1->x, &s2->x, 1, &nd, nullptr, &v, &t), "artp_check_motions_segments");
    if (!v) {
      if (last_valid_t) *last_valid_t = t;
      if (last_valid) *last_valid = interpolateSE3(*s1, *s2, t);
    }
    return v != 0;
  }
  // The batch form with PER-EDGE segment counts nd[e] = SE3StateSpace::validSegmentCount(s1, s2) (OMPL 1.4.2 rule,
  // artp_valid_segment_count) -- what si_->checkMotion does at prm_motion_cost.cpp:652 / lazy_prm_star_min_update.cpp:725.
  void checkMotionSegments(const std::vector<State>& s1, const std::vector<State>& s2, const artp_se3_space& space,
                           std::vector<uint8_t>* valid, std::vector<double>* last_valid_t, std::vector<int32_t>* nd = nullptr) const {
    if (s1.size() != s2.size()) throw std::invalid_argument("checkMotionSegments: size mismatch");
    valid->resize(s1.size());
    last_valid_t->resize(s1.size());
    if (s1.empty()) return;
    std::vector<int32_t> seg(s1.size());
    const auto& h = checker_->handle();
    h->check(artp_valid_segment_count(&space, &s1[0].x, &s2[0].x, s1.size(), seg.data()), "artp_valid_segment_count");
    h->check(artp_check_motions_segments(h->get(), &s1[0].x, &s2[0].x, s1.size(), seg.data(), nullptr, valid->data(),
                                         last_valid_t->data()), "artp_check_motions_segments");
    if (nd) *nd = seg;
  }
  // OMPL 1.4.2 SE3StateSpace::interpolate = RealVector lerp + SO3 slerp
  static State interpolateSE3(const State& a, const State& b, double t) {
    State o;
    o.x = a.x + (b.x - a.x) * t; o.y = a.y + (b.y - a.y) * t; o.z = a.z + (b.z - a.z) * t;
    const double dq = a.qx * b.qx + a.qy * b.qy + a.qz * b.qz + a.qw * b.qw;
    const double dqa = std::fabs(dq);
    const double theta = (dqa > 1.0 - 1e-9) ? 0.0 : std::acos(dqa);
    if (theta > std::numeric_limits<double>::epsilon()) {
      const double d = 1.0 / std::sin(theta), s0 = std::sin((1.0 - t) * theta);
      double s1 = std::sin(t * theta);
      if (dq < 0) s1 = -s1;
      o.qx = (a.qx * s0 + b.qx * s1) * d; o.qy = (a.qy * s0 + b.qy * s1) * d;
      o.qz = (a.qz * s0 + b.qz * s1) * d; o.qw = (a.qw * s0 + b.qw * s1) * d;
    } else {
      o.qx = a.qx; o.qy = a.qy; o.qz = a.qz; o.qw = a.qw;
    }
    return o;
  }
  // PRMMotionCost::addValidMilestone's connection loop (prm_motion_cost.cpp:341-372) for a batch of candidate edges:
  // n_interp[e] = (unsigned)(lateralDistance / max_lateral) interior states, valid_prefix[e] = how many leading ones are
  // valid; the connection holds iff valid_prefix[e] == n_interp[e].
  void checkEdgeInteriors(const std::vector<State>& s1, const std::vector<State>& s2, double max_lateral,
                          std::vector<int32_t>* n_interp, std::vector<int32_t>* valid_prefix) const {
    if (s1.size() != s2.size()) throw std::invalid_argument("checkEdgeInteriors: size mismatch");
    n_interp->resize(s1.size());
    valid_prefix->resize(s1.size());
    if (s1.empty()) return;
    for (size_t e = 0; e < s1.size(); ++e) (*n_interp)[e] = static_cast<int32_t>(lateralCount(s1[e], s2[e], max_lateral));
    const auto& h = checker_->handle();
    h->check(artp_check_edge_interiors(h->get(), &s1[0].x, &s2[0].x, s1.size(), n_interp->data(), max_lateral,
                                       valid_prefix->data()), "artp_check_edge_interiors");
  }
 private:
  StateValidityCheckerPtr checker_;
  int nd_;
};

// art_planner::PathLengthObjective (path_length_objective.cpp:26-70).
class PathLengthObjective {
 public:
  explicit PathLengthObjective(const StateValidityCheckerPtr& checker) : checker_(checker) {}
  double motionCost(const State* s1, const State* s2) const {
    double c = 0;
    const auto& h = checker_->handle();
    h->check(artp_path_length_cost(h->get(), &s1->x, &s2->x, 1, &c), "artp_path_length_cost");
    return c;
  }
  double motionCostHeuristic(const State* s1, const State* s2) const {           // path_length_objective.cpp:58-70
    const double dx = s2->x - s1->x, dy = s2->y - s1->y, dz = s2->z - s1->z;
    return std::sqrt(dx * dx + dy * dy + dz * dz) / checker_->handle()->params().objectives.custom_path_length.max_lon_vel;
  }
  void motionCostBatch(const std::vector<State>& s1, const std::vector<State>& s2, std::vector<double>* cost) const {
    cost->resize(s1.size());
    if (s1.empty()) return;
    const auto& h = checker_->handle();
    h->check(artp_path_length_cost(h->get(), &s1[0].x, &s2[0].x, s1.size(), cost->data()), "artp_path_length_cost");
  }
 private:
  StateValidityCheckerPtr checker_;
};

// Row-major dynamic float matrix, the shape of MotionCostObjective::EdgeMatrix (motion_cost_objective.h:22).
struct EdgeMatrix {
  size_t n_rows{0}, n_cols{0};
  std::vector<float> v;
  void resize(size_t r, size_t c) { n_rows = r; n_cols = c; v.assign(r * c, 0.0f); }
  size_t rows() const { return n_rows; }
  float& operator()(size_t r, size_t c) { return v[r * n_cols + c]; }
  float operator()(size_t r, size_t c) const { return v[r * n_cols + c]; }
  const float* data() const { return v.data(); }
  float* data() { return v.data(); }
};

// art_planner::MotionCostObjective (motion_cost_objective.h:19-78, motion_cost_objective.cpp:28-95). The batch functor
// defaults to the in-process network (artp_motion_cost) instead of the ROS cost-server call of planner_ros.cpp:283-308.
class MotionCostObjective {
 public:
  using MotionCostFunc = std::function<bool(const EdgeMatrix&, EdgeMatrix*)>;

  explicit MotionCostObjective(const StateValidityCheckerPtr& checker, std::unique_ptr<MotionCostFunc> func = nullptr)
      : checker_(checker), motion_cost_func_(std::move(func)) {
    custom_func_ = motion_cost_func_ != nullptr;
    if (!motion_cost_func_) {
      HandlePtr h = checker_->handle();
      motion_cost_func_.reset(new MotionCostFunc([h](const EdgeMatrix& edges, EdgeMatrix* costs) {
        costs->resize(edges.rows(), 3);
        return artp_motion_cost(h->get(), edges.data(), edges.rows(), costs->data()) == ARTP_OK;
      }));
    }
  }
  // Either network's blob (artp.h, above artp_cost_weights_size): its length picks network_light or network.
  void setWeights(const std::vector<float>& blob) {
    checker_->handle()->check(artp_set_cost_weights(checker_->handle()->get(), blob.data(), blob.size()), "artp_set_cost_weights");
  }
  void updateFeatures() { checker_->handle()->check(artp_update_features(checker_->handle()->get()), "artp_update_features"); }
  // CostPredictor.updateFeatures on the map the cost server prepares from the RAW elevation (artp_update_features_raw):
  // the rows x cols column-major layer, the map's resolution and position; no installed map needed.
  void updateFeaturesRaw(const std::vector<float>& elevation, int rows, int cols, double resolution, double position_x,
                         double position_y) {
    if (elevation.size() != (size_t)rows * (size_t)cols)
      throw std::runtime_error("updateFeaturesRaw: layer size is not rows * cols");
    checker_->handle()->check(artp_update_features_raw(checker_->handle()->get(), elevation.data(), rows, cols, resolution,
                                                       position_x, position_y),
                              "artp_update_features_raw");
  }

  double getCost(const float* e3) const {                                        // motion_cost_objective.h:54-61
    const auto& w = checker_->handle()->params().planner.prm_motion_cost.cost_weights;
    // getEnergy/getTime/getRisk return double: the weighted sum is evaluated in double on exact float products
    return static_cast<double>(e3[0]) * w.energy + static_cast<double>(e3[1]) * w.time + static_cast<double>(e3[2]) * w.risk;
  }
  bool isFeasible(const float* e3) const {                                       // motion_cost_objective.h:63-65
    return static_cast<double>(e3[2]) <= checker_->handle()->params().planner.prm_motion_cost.risk_threshold;
  }
  bool costQuery(const EdgeMatrix& edge_matrix, EdgeMatrix* edge_cost) const {   // motion_cost_objective.cpp:28-33
    edge_cost->resize(edge_matrix.rows(), 3);
    return (*motion_cost_func_)(edge_matrix, edge_cost);
  }

  // motion_cost_objective.cpp:36-95: split the edge at max_query_edge_length, query every piece, sum; +inf if any piece
  // is too risky; throws "Motion cost call failed" if the functor fails.
  double motionCost(const State* s1, const State* s2) const {
    const auto& pm = checker_->handle()->params().planner.prm_motion_cost;
    const unsigned n_interp = lateralCount(*s1, *s2, pm.max_query_edge_length);
    const double n_interp_div = 1.0 / (n_interp + 1);
    EdgeMatrix em, ec;
    em.resize(n_interp + 1, 6);
    em(0, 3) = static_cast<float>(s1->x); em(0, 4) = static_cast<float>(s1->y); em(0, 5) = yaw(*s1);
    em(n_interp, 0) = static_cast<float>(s2->x); em(n_interp, 1) = static_cast<float>(s2->y); em(n_interp, 2) = yaw(*s2);
    for (unsigned step = 1; step < n_interp + 1; ++step) {
      const State cur = interpolate(*s1, *s2, step * n_interp_div);
      em(step - 1, 0) = static_cast<float>(cur.x); em(step - 1, 1) = static_cast<float>(cur.y); em(step - 1, 2) = yaw(cur);
      em(step, 3) = static_cast<float>(cur.x); em(step, 4) = static_cast<float>(cur.y); em(step, 5) = yaw(cur);
    }
    if (!costQuery(em, &ec)) throw std::runtime_error("Motion cost call failed");
    double cost = 0;
    for (unsigned i = 0; i < n_interp + 1; ++i) {
      const float* e3 = ec.data() + 3 * i;
      if (static_cast<double>(e3[2]) > pm.risk_threshold) return std::numeric_limits<double>::infinity();
      cost += getCost(e3);
    }
    return cost;
  }
  double motionCostHeuristic(const State*, const State*) const { return 0.0; }   // motion_cost_objective.cpp:99-103

  // motionCost for a batch of edges: split, query and sum on the device in one call (artp_motion_cost_split), the same
  // cost per edge as motionCost. A caller-supplied MotionCostFunc (e.g. the ROS transport) stays the only cost source:
  // the batch then loops over motionCost. Throws "Motion cost call failed" like motionCost.
  void motionCostBatch(const std::vector<State>& s1, const std::vector<State>& s2, std::vector<double>* cost) const {
    if (s1.size() != s2.size()) throw std::invalid_argument("motionCostBatch: size mismatch");
    cost->resize(s1.size());
    if (s1.empty()) return;
    if (custom_func_) {
      for (size_t e = 0; e < s1.size(); ++e) (*cost)[e] = motionCost(&s1[e], &s2[e]);
      return;
    }
    const auto& h = checker_->handle();
    if (artp_motion_cost_split(h->get(), &s1[0].x, &s2[0].x, s1.size(), h->params().planner.prm_motion_cost.max_query_edge_length,
                               cost->data()) != ARTP_OK)
      throw std::runtime_error("Motion cost call failed");
  }
  // ompl::geometric::PathGeometric::cost(obj) (OMPL 1.4.2) for this objective: initial and terminal cost are the identity
  // 0, so the cost is 0 for fewer than two states, else the left-to-right sum of motionCost over consecutive states.
  double pathCost(const std::vector<State>& path) const {
    if (path.size() < 2) return 0.0;
    std::vector<double> c;
    motionCostBatch(std::vector<State>(path.begin(), path.end() - 1), std::vector<State>(path.begin() + 1, path.end()), &c);
    double cost = 0.0;
    for (double v : c) cost += v;
    return cost;
  }

  // PRMMotionCostMaintainer::updateEdges / computeCostForVertexEdges (prm_motion_cost.cpp:27-128) for a batch of graph
  // edges (source = v1, target = v2): edge matrix -> cost query -> per edge isFeasible ? getCost : +inf, in one device call.
  // Returns false where the reference's functor would (then the graph is left alone, :69-72 / :124-127).
  bool updateEdgesBatch(const std::vector<State>& source, const std::vector<State>& target, std::vector<double>* cost,
                        std::vector<uint8_t>* feasible) const {
    if (source.size() != target.size()) throw std::invalid_argument("updateEdgesBatch: size mismatch");
    cost->resize(source.size());
    feasible->resize(source.size());
    if (source.empty()) return true;
    return artp_motion_cost_states(checker_->handle()->get(), &source[0].x, &target[0].x, source.size(), cost->data(),
                                   feasible->data(), nullptr) == ARTP_OK;
  }

  // getYawFromSO3 (utils.h:80-88): double atan2 returned through float
  static float yaw(const State& s) {
    return static_cast<float>(std::atan2(2 * (s.qw * s.qz + s.qx * s.qy), 1 - 2 * (s.qy * s.qy + s.qz * s.qz)));
  }
  static State interpolate(const State& a, const State& b, double t) { return MotionValidator::interpolateSE3(a, b, t); }

 private:
  StateValidityCheckerPtr checker_;
  std::unique_ptr<MotionCostFunc> motion_cost_func_;
  bool custom_func_{false};   // motion_cost_func_ came from the caller
};

}  // namespace artp_host

#ifdef ARTP_WITH_OMPL
// OMPL adapters (compiled only where OMPL >= 1.4.2 is installed): the exact plugin surface of planner.cpp:125-130.
#include <ompl/base/MotionValidator.h>
#include <ompl/base/SpaceInformation.h>
#include <ompl/base/StateValidityChecker.h>
#include <ompl/base/goals/GoalState.h>
#include <ompl/base/objectives/PathLengthOptimizationObjective.h>
#include <ompl/util/RandomNumbers.h>
#include <ompl/base/spaces/SE3StateSpace.h>
#include <ompl/geometric/PathGeometric.h>
namespace artp_host {
namespace ob = ompl::base;
namespace og = ompl::geometric;
inline State fromOmpl(const ob::State* s) {
  const auto* se3 = s->as<ob::SE3StateSpace::StateType>();
  State o;
  o.x = se3->getX(); o.y = se3->getY(); o.z = se3->getZ();
  o.qx = se3->rotation().x; o.qy = se3->rotation().y; o.qz = se3->rotation().z; o.qw = se3->rotation().w;
  return o;
}
class OmplStateValidityChecker : public ob::StateValidityChecker {
 public:
  OmplStateValidityChecker(const ob::SpaceInformationPtr& si, const StateValidityCheckerPtr& c) : ob::StateValidityChecker(si), c_(c) {}
  bool isValid(const ob::State* state) const override { const State s = fromOmpl(state); return c_->isValid(&s); }
 private:
  StateValidityCheckerPtr c_;
};
class OmplMotionValidator : public ob::MotionValidator {
 public:
  OmplMotionValidator(const ob::SpaceInformationPtr& si, const StateValidityCheckerPtr& c) : ob::MotionValidator(si), c_(c) {}
  bool checkMotion(const ob::State* s1, const ob::State* s2) const override {
    const State a = fromOmpl(s1), b = fromOmpl(s2);
    return MotionValidator(c_, si_->getStateSpace()->validSegmentCount(s1, s2)).checkMotion(&a, &b);
  }
  bool checkMotion(const ob::State* s1, const ob::State* s2, std::pair<ob::State*, double>& lastValid) const override {
    const State a = fromOmpl(s1), b = fromOmpl(s2);
    double t = 1.0;
    const bool ok = MotionValidator(c_, si_->getStateSpace()->validSegmentCount(s1, s2)).checkMotion(&a, &b, &t, nullptr);
    if (!ok) {   // DiscreteMotionValidator: lastValid is only written for invalid motions
      lastValid.second = t;
      if (lastValid.first) si_->getStateSpace()->interpolate(s1, s2, t, lastValid.first);
    }
    return ok;
  }
 private:
  StateValidityCheckerPtr c_;
};
// StartState / GoalStateRegion as OMPL goals (start.h, goal.h: ob::GoalState with setThreshold / setMaxNumSamples).
// sampleGoal draws its n_iter offsets from its own ompl::RNG::uniformInBall, as the reference loop does, and checks all
// candidates in one call with those offsets: the result is the reference's for the same RNG. Only the RNG's position
// afterwards differs, since this draws all n_iter offsets every time.
class OmplDiscSearchGoal : public ob::GoalState {
 public:
  OmplDiscSearchGoal(const ob::SpaceInformationPtr& si, const StateValidityCheckerPtr& c) : ob::GoalState(si), c_(c) {}
  void setMaxNumSamples(const unsigned int& num_samples) { max_num_samples_ = num_samples; }
  void sampleGoal(ob::State* state) const override {
    std::vector<double> off(2 * static_cast<size_t>(max_num_samples_)), o(2);
    for (unsigned int i = 0; i < max_num_samples_; ++i) {
      rng_.uniformInBall(threshold_, o);
      off[2 * i] = o[0]; off[2 * i + 1] = o[1];
    }
    const std::vector<State> centre{fromOmpl(state_)};
    std::vector<State> out;
    std::vector<int32_t> index;
    c_->findValidNearBatch(centre, {threshold_}, max_num_samples_, off.data(), 0, 0, &out, &index);
    si_->copyState(state, state_);
    auto* s = state->as<ob::SE3StateSpace::StateType>();
    s->setX(out[0].x);
    s->setY(out[0].y);
  }
 private:
  StateValidityCheckerPtr c_;
  unsigned int max_num_samples_{0};
  mutable ompl::RNG rng_;
};
class OmplStartState : public OmplDiscSearchGoal { public: using OmplDiscSearchGoal::OmplDiscSearchGoal; };
class OmplGoalStateRegion : public OmplDiscSearchGoal { public: using OmplDiscSearchGoal::OmplDiscSearchGoal; };

// Planner::getSolutionPath(simplify) over an og::PathGeometric: the device call, then the returned states as a new path.
inline og::PathGeometric getSolutionPath(const PathSimplifier& simplifier, const og::PathGeometric& path, bool simplify) {
  if (!simplify) return path;
  std::vector<State> in(path.getStateCount());
  for (size_t i = 0; i < in.size(); ++i) in[i] = fromOmpl(path.getState(i));
  const PathSimplifier::Result r = simplifier.getSolutionPath(in);
  og::PathGeometric out(path.getSpaceInformation());
  ob::State* s = out.getSpaceInformation()->allocState();
  for (const State& t : r.path) {
    auto* se3 = s->as<ob::SE3StateSpace::StateType>();
    se3->setXYZ(t.x, t.y, t.z);
    se3->rotation().x = t.qx; se3->rotation().y = t.qy; se3->rotation().z = t.qz; se3->rotation().w = t.qw;
    out.append(s);
  }
  out.getSpaceInformation()->freeState(s);
  return out;
}

// Planner::getSolutionPath(simplify) for the Planner mirror: its last plan's path (simplified as its parameters say) as an
// og::PathGeometric; throws like planner.cpp:268-270 when the plan did not solve.
inline og::PathGeometric getSolutionPath(const Planner& planner, const ob::SpaceInformationPtr& si) {
  og::PathGeometric out(si);
  ob::State* s = si->allocState();
  for (const State& t : planner.getSolutionPath()) {
    auto* se3 = s->as<ob::SE3StateSpace::StateType>();
    se3->setXYZ(t.x, t.y, t.z);
    se3->rotation().x = t.qx; se3->rotation().y = t.qy; se3->rotation().z = t.qz; se3->rotation().w = t.qw;
    out.append(s);
  }
  si->freeState(s);
  return out;
}

class OmplPathLengthObjective : public ob::PathLengthOptimizationObjective {
 public:
  OmplPathLengthObjective(const ob::SpaceInformationPtr& si, const StateValidityCheckerPtr& c)
      : ob::PathLengthOptimizationObjective(si), o_(c) {}
  ob::Cost motionCost(const ob::State* s1, const ob::State* s2) const override {
    const State a = fromOmpl(s1), b = fromOmpl(s2);
    return ob::Cost(o_.motionCost(&a, &b));
  }
 private:
  PathLengthObjective o_;
};
}  // namespace artp_host
#endif
