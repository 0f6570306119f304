// tests/host_cpp/start_goal.cpp -- drives the start / goal search of the C++ host mirror (include/artp_host.hpp) the way
// Planner::setStartAndGoal and OMPL drive StartState / GoalStateRegion (planner.cpp:167-189): one StartState and one
// GoalStateRegion object, sampleGoal once per query, plus the batch call with explicit offsets and the goal projection.
//   start_goal --expect-no-gpu     : construction must fail loudly (no CPU fallback)
//   start_goal <in.bin> <out.bin>  : run the queries in in.bin, write the results (see tests/test_start_goal_host_cpp.py)
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iostream>

#include "artp_host.hpp"

using namespace artp_host;

template <class T> static void rd(std::ifstream& f, T* p, size_t n) { f.read(reinterpret_cast<char*>(p), sizeof(T) * n); }
template <class T> static void wr(std::ofstream& f, const T* p, size_t n) { f.write(reinterpret_cast<const char*>(p), sizeof(T) * n); }

int main(int argc, char** argv) {
  auto params = std::make_shared<Params>();
  if (argc == 2 && !std::strcmp(argv[1], "--expect-no-gpu")) {
    try {
      StateValidityChecker c(params);
    } catch (const std::runtime_error& e) {
      std::cout << "failed loudly: " << e.what() << "\n";
      return 0;
    }
    std::cout << "a handle was created: a CUDA device is present\n";
    return 3;
  }
  if (argc != 3) { std::cerr << "usage\n"; return 2; }
  std::ifstream in(argv[1], std::ios::binary);
  int32_t hdr[4];      // rows, cols, n queries, n_iter
  double geo[5];       // res, cx, cy, start radius, goal radius
  uint64_t seeds[2];   // start seed, goal seed
  rd(in, hdr, 4); rd(in, geo, 5); rd(in, seeds, 2);
  auto map = std::make_shared<Map>();
  map->rows = hdr[0]; map->cols = hdr[1]; map->resolution = geo[0]; map->position_x = geo[1]; map->position_y = geo[2];
  map->elevation.resize((size_t)hdr[0] * hdr[1]); map->elevation_masked.resize(map->elevation.size());
  rd(in, map->elevation.data(), map->elevation.size()); rd(in, map->elevation_masked.data(), map->elevation_masked.size());
  const size_t n = hdr[2];
  const uint32_t n_iter = (uint32_t)hdr[3];
  std::vector<State> starts(n), goals(n);
  rd(in, starts.data(), n); rd(in, goals.data(), n);
  std::vector<double> offsets(n * n_iter * 2);
  rd(in, offsets.data(), offsets.size());
  if (!in) { std::cerr << "short input\n"; return 2; }
  // art_planner_ros/config/params.yaml robot geometry
  params->robot.torso.length = 1.31; params->robot.torso.width = 0.65; params->robot.torso.height = 0.30;
  params->robot.torso.offset.z = 0.04;
  params->robot.feet.offset.x = 0.51; params->robot.feet.offset.y = 0.20; params->robot.feet.offset.z = -0.475;
  params->robot.feet.reach.x = 0.2; params->robot.feet.reach.y = 0.2; params->robot.feet.reach.z = 0.2;
  auto checker = std::make_shared<StateValidityChecker>(params);
  checker->setMap(map);
  checker->updateHeightField();
  // the planner's per-query order: project the goal, repair the start, repair the goal
  checker->estimateNormals();
  std::vector<State> projected;
  std::vector<uint8_t> inside;
  checker->poseFrom2D(goals, &projected, &inside);
  StartState start(checker, seeds[0]);
  start.setThreshold(geo[3]);
  start.setMaxNumSamples(n_iter);
  GoalStateRegion goal(checker, seeds[1]);
  goal.setThreshold(geo[4]);
  goal.setMaxNumSamples(n_iter);
  std::vector<State> s_out(n), g_out(n);
  std::vector<int32_t> s_idx(n), g_idx(n);
  std::vector<uint64_t> s_next(n), g_next(n);
  for (size_t q = 0; q < n; ++q) {
    start.setState(starts[q]);
    s_idx[q] = start.sampleGoal(&s_out[q]);
    s_next[q] = start.nextDraw();
    goal.setState(projected[q]);
    g_idx[q] = goal.sampleGoal(&g_out[q]);
    g_next[q] = goal.nextDraw();
  }
  std::vector<State> b_out;
  std::vector<int32_t> b_idx;
  checker->findValidNearBatch(starts, std::vector<double>(n, geo[3]), n_iter, offsets.data(), 0, 0, &b_out, &b_idx);
  std::ofstream out(argv[2], std::ios::binary);
  wr(out, projected.data(), n); wr(out, inside.data(), n);
  wr(out, s_out.data(), n); wr(out, s_idx.data(), n); wr(out, s_next.data(), n);
  wr(out, g_out.data(), n); wr(out, g_idx.data(), n); wr(out, g_next.data(), n);
  wr(out, b_out.data(), n); wr(out, b_idx.data(), n);
  return out ? 0 : 6;
}
