// tests/host_cpp/roadmap.cpp -- drives the C++ host mirror's PRMRoadmap (include/artp_host.hpp) the way
// PlannerRos::updateMapAndPlanFromCurrentRobotPose drives PRMMotionCost (planner_ros.cpp:370-376): clear, sampleGraph,
// then baseSolve's start / goal milestones, with the copy-out after each step.
//   roadmap --expect-no-gpu     : construction must fail loudly (no CPU fallback)
//   roadmap <in.bin> <out.bin>  : build the roadmap of the map in in.bin, write it (see tests/test_roadmap_host_cpp.py)
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
      auto c = std::make_shared<StateValidityChecker>(params);
      PRMRoadmap rm(c);
    } catch (const std::runtime_error& e) {
      std::cout << "failed loudly: " << e.what() << "\n";
      return 0;
    }
    std::cout << "a handle was created: a CUDA device is present\n";
    return 3;
  }
  if (argc != 3) { std::cerr << "usage\n"; return 2; }
  std::ifstream in(argv[1], std::ios::binary);
  int32_t hdr[5];      // rows, cols, max_n_vertices, max_n_edges, recompute interval
  double geo[7];       // res, cx, cy, low x, low y, high x, high y
  uint64_t seed;
  rd(in, hdr, 5); rd(in, geo, 7); rd(in, &seed, 1);
  auto map = std::make_shared<Map>();
  map->rows = hdr[0]; map->cols = hdr[1]; map->resolution = geo[0]; map->position_x = geo[1]; map->position_y = geo[2];
  map->elevation.resize((size_t)hdr[0] * hdr[1]); map->elevation_masked.resize(map->elevation.size());
  rd(in, map->elevation.data(), map->elevation.size()); rd(in, map->elevation_masked.data(), map->elevation_masked.size());
  State q[2];
  rd(in, q, 2);
  if (!in) { std::cerr << "short input\n"; return 2; }
  // art_planner_ros/config/params.yaml robot geometry, uniform sampling inside the given bounds
  params->robot.torso.length = 1.31; params->robot.torso.width = 0.65; params->robot.torso.height = 0.30;
  params->robot.torso.offset.z = 0.04;
  params->robot.feet.offset.x = 0.51; params->robot.feet.offset.y = 0.20; params->robot.feet.offset.z = -0.475;
  params->robot.feet.reach.x = 0.2; params->robot.feet.reach.y = 0.2; params->robot.feet.reach.z = 0.2;
  params->sampler.sample_from_distribution = false;
  params->planner.prm_motion_cost.max_n_vertices = (unsigned)hdr[2];
  params->planner.prm_motion_cost.max_n_edges = (unsigned)hdr[3];
  params->planner.prm_motion_cost.recompute_density_after_n_samples = (unsigned)hdr[4];
  auto checker = std::make_shared<StateValidityChecker>(params);
  checker->setMap(map);
  checker->updateHeightField();
  checker->estimateNormals();
  const double low[2] = {geo[3], geo[4]}, high[2] = {geo[5], geo[6]};
  SE3FromSE2Sampler sampler(checker, map, seed, low, high);
  PRMRoadmap rm(checker, 20000, 40000);
  const uint64_t used = rm.sampleGraph(sampler, 1ull << 24, false);
  size_t nv0 = 0, ne0 = 0;
  rm.counts(&nv0, &ne0);
  rm.addValidMilestones(std::vector<State>(q, q + 2));
  std::vector<State> st, st_tail;
  std::vector<uint8_t> kinds, kinds_tail;
  std::vector<uint32_t> uv, uv_tail;
  rm.vertices(0, &st, &kinds);
  rm.edges(0, &uv);
  rm.vertices(nv0, &st_tail, &kinds_tail);
  rm.edges(ne0, &uv_tail);
  if (st_tail.size() != st.size() - nv0 || uv_tail.size() != uv.size() - 2 * ne0) return 4;
  if (std::memcmp(st_tail.data(), st.data() + nv0, st_tail.size() * sizeof(State))) return 5;
  const uint64_t nv = st.size(), ne = uv.size() / 2;
  std::ofstream out(argv[2], std::ios::binary);
  wr(out, &used, 1); wr(out, &nv, 1); wr(out, &ne, 1);
  wr(out, st.data(), nv); wr(out, kinds.data(), nv); wr(out, uv.data(), 2 * ne);
  return out ? 0 : 6;
}
