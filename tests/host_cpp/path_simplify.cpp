// tests/host_cpp/path_simplify.cpp -- drives the C++ host mirror's PathSimplifier (include/artp_host.hpp) the way
// PlannerRos publishes a plan: Planner::getSolutionPath(params_->planner.simplify_solution) on a solved path.
//   path_simplify --expect-no-gpu     : construction must fail loudly (no CPU fallback)
//   path_simplify <in.bin> <out.bin>  : getSolutionPath of the path in in.bin on its map (see
//                                       tests/test_path_simplify_host_cpp.py), the result and its info to out.bin
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
      PathSimplifier ps(c, artp_se3_space{});
    } catch (const std::runtime_error& e) {
      std::cout << "failed loudly: " << e.what() << "\n";
      return 0;
    }
    std::cout << "a handle was created: a CUDA device is present\n";
    return 3;
  }
  if (argc != 3) { std::cerr << "usage\n"; return 2; }
  std::ifstream in(argv[1], std::ios::binary);
  int32_t hdr[5];      // rows, cols, path states, unknown_space_untraversable, use_directional_cost
  double geo[3];       // res, cx, cy
  double robot[15];    // torso l w h, torso offset xyz, feet offset xyz, reach xyz, max lon / lat / ang velocity
  double space[7];     // artp_se3_space: low[3], high[3], fraction
  uint64_t seed;
  rd(in, hdr, 5); rd(in, geo, 3); rd(in, robot, 15); rd(in, space, 7); rd(in, &seed, 1);
  auto map = std::make_shared<Map>();
  map->rows = hdr[0]; map->cols = hdr[1]; map->resolution = geo[0]; map->position_x = geo[1]; map->position_y = geo[2];
  map->elevation.resize((size_t)hdr[0] * hdr[1]); map->elevation_masked.resize(map->elevation.size());
  rd(in, map->elevation.data(), map->elevation.size()); rd(in, map->elevation_masked.data(), map->elevation_masked.size());
  std::vector<State> path((size_t)hdr[2]);
  rd(in, path.data(), path.size());
  if (!in) { std::cerr << "short input\n"; return 2; }
  auto& r = params->robot;
  r.torso.length = robot[0]; r.torso.width = robot[1]; r.torso.height = robot[2];
  r.torso.offset.x = robot[3]; r.torso.offset.y = robot[4]; r.torso.offset.z = robot[5];
  r.feet.offset.x = robot[6]; r.feet.offset.y = robot[7]; r.feet.offset.z = robot[8];
  r.feet.reach.x = robot[9]; r.feet.reach.y = robot[10]; r.feet.reach.z = robot[11];
  params->planner.unknown_space_untraversable = hdr[3] != 0;
  auto& pl = params->objectives.custom_path_length;
  pl.use_directional_cost = hdr[4] != 0; pl.max_lon_vel = robot[12]; pl.max_lat_vel = robot[13]; pl.max_ang_vel = robot[14];
  auto checker = std::make_shared<StateValidityChecker>(params);
  checker->setMap(map);
  checker->updateHeightField();
  artp_se3_space sp{};
  for (int i = 0; i < 3; ++i) { sp.low[i] = space[i]; sp.high[i] = space[3 + i]; }
  sp.longest_valid_segment_fraction = space[6];
  // getObjective's PathLengthObjective (planner.cpp:27-35): the planners other than prm_motion_cost
  PathSimplifier ps(checker, sp, PathSimplifier::PATH_LENGTH, seed);
  const PathSimplifier::Result res = ps.getSolutionPath(path, true);
  const PathSimplifier::Result kept = ps.getSolutionPath(path, false);
  if (kept.path.size() != path.size()) { std::cerr << "simplify=false changed the path\n"; return 1; }
  std::ofstream out(argv[2], std::ios::binary);
  const uint64_t n = res.path.size();
  wr(out, &n, 1);
  wr(out, res.path.data(), res.path.size());
  wr(out, &res.info, 1);
  std::cout << "path " << path.size() << " -> " << n << " states\n";
  return 0;
}
