// tests/host_cpp/planner.cpp -- drives the C++ host mirror's Planner (include/artp_host.hpp) the way
// PlannerRos::updateMapAndPlanFromCurrentRobotPose replans: setMap, then plan and getSolutionPath.
//   planner --expect-no-gpu     : construction must fail loudly (no CPU fallback)
//   planner <in.bin> <out.bin>  : one replan of the map and query in in.bin (see tests/test_planner_host_cpp.py); the
//                                 path and the info to out.bin
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
      Planner planner(c);
    } catch (const std::runtime_error& e) {
      std::cout << "failed loudly: " << e.what() << "\n";
      return 0;
    }
    std::cout << "a handle was created: a CUDA device is present\n";
    return 3;
  }
  if (argc != 3) { std::cerr << "usage\n"; return 2; }
  std::ifstream in(argv[1], std::ios::binary);
  int32_t hdr[2];              // rows, cols
  double geo[3];               // res, cx, cy
  double robot[12];            // torso l w h, torso offset xyz, feet offset xyz, reach xyz
  artp_planner_params pp{};
  double query[14];            // start, goal
  rd(in, hdr, 2); rd(in, geo, 3); rd(in, robot, 12); rd(in, &pp, 1); rd(in, query, 14);
  const size_t n = (size_t)hdr[0] * hdr[1];
  std::vector<float> e(n), t(n), ei(n), ti(n);
  rd(in, e.data(), n); rd(in, t.data(), n); rd(in, ei.data(), n); rd(in, ti.data(), n);
  std::vector<float> blob;
  uint64_t nb = 0;
  rd(in, &nb, 1);
  blob.resize(nb);
  rd(in, blob.data(), nb);
  if (!in) { std::cerr << "short input\n"; return 2; }
  auto& r = params->robot;
  r.torso.length = robot[0]; r.torso.width = robot[1]; r.torso.height = robot[2];
  r.torso.offset.x = robot[3]; r.torso.offset.y = robot[4]; r.torso.offset.z = robot[5];
  r.feet.offset.x = robot[6]; r.feet.offset.y = robot[7]; r.feet.offset.z = robot[8];
  r.feet.reach.x = robot[9]; r.feet.reach.y = robot[10]; r.feet.reach.z = robot[11];
  params->planner.prm_motion_cost.risk_threshold = 0.6f;
  auto checker = std::make_shared<StateValidityChecker>(params);
  checker->handle()->check(artp_set_cost_weights(checker->handle()->get(), blob.data(), blob.size()), "artp_set_cost_weights");
  Planner planner(checker);
  planner.parameters() = pp;
  Map map;
  map.rows = hdr[0]; map.cols = hdr[1]; map.resolution = geo[0]; map.position_x = geo[1]; map.position_y = geo[2];
  planner.setMap(map, e, t, ei, ti);
  State start, goal;
  std::memcpy(&start.x, query, 7 * sizeof(double));
  std::memcpy(&goal.x, query + 7, 7 * sizeof(double));
  const PlannerStatus status = planner.plan(start, goal);
  std::vector<State> path;
  if (status == SOLVED) path = planner.getSolutionPath();
  else {
    try { planner.getSolutionPath(); std::cerr << "an unsolved plan returned a path\n"; return 1; } catch (const std::runtime_error&) {}
  }
  std::ofstream out(argv[2], std::ios::binary);
  const uint64_t np = path.size();
  wr(out, &np, 1);
  wr(out, path.data(), path.size());
  wr(out, &planner.info(), 1);
  std::cout << "status " << status << ", " << np << " states\n";
  return 0;
}
