// tests/host_cpp/inpaint.cpp -- drives the C++ host mirror's inpaintMatrix and raw-layer Planner::setMap
// (include/artp_host.hpp) the way processors::Basic and PlannerRos::updateMapAndPlanFromCurrentRobotPose use them.
//   inpaint --expect-no-gpu     : construction must fail loudly (no CPU fallback)
//   inpaint <in.bin> <out.bin>  : in.bin holds the map, the robot, the planner parameters, one query, the raw elevation
//                                 and traversability and the weights (see tests/test_inpaint_host_cpp.py); out.bin gets
//                                 inpaintMatrix of both layers, then the path and info of one replan after the raw setMap
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
      inpaintMatrix(*c->handle(), std::vector<float>(4, 1.0f), 2, 2);
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
  std::vector<float> e(n), t(n);
  rd(in, e.data(), n); rd(in, t.data(), n);
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
  const std::vector<float> ei = inpaintMatrix(*checker->handle(), e, hdr[0], hdr[1]);
  const std::vector<float> ti = inpaintMatrix(*checker->handle(), t, hdr[0], hdr[1]);
  Planner planner(checker);
  planner.parameters() = pp;
  Map map;
  map.rows = hdr[0]; map.cols = hdr[1]; map.resolution = geo[0]; map.position_x = geo[1]; map.position_y = geo[2];
  planner.setMap(map, e, t);
  State start, goal;
  std::memcpy(&start.x, query, 7 * sizeof(double));
  std::memcpy(&goal.x, query + 7, 7 * sizeof(double));
  const PlannerStatus status = planner.plan(start, goal);
  std::vector<State> path;
  if (status == SOLVED) path = planner.getSolutionPath();
  std::ofstream out(argv[2], std::ios::binary);
  wr(out, ei.data(), n);
  wr(out, ti.data(), n);
  const uint64_t np = path.size();
  wr(out, &np, 1);
  wr(out, path.data(), path.size());
  wr(out, &planner.info(), 1);
  wr(out, &planner.mapInfo(), 1);
  std::cout << "status " << status << ", " << np << " states\n";
  return 0;
}
