// tests/host_cpp/box_verdicts.cpp -- drives the box verdicts of the C++ host mirror (include/artp_host.hpp):
// StateValidityChecker::boxVerdicts and boxVerdictLayer after setMap, updateHeightField and estimateNormals.
//   box_verdicts --expect-no-gpu     : construction must fail loudly (no CPU fallback)
//   box_verdicts <in.bin> <out.bin>  : the words of the states and the layer at the yaw in in.bin
//                                      (see tests/test_box_verdicts_host_cpp.py)
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iostream>

#include "artp_host.hpp"

using namespace artp_host;

template <class T> static void rd(std::ifstream& f, T* p, size_t n) { f.read(reinterpret_cast<char*>(p), sizeof(T) * n); }

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
  int32_t hdr[3];      // rows, cols, number of states
  double geo[4];       // res, cx, cy, yaw
  rd(in, hdr, 3); rd(in, geo, 4);
  auto map = std::make_shared<Map>();
  map->rows = hdr[0]; map->cols = hdr[1]; map->resolution = geo[0]; map->position_x = geo[1]; map->position_y = geo[2];
  map->elevation.resize((size_t)hdr[0] * hdr[1]); map->elevation_masked.resize(map->elevation.size());
  rd(in, map->elevation.data(), map->elevation.size()); rd(in, map->elevation_masked.data(), map->elevation_masked.size());
  std::vector<State> states(hdr[2]);
  rd(in, &states[0].x, 7 * states.size());
  if (!in) { std::cerr << "short input\n"; return 2; }
  // art_planner_ros/config/params.yaml robot geometry
  params->robot.torso.length = 1.31; params->robot.torso.width = 0.65; params->robot.torso.height = 0.30;
  params->robot.torso.offset.z = 0.04;
  params->robot.feet.offset.x = 0.51; params->robot.feet.offset.y = 0.20; params->robot.feet.offset.z = -0.475;
  params->robot.feet.reach.x = 0.2; params->robot.feet.reach.y = 0.2; params->robot.feet.reach.z = 0.2;
  auto checker = std::make_shared<StateValidityChecker>(params);
  checker->setMap(map);
  checker->updateHeightField();
  checker->estimateNormals();
  const std::vector<uint16_t> why = checker->boxVerdicts(states);
  const std::vector<uint16_t> layer = checker->boxVerdictLayer(geo[3]);
  std::ofstream out(argv[2], std::ios::binary);
  out.write(reinterpret_cast<const char*>(why.data()), sizeof(uint16_t) * why.size());
  out.write(reinterpret_cast<const char*>(layer.data()), sizeof(uint16_t) * layer.size());
  return out ? 0 : 6;
}
