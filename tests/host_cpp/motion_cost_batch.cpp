// tests/host_cpp/motion_cost_batch.cpp -- the C++ host mirror's batched learned edge cost against its per-edge form:
// MotionCostObjective::motionCostBatch / pathCost (one device call) next to motionCost (one functor call per edge).
//   motion_cost_batch <in.bin> <out.bin>   (see tests/test_motion_cost_split_gpu.py for the layout)
#include <fstream>
#include <iostream>

#include "artp_host.hpp"

using namespace artp_host;

template <class T> static void rd(std::ifstream& f, T* p, size_t n) { f.read(reinterpret_cast<char*>(p), sizeof(T) * n); }
template <class T> static void wr(std::ofstream& f, const T* p, size_t n) { f.write(reinterpret_cast<const char*>(p), sizeof(T) * n); }

int main(int argc, char** argv) {
  if (argc != 3) { std::cerr << "usage: motion_cost_batch <in.bin> <out.bin>\n"; return 2; }
  std::ifstream in(argv[1], std::ios::binary);
  int32_t hdr[5];   // rows, cols, n_edges, n_path, n_weights
  double geo[4];    // res, cx, cy, risk_threshold
  rd(in, hdr, 5); rd(in, geo, 4);
  auto map = std::make_shared<Map>();
  map->rows = hdr[0]; map->cols = hdr[1]; map->resolution = geo[0]; map->position_x = geo[1]; map->position_y = geo[2];
  map->elevation.resize((size_t)hdr[0] * hdr[1]); map->elevation_masked.resize(map->elevation.size());
  rd(in, map->elevation.data(), map->elevation.size()); rd(in, map->elevation_masked.data(), map->elevation_masked.size());
  std::vector<State> s1(hdr[2]), s2(hdr[2]), path(hdr[3]);
  rd(in, s1.data(), s1.size()); rd(in, s2.data(), s2.size()); rd(in, path.data(), path.size());
  std::vector<float> blob(hdr[4]);
  rd(in, blob.data(), blob.size());
  if (!in) { std::cerr << "short input\n"; return 2; }

  auto params = std::make_shared<Params>();
  params->planner.prm_motion_cost.risk_threshold = static_cast<float>(geo[3]);
  auto checker = std::make_shared<StateValidityChecker>(params);
  checker->setMap(map);
  checker->updateHeightField();
  MotionCostObjective obj(checker);
  obj.setWeights(blob);
  obj.updateFeatures();

  std::vector<double> single(s1.size()), batch, seg(path.size() > 1 ? path.size() - 1 : 0);
  for (size_t e = 0; e < s1.size(); ++e) single[e] = obj.motionCost(&s1[e], &s2[e]);
  obj.motionCostBatch(s1, s2, &batch);
  for (size_t i = 0; i < seg.size(); ++i) seg[i] = obj.motionCost(&path[i], &path[i + 1]);
  const double path_cost = obj.pathCost(path);
  const double short_paths[2] = {obj.pathCost(std::vector<State>(path.begin(), path.begin() + 1)), obj.pathCost({})};

  // a caller-supplied functor stays the only cost source: the batch goes through it once per edge
  uint64_t functor_calls = 0;
  HandlePtr h = checker->handle();
  std::unique_ptr<MotionCostObjective::MotionCostFunc> func(new MotionCostObjective::MotionCostFunc(
      [h, &functor_calls](const EdgeMatrix& edges, EdgeMatrix* costs) {
        ++functor_calls;
        costs->resize(edges.rows(), 3);
        return artp_motion_cost(h->get(), edges.data(), edges.rows(), costs->data()) == ARTP_OK;
      }));
  MotionCostObjective custom(checker, std::move(func));
  std::vector<double> custom_batch;
  custom.motionCostBatch(s1, s2, &custom_batch);

  std::ofstream out(argv[2], std::ios::binary);
  wr(out, single.data(), single.size()); wr(out, batch.data(), batch.size()); wr(out, seg.data(), seg.size());
  wr(out, &path_cost, 1); wr(out, short_paths, 2);
  wr(out, custom_batch.data(), custom_batch.size()); wr(out, &functor_calls, 1);
  std::cout << "ok " << s1.size() << " edges, path of " << path.size() << " states\n";
  return 0;
}
