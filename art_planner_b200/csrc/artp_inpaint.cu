// art_planner_b200/csrc/artp_inpaint.cu -- inpaintMatrix on the device (artp_inpaint.cuh) behind the C ABI:
// artp_inpaint_layer (host buffers), artp_inpaint_layer_device (device buffers), and artp_api::inpaint_layer, the body
// artp_planner_set_map_raw runs on the layers it has uploaded. Beside it the cost server's preparation of the same raw
// layer over the same march: artp_cost_map_layer[_device], and artp_update_features_raw[_device], which runs the trunk on
// it (cost_map_features, also what artp_planner_set_map[_raw] run with cost_map_from_raw).
#include <algorithm>
#include <cmath>

#include "artp_internal.h"
#include "artp_inpaint.cuh"

using namespace artp_api;
using namespace artp_inpaint;

namespace {

int inpaint_args(Handle* h, const void* in, int rows, int cols, const void* out, const char* what = "inpaint") {
  if (!in || !out) return null_buffer(h);
  if (rows < 2 || cols < 2 || (size_t)rows * cols >= 0x7FFFFFFFull) {
    h->err = std::string(what) + ": rows and cols must be >= 2 and rows * cols < 2^31"; return ARTP_E_INVALID;
  }
  return ARTP_OK;
}

// artp_update_features_raw[_device]'s checks before any work: arguments, geometry, weights.
int features_raw_args(Handle* h, const float* raw, int rows, int cols, double res, double cx, double cy) {
  TRY(inpaint_args(h, raw, rows, cols, raw, "cost map"));
  if (!(res > 0) || !std::isfinite(cx) || !std::isfinite(cy)) { h->err = "bad map arguments"; return ARTP_E_INVALID; }
  return check_cost_weights(h);
}

// The stages from region to march (artp_inpaint.cuh) on the H x W image that prep(img, flag) fills, then finish(img);
// stream-ordered scratch.
template <class Prep, class Finish>
int march(Handle* h, int H, int W, cudaStream_t s, Prep prep, Finish finish) {
  const size_t n = (size_t)H * W;
  // Components: their regions are disjoint and each holds the clipped 7 x 7 square around one of its mask cells, so
  // there are at most n / (min(4, H) * min(4, W)) of them.
  const size_t max_comp = n / ((size_t)std::min(4, H) * std::min(4, W)) + 1;
  const size_t bytes[10] = {n /* img */, n /* flag */, n * 4 /* t */, n * 4 /* label */, n * 4 /* slot */,
                            max_comp * sizeof(Comp), max_comp * 4 /* order */, n * 8 /* heap keys */, n * 4 /* heap cells */,
                            512 /* counters */};
  size_t pos[10], end = 0;
  for (int i = 0; i < 10; ++i) { end = (end + 255) & ~(size_t)255; pos[i] = end; end += bytes[i]; }
  char* base = nullptr;
  CU_TRY(h, cudaMallocAsync(reinterpret_cast<void**>(&base), end, s));
  uint8_t* img = (uint8_t*)(base + pos[0]);
  uint8_t* flag = (uint8_t*)(base + pos[1]);
  float* t = (float*)(base + pos[2]);
  int* label = (int*)(base + pos[3]);
  int* slot = (int*)(base + pos[4]);
  Comp* comps = (Comp*)(base + pos[5]);
  int* order = (int*)(base + pos[6]);
  unsigned long long* key = (unsigned long long*)(base + pos[7]);
  int* cell = (int*)(base + pos[8]);
  int* cnt = (int*)(base + pos[9]);
  int rc = ARTP_OK;
  const unsigned g = grid_for(h, n, 256, 8);
  auto run = [&]() -> int {
    CU_TRY(h, cudaMemsetAsync(cnt, 0, bytes[9], s));
    TRY(prep(img, flag));
    TRY(launch(h, inp_region_kernel, g, 256, 0, s, H, W, flag, t, label));
    TRY(launch(h, inp_union_kernel, g, 256, 0, s, H, W, label));
    TRY(launch(h, inp_root_kernel, g, 256, 0, s, n, label, slot, comps, cnt));
    TRY(launch(h, inp_flatten_kernel, g, 256, 0, s, n, label));
    TRY(launch(h, inp_bbox_kernel, g, 256, 0, s, H, W, (const int*)label, (const int*)slot, comps));
    const unsigned gc = grid_for(h, max_comp, 256, 4);
    TRY(launch(h, inp_class_count_kernel, gc, 256, 0, s, (const Comp*)comps, cnt));
    TRY(launch(h, inp_class_scatter_kernel, gc, 256, 0, s, (const Comp*)comps, cnt, order));
    Grid gr{H, W, img, flag, t};
    TRY(launch(h, inp_march_kernel, (unsigned)h->sm_count * 8, 32 * kWarps, 0, s, gr, (const int*)label, (const Comp*)comps,
               (const int*)order, (const int*)cnt, cnt, key, cell));
    return finish((const uint8_t*)img);
  };
  rc = run();
  const cudaError_t fe = cudaFreeAsync(base, s);
  if (rc == ARTP_OK && fe != cudaSuccess) CU_TRY(h, fe);
  return rc;
}

// The body both forms of an entry point share, on s: scan the rows x cols layer d_in into the words at d_w (64 bytes of
// device memory), read them back (one synchronisation of s), then refuse the layer or run the work. A host-buffer call
// (host_call) ends (host_call_end) before it returns a refusal; on an error it returns at once.
int inpaint_body(Handle* h, const float* d_in, int rows, int cols, uint32_t* d_mm, float* d_out, cudaStream_t s,
                 bool host_call) {
  TRY(finite_min_max(h, d_in, (size_t)rows * cols, d_mm, s));
  uint32_t mm[3];
  TRY(copy_async(h, mm, d_mm, sizeof(mm), cudaMemcpyDeviceToHost, s));
  TRY(sync_stream(h, s));
  if (!mm[2]) { if (host_call) host_call_end(h); h->err = "inpaint: the layer has no finite cell"; return ARTP_E_INVALID; }
  return inpaint_layer(h, d_in, rows, cols, d_mm, d_out, s);
}

// The cost-map pairs' scan, read-back and verdict (cost_map_verdict) into w.
int cost_map_check(Handle* h, const float* d_in, int rows, int cols, uint32_t* d_w, uint32_t (&w)[kCostMapWords],
                   cudaStream_t s, bool host_call) {
  TRY(cost_map_scan(h, d_in, (size_t)rows * cols, d_w, s));
  TRY(copy_async(h, w, d_w, sizeof(w), cudaMemcpyDeviceToHost, s));
  TRY(sync_stream(h, s));
  const int rc = cost_map_verdict(h, w);
  if (rc && host_call) host_call_end(h);
  return rc;
}

int cost_map_body(Handle* h, const float* d_in, int rows, int cols, uint32_t* d_w, float* d_out, cudaStream_t s,
                  bool host_call) {
  uint32_t w[kCostMapWords];
  TRY(cost_map_check(h, d_in, rows, cols, d_w, w, s, host_call));
  return cost_map_layer(h, d_in, rows, cols, d_w, w[3] != 0, false, d_out, s);
}

int features_raw_body(Handle* h, const float* d_in, int rows, int cols, uint32_t* d_w, double res, double cx, double cy,
                      cudaStream_t s, bool host_call) {
  uint32_t w[kCostMapWords];
  TRY(cost_map_check(h, d_in, rows, cols, d_w, w, s, host_call));
  return cost_map_features(h, d_in, rows, cols, d_w, w[3] != 0, res, cx, cy, s);
}

}  // namespace

// The march on a layer whose finite min / max keys (finite_min_max) are at d_mm, on the cols x rows image.
int artp_api::inpaint_layer(Handle* h, const float* d_in, int rows, int cols, const uint32_t* d_mm, float* d_out,
                            cudaStream_t s) {
  const size_t n = (size_t)rows * cols;
  const unsigned g = grid_for(h, n, 256, 8);
  return march(h, cols, rows, s,
               [&](uint8_t* img, uint8_t* flag) { return launch(h, inp_prep_kernel, g, 256, 0, s, d_in, n, d_mm, img, flag); },
               [&](const uint8_t* img) { return launch(h, inp_finish_kernel, g, 256, 0, s, img, rows, cols, d_mm, d_out); });
}

int artp_api::cost_map_scan(Handle* h, const float* d_in, size_t n, uint32_t* d_w, cudaStream_t s) {
  TRY(finite_min_max(h, d_in, n, d_w, s));
  return nonfinite_any(h, d_in, n, d_w + 3, s);
}

int artp_api::cost_map_verdict(Handle* h, const uint32_t* w) {
  if (w[4]) { h->err = "cost map: the layer has a +-inf cell"; return ARTP_E_INVALID; }
  if (!w[2]) { h->err = "cost map: the layer has no finite cell"; return ARTP_E_INVALID; }
  if (!w[3]) return ARTP_OK;   // no hole: the layer itself
  const float mn = key_float(w[0]), d = key_float(w[1]) - mn;
  if (!std::isfinite(d * 255.0f)) { h->err = "cost map: the finite range times 255 overflows float"; return ARTP_E_INVALID; }
  return ARTP_OK;
}

int artp_api::cost_map_layer(Handle* h, const float* d_in, int rows, int cols, const uint32_t* d_w, bool holes,
                             bool reverse_cols, float* d_out, cudaStream_t s) {
  const size_t n = (size_t)rows * cols;
  const unsigned g = grid_for(h, n, 256, 8);
  if (!holes) return launch(h, cm_finish_kernel, g, 256, 0, s, (const uint8_t*)nullptr, d_in, rows, cols, d_w, reverse_cols, d_out);
  return march(h, rows, cols, s,
               [&](uint8_t* img, uint8_t* flag) { return launch(h, cm_prep_kernel, g, 256, 0, s, d_in, rows, cols, d_w, img, flag); },
               [&](const uint8_t* img) {
                 return launch(h, cm_finish_kernel, g, 256, 0, s, img, d_in, rows, cols, d_w, reverse_cols, d_out);
               });
}

int artp_api::cost_map_features(Handle* h, const float* d_in, int rows, int cols, const uint32_t* d_w, bool holes,
                                double res, double cx, double cy, cudaStream_t s) {
  float* d_map = nullptr;
  CU_TRY(h, cudaMallocAsync(reinterpret_cast<void**>(&d_map), (size_t)rows * cols * sizeof(float), s));
  int rc = cost_map_layer(h, d_in, rows, cols, d_w, holes, true, d_map, s);
  if (rc == ARTP_OK)
    rc = update_features(h, d_map, rows, cols, rows, res, cx, cy, s);
  const cudaError_t fe = cudaFreeAsync(d_map, s);
  if (rc == ARTP_OK && fe != cudaSuccess) CU_TRY(h, fe);
  return rc;
}

extern "C" {

int artp_inpaint_layer(artp_handle* hh, const float* layer, int rows, int cols, float* out) {
  LOCK_CALL(h, hh);
  TRY(inpaint_args(h, layer, rows, cols, out));
  const size_t n = (size_t)rows * cols, lb = n * sizeof(float);
  char* r[3];
  TRY(host_call_begin(h, {lb, lb, 64}, r));
  float *d_in = (float*)r[0], *d_out = (float*)r[1];
  TRY(copy_async(h, d_in, layer, lb, cudaMemcpyHostToDevice, h->stream));
  TRY(inpaint_body(h, d_in, rows, cols, (uint32_t*)r[2], d_out, h->stream, true));
  TRY(copy_async(h, out, d_out, lb, cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h);
}

int artp_inpaint_layer_device(artp_handle* hh, const float* d_layer, int rows, int cols, float* d_out, void* stream) {
  LOCK_CALL(h, hh);
  TRY(inpaint_args(h, d_layer, rows, cols, d_out));
  CU_TRY(h, cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  uint32_t* d_mm = nullptr;
  CU_TRY(h, cudaMallocAsync(reinterpret_cast<void**>(&d_mm), 64, s));
  const int rc = inpaint_body(h, d_layer, rows, cols, d_mm, d_out, s, false);
  cudaFreeAsync(d_mm, s);
  return rc;
}

int artp_cost_map_layer(artp_handle* hh, const float* raw, int rows, int cols, float* out) {
  LOCK_CALL(h, hh);
  TRY(inpaint_args(h, raw, rows, cols, out, "cost map"));
  const size_t n = (size_t)rows * cols, lb = n * sizeof(float);
  char* r[3];
  TRY(host_call_begin(h, {lb, lb, 64}, r));
  float *d_in = (float*)r[0], *d_out = (float*)r[1];
  TRY(copy_async(h, d_in, raw, lb, cudaMemcpyHostToDevice, h->stream));
  TRY(cost_map_body(h, d_in, rows, cols, (uint32_t*)r[2], d_out, h->stream, true));
  TRY(copy_async(h, out, d_out, lb, cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h);
}

int artp_cost_map_layer_device(artp_handle* hh, const float* d_raw, int rows, int cols, float* d_out, void* stream) {
  LOCK_CALL(h, hh);
  TRY(inpaint_args(h, d_raw, rows, cols, d_out, "cost map"));
  CU_TRY(h, cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  uint32_t* d_w = nullptr;
  CU_TRY(h, cudaMallocAsync(reinterpret_cast<void**>(&d_w), 64, s));
  const int rc = cost_map_body(h, d_raw, rows, cols, d_w, d_out, s, false);
  cudaFreeAsync(d_w, s);
  return rc;
}

int artp_update_features_raw(artp_handle* hh, const float* raw, int rows, int cols, double res, double cx, double cy) {
  LOCK_CALL(h, hh);
  TRY(features_raw_args(h, raw, rows, cols, res, cx, cy));
  const size_t n = (size_t)rows * cols, lb = n * sizeof(float);
  char* r[2];
  TRY(host_call_begin(h, {lb, 64}, r));
  float* d_in = (float*)r[0];
  TRY(copy_async(h, d_in, raw, lb, cudaMemcpyHostToDevice, h->stream));
  TRY(features_raw_body(h, d_in, rows, cols, (uint32_t*)r[1], res, cx, cy, h->stream, true));
  return host_call_end(h);
}

int artp_update_features_raw_device(artp_handle* hh, const float* d_raw, int rows, int cols, double res, double cx,
                                    double cy, void* stream) {
  LOCK_CALL(h, hh);
  TRY(features_raw_args(h, d_raw, rows, cols, res, cx, cy));
  CU_TRY(h, cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  uint32_t* d_w = nullptr;
  CU_TRY(h, cudaMallocAsync(reinterpret_cast<void**>(&d_w), 64, s));
  const int rc = features_raw_body(h, d_raw, rows, cols, d_w, res, cx, cy, s, false);
  cudaFreeAsync(d_w, s);
  return rc;
}

}  // extern "C"
