// art_planner_b200/csrc/artp_inpaint.cu -- inpaintMatrix on the device (artp_inpaint.cuh) behind the C ABI:
// artp_inpaint_layer (host buffers), artp_inpaint_layer_device (device buffers), and artp_api::inpaint_layer, the body
// artp_planner_set_map_raw runs on the layers it has uploaded.
#include <algorithm>

#include "artp_internal.h"
#include "artp_inpaint.cuh"

using namespace artp_api;
using namespace artp_inpaint;

namespace {

int inpaint_args(Handle* h, const void* in, int rows, int cols, const void* out) {
  if (!in || !out) return null_buffer(h);
  if (rows < 2 || cols < 2 || (size_t)rows * cols >= 0x7FFFFFFFull) {
    h->err = "inpaint: rows and cols must be >= 2 and rows * cols < 2^31"; return ARTP_E_INVALID;
  }
  return ARTP_OK;
}

}  // namespace

// The march on a layer whose finite min / max keys (finite_min_max) are at d_mm; stream-ordered scratch.
int artp_api::inpaint_layer(Handle* h, const float* d_in, int rows, int cols, const uint32_t* d_mm, float* d_out,
                            cudaStream_t s) {
  const size_t n = (size_t)rows * cols;
  const int H = cols, W = rows;
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
    TRY(launch(h, inp_prep_kernel, g, 256, 0, s, d_in, n, d_mm, img, flag));
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
    return launch(h, inp_finish_kernel, g, 256, 0, s, (const uint8_t*)img, rows, cols, d_mm, d_out);
  };
  rc = run();
  const cudaError_t fe = cudaFreeAsync(base, s);
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
  cudaStream_t s = h->stream;
  float *d_in = (float*)r[0], *d_out = (float*)r[1];
  uint32_t* d_mm = (uint32_t*)r[2];
  TRY(copy_async(h, d_in, layer, lb, cudaMemcpyHostToDevice, s));
  TRY(finite_min_max(h, d_in, n, d_mm, s));
  uint32_t mm[3];
  TRY(copy_async(h, mm, d_mm, sizeof(mm), cudaMemcpyDeviceToHost, s));
  TRY(sync_stream(h, s));
  if (!mm[2]) { host_call_end(h); h->err = "inpaint: the layer has no finite cell"; return ARTP_E_INVALID; }
  TRY(inpaint_layer(h, d_in, rows, cols, d_mm, d_out, s));
  TRY(copy_async(h, out, d_out, lb, cudaMemcpyDeviceToHost, s));
  return host_call_end(h);
}

int artp_inpaint_layer_device(artp_handle* hh, const float* d_layer, int rows, int cols, float* d_out, void* stream) {
  LOCK_CALL(h, hh);
  TRY(inpaint_args(h, d_layer, rows, cols, d_out));
  CU_TRY(h, cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  const size_t n = (size_t)rows * cols;
  uint32_t* d_mm = nullptr;
  CU_TRY(h, cudaMallocAsync(reinterpret_cast<void**>(&d_mm), 64, s));
  int rc = finite_min_max(h, d_layer, n, d_mm, s);
  uint32_t mm[3] = {0, 0, 0};
  if (rc == ARTP_OK) rc = copy_async(h, mm, d_mm, sizeof(mm), cudaMemcpyDeviceToHost, s);
  if (rc == ARTP_OK) rc = sync_stream(h, s);
  if (rc == ARTP_OK && !mm[2]) { h->err = "inpaint: the layer has no finite cell"; rc = ARTP_E_INVALID; }
  if (rc == ARTP_OK) rc = inpaint_layer(h, d_layer, rows, cols, d_mm, d_out, s);
  cudaFreeAsync(d_mm, s);
  return rc;
}

}  // extern "C"
