// art_planner_b200/csrc/artp_capi.cu -- C ABI (include/artp.h) over the sm_90a kernels.
// Host side mirrors the reference's checker objects: artp_create ~ StateValidityChecker ctor,
// artp_set_map ~ setMap + updateHeightField (HeightMapBoxChecker::setHeightField,
// art_planner/src/validity_checker/height_map_box_checker.cpp:38-54), artp_check_* ~ isValid / checkMotion.
// No CPU fallback: every entry point fails with ARTP_E_CUDA if the device or the kernel image is unusable.
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cassert>
#include <climits>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <initializer_list>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/artp.h"
#include "artp_cnn.h"
#include "artp_kernels.cuh"
#include "artp_tiles.cuh"
#include "artp_sampler.cuh"
#include "artp_basic.cuh"
#include "artp_distribution.cuh"

namespace {

thread_local std::string g_create_error;
constexpr int kMaxSlices = 9;   // H2D slices per host-fed round: at most 8 scheduled fractions and the remainder

// One box queue: the classify stage appends records up to `end`, the queue's box kernel claims them from `claim`.
struct QueueCtr { uint32_t end, claim; };
// The three box queues of a round (Handle::d_ctr), or the entries one slice of a host-fed round appended (Handle::d_slices).
// One 32-byte sector each: the box kernels of consecutive slices claim from their records at the same time.
struct alignas(32) BoxQueues { QueueCtr big, reach, group; };
// Per-handle device counters: the round's queues, the boxes deferred to the grouping stage, and the sampler's CDF check.
struct Counters { BoxQueues q; uint32_t defer, scratch; };

struct Handle {
  artp_params p;
  int device = 0;
  int sm_count = 0;
  artp::Checker chk;
  float* d_H[2] = {nullptr, nullptr};
  float2* d_T[2][artp::kMaxLevel + 1] = {};
  uint32_t* d_C[2][artp::kMaxLevel + 1] = {};    // compact conservative copies of d_T (Field::C)
  int pitch = 0;
  int rows = 0, cols = 0;           // full map
  int win_row0 = 0, win_rows = 0;   // rows held by this handle (artp_set_map_window); whole map: 0, rows
  bool has_map = false;
  Counters* d_ctr = nullptr;
  uint32_t* d_defer = nullptr;      // deferred record list (bit 31: reach-box queue)
  artp::BoxRec* d_recs = nullptr;   // classify -> warp-stage box queue (torso boxes, reach boxes of unusual size)
  artp::BoxRec* d_recs_f = nullptr; // classify -> reach-box queue (one warp per box: zones with -inf or mergeable planes)
  artp::BoxRec* d_recs_g = nullptr; // classify -> reach-box queue of the 8-lane-group kernel (all-finite, merge-free zones)
  int group_grid = 0, group_smem = 0;
  size_t recs_cap = 0;
  uint32_t* d_block_counts = nullptr;
  size_t block_counts_cap = 0;
  char* d_stage = nullptr;          // device staging for the host-buffer API
  size_t stage_cap = 0;
  cudaStream_t stream = nullptr;    // internal compute stream for the host-buffer API
  cudaStream_t copy_stream = nullptr;   // H2D slices of the host-buffer API
  cudaStream_t group_stream = nullptr;  // the 8-lane-group kernel of slice i (host-fed rounds), beside the other box kernels
  cudaEvent_t group_ev = nullptr;
  cudaStream_t box_stream = nullptr;    // box stages of slice i, concurrent with the copy + classify of slice i + 1
  cudaEvent_t copy_ev[kMaxSlices] = {};    // H2D of slice i landed (the call's stream waits on it)
  cudaEvent_t slice_ev[kMaxSlices] = {};   // classify of slice i done (box_stream waits on it)
  cudaEvent_t box_ev = nullptr;            // box stages of a round done (stream waits on it)
  BoxQueues* d_slices = nullptr;           // per slice of a host-fed round: its share of the three queues
  int k2_grid = 0, k2_smem = 0, k2_tcap = 0;
  // stage B (artp_tiles.cuh): [0] big tiles (torso queue, 4 warps per CTA), [1] small tiles (reach-box queue, 8 warps)
  artp::TileCfg tile_cfg[2] = {};
  int tile_grid[2] = {0, 0}, tile_smem[2] = {0, 0}, tile_warps[2] = {8, 8};
  CUtensorMap tile_map[2][2];       // [cfg][layer]: 2-D tile maps over elevation / elevation_masked
  int mode = 0;
  artp_cnn::State* cnn = nullptr;
  int cnn_mode = 0;
  // sampler (artp_set_sampler): device copies of the per-cell layers, scratch of the fused sample->check->compact path
  artp::SamplerDev samp{};
  float* d_samp_layers = nullptr;   // normal_x | normal_y | normal_z | std_dev | cum_prob | cum_row
  size_t samp_layers_cap = 0;       // floats
  bool has_sampler = false;
  bool has_device_normals = false;  // artp_estimate_normals filled normal_x/y/z/std_dev of d_samp_layers for this map
  bool has_device_cdf = false;      // artp_compute_sample_cdf filled cum_prob / cum_row of d_samp_layers for this map
  bool has_normals = false;         // normal_x/y/z of d_samp_layers hold this map's normals (device-estimated or the caller's)
  char* d_samp_scratch = nullptr;
  size_t samp_scratch_cap = 0;
  double res = 0.0;                 // map resolution as artp_set_map received it
  // sampling distribution (artp_distribution.cuh): the layers artp_set_sample_filter keeps for this map ...
  float* d_dist_layers = nullptr;   // traversability_sample_filter | observed
  size_t dist_layers_cap = 0;       // floats
  bool has_sample_filter = false, has_dist_observed = false;
  char* d_dist_scratch = nullptr;   // n_samples | blur pass | sample_probability | cap row sums | words (artp_update_sample_distribution)
  size_t dist_scratch_cap = 0;
  // ... and the layers of the last artp_process_basic, its NULL-layer inputs
  float* d_basic_keep = nullptr;    // observed | traversability_thresholded
  size_t basic_keep_cap = 0;        // floats
  int basic_rows = 0, basic_cols = 0;
  bool has_basic_layers = false, has_basic_observed = false;
  uint8_t* h_small_out = nullptr;   // mapped pinned host bytes the latency-path kernel writes its verdicts to
  int timing = 0;
  cudaEvent_t ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};   // classify | warp | reach vertex | reach plane | group
  bool ev_valid = false;
  bool deferred_unread = false;
  // Cross-stream ordering of the per-handle scratch (ADVICE r1): calls may come on different streams; every call that
  // uses a scratch group first makes its stream wait for the previous user of that group, and records an event after.
  // group 0: d_ctr / d_recs / d_defer / d_stage / d_samp_scratch (check, sampler);  group 1: d_block_counts (compaction)
  cudaEvent_t chain_ev[2] = {nullptr, nullptr};
  cudaStream_t chain_stream[2] = {nullptr, nullptr};
  bool chain_busy[2] = {false, false};
  // Sticky error word in mapped pinned host memory: the plane-grouping stage sets it when a zone does not fit its
  // shared-memory store (the item is then marked INVALID -- fail closed). Host-buffer calls return ARTP_E_LIMIT from the
  // call that caused it; device-buffer (asynchronous) calls surface it through artp_poll_error().
  uint32_t* h_err = nullptr;        // host view
  uint32_t* d_err = nullptr;        // device view of the same word
  int tcap_override = 0;            // test hook (artp_debug_set_group_capacity)
  artp_stats stats{};
  std::string err;
  std::recursive_mutex mtx;   // recursive: host-buffer entry points hold it across their nested *_device call
};

#define CU_TRY(h, expr)                                                                          \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) {                                                                     \
      (h)->err = std::string(#expr) + ": " + cudaGetErrorString(_e);                             \
      return ARTP_E_CUDA;                                                                        \
    }                                                                                            \
  } while (0)

// Opens an entry point that takes a handle: a null handle is ARTP_E_INVALID; otherwise `h` is the handle, and its lock is
// held until the entry point returns, across staging copies and nested *_device calls (the mutex is recursive).
#define LOCK_HANDLE(h, hh)                                                                       \
  if (!(hh)) return ARTP_E_INVALID;                                                              \
  Handle* h = reinterpret_cast<Handle*>(hh);                                                     \
  std::lock_guard<std::recursive_mutex> h##_lock(h->mtx)

// H[x + z*nx] = layer[x + (nz-1-z)*nx] (+0.0f canonicalises -0 like GetHeight's (h*scale)+offset,
// ode/ode/src/heightfield.cpp:383).
__global__ void reverse_columns_kernel(const float* __restrict__ layer, float* __restrict__ H, int nx, int nz, int pitch) {
  const size_t total = (size_t)pitch * nz;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int z = (int)(i / pitch), x = (int)(i - (size_t)z * pitch);
    H[i] = (x < nx) ? layer[x + (size_t)(nz - 1 - z) * nx] * 1.0f + 0.0f : 0.0f;   // pad columns are never read
  }
}

// Range-table level k from level k-1 (level 0 = the heights themselves): reduction over the 2^k x 2^k window
// starting at (x,z) = op of the four 2^(k-1) windows at offsets {0,half} (clamped at the border; clamped windows
// are never queried). (max over all h, min over finite h or +inf, any non-finite).
__global__ void build_level_kernel(const float* __restrict__ H, const float2* __restrict__ prevT,
                                   const unsigned char* __restrict__ prevNF, const unsigned char* __restrict__ mergeable,
                                   float2* __restrict__ T, unsigned char* __restrict__ NF, int nx, int nz, int pitch, int half) {
  const size_t total = (size_t)pitch * nz;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int z = (int)(i / pitch), x = (int)(i - (size_t)z * pitch);
    if (x >= nx) { T[i] = make_float2(0.f, 0.f); NF[i] = 0; continue; }
    const int x2 = min(x + half, nx - 1), z2 = min(z + half, nz - 1);
    const size_t id[4] = {(size_t)z * pitch + x, (size_t)z * pitch + x2, (size_t)z2 * pitch + x, (size_t)z2 * pitch + x2};
    float mx = -CUDART_INF_F, mn = CUDART_INF_F;
    unsigned char nf = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if (prevT) {
        const float2 v = prevT[id[q]];
        mx = fmaxf(mx, v.x); mn = fminf(mn, v.y); nf |= prevNF[id[q]];
      } else {
        const float h = H[id[q]];
        mx = fmaxf(mx, h);
        if (fabsf(h) < CUDART_INF_F) mn = fminf(mn, h); else nf |= 1;
        nf |= mergeable[id[q]];      // 0 or 2: the cell starting at this vertex holds a mergeable triangle
      }
    }
    T[i] = make_float2(mx, mn);
    NF[i] = nf;
  }
}

// Compact table level from T and the window flags NF (encoding at artp::Field::C): maxCode = the smallest code c >= 1 with
// dec(c) >= max, minCode = the largest c with dec(c) <= min, both found by bisection over the non-decreasing dec(). A height
// the codes cannot cover (above dec(kCodeMax)) takes the reserved code kCodeNone, which sends its zones to the exact tables.
__global__ void build_codes_kernel(const float2* __restrict__ T, const unsigned char* __restrict__ NF, uint32_t* __restrict__ C,
                                   size_t n, float base, float step) {
  const float top = artp::code_dec(base, step, artp::kCodeMax);
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float2 v = T[i];
    uint32_t cM = 0, cm = artp::kCodeNone;
    if (v.x > top) cM = artp::kCodeNone;
    else if (v.x > -CUDART_INF_F) {
      uint32_t lo = 1, hi = artp::kCodeMax;
      while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (artp::code_dec(base, step, mid) >= v.x) hi = mid; else lo = mid + 1;
      }
      cM = lo;
    }
    if (v.y <= top) {
      uint32_t lo = 0, hi = artp::kCodeMax;
      while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (artp::code_dec(base, step, mid) <= v.y) lo = mid; else hi = mid - 1;
      }
      cm = lo;
    }
    C[i] = artp::code_word(cM, cm, NF[i] & 3u);
  }
}

// Encoding of the compact tables of one layer: base = the smallest finite height, step = the smallest power of two
// with dec(kCodeMax) >= the largest finite height (checked with the device's own dec()).
void code_scale(const float* layer, size_t n, float& base, float& step) {
  float lo = HUGE_VALF, hi = -HUGE_VALF;
  for (size_t i = 0; i < n; ++i) {
    const float v = layer[i] * 1.0f + 0.0f;   // the stored height (reverse_columns_kernel)
    if (std::fabs(v) < HUGE_VALF) { lo = std::min(lo, v); hi = std::max(hi, v); }
  }
  base = lo <= hi ? lo : 0.0f;
  int e = -126;
  while (e < 127 && artp::code_dec(base, std::ldexp(1.0f, e), artp::kCodeMax) < hi) ++e;
  step = std::ldexp(1.0f, e);
}

// ---------------------------------------------------------------------------------------------------------------
// Plane tables: which cells hold a triangle whose plane equals (within eps, the greedy grouping's test,
// heightfield.cpp:1541-1546) the plane of ANOTHER triangle of the layer? A zone without such a cell cannot merge
// anything: every kept triangle is its own plane group whatever the box, and the warp stage skips its merge screen.
// All triangle planes (exact, the collider's arithmetic) go into a hash table keyed by their (n0, n2, d) buckets; a
// second pass looks every triangle's +-2 eps neighbour buckets up. Natural terrain flags nothing; flat or terraced
// maps flag almost everything and keep the screen / the exact grouping stage.
struct PlaneSlot { unsigned long long key; uint32_t lo, hi; };
constexpr unsigned long long kEmptyKey = ~0ull;
__device__ __forceinline__ unsigned long long plane_key(int kx, int kz, int kd) {
  return ((unsigned long long)(uint32_t)(kx & 0xffff) << 48) | ((unsigned long long)(uint32_t)(kz & 0xffff) << 32) | (uint32_t)kd;
}
__device__ __forceinline__ uint32_t plane_slot_hash(unsigned long long k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
  return (uint32_t)k;
}
__global__ void plane_table_clear_kernel(PlaneSlot* tab, size_t cap) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < cap; i += (size_t)gridDim.x * blockDim.x) {
    tab[i].key = kEmptyKey; tab[i].lo = 0xffffffffu; tab[i].hi = 0u;
  }
}
// Exact plane of triangle u of cell (x, z), or false if one of its vertices is not finite (never kept).
__device__ __forceinline__ bool cell_tri_plane(const artp::Field& f, int x, int x_off, int z, int u, float pl[4]) {
  float hA, hB, hC, hD;
  artp::load_cell(f, x, z, hA, hB, hC, hD);
  const bool ok = u == 0 ? (artp::finitef(hA) && artp::finitef(hB) && artp::finitef(hC))
                         : (artp::finitef(hD) && artp::finitef(hB) && artp::finitef(hC));
  if (!ok) return false;
  artp::cell_plane(f, u == 0, x + x_off, z, hA, hB, hC, hD, pl);   // vertex coordinates are those of the full map
  return true;
}
__global__ void plane_table_insert_kernel(const artp::Field f, int x_off, PlaneSlot* tab, uint32_t mask) {
  const size_t ncell = (size_t)(f.nx - 1) * (f.nz - 1);
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < 2 * ncell; i += (size_t)gridDim.x * blockDim.x) {
    const size_t c = i >> 1;
    const int u = (int)(i & 1), z = (int)(c / (f.nx - 1)), x = (int)(c - (size_t)z * (f.nx - 1));
    float pl[4];
    if (!cell_tri_plane(f, x, x_off, z, u, pl)) continue;
    const uint32_t id = (uint32_t)(((size_t)z * f.pitch + x) * 2 + u);
    const unsigned long long key = plane_key((int)floorf((pl[0] + 1.0f) * artp::kKeyScale), (int)floorf((pl[2] + 1.0f) * artp::kKeyScale),
                                             artp::dkey(pl[3]));
    uint32_t s = plane_slot_hash(key) & mask;
    for (;;) {
      const unsigned long long old = atomicCAS(&tab[s].key, kEmptyKey, key);
      if (old == kEmptyKey || old == key) {
        // (lo, hi) only has to tell "one triangle" from "several": skip the atomics once id lies strictly inside
        if (!(tab[s].lo < id && tab[s].hi > id)) { atomicMin(&tab[s].lo, id); atomicMax(&tab[s].hi, id); }
        break;
      }
      s = (s + 1) & mask;
    }
  }
}
__global__ void plane_table_query_kernel(const artp::Field f, int x_off, const PlaneSlot* __restrict__ tab, uint32_t mask,
                                         unsigned char* __restrict__ mergeable) {
  const size_t ncell = (size_t)(f.nx - 1) * (f.nz - 1);
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < 2 * ncell; i += (size_t)gridDim.x * blockDim.x) {
    const size_t c = i >> 1;
    const int u = (int)(i & 1), z = (int)(c / (f.nx - 1)), x = (int)(c - (size_t)z * (f.nx - 1));
    float pl[4];
    if (!cell_tri_plane(f, x, x_off, z, u, pl)) continue;
    const uint32_t id = (uint32_t)(((size_t)z * f.pitch + x) * 2 + u);
    const float e2 = 2.0f * ARTP_EPS;
    const int kx0 = (int)floorf((pl[0] - e2 + 1.0f) * artp::kKeyScale), kx1 = (int)floorf((pl[0] + e2 + 1.0f) * artp::kKeyScale);
    const int kz0 = (int)floorf((pl[2] - e2 + 1.0f) * artp::kKeyScale), kz1 = (int)floorf((pl[2] + e2 + 1.0f) * artp::kKeyScale);
    const int kd0 = artp::dkey(pl[3] - e2), kd1 = artp::dkey(pl[3] + e2);
    bool dup = false;
    for (int kx = kx0; kx <= kx1 && !dup; ++kx)
      for (int kz = kz0; kz <= kz1 && !dup; ++kz)
        for (int kd = kd0; kd <= kd1 && !dup; ++kd) {
          const unsigned long long key = plane_key(kx, kz, kd);
          uint32_t s = plane_slot_hash(key) & mask;
          for (;;) {
            const unsigned long long k = tab[s].key;
            if (k == kEmptyKey) break;
            if (k == key) { dup = tab[s].lo != id || tab[s].hi != id; break; }
            s = (s + 1) & mask;
          }
        }
    if (dup) mergeable[(size_t)z * f.pitch + x] = 2;   // races write the same value
  }
}

__global__ void fill_u8_kernel(uint8_t* p, size_t n, uint8_t v) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}

// PathLengthObjective::motionCost (art_planner/src/objectives/path_length_objective.cpp:26-70), double.
__global__ void path_length_kernel(const double* __restrict__ s1, const double* __restrict__ s2, size_t n,
                                   double* __restrict__ cost, int directional, double v_lon, double v_lat,
                                   double v_ang) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const double* a = s1 + 7 * i;
    const double* b = s2 + 7 * i;
    const double x_dif = b[0] - a[0], y_dif = b[1] - a[1], z_dif = b[2] - a[2];
    if (!directional) {
      cost[i] = sqrt(x_dif * x_dif + y_dif * y_dif + z_dif * z_dif) / v_lon;
      continue;
    }
    // getYawFromSO3 returns `Scalar` = float (utils.h:80-88)
    const double yaw1 = (double)(float)atan2(2 * (a[6] * a[5] + a[3] * a[4]), 1 - 2 * (a[4] * a[4] + a[5] * a[5]));
    const double yaw2 = (double)(float)atan2(2 * (b[6] * b[5] + b[3] * b[4]), 1 - 2 * (b[4] * b[4] + b[5] * b[5]));
    const double d = fabs(yaw1 - yaw2);
    const double yaw_dif = (d > 3.14159265358979323846) ? 2.0 * 3.14159265358979323846 - d : d;
    const double lon_dif = cos(yaw1) * x_dif + sin(yaw1) * y_dif;
    const double lat_dif = -sin(yaw1) * x_dif + cos(yaw1) * y_dif;
    const double t_yaw = fabs(yaw_dif) / v_ang, t_lon = fabs(lon_dif) / v_lon, t_lat = fabs(lat_dif) / v_lat;
    const double m = t_lon > t_lat ? t_lon : t_lat;
    cost[i] = m > t_yaw ? m : t_yaw;
  }
}

// Ordered compaction: (A) per-block counts, (B) single-block exclusive scan, (C) scatter.
constexpr int kCompactBlock = 1024;
// BITS: the mask is bit-packed (item i = bit i&31 of word i>>5, artp_pack_valid_bits_device), else one byte per item.
template <bool BITS>
__device__ __forceinline__ int mask_at(const uint8_t* __restrict__ valid, size_t i) {
  if (BITS) return (int)((reinterpret_cast<const uint32_t*>(valid)[i >> 5] >> (i & 31)) & 1u);
  return valid[i] != 0;
}
template <bool BITS>
__global__ void compact_count_kernel(const uint8_t* __restrict__ valid, size_t n, uint32_t* __restrict__ counts) {
  const size_t i = (size_t)blockIdx.x * kCompactBlock + threadIdx.x;
  const int v = (i < n) && mask_at<BITS>(valid, i);
  const int c = __syncthreads_count(v);
  if (threadIdx.x == 0) counts[blockIdx.x] = (uint32_t)c;
}
__global__ void compact_scan_kernel(uint32_t* counts, size_t nb, uint32_t* total) {
  __shared__ uint32_t carry;
  __shared__ uint32_t wsum[32];
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (size_t b0 = 0; b0 < nb; b0 += blockDim.x) {
    const size_t i = b0 + threadIdx.x;
    const uint32_t v = i < nb ? counts[i] : 0u;
    uint32_t x = v;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) wsum[wid] = x;
    __syncthreads();
    if (wid == 0) {
      uint32_t s = lane < (int)(blockDim.x >> 5) ? wsum[lane] : 0u;
      for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += y; }
      wsum[lane] = s;
    }
    __syncthreads();
    const uint32_t before = carry + (wid ? wsum[wid - 1] : 0u) + x - v;
    if (i < nb) counts[i] = before;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) carry = before + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = carry;
}
template <bool BITS, typename IndexT>
__global__ void compact_scatter_kernel(const uint8_t* __restrict__ valid, size_t n, int64_t base,
                                       const uint32_t* __restrict__ offsets, IndexT* __restrict__ out) {
  __shared__ uint32_t wsum[32];
  const size_t i = (size_t)blockIdx.x * kCompactBlock + threadIdx.x;
  const int v = (i < n) && mask_at<BITS>(valid, i);
  const unsigned bal = __ballot_sync(0xffffffffu, v);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) wsum[wid] = __popc(bal);
  __syncthreads();
  if (wid == 0) {
    uint32_t s = wsum[lane];
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += y; }
    wsum[lane] = s;
  }
  __syncthreads();
  if (v) {
    const uint32_t pos = offsets[blockIdx.x] + (wid ? wsum[wid - 1] : 0u) + __popc(bal & ((1u << lane) - 1u));
    out[pos] = (IndexT)(base + (int64_t)i);
  }
}

// bits[w] bit b = valid[32*w + b] != 0; one warp ballot per word, tail bits zero.
__global__ void pack_bits_kernel(const uint8_t* __restrict__ valid, size_t n, uint32_t* __restrict__ bits) {
  const size_t words = (n + 31) / 32;
  const size_t warps = ((size_t)gridDim.x * blockDim.x) >> 5, wid = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  for (size_t w = wid; w < words; w += warps) {
    const size_t i = w * 32 + lane;
    const unsigned bal = __ballot_sync(0xffffffffu, i < n && valid[i] != 0);
    if (lane == 0) bits[w] = bal;
  }
}

constexpr size_t kChunkItems = 1u << 20;   // work items per internal launch round (bounds the box queue)

// Grow a per-handle device buffer to hold `count` elements (cap counts them too); the contents are not kept. Rare (growth
// only): the device is synchronised before the free, because a call on any stream may still read the old buffer.
template <typename T>
int grow(Handle* h, T*& buf, size_t& cap, size_t count) {
  if (cap >= count) return ARTP_OK;
  CU_TRY(h, cudaDeviceSynchronize());
  cudaFree(buf);
  buf = nullptr;
  cap = 0;
  CU_TRY(h, cudaMalloc(&buf, count * sizeof(T)));
  cap = count;
  return ARTP_OK;
}

int ensure_queues(Handle* h, size_t n_items) {
  const size_t need = 5 * std::min(n_items, kChunkItems);
  if (h->recs_cap >= need) return ARTP_OK;
  const size_t cap = std::max<size_t>(need, 1u << 16);
  h->recs_cap = 0;   // the four queues share it: set once all four have grown
  size_t had[4] = {0, 0, 0, 0};
  int rc;
  if ((rc = grow(h, h->d_recs, had[0], cap)) || (rc = grow(h, h->d_recs_f, had[1], cap)) ||
      (rc = grow(h, h->d_recs_g, had[2], cap)) || (rc = grow(h, h->d_defer, had[3], cap)))
    return rc;
  h->recs_cap = cap;
  return ARTP_OK;
}

// Scratch-group ordering across streams (see Handle::chain_ev).
int chain_begin(Handle* h, int g, cudaStream_t s) {
  if (h->chain_busy[g] && h->chain_stream[g] != s) CU_TRY(h, cudaStreamWaitEvent(s, h->chain_ev[g], 0));
  return ARTP_OK;
}
int chain_end(Handle* h, int g, cudaStream_t s) {
  CU_TRY(h, cudaEventRecord(h->chain_ev[g], s));
  h->chain_stream[g] = s;
  h->chain_busy[g] = true;
  return ARTP_OK;
}
struct ChainScope {   // begin on construction, end on destruction (every return path)
  Handle* h; int g; cudaStream_t s; int rc;
  ChainScope(Handle* h_, int g_, cudaStream_t s_) : h(h_), g(g_), s(s_), rc(chain_begin(h_, g_, s_)) {}
  ~ChainScope() { if (rc == ARTP_OK) chain_end(h, g, s); }
};

// Sticky plane-grouping overflow (set by the device, see Handle::h_err): read and clear.
int take_sticky_error(Handle* h) {
  if (h->h_err && *(volatile uint32_t*)h->h_err) {
    const uint32_t e = *(volatile uint32_t*)h->h_err;
    *(volatile uint32_t*)h->h_err = 0;
    if (e & 2u) {
      h->err = "a box reached outside this handle's map window (artp_set_map_window: route samples to the shard that holds them, "
               "halo >= box half-diagonal + offsets); affected poses were marked invalid";
      return ARTP_E_WINDOW;
    }
    h->err = "plane-grouping stage overflow: a zone exceeded its shared-memory store; affected poses were marked invalid";
    return ARTP_E_LIMIT;
  }
  return ARTP_OK;
}

// Host-buffer calls run on h->stream as users of scratch group 0. host_call_begin waits for the group's previous user and
// hands out region[i] = bytes[i] bytes of d_stage at a 256-byte boundary (d_stage is grown for all of them first: growth
// reallocates it). host_call_end waits for the call's work, after which the group is idle. For a call that ran the validity
// pipeline (`pipeline`) it then returns the sticky device error (Handle::h_err) of the call; the verdicts are complete
// (fail closed) then, so only ARTP_E_CUDA from host_call_end means the call's outputs are not there.
int host_call_begin(Handle* h, std::initializer_list<size_t> bytes = {}, char** region = nullptr) {
  CU_TRY(h, cudaSetDevice(h->device));
  int rc = chain_begin(h, 0, h->stream);
  if (rc) return rc;
  size_t end = 0;
  for (size_t b : bytes) end = ((end + 255) & ~(size_t)255) + b;
  if ((rc = grow(h, h->d_stage, h->stage_cap, end))) return rc;
  end = 0;
  for (size_t b : bytes) {
    end = (end + 255) & ~(size_t)255;
    *region++ = h->d_stage + end;
    end += b;
  }
  return ARTP_OK;
}
int host_call_end(Handle* h, bool pipeline = false) {
  CU_TRY(h, cudaStreamSynchronize(h->stream));
  h->chain_busy[0] = false;
  return pipeline ? take_sticky_error(h) : ARTP_OK;
}

// Host feed of a call: the states are copied H2D in slices on the copy stream while the kernels of the previous slice run.
struct HostFeed {
  const char* host;        // host states
  char* dev;               // device destination (same layout)
  size_t bytes_per_item;
  size_t slice_items;      // rounds up to this size run unsliced; equal slices of this size below kScheduleItems
  // Slice schedule of a round as fractions (0-terminated): a small first slice so that the kernels start early, then equal
  // ones. Every slice costs its kernels' latency floors (~0.1 ms of chain per slice, profiles/stage_vs_n.py), which is why
  // five or six slices beat both fewer (long tail after the last byte) and more, and why shrinking the last slices below
  // ~15 % buys nothing.
  float schedule[8];
};
constexpr size_t kScheduleItems = 1u << 18;   // rounds from this size on are cut by the schedule
// Host-fed rounds cap the grids of the two per-slice reach kernels at two CTAs per SM each: the box kernels are persistent
// and fill the SMs, so without the cap the next slice's classify crawls in the leftover registers.
constexpr int kPipeReachCtasPerSm = 2;

// Slice i of a piped round is closed: its box stages consume the queue entries [end of slice i-1, current end).
__global__ void close_slice_kernel(const BoxQueues* round, BoxQueues* slices, int i) {
  const BoxQueues prev = i ? slices[i - 1] : BoxQueues{};
  slices[i].group = {round->group.end, prev.group.end};   // the claim counter starts at the slice's begin
  slices[i].reach = {round->reach.end, prev.reach.end};
  slices[i].big = {round->big.end, prev.big.end};
}

// Stage launchers shared by both rounds. Each launches its kernels over the items [lo, hi) and counts them in
// stats.kernel_launches.
int launch_classify(Handle* h, artp::Work w, size_t lo, size_t hi, cudaStream_t s) {
  w.item_base = (uint32_t)lo;
  w.n_items = (uint32_t)hi;
  BoxQueues* q = &h->d_ctr->q;   // every round appends to the round's queues
  artp::classify_items_kernel<<<(unsigned)((hi - lo + artp::kClassifyItems - 1) / artp::kClassifyItems), artp::kClassifyItems, 0, s>>>(
      h->chk, w, h->d_recs, h->d_recs_f, h->group_grid ? h->d_recs_g : nullptr, &q->big.end, &q->reach.end, &q->group.end,
      h->mode == 1);
  CU_TRY(h, cudaGetLastError());
  h->stats.kernel_launches += 1;
  return ARTP_OK;
}

// The box kernels over the queue entries q, one launcher per queue: the big-tile queue, and the two reach-box queues (one
// warp per box; 8-lane groups), which exist only for some box sizes. reach_cap caps the grids of the two reach kernels.
int launch_big_tile(Handle* h, artp::Work w, size_t lo, size_t hi, BoxQueues* q, cudaStream_t s) {
  w.item_base = (uint32_t)lo;
  w.n_items = (uint32_t)hi;
  const int wpc = h->tile_warps[0];   // no more CTAs than there can be boxes: up to five big-tile boxes per item
  const unsigned grid = (unsigned)std::min<size_t>((size_t)h->tile_grid[0], (5 * (hi - lo) + wpc - 1) / wpc);
  artp::box_tiles_warp_kernel<<<grid, wpc * 32, h->tile_smem[0], s>>>(h->chk, h->tile_map[0][0], h->tile_map[0][1], h->tile_cfg[0], w,
                                                                     h->d_recs, &q->big.end, &q->big.claim, &h->d_ctr->defer,
                                                                     h->d_defer, 0u, h->mode == 1);
  CU_TRY(h, cudaGetLastError());
  h->stats.kernel_launches += 1;
  return ARTP_OK;
}
int launch_reach_warp(Handle* h, artp::Work w, size_t lo, size_t hi, BoxQueues* q, cudaStream_t s, unsigned reach_cap) {
  if (!h->chk.reach_tw) return ARTP_OK;
  w.item_base = (uint32_t)lo;
  w.n_items = (uint32_t)hi;
  const int wpc = h->tile_warps[1];
  const unsigned grid = (unsigned)std::min<size_t>({(size_t)h->tile_grid[1], (4 * (hi - lo) + wpc - 1) / wpc, reach_cap});
  artp::box_tiles_warp_kernel<<<grid, wpc * 32, h->tile_smem[1], s>>>(h->chk, h->tile_map[1][1], h->tile_map[1][1], h->tile_cfg[1], w,
                                                                     h->d_recs_f, &q->reach.end, &q->reach.claim, &h->d_ctr->defer,
                                                                     h->d_defer, artp::kDeferReachBit, h->mode == 1);
  CU_TRY(h, cudaGetLastError());
  h->stats.kernel_launches += 1;
  return ARTP_OK;
}
int launch_reach_groups(Handle* h, artp::Work w, size_t lo, size_t hi, BoxQueues* q, cudaStream_t s, unsigned reach_cap) {
  if (!h->group_grid) return ARTP_OK;
  w.item_base = (uint32_t)lo;
  w.n_items = (uint32_t)hi;
  const unsigned grid = (unsigned)std::min<size_t>({(size_t)h->group_grid, (hi - lo + 7) / 8, reach_cap});
  artp::reach_groups_kernel<<<grid, artp::kMaxTileWarps * 32, h->group_smem, s>>>(h->chk, h->tile_map[1][1], h->tile_cfg[1], w,
                                                                                 h->d_recs_g, &q->group.end, &q->group.claim);
  CU_TRY(h, cudaGetLastError());
  h->stats.kernel_launches += 1;
  return ARTP_OK;
}

// The plane-grouping stage over every box the round [lo, hi) deferred.
int launch_grouping(Handle* h, artp::Work w, size_t lo, size_t hi, cudaStream_t s) {
  w.item_base = (uint32_t)lo;
  w.n_items = (uint32_t)hi;
  const unsigned grid = (unsigned)std::min<size_t>((size_t)h->k2_grid, 5 * (hi - lo));
  artp::box_items_block_kernel<<<grid, artp::kBlockStageThreads, h->k2_smem, s>>>(h->chk, w, h->d_recs, h->d_recs_f, &h->d_ctr->defer,
                                                                                  h->d_defer, h->k2_tcap, h->d_err);
  CU_TRY(h, cudaGetLastError());
  h->stats.kernel_launches += 1;
  return ARTP_OK;
}

// Device round: the items [base, end) are on the device. Classify, the three box kernels, then the grouping stage. The box
// kernels only ever clear verdicts of different boxes, so the two reach kernels fork onto box_stream / group_stream after
// the classify stage and join before the grouping stage (each kernel has a latency floor of 20-30 us). With stage timing
// on, everything runs in order on s, and a timed round records the per-stage events.
int run_round_device(Handle* h, const artp::Work& w, cudaStream_t s, size_t base, size_t end, bool timed) {
  CU_TRY(h, cudaMemsetAsync(h->d_ctr, 0, sizeof(Counters), s));
  if (timed) CU_TRY(h, cudaEventRecord(h->ev[0], s));
  int rc = launch_classify(h, w, base, end, s);
  if (rc) return rc;
  if (timed) CU_TRY(h, cudaEventRecord(h->ev[1], s));
  const bool fork = !h->timing && h->chk.reach_tw;
  if (fork) {
    CU_TRY(h, cudaEventRecord(h->slice_ev[0], s));
    CU_TRY(h, cudaStreamWaitEvent(h->box_stream, h->slice_ev[0], 0));
    if (h->group_grid) CU_TRY(h, cudaStreamWaitEvent(h->group_stream, h->slice_ev[0], 0));
  }
  BoxQueues* q = &h->d_ctr->q;
  if ((rc = launch_big_tile(h, w, base, end, q, s))) return rc;
  if (timed) CU_TRY(h, cudaEventRecord(h->ev[2], s));
  if ((rc = launch_reach_warp(h, w, base, end, q, fork ? h->box_stream : s, UINT_MAX))) return rc;
  if (timed) CU_TRY(h, cudaEventRecord(h->ev[3], s));
  if ((rc = launch_reach_groups(h, w, base, end, q, fork ? h->group_stream : s, UINT_MAX))) return rc;
  if (fork) {
    CU_TRY(h, cudaEventRecord(h->box_ev, h->box_stream));
    CU_TRY(h, cudaStreamWaitEvent(s, h->box_ev, 0));
    if (h->group_grid) {
      CU_TRY(h, cudaEventRecord(h->group_ev, h->group_stream));
      CU_TRY(h, cudaStreamWaitEvent(s, h->group_ev, 0));
    }
  }
  if (timed) CU_TRY(h, cudaEventRecord(h->ev[4], s));
  rc = launch_grouping(h, w, base, end, s);
  if (rc) return rc;
  if (timed) { CU_TRY(h, cudaEventRecord(h->ev[5], s)); h->ev_valid = true; }
  return ARTP_OK;
}

// Host-fed round (the host-buffer entry points): the states arrive in slices over PCIe. Four streams:
//   copy_stream    H2D of slice i+1
//   s              classify of slice i as soon as its copy has landed (appends to the three box queues)
//   box_stream     one-warp-per-box kernels of slice i (reach-box queue, then big-tile queue) over exactly the queue entries
//                  its classify appended (per-slice claim counters, close_slice_kernel), then the grouping stage once per round
//   group_stream   the 8-lane-group kernel of slice i, beside them
// so the copy, the classify stage and the box stages of consecutive slices overlap; s waits for box_stream at the end.
int run_round_piped(Handle* h, const artp::Work& w, cudaStream_t s, const HostFeed& feed, size_t base, size_t end) {
  size_t cut[kMaxSlices + 1];
  int ncut = 0;
  cut[0] = base;
  if (end - base >= kScheduleItems) {
    double acc = 0.0;
    for (int i = 0; i < 8 && feed.schedule[i] > 0.0f; ++i) {
      acc += feed.schedule[i];
      const size_t c = std::min(end, (base + (size_t)((double)(end - base) * acc) + 127) & ~(size_t)127);
      if (c > cut[ncut]) cut[++ncut] = c;
    }
    if (cut[ncut] != end) cut[++ncut] = end;
  } else {
    for (size_t lo = base; lo < end; lo += feed.slice_items) cut[++ncut] = std::min(end, lo + feed.slice_items);
  }
  assert(ncut <= kMaxSlices);
  CU_TRY(h, cudaMemsetAsync(h->d_ctr, 0, sizeof(Counters), s));
  const unsigned reach_cap = (unsigned)(kPipeReachCtasPerSm * h->sm_count);
  for (int si = 0; si < ncut; ++si) {
    const size_t lo = cut[si], hi = cut[si + 1];
    CU_TRY(h, cudaMemcpyAsync(feed.dev + lo * feed.bytes_per_item, feed.host + lo * feed.bytes_per_item,
                              (hi - lo) * feed.bytes_per_item, cudaMemcpyHostToDevice, h->copy_stream));
    CU_TRY(h, cudaEventRecord(h->copy_ev[si], h->copy_stream));
    CU_TRY(h, cudaStreamWaitEvent(s, h->copy_ev[si], 0));
    int rc = launch_classify(h, w, lo, hi, s);
    if (rc) return rc;
    close_slice_kernel<<<1, 1, 0, s>>>(&h->d_ctr->q, h->d_slices, si);
    CU_TRY(h, cudaGetLastError());
    h->stats.kernel_launches += 1;
    CU_TRY(h, cudaEventRecord(h->slice_ev[si], s));
    CU_TRY(h, cudaStreamWaitEvent(h->box_stream, h->slice_ev[si], 0));
    if (h->group_grid) CU_TRY(h, cudaStreamWaitEvent(h->group_stream, h->slice_ev[si], 0));
    // the big-tile queue (torso boxes: few) of this slice behind its reach-box queue: issued ahead of the reach kernels,
    // it made host-fed calls 2-4 % slower (H100 80GB HBM3, 400 W power limit)
    if ((rc = launch_reach_groups(h, w, lo, hi, h->d_slices + si, h->group_stream, reach_cap))) return rc;
    if ((rc = launch_reach_warp(h, w, lo, hi, h->d_slices + si, h->box_stream, reach_cap))) return rc;
    if ((rc = launch_big_tile(h, w, lo, hi, h->d_slices + si, h->box_stream))) return rc;
  }
  if (h->group_grid) {
    // the grouping stage (box_stream) runs last: the group kernels must not clear a verdict after it has been copied out
    CU_TRY(h, cudaEventRecord(h->group_ev, h->group_stream));
    CU_TRY(h, cudaStreamWaitEvent(h->box_stream, h->group_ev, 0));
  }
  int rc = launch_grouping(h, w, base, end, h->box_stream);
  if (rc) return rc;
  CU_TRY(h, cudaEventRecord(h->box_ev, h->box_stream));
  CU_TRY(h, cudaStreamWaitEvent(s, h->box_ev, 0));
  return ARTP_OK;
}

// Launch the pipeline for a prepared Work (items 0 .. w.n_items = the whole call) on stream s, in rounds of kChunkItems
// work items (bounds the box queues). With a host feed, a round larger than one slice is piped; any other round (and
// every round while stage timing is on) has its states copied on s and runs as a device round.
int run_items(Handle* h, artp::Work w, cudaStream_t s, const HostFeed* feed = nullptr) {
  const size_t n_total = w.n_items;
  int rc = ensure_queues(h, n_total);
  if (rc) return rc;
  const uint64_t launches0 = h->stats.kernel_launches;
  for (size_t base = 0; base < n_total; base += kChunkItems) {
    const size_t end = std::min(n_total, base + kChunkItems);
    if (feed && feed->slice_items < end - base && !h->timing) {
      rc = run_round_piped(h, w, s, *feed, base, end);
    } else {
      if (feed)
        CU_TRY(h, cudaMemcpyAsync(feed->dev + base * feed->bytes_per_item, feed->host + base * feed->bytes_per_item,
                                  (end - base) * feed->bytes_per_item, cudaMemcpyHostToDevice, s));
      rc = run_round_device(h, w, s, base, end, h->timing && end == n_total);
    }
    if (rc) return rc;
  }
  h->stats.last_launches = (uint32_t)(h->stats.kernel_launches - launches0);
  h->deferred_unread = true;
  return ARTP_OK;
}

int check_common(Handle* h, size_t n) {
  if (!h->has_map) { h->err = "no map set"; return ARTP_E_NOMAP; }
  if (n >= (size_t)0xFFFFFFF0u) { h->err = "too many items for one call"; return ARTP_E_LIMIT; }
  return ARTP_OK;
}

// Latency path for n <= kSmallBatch host states (doubles): one launch, verdicts through mapped host memory.
int check_poses_small(Handle* h, const artp::SmallBatch& sb, size_t n, uint8_t* valid, int steps = -1) {
  int rc = host_call_begin(h);
  if (rc) return rc;
  if (!h->h_small_out) {
    CU_TRY(h, cudaHostAlloc((void**)&h->h_small_out, 64, cudaHostAllocMapped));
    CU_TRY(h, cudaFuncSetAttribute(artp::pose_small_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  }
  uint8_t* d_out = nullptr;
  CU_TRY(h, cudaHostGetDevicePointer((void**)&d_out, h->h_small_out, 0));
  artp::pose_small_kernel<<<(unsigned)n, 256, h->k2_smem, h->stream>>>(h->chk, sb, d_out, h->k2_tcap, h->d_err,
                                                                        h->mode == 1, steps);
  CU_TRY(h, cudaGetLastError());
  rc = host_call_end(h, true);
  if (rc == ARTP_E_CUDA) return rc;
  if (steps < 0) {
    std::memcpy(valid, h->h_small_out, n);
  } else {   // n = edges * (steps + 1) state verdicts -> one flag per edge
    const size_t per = (size_t)steps + 1;
    for (size_t e = 0; e < n / per; ++e) {
      uint8_t ok = 1;
      for (size_t j = 0; j < per; ++j) ok &= h->h_small_out[e * per + j];
      valid[e] = ok;
    }
  }
  h->stats.kernel_launches += 1;
  h->stats.last_launches = 1;
  h->stats.poses_checked += n;
  h->ev_valid = false;
  return rc;
}

// The pose entry points. T is double, or float: the caller has already applied the double -> float cast that
// Pose3FromSE3 (utils.h:25-38) performs first, so the result is identical to the double entry point while the H2D stream
// is 28 B/pose instead of 56. With on_device, states and valid are device buffers and the call is asynchronous on stream;
// otherwise they are host buffers: up to kSmallBatch states take the latency path, more are fed to the device in slices.
template <typename T>
int check_poses(artp_handle* hh, const T* states, size_t n, uint8_t* valid, bool on_device, cudaStream_t stream) {
  LOCK_HANDLE(h, hh);
  int rc = check_common(h, n);
  if (rc) return rc;
  if (n == 0) return ARTP_OK;
  if (!states || !valid) { h->err = "null buffer"; return ARTP_E_INVALID; }
  auto work = [n](const T* d_states, uint8_t* d_valid) {
    artp::Work w;
    w.s1 = nullptr; w.s2 = nullptr; w.s2f = nullptr; w.valid = d_valid; w.item_base = 0; w.n_items = (uint32_t)n;
    w.steps = 0; w.edge_mode = 0;
    if constexpr (std::is_same_v<T, float>) w.s2f = d_states; else w.s2 = d_states;
    return w;
  };
  if (on_device) {
    CU_TRY(h, cudaSetDevice(h->device));
    ChainScope cs(h, 0, stream);
    if (cs.rc) return cs.rc;
    rc = run_items(h, work(states, valid), stream);
    if (rc) return rc;
    h->stats.poses_checked += n;
    return ARTP_OK;
  }
  if (n <= (size_t)artp::kSmallBatch && !h->timing) {
    artp::SmallBatch sb;
    for (size_t i = 0; i < n * 7; ++i) (&sb.s[0][0])[i] = (double)states[i];   // exact; a float state is cast back in the kernel
    return check_poses_small(h, sb, n, valid);
  }
  char* r[2];
  if ((rc = host_call_begin(h, {n * 7 * sizeof(T), n}, r))) return rc;
  const HostFeed feed = std::is_same_v<T, float>
                            ? HostFeed{(const char*)states, r[0], 7 * sizeof(T), 256 * 1024, {0.08f, 0.17f, 0.25f, 0.25f, 0.25f}}
                            : HostFeed{(const char*)states, r[0], 7 * sizeof(T), 128 * 1024, {0.06f, 0.14f, 0.20f, 0.20f, 0.20f, 0.20f}};
  rc = run_items(h, work((const T*)r[0], (uint8_t*)r[1]), h->stream, &feed);
  if (rc) return rc;
  CU_TRY(h, cudaMemcpyAsync(valid, r[1], n, cudaMemcpyDeviceToHost, h->stream));
  h->stats.poses_checked += n;
  return host_call_end(h, true);
}

}  // namespace

extern "C" {

const char* artp_version(void) { return "artp 0.1 sm_90a"; }

const char* artp_last_error(const artp_handle* hh) {
  if (!hh) return g_create_error.c_str();
  return reinterpret_cast<const Handle*>(hh)->err.c_str();
}

int artp_create(const artp_params* params, artp_handle** out) {
  if (!params || !out) { g_create_error = "null argument"; return ARTP_E_INVALID; }
  *out = nullptr;
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    g_create_error = std::string("no CUDA device: ") + cudaGetErrorString(e);
    return ARTP_E_CUDA;
  }
  if (params->device < 0 || params->device >= ndev) { g_create_error = "bad device ordinal"; return ARTP_E_INVALID; }
  if (!(params->torso_length > 0 && params->torso_width > 0 && params->torso_height > 0 && params->reach_x > 0 &&
        params->reach_y > 0 && params->reach_z > 0)) {
    g_create_error = "box dimensions must be positive";
    return ARTP_E_INVALID;
  }
  Handle* h = new Handle();
  h->p = *params;
  h->device = params->device;
  auto fail = [&](const char* what, cudaError_t ce) {
    g_create_error = std::string(what) + ": " + cudaGetErrorString(ce);
    artp_destroy(reinterpret_cast<artp_handle*>(h));   // releases whatever was created before the failing call
    return ARTP_E_CUDA;
  };
  if ((e = cudaSetDevice(h->device)) != cudaSuccess) return fail("cudaSetDevice", e);
  cudaDeviceProp prop;
  if ((e = cudaGetDeviceProperties(&prop, h->device)) != cudaSuccess) return fail("cudaGetDeviceProperties", e);
  h->sm_count = prop.multiProcessorCount;
  cudaFuncAttributes fa;
  if ((e = cudaFuncGetAttributes(&fa, artp::box_tiles_warp_kernel)) != cudaSuccess)
    return fail("no usable kernel image (built for sm_90a)", e);
  for (cudaStream_t* st : {&h->stream, &h->copy_stream, &h->box_stream, &h->group_stream})
    if ((e = cudaStreamCreateWithFlags(st, cudaStreamNonBlocking)) != cudaSuccess) return fail("cudaStreamCreate", e);
  if ((e = cudaEventCreateWithFlags(&h->group_ev, cudaEventDisableTiming)) != cudaSuccess) return fail("cudaEventCreate", e);
  for (int i = 0; i < kMaxSlices; ++i) {
    if ((e = cudaEventCreateWithFlags(&h->copy_ev[i], cudaEventDisableTiming)) != cudaSuccess) return fail("cudaEventCreate", e);
    if ((e = cudaEventCreateWithFlags(&h->slice_ev[i], cudaEventDisableTiming)) != cudaSuccess) return fail("cudaEventCreate", e);
  }
  if ((e = cudaEventCreateWithFlags(&h->box_ev, cudaEventDisableTiming)) != cudaSuccess) return fail("cudaEventCreate", e);
  if ((e = cudaMalloc(&h->d_slices, kMaxSlices * sizeof(BoxQueues))) != cudaSuccess) return fail("cudaMalloc", e);
  if ((e = cudaMalloc(&h->d_ctr, sizeof(Counters))) != cudaSuccess) return fail("cudaMalloc", e);
  for (int g = 0; g < 2; ++g)
    if ((e = cudaEventCreateWithFlags(&h->chain_ev[g], cudaEventDisableTiming)) != cudaSuccess) return fail("cudaEventCreate", e);
  if ((e = cudaHostAlloc((void**)&h->h_err, 64, cudaHostAllocMapped)) != cudaSuccess) return fail("cudaHostAlloc", e);
  *h->h_err = 0;
  if ((e = cudaHostGetDevicePointer((void**)&h->d_err, h->h_err, 0)) != cudaSuccess) return fail("cudaHostGetDevicePointer", e);
  h->cnn = artp_cnn::create(h->device, h->sm_count);
  // checker constants (float casts as the reference's ctor/Pose3FromXYZ arguments make them)
  artp::Checker& c = h->chk;
  std::memset(&c, 0, sizeof(c));
  c.side[0][0] = (float)params->torso_length; c.side[0][1] = (float)params->torso_width; c.side[0][2] = (float)params->torso_height;
  c.side[1][0] = (float)params->reach_x; c.side[1][1] = (float)params->reach_y; c.side[1][2] = (float)params->reach_z;
  c.torso_off[0] = (float)params->torso_off_x; c.torso_off[1] = (float)params->torso_off_y;
  c.torso_off[2] = (float)(params->torso_off_z - params->feet_off_z);
  c.feet_ox = (float)params->feet_off_x; c.feet_oy = (float)params->feet_off_y;
  c.unknown_untraversable = params->unknown_space_untraversable ? 1 : 0;
  *out = reinterpret_cast<artp_handle*>(h);
  return ARTP_OK;
}

void artp_destroy(artp_handle* hh) {
  if (!hh) return;
  Handle* h = reinterpret_cast<Handle*>(hh);
  cudaSetDevice(h->device);
  if (h->stream) { cudaStreamSynchronize(h->stream); cudaStreamDestroy(h->stream); }
  if (h->copy_stream) { cudaStreamSynchronize(h->copy_stream); cudaStreamDestroy(h->copy_stream); }
  if (h->box_stream) { cudaStreamSynchronize(h->box_stream); cudaStreamDestroy(h->box_stream); }
  if (h->group_stream) { cudaStreamSynchronize(h->group_stream); cudaStreamDestroy(h->group_stream); }
  if (h->group_ev) cudaEventDestroy(h->group_ev);
  for (int i = 0; i < kMaxSlices; ++i) {
    if (h->copy_ev[i]) cudaEventDestroy(h->copy_ev[i]);
    if (h->slice_ev[i]) cudaEventDestroy(h->slice_ev[i]);
  }
  if (h->box_ev) cudaEventDestroy(h->box_ev);
  cudaFree(h->d_slices);
  for (int k = 0; k < 2; ++k) for (int l = 0; l <= artp::kMaxLevel; ++l) { cudaFree(h->d_T[k][l]); cudaFree(h->d_C[k][l]); }
  cudaFree(h->d_H[0]); cudaFree(h->d_H[1]); cudaFree(h->d_ctr); cudaFree(h->d_defer); cudaFree(h->d_stage);
  cudaFree(h->d_block_counts); cudaFree(h->d_recs); cudaFree(h->d_recs_f); cudaFree(h->d_recs_g); cudaFree(h->d_samp_layers); cudaFree(h->d_samp_scratch);
  cudaFree(h->d_dist_layers); cudaFree(h->d_dist_scratch); cudaFree(h->d_basic_keep);
  if (h->h_small_out) cudaFreeHost(h->h_small_out);
  if (h->h_err) cudaFreeHost(h->h_err);
  for (int g = 0; g < 2; ++g) if (h->chain_ev[g]) cudaEventDestroy(h->chain_ev[g]);
  artp_cnn::destroy(h->cnn);
  for (int i = 0; i < 6; ++i) if (h->ev[i]) cudaEventDestroy(h->ev[i]);
  delete h;
}

int artp_has_map(const artp_handle* hh) { return hh && reinterpret_cast<const Handle*>(hh)->has_map ? 1 : 0; }

int artp_set_mode(artp_handle* hh, int mode) {
  if (!hh || mode < 0 || mode > 1) return ARTP_E_INVALID;
  reinterpret_cast<Handle*>(hh)->mode = mode;
  return ARTP_OK;
}

int artp_set_timing(artp_handle* hh, int enable) {
  LOCK_HANDLE(h, hh);
  CU_TRY(h, cudaSetDevice(h->device));
  if (enable && !h->ev[0]) for (int i = 0; i < 6; ++i) CU_TRY(h, cudaEventCreate(&h->ev[i]));
  h->timing = enable ? 1 : 0;
  h->ev_valid = false;
  return ARTP_OK;
}

int artp_get_last_timing(artp_handle* hh, float* ms3) {
  LOCK_HANDLE(h, hh);
  if (!ms3) return ARTP_E_INVALID;
  if (!h->timing || !h->ev_valid) { h->err = "timing not enabled or no call recorded"; return ARTP_E_INVALID; }
  CU_TRY(h, cudaSetDevice(h->device));
  CU_TRY(h, cudaEventSynchronize(h->ev[5]));
  CU_TRY(h, cudaEventElapsedTime(ms3 + 0, h->ev[0], h->ev[1]));   // classify
  CU_TRY(h, cudaEventElapsedTime(ms3 + 1, h->ev[1], h->ev[4]));   // box stages: warp + reach vertex + reach plane
  CU_TRY(h, cudaEventElapsedTime(ms3 + 2, h->ev[4], h->ev[5]));   // plane grouping
  return ARTP_OK;
}

int artp_get_last_stage_timing(artp_handle* hh, float* ms5) {
  LOCK_HANDLE(h, hh);
  if (!ms5) return ARTP_E_INVALID;
  if (!h->timing || !h->ev_valid) { h->err = "timing not enabled or no call recorded"; return ARTP_E_INVALID; }
  CU_TRY(h, cudaSetDevice(h->device));
  CU_TRY(h, cudaEventSynchronize(h->ev[5]));
  for (int i = 0; i < 5; ++i) CU_TRY(h, cudaEventElapsedTime(ms5 + i, h->ev[i], h->ev[i + 1]));
  return ARTP_OK;
}

// Pinned host memory for the adapter's staging buffers (the contiguous n x 7 state batch it gathers the OMPL states into,
// the verdict bytes): cudaHostAlloc'd pages are allocated pinned and portable, so the copies run as DMA at PCIe line
// rate without a staging copy.
void* artp_host_alloc(size_t bytes) {
  void* p = nullptr;
  if (bytes == 0 || cudaHostAlloc(&p, bytes, cudaHostAllocPortable) != cudaSuccess) return nullptr;
  return p;
}
void artp_host_free(void* p) { if (p) cudaFreeHost(p); }

int artp_poll_error(artp_handle* hh) {
  LOCK_HANDLE(h, hh);
  return take_sticky_error(h);
}

int artp_debug_set_group_capacity(artp_handle* hh, int max_triangles) {
  LOCK_HANDLE(h, hh);
  if (max_triangles < 0) return ARTP_E_INVALID;
  h->tcap_override = max_triangles;   // takes effect at the next artp_set_map
  return ARTP_OK;
}

int artp_get_stats(artp_handle* hh, artp_stats* out) {
  LOCK_HANDLE(h, hh);
  if (!out) return ARTP_E_INVALID;
  CU_TRY(h, cudaSetDevice(h->device));
  Counters ctr{};
  CU_TRY(h, cudaMemcpy(&ctr, h->d_ctr, sizeof(ctr), cudaMemcpyDeviceToHost));   // synchronises the device
  h->stats.last_deferred = ctr.defer;
  h->stats.last_queued_boxes = ctr.q.big.end + ctr.q.reach.end + ctr.q.group.end;
  h->stats.last_queued_warp_stage = ctr.q.big.end;
  h->stats.last_queued_reach_stage = ctr.q.reach.end;
  h->stats.last_reach_plane_stage = ctr.q.group.end;
  if (h->deferred_unread) { h->stats.poses_deferred += ctr.defer; h->deferred_unread = false; }
  *out = h->stats;
  return take_sticky_error(h);
}

int artp_set_map(artp_handle* hh, const float* elevation, const float* elevation_masked, int rows, int cols, double res,
                 double cx, double cy) {
  return artp_set_map_window(hh, elevation, elevation_masked, rows, cols, res, cx, cy, 0, rows);
}

// Spatial shard of a map (SURVEY 8e): this handle holds only rows [row0, row0 + nrows) of the rows x cols layers --
// its slab plus the halo the caller chose -- but keeps the geometry of the FULL map (sample spacing L / (N - 1), vertex
// coordinates, isInside), so every verdict is bit-identical to a handle holding the whole map. The device pointers
// of the layer / range tables are shifted by -row0, so the kernels keep indexing with global vertex indices.
int artp_set_map_window(artp_handle* hh, const float* elevation, const float* elevation_masked, int rows, int cols, double res,
                        double cx, double cy, int row0, int nrows) {
  LOCK_HANDLE(h, hh);
  if (!elevation || !elevation_masked || rows < 2 || cols < 2 || !(res > 0)) { h->err = "bad map arguments"; return ARTP_E_INVALID; }
  if (row0 < 0 || nrows < 2 || row0 + nrows > rows || (row0 & 3)) {
    h->err = "bad map window (row0 must be a multiple of 4, 0 <= row0, row0 + nrows <= rows, nrows >= 2)"; return ARTP_E_INVALID;
  }
  CU_TRY(h, cudaSetDevice(h->device));
  const size_t ncell = (size_t)nrows * cols;
  // geometry exactly as dxHeightfieldData::SetData computes it in fp32 (heightfield.cpp:130-169)
  const double Lx = rows * res, Ly = cols * res;   // grid_map: length = size * resolution
  artp::Field f;
  f.nx = rows; f.nz = cols;
  f.W = (float)Lx; f.D = (float)Ly;
  f.hW = f.W / 2.0f; f.hD = f.D / 2.0f;
  f.sW = f.W / (f.nx - 1.0f);
  f.sD = f.D / (f.nz - 1.0f);
  f.asp = f.sD / f.sW;
  f.iW = 1.0f / f.sW;
  f.iD = 1.0f / f.sD;
  f.px = (float)cx; f.py = (float)cy;
  // K2 shared-memory plane store: bound the zone of either box by its half-diagonal; same bound -> table levels
  int tcap = 0, kmax[2] = {0, 0};
  for (int k = 0; k < 2; ++k) {
    const float* sd = h->chk.side[k];
    const double r = 0.5 * std::sqrt((double)sd[0] * sd[0] + (double)sd[1] * sd[1] + (double)sd[2] * sd[2]);
    const int nxm = std::min(rows, (int)std::ceil(2.0 * r * f.iW) + 4), nzm = std::min(cols, (int)std::ceil(2.0 * r * f.iD) + 4);
    tcap = std::max(tcap, 2 * (nxm - 1) * (nzm - 1));
    int kk = 0;
    while ((2 << kk) <= std::min(nxm, nzm) && kk < artp::kMaxLevel) ++kk;   // floor(log2(min dim bound))
    kmax[k] = kk;
  }
  if (h->tcap_override > 0) tcap = std::min(tcap, h->tcap_override);   // test hook: force the overflow path
  tcap = (tcap + 3) & ~3;
  const int smem = tcap * 21 + 64;
  if (smem > 200 * 1024) {
    h->err = "box/map resolution combination exceeds the plane-grouping kernel's shared-memory store";
    return ARTP_E_LIMIT;
  }
  CU_TRY(h, cudaFuncSetAttribute(artp::box_items_block_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  int per_sm = 0;
  CU_TRY(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, artp::box_items_block_kernel, artp::kBlockStageThreads, smem));
  h->k2_smem = smem; h->k2_tcap = tcap; h->k2_grid = h->sm_count * std::max(per_sm, 1);
  // upload (the previous map may still be in use by asynchronous calls on the caller's streams)
  CU_TRY(h, cudaDeviceSynchronize());
  h->chain_busy[0] = h->chain_busy[1] = false;
  const int pitch = (nrows + 3) & ~3;
  const size_t npad = (size_t)pitch * cols;
  if (h->win_rows != nrows || h->cols != cols) {
    for (int k = 0; k < 2; ++k) {
      cudaFree(h->d_H[k]); h->d_H[k] = nullptr;
      for (int l = 0; l <= artp::kMaxLevel; ++l) {
        cudaFree(h->d_T[k][l]); cudaFree(h->d_C[k][l]);
        h->d_T[k][l] = nullptr; h->d_C[k][l] = nullptr;
      }
      CU_TRY(h, cudaMalloc(&h->d_H[k], npad * sizeof(float)));
    }
  }
  for (int k = 0; k < 2; ++k)
    for (int l = 1; l <= kmax[k]; ++l)
      if (!h->d_T[k][l]) {
        CU_TRY(h, cudaMalloc(&h->d_T[k][l], npad * sizeof(float2)));
        CU_TRY(h, cudaMalloc(&h->d_C[k][l], npad * sizeof(uint32_t)));
      }
  int rc = grow(h, h->d_stage, h->stage_cap, ncell * sizeof(float));
  if (rc) return rc;
  const float* src[2] = {elevation, elevation_masked};
  float cbase[2], cstep[2];
  for (int k = 0; k < 2; ++k) code_scale(src[k], ncell, cbase[k], cstep[k]);
  // plane tables (temporary): 4 slots per cell = load factor 0.5 for the 2 triangles of a cell
  size_t cap = 1;
  while (cap < 4 * ncell) cap <<= 1;
  PlaneSlot* d_tab = nullptr;
  unsigned char* d_merge = nullptr;   // [0, npad): mergeable cells; [npad, 3 npad): two byte-flag levels (ping-pong while building)
  CU_TRY(h, cudaMalloc(&d_tab, cap * sizeof(PlaneSlot)));
  if (cudaMalloc(&d_merge, 3 * npad) != cudaSuccess) { cudaFree(d_tab); h->err = "cudaMalloc (plane tables)"; return ARTP_E_CUDA; }
  for (int k = 0; k < 2; ++k) {
    CU_TRY(h, cudaMemcpyAsync(h->d_stage, src[k], ncell * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    reverse_columns_kernel<<<h->sm_count * 4, 256, 0, h->stream>>>((const float*)h->d_stage, h->d_H[k], nrows, cols, pitch);
    CU_TRY(h, cudaGetLastError());
    artp::Field fk = f;                     // local storage, global geometry: cell x of the window is global cell x + row0
    fk.H = h->d_H[k]; fk.pitch = pitch; fk.nx = nrows;
    plane_table_clear_kernel<<<h->sm_count * 8, 256, 0, h->stream>>>(d_tab, cap);
    CU_TRY(h, cudaMemsetAsync(d_merge, 0, npad, h->stream));
    plane_table_insert_kernel<<<h->sm_count * 8, 256, 0, h->stream>>>(fk, row0, d_tab, (uint32_t)(cap - 1));
    plane_table_query_kernel<<<h->sm_count * 8, 256, 0, h->stream>>>(fk, row0, d_tab, (uint32_t)(cap - 1), d_merge);
    CU_TRY(h, cudaGetLastError());
    h->stats.kernel_launches += 4;
    for (int l = 1; l <= kmax[k]; ++l) {
      unsigned char* nf_prev = d_merge + npad * (size_t)(1 + ((l - 1) & 1));
      unsigned char* nf_cur = d_merge + npad * (size_t)(1 + (l & 1));
      build_level_kernel<<<h->sm_count * 4, 256, 0, h->stream>>>(h->d_H[k], l > 1 ? h->d_T[k][l - 1] : nullptr,
                                                                  l > 1 ? nf_prev : nullptr, d_merge, h->d_T[k][l], nf_cur, nrows,
                                                                  cols, pitch, 1 << (l - 1));
      build_codes_kernel<<<h->sm_count * 4, 256, 0, h->stream>>>(h->d_T[k][l], nf_cur, h->d_C[k][l], npad, cbase[k], cstep[k]);
      CU_TRY(h, cudaGetLastError());
      h->stats.kernel_launches += 2;
    }
  }
  CU_TRY(h, cudaStreamSynchronize(h->stream));
  cudaFree(d_tab); cudaFree(d_merge);
  h->rows = rows; h->cols = cols; h->pitch = pitch; h->win_row0 = row0; h->win_rows = nrows;
  f.pitch = pitch;
  f.x_lo = row0; f.x_hi = row0 + nrows - 1;
  for (int k = 0; k < 2; ++k) {
    f.H = h->d_H[k] - row0;                 // indexed with GLOBAL vertex indices x in [x_lo, x_hi]
    f.kmax = kmax[k];
    f.cbase = cbase[k]; f.cstep = cstep[k];
    for (int l = 0; l <= artp::kMaxLevel; ++l) {
      f.T[l] = (l >= 1 && l <= kmax[k]) ? h->d_T[k][l] - row0 : nullptr;
      f.C[l] = (l >= 1 && l <= kmax[k]) ? h->d_C[k][l] - row0 : nullptr;
    }
    h->chk.f[k] = f;
  }
  h->chk.err_word = h->d_err;
  h->chk.Lx = Lx; h->chk.Ly = Ly; h->chk.cx = cx; h->chk.cy = cy;
  h->chk.cell_margin = 0.02f + 2e-6f * (float)std::max(rows, cols);
  // Stage B tiles (artp_tiles.cuh): a zone spans at most ceil(2 r / s) + 3 vertices per axis (r = box half-diagonal);
  // + 3 columns because the tile starts at x0 & ~3; width rounded up to a multiple of 4 floats (16-byte rows).
  {
    typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                      const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                      CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn) {
      h->err = "cuTensorMapEncodeTiled not available from the driver"; return ARTP_E_CUDA;
    }
    h->chk.reach_tw = 0; h->chk.reach_th = 0;
    for (int q = 0; q < 2; ++q) {          // 0: big tiles (torso box bound), 1: small tiles (reach box bound)
      const float* sd = h->chk.side[q];
      const double r = 0.5 * std::sqrt((double)sd[0] * sd[0] + (double)sd[1] * sd[1] + (double)sd[2] * sd[2]);
      int tw = ((int)std::ceil(2.0 * r * f.iW) + 3 + 3 + 3) & ~3, th = (int)std::ceil(2.0 * r * f.iD) + 3;
      tw = std::min(tw, 256); th = std::min(th, 256);
      artp::TileCfg tc;
      tc.tw = tw; tc.th = th; tc.bytes = (uint32_t)tw * th * 4; tc.stride = (tc.bytes + 127u) & ~127u;
      // big tiles: one slot per warp (three 8-warp CTAs per SM hide the copy latency better than a second 7 KB slot);
      // small tiles: two slots, the next box's tile is in flight while this one is decided
      tc.slots = (tc.stride > 2048) ? 1 : 2;
      int wpc = 8;
      while (wpc > 1 && (size_t)wpc * tc.slots * tc.stride + 128 > 72 * 1024) wpc >>= 1;
      if ((size_t)wpc * tc.slots * tc.stride + 128 > 200 * 1024) {
        if (q == 1) continue;              // no reach-box queue: everything takes the big-tile queue
        // boxes this large relative to the cells: tiles capped, oversized zones go to the grouping stage
        tc.tw = 64; tc.th = 64; tc.bytes = 64 * 64 * 4; tc.stride = tc.bytes; tc.slots = 1; wpc = 4;
      }
      const cuuint64_t gdim[2] = {(cuuint64_t)pitch, (cuuint64_t)cols};
      const cuuint64_t gstr[1] = {(cuuint64_t)pitch * sizeof(float)};
      const cuuint32_t box[2] = {(cuuint32_t)tc.tw, (cuuint32_t)tc.th};
      const cuuint32_t one[2] = {1, 1};
      for (int layer = 0; layer < 2; ++layer) {
        const CUresult cr = reinterpret_cast<EncodeTiledFn>(fn)(&h->tile_map[q][layer], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, h->d_H[layer], gdim,
                                                                gstr, box, one, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                                                                CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (cr != CUDA_SUCCESS) { h->err = "cuTensorMapEncodeTiled failed (" + std::to_string((int)cr) + ")"; return ARTP_E_CUDA; }
      }
      tc.x_off = row0;
      h->tile_cfg[q] = tc; h->tile_warps[q] = wpc;
      h->tile_smem[q] = (int)((size_t)wpc * tc.slots * tc.stride + 128);
      if (q == 1) { h->chk.reach_tw = tc.tw; h->chk.reach_th = tc.th; }
    }
    h->group_grid = 0;
    if (h->chk.reach_tw && h->tile_cfg[1].tw <= 127 && h->tile_cfg[1].th <= 255) {   // task packing: 7 + 8 bits of cell coordinates
      const int gsm = artp::kMaxTileWarps * 8 * (int)h->tile_cfg[1].stride + 128;
      if (gsm <= 160 * 1024 && !std::getenv("ARTP_NO_GROUPS")) {   // ARTP_NO_GROUPS: every reach box takes the one-warp-per-box queue
        CU_TRY(h, cudaFuncSetAttribute(artp::reach_groups_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, gsm));
        int ps = 0;
        CU_TRY(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ps, artp::reach_groups_kernel, artp::kMaxTileWarps * 32, gsm));
        h->group_grid = h->sm_count * std::max(ps, 1);
        h->group_smem = gsm;
      }
    }
    const int smax = std::max(h->tile_smem[0], h->tile_smem[1]);
    CU_TRY(h, cudaFuncSetAttribute(artp::box_tiles_warp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smax));
    for (int q = 0; q < 2; ++q) {
      int ps = 0;
      CU_TRY(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ps, artp::box_tiles_warp_kernel, h->tile_warps[q] * 32, h->tile_smem[q]));
      h->tile_grid[q] = h->sm_count * std::max(ps, 1);
    }
  }
  h->has_map = true;
  h->has_sampler = false;      // its layers belong to the previous map
  h->has_device_normals = false;
  h->has_device_cdf = false;
  h->has_normals = false;
  h->has_sample_filter = false;
  h->has_dist_observed = false;
  h->res = res;
  return ARTP_OK;
}

int artp_check_poses(artp_handle* hh, const double* states, size_t n, uint8_t* valid) {
  return check_poses(hh, states, n, valid, false, nullptr);
}
int artp_check_poses_f32(artp_handle* hh, const float* states, size_t n, uint8_t* valid) {
  return check_poses(hh, states, n, valid, false, nullptr);
}
int artp_check_poses_device(artp_handle* hh, const double* d_states, size_t n, uint8_t* d_valid, void* stream) {
  return check_poses(hh, d_states, n, d_valid, true, (cudaStream_t)stream);
}
int artp_check_poses_f32_device(artp_handle* hh, const float* d_states, size_t n, uint8_t* d_valid, void* stream) {
  return check_poses(hh, d_states, n, d_valid, true, (cudaStream_t)stream);
}

int artp_check_motions_device(artp_handle* hh, const double* d_s1, const double* d_s2, size_t n, int n_steps,
                              uint8_t* d_valid, void* stream) {
  LOCK_HANDLE(h, hh);
  if (n_steps < 0) { h->err = "n_steps < 0"; return ARTP_E_INVALID; }
  const size_t items = n * ((size_t)n_steps + 1);
  int rc = check_common(h, items);
  if (rc) return rc;
  if (n == 0) return ARTP_OK;
  if (!d_s1 || !d_s2 || !d_valid) { h->err = "null buffer"; return ARTP_E_INVALID; }
  CU_TRY(h, cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  ChainScope cs(h, 0, s);
  if (cs.rc) return cs.rc;
  fill_u8_kernel<<<std::min<size_t>((n + 255) / 256, (size_t)h->sm_count * 8), 256, 0, s>>>(d_valid, n, 1);
  CU_TRY(h, cudaGetLastError());
  artp::Work w;
  w.s1 = d_s1; w.s2 = d_s2; w.s2f = nullptr; w.valid = d_valid; w.item_base = 0; w.n_items = (uint32_t)items; w.steps = n_steps; w.edge_mode = 1;
  rc = run_items(h, w, s);
  if (rc) return rc;
  h->stats.kernel_launches += 1;
  h->stats.last_launches += 1;
  h->stats.poses_checked += items;
  return ARTP_OK;
}

int artp_check_motions(artp_handle* hh, const double* s1, const double* s2, size_t n, int n_steps, uint8_t* valid) {
  LOCK_HANDLE(h, hh);
  if (!h->has_map) { h->err = "no map set"; return ARTP_E_NOMAP; }
  if (n == 0) return ARTP_OK;
  if (!s1 || !s2 || !valid) { h->err = "null buffer"; return ARTP_E_INVALID; }
  if (n_steps >= 0 && n * ((size_t)n_steps + 1) <= (size_t)artp::kSmallBatch && 2 * n <= (size_t)artp::kSmallBatch &&
      !h->timing) {
    // latency path (a single checkMotion call): one fused launch, interpolation on the device as in the pipeline
    artp::SmallBatch sb;
    for (size_t e = 0; e < n; ++e) {
      std::memcpy(sb.s[2 * e], s1 + 7 * e, 7 * sizeof(double));
      std::memcpy(sb.s[2 * e + 1], s2 + 7 * e, 7 * sizeof(double));
    }
    return check_poses_small(h, sb, n * ((size_t)n_steps + 1), valid, n_steps);
  }
  const size_t sb = n * 7 * sizeof(double);
  char* r[3];
  int rc = host_call_begin(h, {sb, sb, n}, r);
  if (rc) return rc;
  CU_TRY(h, cudaMemcpyAsync(r[0], s1, sb, cudaMemcpyHostToDevice, h->stream));
  CU_TRY(h, cudaMemcpyAsync(r[1], s2, sb, cudaMemcpyHostToDevice, h->stream));
  rc = artp_check_motions_device(hh, (const double*)r[0], (const double*)r[1], n, n_steps, (uint8_t*)r[2], h->stream);
  if (rc) return rc;
  CU_TRY(h, cudaMemcpyAsync(valid, r[2], n, cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h, true);
}

// valid_prefix[e] = number of leading 1s in item_valid[item_off[e] .. item_off[e+1])
__global__ void edge_prefix_kernel(const uint8_t* __restrict__ item_valid, const uint32_t* __restrict__ item_off, size_t n,
                                   int32_t* __restrict__ valid_prefix) {
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x) {
    const uint32_t o0 = item_off[e], o1 = item_off[e + 1];
    uint32_t k = o0;
    while (k < o1 && item_valid[k]) ++k;
    valid_prefix[e] = (int32_t)(k - o0);
  }
}

// Edge e checks the items d_item_off[e] .. d_item_off[e+1] between d_s1[e] and d_s2[e] (interior states, or with
// `quotient` the segment states of the motion) and gets the number of leading valid ones in d_valid_prefix[e].
static int check_items_prefix(Handle* h, const double* d_s1, const double* d_s2, size_t n, const uint32_t* d_item_off,
                              size_t total_items, uint8_t* d_item_valid, int32_t* d_valid_prefix, void* stream, int quotient) {
  int rc = check_common(h, total_items);
  if (rc) return rc;
  if (n == 0) return ARTP_OK;
  if (!d_s1 || !d_s2 || !d_item_off || !d_valid_prefix || (total_items && !d_item_valid)) {
    h->err = "null buffer"; return ARTP_E_INVALID;
  }
  if (n >= 0xFFFFFFFFull) { h->err = "too many edges"; return ARTP_E_INVALID; }
  CU_TRY(h, cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  ChainScope cs(h, 0, s);
  if (cs.rc) return cs.rc;
  h->stats.last_launches = 0;
  if (total_items) {
    artp::Work w;
    w.s1 = d_s1; w.s2 = d_s2; w.s2f = nullptr; w.valid = d_item_valid; w.item_base = 0; w.n_items = (uint32_t)total_items;
    w.steps = 0; w.edge_mode = 0; w.item_off = d_item_off; w.n_edges = (uint32_t)n; w.quotient = quotient;
    rc = run_items(h, w, s);
    if (rc) return rc;
  }
  edge_prefix_kernel<<<std::min<size_t>((n + 255) / 256, (size_t)h->sm_count * 8), 256, 0, s>>>(d_item_valid, d_item_off, n,
                                                                                                  d_valid_prefix);
  CU_TRY(h, cudaGetLastError());
  h->stats.kernel_launches += 1;
  h->stats.last_launches += 1;
  h->stats.poses_checked += total_items;
  return ARTP_OK;
}

// check_items_prefix over host buffers: the n = off.size() - 1 edges (s1[e], s2[e]) with their item offsets `off`;
// valid_prefix[e] receives edge e's number of leading valid items.
static int check_items_prefix_host(Handle* h, const double* s1, const double* s2, const std::vector<uint32_t>& off,
                                   int quotient, int32_t* valid_prefix) {
  const size_t n = off.size() - 1, total = off[n], sb = n * 7 * sizeof(double);
  char* r[5];   // s1 | s2 | off | prefix | item flags
  int rc = host_call_begin(h, {sb, sb, (n + 1) * sizeof(uint32_t), n * sizeof(int32_t), total}, r);
  if (rc) return rc;
  CU_TRY(h, cudaMemcpyAsync(r[0], s1, sb, cudaMemcpyHostToDevice, h->stream));
  CU_TRY(h, cudaMemcpyAsync(r[1], s2, sb, cudaMemcpyHostToDevice, h->stream));
  CU_TRY(h, cudaMemcpyAsync(r[2], off.data(), (n + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
  rc = check_items_prefix(h, (const double*)r[0], (const double*)r[1], n, (const uint32_t*)r[2], total, (uint8_t*)r[4],
                          (int32_t*)r[3], h->stream, quotient);
  if (rc) return rc;
  CU_TRY(h, cudaMemcpyAsync(valid_prefix, r[3], n * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h, true);   // `off` outlives its H2D copy: the call synchronises before it returns
}

int artp_check_edge_interiors_device(artp_handle* hh, const double* d_s1, const double* d_s2, size_t n,
                                     const uint32_t* d_item_off, size_t total_items, uint8_t* d_item_valid,
                                     int32_t* d_valid_prefix, void* stream) {
  LOCK_HANDLE(h, hh);
  return check_items_prefix(h, d_s1, d_s2, n, d_item_off, total_items, d_item_valid, d_valid_prefix, stream, 0);
}

int artp_check_edge_interiors(artp_handle* hh, const double* s1, const double* s2, size_t n, const int32_t* n_interp,
                              double max_lateral, int32_t* valid_prefix) {
  LOCK_HANDLE(h, hh);
  if (!h->has_map) { h->err = "no map set"; return ARTP_E_NOMAP; }
  if (n == 0) return ARTP_OK;
  if (!s1 || !s2 || !valid_prefix) { h->err = "null buffer"; return ARTP_E_INVALID; }
  if (!n_interp && !(max_lateral > 0.0)) { h->err = "n_interp == NULL needs max_lateral > 0"; return ARTP_E_INVALID; }
  std::vector<uint32_t> off(n + 1);
  size_t total = 0;
  for (size_t e = 0; e < n; ++e) {
    off[e] = (uint32_t)total;
    long long ne;
    if (n_interp) {
      ne = n_interp[e];
    } else {   // lateralDistance (utils.h:52-61) / max_lateral truncated like prm_motion_cost.cpp:341-343
      const double dx = s2[7 * e] - s1[7 * e], dy = s2[7 * e + 1] - s1[7 * e + 1];
      ne = (long long)(unsigned int)(std::sqrt(dx * dx + dy * dy) / max_lateral);
    }
    if (ne < 0) { h->err = "n_interp < 0"; return ARTP_E_INVALID; }
    total += (size_t)ne;
    if (total >= 0xFFFFFFFFull) { h->err = "too many interior states (>= 2^32)"; return ARTP_E_INVALID; }
  }
  off[n] = (uint32_t)total;
  return check_items_prefix_host(h, s1, s2, off, 0, valid_prefix);
}

// ompl::base::CompoundStateSpace::validSegmentCount for SE3 = max over the R^3 and SO(3) sub-spaces of
// (unsigned)ceil(distance / (maximum extent * longest valid segment fraction)) (OMPL 1.4.2 StateSpace.cpp;
// RealVectorStateSpace: Euclidean distance, extent = |high - low|; SO3StateSpace: arc length acos(|q1.q2|) with
// the 1e-9 clamp, extent pi/2). Host arithmetic, doubles, like OMPL.
int artp_valid_segment_count(const artp_se3_space* sp, const double* s1, const double* s2, size_t n, int32_t* nd) {
  if (!sp || (n && (!s1 || !s2 || !nd))) return ARTP_E_INVALID;
  const double frac = sp->longest_valid_segment_fraction > 0 ? sp->longest_valid_segment_fraction : 0.01;
  double e2 = 0;
  for (int i = 0; i < 3; ++i) e2 += (sp->high[i] - sp->low[i]) * (sp->high[i] - sp->low[i]);
  const double seg_r3 = std::sqrt(e2) * frac, seg_so3 = 0.5 * 3.14159265358979323846 * frac;
  if (!(seg_r3 > 0)) return ARTP_E_INVALID;
  for (size_t i = 0; i < n; ++i) {
    const double* a = s1 + 7 * i;
    const double* b = s2 + 7 * i;
    const double dx = a[0] - b[0], dy = a[1] - b[1], dz = a[2] - b[2];
    const double d3 = std::sqrt(dx * dx + dy * dy + dz * dz);
    const double dq = std::fabs(a[3] * b[3] + a[4] * b[4] + a[5] * b[5] + a[6] * b[6]);
    const double ds = (dq > 1.0 - 1e-9) ? 0.0 : std::acos(dq);
    const unsigned n3 = (unsigned)std::ceil(d3 / seg_r3), ns = (unsigned)std::ceil(ds / seg_so3);
    nd[i] = (int32_t)std::max(n3, ns);
  }
  return ARTP_OK;
}

int artp_check_motions_segments(artp_handle* hh, const double* s1, const double* s2, size_t n, const int32_t* nd,
                                const artp_se3_space* sp, uint8_t* valid, double* last_valid_t) {
  LOCK_HANDLE(h, hh);
  if (!h->has_map) { h->err = "no map set"; return ARTP_E_NOMAP; }
  if (n == 0) return ARTP_OK;
  if (!s1 || !s2 || !valid || (!nd && !sp)) { h->err = "null buffer (nd == NULL needs the space parameters)"; return ARTP_E_INVALID; }
  std::vector<int32_t> seg(n);
  if (nd) std::copy(nd, nd + n, seg.begin());
  else { const int rc = artp_valid_segment_count(sp, s1, s2, n, seg.data()); if (rc) { h->err = "bad SE3 space parameters"; return rc; } }
  std::vector<uint32_t> off(n + 1);
  size_t total = 0;
  for (size_t e = 0; e < n; ++e) {
    if (seg[e] < 0) { h->err = "segment count < 0"; return ARTP_E_INVALID; }
    if (seg[e] < 1) seg[e] = 1;                 // nd = 0 (identical states): only s2 is checked
    off[e] = (uint32_t)total;
    total += (size_t)seg[e];
    if (total >= 0xFFFFFFFFull) { h->err = "too many states (>= 2^32)"; return ARTP_E_INVALID; }
  }
  off[n] = (uint32_t)total;
  std::vector<int32_t> prefix(n);
  const int rc = check_items_prefix_host(h, s1, s2, off, 1, prefix.data());
  if (rc == ARTP_E_CUDA) return rc;
  for (size_t e = 0; e < n; ++e) {
    // DiscreteMotionValidator::checkMotion(s1, s2, lastValid): the first invalid state in the order j = 1 .. nd-1, s2
    // is state index p (0-based) => lastValid.second = p / nd  ((j-1)/nd for an interior state, (nd-1)/nd for s2)
    valid[e] = prefix[e] == seg[e] ? 1 : 0;
    if (last_valid_t) last_valid_t[e] = valid[e] ? 1.0 : (double)prefix[e] / (double)seg[e];
  }
  return rc;
}

// Rows [tx, ty, tyaw, sx, sy, syaw] of the MotionCostFunc edge matrix from SE(3) states exactly as
// PRMMotionCostMaintainer::updateEdges / computeCostForVertexEdges fill them (prm_motion_cost.cpp:27-128): x, y cast
// double -> float by the assignment into the float matrix, yaw = getYawFromSO3 (utils.h:80-88: double atan2, float result).
__global__ void edge_matrix_kernel(const double* __restrict__ s_start, const double* __restrict__ s_target, size_t n,
                                   float* __restrict__ edges) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const double* a = s_start + 7 * i;
    const double* b = s_target + 7 * i;
    float* o = edges + 6 * i;
    o[0] = (float)b[0]; o[1] = (float)b[1];
    o[2] = (float)atan2(2 * (b[6] * b[5] + b[3] * b[4]), 1 - 2 * (b[4] * b[4] + b[5] * b[5]));
    o[3] = (float)a[0]; o[4] = (float)a[1];
    o[5] = (float)atan2(2 * (a[6] * a[5] + a[3] * a[4]), 1 - 2 * (a[4] * a[4] + a[5] * a[5]));
  }
}
// getCost / isFeasible per row (motion_cost_objective.h:54-66); infeasible edges get +inf like updateEdges (:56-59)
__global__ void combine_cost_kernel(const float* __restrict__ cost3, size_t n, float we, float wt, float wr, float thr,
                                    double* __restrict__ cost, uint8_t* __restrict__ feasible) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float ce = cost3[3 * i], ct = cost3[3 * i + 1], cr = cost3[3 * i + 2];
    const bool ok = (double)cr <= (double)thr;
    feasible[i] = ok ? 1 : 0;
    cost[i] = ok ? (double)ce * (double)we + (double)ct * (double)wt + (double)cr * (double)wr : CUDART_INF;
  }
}

// MotionCostObjective::motionCost (motion_cost_objective.cpp:36-95) splits edge e into the pieces piece_off[e] ..
// piece_off[e+1] - 1 (n_interp + 1 of them). Knot j of the edge is s1 for j = 0, s2 for j = n_interp + 1 (copied, not
// interpolated) and interpolate(s1, s2, j * (1.0 / (n_interp + 1))) in between (:49, :67); piece i's row is
// [x y yaw](knot i+1) ++ [x y yaw](knot i) with the casts of edge_matrix_kernel. Built here, in the translation unit
// without FMA contraction, so that the rows equal the host's bit for bit; the head's translation unit contracts.
__device__ __forceinline__ void knot_row(const double* s, float* o) {
  o[0] = (float)s[0]; o[1] = (float)s[1];
  o[2] = (float)atan2(2 * (s[6] * s[5] + s[3] * s[4]), 1 - 2 * (s[4] * s[4] + s[5] * s[5]));
}
__device__ __forceinline__ void split_knot_row(const double* a, const double* b, uint32_t j, uint32_t n_pieces, float* o) {
  if (j == 0) {
    knot_row(a, o);
  } else if (j == n_pieces) {
    knot_row(b, o);
  } else {   // no pointer select between a, b and k: that would put all three in local memory
    double k[7];
    artp::se3_interpolate(a, b, (double)j * (1.0 / (double)n_pieces), k);
    knot_row(k, o);
  }
}
__global__ void split_rows_kernel(const double* __restrict__ s1, const double* __restrict__ s2, uint32_t n_edges,
                                  const uint32_t* __restrict__ piece_off, size_t total, float* __restrict__ rows) {
  for (size_t p = blockIdx.x * (size_t)blockDim.x + threadIdx.x; p < total; p += (size_t)gridDim.x * blockDim.x) {
    uint32_t lo = 0, hi = n_edges;          // largest e with piece_off[e] <= p, as load_item_state
    while (hi - lo > 1) {
      const uint32_t mid = (lo + hi) >> 1;
      if (__ldg(piece_off + mid) <= p) lo = mid; else hi = mid;
    }
    const uint32_t o0 = __ldg(piece_off + lo), n_pieces = __ldg(piece_off + lo + 1) - o0, i = (uint32_t)p - o0;
    double a[7], b[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) { a[k] = s1[(size_t)lo * 7 + k]; b[k] = s2[(size_t)lo * 7 + k]; }
    split_knot_row(a, b, i + 1, n_pieces, rows + 6 * p);
    split_knot_row(a, b, i, n_pieces, rows + 6 * p + 3);
  }
}
// The rest of motionCost per edge, one thread walking its pieces in order: +inf at the first piece whose risk is above
// the threshold (isFeasible), else the left-to-right double sum of getCost from 0.0, the expression of combine_cost_kernel.
__global__ void split_reduce_kernel(const float* __restrict__ cost3, const uint32_t* __restrict__ piece_off, size_t n,
                                    float we, float wt, float wr, float thr, double* __restrict__ cost) {
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x) {
    const uint32_t o0 = piece_off[e], o1 = piece_off[e + 1];
    double c = 0.0;
    for (uint32_t k = o0; k < o1; ++k) {
      const float ce = cost3[3 * (size_t)k], ct = cost3[3 * (size_t)k + 1], cr = cost3[3 * (size_t)k + 2];
      if ((double)cr > (double)thr) { c = CUDART_INF; break; }
      c += (double)ce * (double)we + (double)ct * (double)wt + (double)cr * (double)wr;
    }
    cost[e] = c;
  }
}

int artp_edge_matrix_from_states(const double* s_start, const double* s_target, size_t n, float* edges) {
  if (n && (!s_start || !s_target || !edges)) return ARTP_E_INVALID;
  for (size_t i = 0; i < n; ++i) {
    const double* a = s_start + 7 * i;
    const double* b = s_target + 7 * i;
    float* o = edges + 6 * i;
    o[0] = (float)b[0]; o[1] = (float)b[1];
    o[2] = (float)std::atan2(2 * (b[6] * b[5] + b[3] * b[4]), 1 - 2 * (b[4] * b[4] + b[5] * b[5]));
    o[3] = (float)a[0]; o[4] = (float)a[1];
    o[5] = (float)std::atan2(2 * (a[6] * a[5] + a[3] * a[4]), 1 - 2 * (a[4] * a[4] + a[5] * a[5]));
  }
  return ARTP_OK;
}

int artp_motion_cost_states(artp_handle* hh, const double* s_start, const double* s_target, size_t n, double* cost,
                            uint8_t* feasible, float* cost3) {
  LOCK_HANDLE(h, hh);
  if (n == 0) return ARTP_OK;
  if (!s_start || !s_target || !cost || !feasible) { h->err = "null buffer"; return ARTP_E_INVALID; }
  const size_t sb = n * 7 * sizeof(double);
  char* r[6];   // s_start | s_target | edge matrix | cost3 | cost | feasible
  int rc = host_call_begin(h, {sb, sb, n * 6 * sizeof(float), n * 3 * sizeof(float), n * sizeof(double), n}, r);
  if (rc) return rc;
  float* d_edges = (float*)r[2];
  float* d_c3 = (float*)r[3];
  CU_TRY(h, cudaMemcpyAsync(r[0], s_start, sb, cudaMemcpyHostToDevice, h->stream));
  CU_TRY(h, cudaMemcpyAsync(r[1], s_target, sb, cudaMemcpyHostToDevice, h->stream));
  const unsigned grid = (unsigned)std::min<size_t>((n + 255) / 256, (size_t)h->sm_count * 8);
  edge_matrix_kernel<<<grid, 256, 0, h->stream>>>((const double*)r[0], (const double*)r[1], n, d_edges);
  CU_TRY(h, cudaGetLastError());
  rc = artp_cnn::motion_cost(h->cnn, d_edges, n, d_c3, h->stream, h->err);
  if (rc) return rc;
  combine_cost_kernel<<<grid, 256, 0, h->stream>>>(d_c3, n, h->p.cost_w_energy, h->p.cost_w_time, h->p.cost_w_risk, h->p.risk_threshold,
                                                   (double*)r[4], (uint8_t*)r[5]);
  CU_TRY(h, cudaGetLastError());
  CU_TRY(h, cudaMemcpyAsync(cost, r[4], n * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(h, cudaMemcpyAsync(feasible, r[5], n, cudaMemcpyDeviceToHost, h->stream));
  if (cost3) CU_TRY(h, cudaMemcpyAsync(cost3, d_c3, n * 3 * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  if ((rc = host_call_end(h))) return rc;
  h->stats.kernel_launches += 3;
  h->stats.last_launches = 3;
  return ARTP_OK;
}

int artp_path_length_cost_device(artp_handle* hh, const double* d_s1, const double* d_s2, size_t n, double* d_cost,
                                 void* stream) {
  LOCK_HANDLE(h, hh);
  if (n == 0) return ARTP_OK;
  if (!d_s1 || !d_s2 || !d_cost) { h->err = "null buffer"; return ARTP_E_INVALID; }
  CU_TRY(h, cudaSetDevice(h->device));
  path_length_kernel<<<std::min<size_t>((n + 255) / 256, (size_t)h->sm_count * 8), 256, 0, (cudaStream_t)stream>>>(
      d_s1, d_s2, n, d_cost, h->p.use_directional_cost, h->p.max_lon_vel, h->p.max_lat_vel, h->p.max_ang_vel);
  CU_TRY(h, cudaGetLastError());
  h->stats.kernel_launches += 1;
  h->stats.last_launches = 1;
  return ARTP_OK;
}

int artp_path_length_cost(artp_handle* hh, const double* s1, const double* s2, size_t n, double* cost) {
  LOCK_HANDLE(h, hh);
  if (n == 0) return ARTP_OK;
  if (!s1 || !s2 || !cost) { h->err = "null buffer"; return ARTP_E_INVALID; }
  const size_t sb = n * 7 * sizeof(double);
  char* r[3];
  int rc = host_call_begin(h, {sb, sb, n * sizeof(double)}, r);
  if (rc) return rc;
  CU_TRY(h, cudaMemcpyAsync(r[0], s1, sb, cudaMemcpyHostToDevice, h->stream));
  CU_TRY(h, cudaMemcpyAsync(r[1], s2, sb, cudaMemcpyHostToDevice, h->stream));
  rc = artp_path_length_cost_device(hh, (const double*)r[0], (const double*)r[1], n, (double*)r[2], h->stream);
  if (rc) return rc;
  CU_TRY(h, cudaMemcpyAsync(cost, r[2], n * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h);
}

static int compact_valid_impl(Handle* h, const uint8_t* d_valid, size_t n, int64_t base, void* d_indices,
                              uint32_t* d_count, cudaStream_t s, bool bits = false, bool u32 = false) {
  if (n == 0) { CU_TRY(h, cudaMemsetAsync(d_count, 0, sizeof(uint32_t), s)); return ARTP_OK; }
  ChainScope cs(h, 1, s);
  if (cs.rc) return cs.rc;
  const size_t nb = (n + kCompactBlock - 1) / kCompactBlock;
  const int rc = grow(h, h->d_block_counts, h->block_counts_cap, nb);
  if (rc) return rc;
  if (bits) compact_count_kernel<true><<<(unsigned)nb, kCompactBlock, 0, s>>>(d_valid, n, h->d_block_counts);
  else compact_count_kernel<false><<<(unsigned)nb, kCompactBlock, 0, s>>>(d_valid, n, h->d_block_counts);
  compact_scan_kernel<<<1, 1024, 0, s>>>(h->d_block_counts, nb, d_count);
  if (bits) compact_scatter_kernel<true, int64_t><<<(unsigned)nb, kCompactBlock, 0, s>>>(d_valid, n, base, h->d_block_counts, (int64_t*)d_indices);
  else if (u32) compact_scatter_kernel<false, uint32_t><<<(unsigned)nb, kCompactBlock, 0, s>>>(d_valid, n, base, h->d_block_counts, (uint32_t*)d_indices);
  else compact_scatter_kernel<false, int64_t><<<(unsigned)nb, kCompactBlock, 0, s>>>(d_valid, n, base, h->d_block_counts, (int64_t*)d_indices);
  CU_TRY(h, cudaGetLastError());
  h->stats.kernel_launches += 3;
  h->stats.last_launches = 3;
  return ARTP_OK;
}

int artp_compact_valid_device(artp_handle* hh, const uint8_t* d_valid, size_t n, int64_t base, int64_t* d_indices,
                              uint32_t* d_count, void* stream) {
  LOCK_HANDLE(h, hh);
  if (!d_valid || !d_indices || !d_count) { h->err = "null buffer"; return ARTP_E_INVALID; }
  CU_TRY(h, cudaSetDevice(h->device));
  return compact_valid_impl(h, d_valid, n, base, d_indices, d_count, (cudaStream_t)stream);
}

int artp_compact_valid_u32_device(artp_handle* hh, const uint8_t* d_valid, size_t n, uint32_t base, uint32_t* d_indices,
                                  uint32_t* d_count, void* stream) {
  LOCK_HANDLE(h, hh);
  if (!d_valid || !d_indices || !d_count) { h->err = "null buffer"; return ARTP_E_INVALID; }
  if (n + (size_t)base > 0xFFFFFFFFull) { h->err = "indices do not fit 32 bits"; return ARTP_E_INVALID; }
  CU_TRY(h, cudaSetDevice(h->device));
  return compact_valid_impl(h, d_valid, n, (int64_t)base, d_indices, d_count, (cudaStream_t)stream, false, true);
}

// isValid for a shard + the bit-packed verdicts the multi-GPU exchange sends, in one call on one stream.
int artp_check_poses_bits_device(artp_handle* hh, const double* d_states, size_t n, uint8_t* d_valid, uint32_t* d_bits, void* stream) {
  LOCK_HANDLE(h, hh);
  int rc = artp_check_poses_device(hh, d_states, n, d_valid, stream);
  if (rc) return rc;
  return artp_pack_valid_bits_device(hh, d_valid, n, d_bits, stream);
}

int artp_pack_valid_bits_device(artp_handle* hh, const uint8_t* d_valid, size_t n, uint32_t* d_bits, void* stream) {
  LOCK_HANDLE(h, hh);
  if (n == 0) return ARTP_OK;
  if (!d_valid || !d_bits) { h->err = "null buffer"; return ARTP_E_INVALID; }
  CU_TRY(h, cudaSetDevice(h->device));
  const size_t words = (n + 31) / 32;
  pack_bits_kernel<<<(unsigned)std::min<size_t>((words * 32 + 255) / 256, (size_t)h->sm_count * 8), 256, 0,
                     (cudaStream_t)stream>>>(d_valid, n, d_bits);
  CU_TRY(h, cudaGetLastError());
  h->stats.kernel_launches += 1;
  h->stats.last_launches = 1;
  return ARTP_OK;
}

int artp_compact_bits_device(artp_handle* hh, const uint32_t* d_bits, size_t n, int64_t base, int64_t* d_indices,
                             uint32_t* d_count, void* stream) {
  LOCK_HANDLE(h, hh);
  if (!d_bits || !d_indices || !d_count) { h->err = "null buffer"; return ARTP_E_INVALID; }
  CU_TRY(h, cudaSetDevice(h->device));
  return compact_valid_impl(h, reinterpret_cast<const uint8_t*>(d_bits), n, base, d_indices, d_count, (cudaStream_t)stream, true);
}

// ---------------------------------------------------------------------------------------------------------------
// Sampler: SE3FromSE2Sampler::sampleUniform on the device (artp_sampler.cuh)
// ---------------------------------------------------------------------------------------------------------------
static int ensure_sampler_layers(Handle* h) {
  const size_t need = 5 * (size_t)h->rows * h->cols + (size_t)h->rows + 64;
  if (h->samp_layers_cap < need) {   // the layers computed on the device go with the old buffer
    h->has_device_normals = false;
    h->has_device_cdf = false;
    h->has_normals = false;
  }
  return grow(h, h->d_samp_layers, h->samp_layers_cap, need);
}

// The map fields of the sampler's view (geometry, elevation, normal and plane-fit layers of d_samp_layers).
static void sampler_map_view(Handle* h, artp::SamplerDev& m) {
  const size_t ncell = (size_t)h->rows * h->cols;
  float* base = h->d_samp_layers;
  m.elevation_rev = h->d_H[0]; m.pitch = h->pitch;
  m.normal_x = base; m.normal_y = base + ncell; m.normal_z = base + 2 * ncell; m.std_dev = base + 3 * ncell;
  m.rows = h->rows; m.cols = h->cols;
  m.res = h->chk.Lx / h->rows; m.cx = h->chk.cx; m.cy = h->chk.cy;
}

int artp_estimate_normals(artp_handle* hh, double estimation_radius, float* normal_x, float* normal_y, float* normal_z,
                          float* plane_fit_std_dev) {
  LOCK_HANDLE(h, hh);
  if (!h->has_map) { h->err = "no map set"; return ARTP_E_NOMAP; }
  if (h->win_rows != h->rows) { h->err = "not available on a map window (artp_set_map_window)"; return ARTP_E_INVALID; }
  if (!(estimation_radius >= 0.0)) { h->err = "estimation_radius < 0"; return ARTP_E_INVALID; }
  int rc = host_call_begin(h);
  if (rc) return rc;
  rc = ensure_sampler_layers(h);
  if (rc) return rc;
  const size_t ncell = (size_t)h->rows * h->cols;
  const double res = h->chk.Lx / h->rows;
  float* base = h->d_samp_layers;
  const int r_cells = (int)(estimation_radius / res), r_diag = (int)(estimation_radius * 0.70710678118 / res);   // utils.cpp:226-227
  artp::estimate_normals_kernel<<<(unsigned)std::min<size_t>((ncell + 127) / 128, (size_t)h->sm_count * 32), 128, 0, h->stream>>>(
      h->d_H[0], h->pitch, h->rows, h->cols, res, h->chk.cx, h->chk.cy, r_cells, r_diag, base, base + ncell, base + 2 * ncell,
      base + 3 * ncell);
  CU_TRY(h, cudaGetLastError());
  float* dst[4] = {normal_x, normal_y, normal_z, plane_fit_std_dev};
  for (int k = 0; k < 4; ++k)
    if (dst[k]) CU_TRY(h, cudaMemcpyAsync(dst[k], base + k * ncell, ncell * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  if ((rc = host_call_end(h))) return rc;
  h->has_device_normals = true;
  h->has_normals = true;
  h->has_sampler = false;          // the sampler must be (re)armed with artp_set_sampler
  h->stats.kernel_launches += 1;
  h->stats.last_launches = 1;
  return ARTP_OK;
}

// computeCumulativeProbabilityDistribution of a device-resident probability layer into cum_prob / cum_row of
// d_samp_layers (ensure_sampler_layers first). Two launches on s.
static int launch_sample_cdf(Handle* h, const float* d_prob, cudaStream_t s) {
  const size_t ncell = (size_t)h->rows * h->cols;
  float* d_cum = h->d_samp_layers + 4 * ncell;
  float* d_row = h->d_samp_layers + 5 * ncell;
  artp::cdf_rows_kernel<<<(h->rows + 63) / 64, 64, 0, s>>>(d_prob, h->rows, h->cols, d_cum, d_row);
  artp::cdf_rowwise_kernel<<<1, 32, 0, s>>>(d_row, h->rows);
  CU_TRY(h, cudaGetLastError());
  return ARTP_OK;
}

int artp_compute_sample_cdf(artp_handle* hh, const float* sample_probability, float* cum_prob, float* cum_prob_rowwise) {
  LOCK_HANDLE(h, hh);
  if (!h->has_map) { h->err = "no map set"; return ARTP_E_NOMAP; }
  if (h->win_rows != h->rows) { h->err = "not available on a map window (artp_set_map_window)"; return ARTP_E_INVALID; }
  if (!sample_probability) { h->err = "null buffer"; return ARTP_E_INVALID; }
  const size_t ncell = (size_t)h->rows * h->cols;
  char* d_prob;
  int rc = host_call_begin(h, {ncell * sizeof(float)}, &d_prob);
  if (rc) return rc;
  rc = ensure_sampler_layers(h);
  if (rc) return rc;
  float* d_cum = h->d_samp_layers + 4 * ncell;
  float* d_row = h->d_samp_layers + 5 * ncell;
  CU_TRY(h, cudaMemcpyAsync(d_prob, sample_probability, ncell * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  if ((rc = launch_sample_cdf(h, (const float*)d_prob, h->stream))) return rc;
  if (cum_prob) CU_TRY(h, cudaMemcpyAsync(cum_prob, d_cum, ncell * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  if (cum_prob_rowwise)
    CU_TRY(h, cudaMemcpyAsync(cum_prob_rowwise, d_row, (size_t)h->rows * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  if ((rc = host_call_end(h))) return rc;
  h->has_device_cdf = true;
  h->has_sampler = false;          // the sampler must be (re)armed with artp_set_sampler
  h->stats.kernel_launches += 2;
  h->stats.last_launches = 2;
  return ARTP_OK;
}

int artp_set_sampler(artp_handle* hh, const artp_sampler_params* sp, const float* normal_x, const float* normal_y,
                     const float* normal_z, const float* plane_fit_std_dev, const float* cum_prob,
                     const float* cum_prob_rowwise) {
  LOCK_HANDLE(h, hh);
  if (!h->has_map) { h->err = "no map set"; return ARTP_E_NOMAP; }
  if (h->win_rows != h->rows) { h->err = "not available on a map window (artp_set_map_window)"; return ARTP_E_INVALID; }
  const bool host_normals = normal_x && normal_y && normal_z && plane_fit_std_dev;
  if (!sp) { h->err = "null sampler params"; return ARTP_E_INVALID; }
  if (!host_normals && (normal_x || normal_y || normal_z || plane_fit_std_dev)) {
    h->err = "pass all four normal / plane-fit layers or none"; return ARTP_E_INVALID;
  }
  if (!host_normals && !h->has_device_normals) {
    h->err = "no normal layers: pass them or call artp_estimate_normals after artp_set_map"; return ARTP_E_INVALID;
  }
  const bool host_cdf = cum_prob && cum_prob_rowwise;
  if (sp->sample_from_distribution && !host_cdf && !(h->has_device_cdf && !cum_prob && !cum_prob_rowwise)) {
    h->err = "sample_from_distribution needs the cum_prob layers (pass both, or call artp_compute_sample_cdf first)";
    return ARTP_E_INVALID;
  }
  if (!sp->sample_from_distribution && !(sp->high[0] > sp->low[0] && sp->high[1] > sp->low[1])) {
    h->err = "empty sampling bounds"; return ARTP_E_INVALID;
  }
  const size_t ncell = (size_t)h->rows * h->cols;
  int rc = host_call_begin(h);
  if (rc) return rc;
  rc = ensure_sampler_layers(h);
  if (rc) return rc;
  float* base = h->d_samp_layers;
  if (host_normals) {
    const float* src[4] = {normal_x, normal_y, normal_z, plane_fit_std_dev};
    for (int k = 0; k < 4; ++k)
      CU_TRY(h, cudaMemcpyAsync(base + k * ncell, src[k], ncell * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    h->has_device_normals = false;   // overwritten by the caller's layers
    h->has_normals = true;
  }
  artp::SamplerDev& m = h->samp;
  sampler_map_view(h, m);
  m.cum_prob = nullptr; m.cum_row = nullptr;
  m.max_roll_pert = sp->max_roll_pert; m.max_pitch_pert = sp->max_pitch_pert;
  m.from_distribution = sp->sample_from_distribution ? 1 : 0;
  m.low[0] = sp->low[0]; m.low[1] = sp->low[1]; m.high[0] = sp->high[0]; m.high[1] = sp->high[1];
  m.reach_z = h->p.reach_z;
  uint32_t bad = 0;
  if (m.from_distribution) {
    if (host_cdf) {
      CU_TRY(h, cudaMemcpyAsync(base + 4 * ncell, cum_prob, ncell * sizeof(float), cudaMemcpyHostToDevice, h->stream));
      CU_TRY(h, cudaMemcpyAsync(base + 5 * ncell, cum_prob_rowwise, (size_t)h->rows * sizeof(float), cudaMemcpyHostToDevice,
                                h->stream));
      h->has_device_cdf = false;   // overwritten by the caller's layers
    }
    m.cum_prob = base + 4 * ncell; m.cum_row = base + 5 * ncell;
    // the binary searches need monotone (or all-NaN) CDF rows: refuse anything else
    uint32_t* d_bad = &h->d_ctr->scratch;
    CU_TRY(h, cudaMemsetAsync(d_bad, 0, sizeof(uint32_t), h->stream));
    artp::validate_cdf_kernel<<<(h->rows + 127) / 128, 128, 0, h->stream>>>(m.cum_prob, h->rows, h->cols, (size_t)h->rows, 1, d_bad);
    artp::validate_cdf_kernel<<<1, 32, 0, h->stream>>>(m.cum_row, 1, h->rows, 1, 0, d_bad);
    CU_TRY(h, cudaGetLastError());
    CU_TRY(h, cudaMemcpyAsync(&bad, d_bad, sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
  }
  if ((rc = host_call_end(h))) return rc;
  if (m.from_distribution) h->stats.kernel_launches += 2;
  if (bad) { h->err = "cum_prob layers are not cumulative distributions (rows must be non-decreasing or all NaN)"; return ARTP_E_INVALID; }
  h->has_sampler = true;
  return ARTP_OK;
}

static int sampler_ready(Handle* h) {
  if (!h->has_map) { h->err = "no map set"; return ARTP_E_NOMAP; }
  if (!h->has_sampler) { h->err = "no sampler layers set (artp_set_sampler after artp_set_map)"; return ARTP_E_NOMAP; }
  return ARTP_OK;
}

static inline unsigned grid_for(Handle* h, size_t n, int block) {
  return (unsigned)std::min<size_t>((n + block - 1) / block, (size_t)h->sm_count * 16);
}

int artp_sampler_uniforms(artp_handle* hh, uint64_t seed, uint64_t first_sample, size_t n, double* u) {
  LOCK_HANDLE(h, hh);
  if (n == 0) return ARTP_OK;
  if (!u) { h->err = "null buffer"; return ARTP_E_INVALID; }
  char* d_u;
  int rc = host_call_begin(h, {n * 6 * sizeof(double)}, &d_u);
  if (rc) return rc;
  artp::sampler_uniforms_kernel<<<grid_for(h, n, 256), 256, 0, h->stream>>>(seed, first_sample, n, (double*)d_u);
  CU_TRY(h, cudaGetLastError());
  CU_TRY(h, cudaMemcpyAsync(u, d_u, n * 6 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  if ((rc = host_call_end(h))) return rc;
  h->stats.kernel_launches += 1;
  return ARTP_OK;
}

int artp_sample_states_device(artp_handle* hh, const double* d_u, uint64_t seed, uint64_t first_sample, size_t n,
                              double* d_states, int32_t* d_rowcol, void* stream) {
  LOCK_HANDLE(h, hh);
  int rc = sampler_ready(h);
  if (rc) return rc;
  if (n == 0) return ARTP_OK;
  if (!d_states) { h->err = "null buffer"; return ARTP_E_INVALID; }
  CU_TRY(h, cudaSetDevice(h->device));
  artp::sample_states_kernel<<<grid_for(h, n, 128), 128, 0, (cudaStream_t)stream>>>(h->samp, d_u, seed, first_sample, n, d_states,
                                                                                   nullptr, d_rowcol);
  CU_TRY(h, cudaGetLastError());
  h->stats.kernel_launches += 1;
  h->stats.last_launches = 1;
  return ARTP_OK;
}

int artp_sample_states(artp_handle* hh, const double* u, uint64_t seed, uint64_t first_sample, size_t n, double* states,
                       int32_t* rowcol) {
  LOCK_HANDLE(h, hh);
  int rc = sampler_ready(h);
  if (rc) return rc;
  if (n == 0) return ARTP_OK;
  if (!states) { h->err = "null buffer"; return ARTP_E_INVALID; }
  char* r[3];   // u | states | rowcol
  if ((rc = host_call_begin(h, {n * 6 * sizeof(double), n * 7 * sizeof(double), n * 2 * sizeof(int32_t)}, r))) return rc;
  if (u) CU_TRY(h, cudaMemcpyAsync(r[0], u, n * 6 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  rc = artp_sample_states_device(hh, u ? (const double*)r[0] : nullptr, seed, first_sample, n, (double*)r[1],
                                 rowcol ? (int32_t*)r[2] : nullptr, h->stream);
  if (rc) return rc;
  CU_TRY(h, cudaMemcpyAsync(states, r[1], n * 7 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  if (rowcol) CU_TRY(h, cudaMemcpyAsync(rowcol, r[2], n * 2 * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h);
}

// running total += chunk count (device-side, stream ordered)
__global__ void add_count_kernel(uint32_t* total, const uint32_t* chunk) { *total += *chunk; }

// out + 7 * (*total) .. : ordered gather of this chunk's valid candidates behind the previous chunks'
__global__ void gather_chunk_kernel(const double* __restrict__ states, const int64_t* __restrict__ idx,
                                    const uint32_t* __restrict__ chunk_count, const uint32_t* __restrict__ total_before,
                                    size_t capacity, double* __restrict__ out) {
  const size_t before = *total_before;
  const size_t room = capacity > before ? capacity - before : 0;
  const size_t cc = *chunk_count;
  const size_t keep = cc < room ? cc : room;
  const size_t n = keep * 7;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const size_t k = i / 7, c = i - k * 7;
    out[before * 7 + i] = states[(size_t)idx[k] * 7 + c];
  }
}

static constexpr size_t kSampleChunk = (size_t)1 << 21;

int artp_sample_valid_device(artp_handle* hh, uint64_t seed, uint64_t first_sample, size_t n_draw, double* d_states_out,
                             size_t capacity, uint32_t* d_count, void* stream) {
  LOCK_HANDLE(h, hh);
  int rc = sampler_ready(h);
  if (rc) return rc;
  if (!d_count || (capacity && !d_states_out)) { h->err = "null buffer"; return ARTP_E_INVALID; }
  CU_TRY(h, cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  CU_TRY(h, cudaMemsetAsync(d_count, 0, sizeof(uint32_t), s));
  if (n_draw == 0) return ARTP_OK;
  ChainScope cs(h, 0, s);
  if (cs.rc) return cs.rc;
  const size_t chunk = std::min(n_draw, kSampleChunk);
  // scratch: states f64 | states f32 | indices | valid | chunk count
  const size_t o_f32 = chunk * 7 * sizeof(double), o_idx = o_f32 + ((chunk * 7 * sizeof(float) + 255) & ~(size_t)255),
               o_val = o_idx + chunk * sizeof(int64_t), o_cnt = o_val + ((chunk + 255) & ~(size_t)255), total = o_cnt + 256;
  if ((rc = grow(h, h->d_samp_scratch, h->samp_scratch_cap, total))) return rc;
  char* sc = h->d_samp_scratch;
  double* d_st = (double*)sc;
  float* d_sf = (float*)(sc + o_f32);
  int64_t* d_idx = (int64_t*)(sc + o_idx);
  uint8_t* d_val = (uint8_t*)(sc + o_val);
  uint32_t* d_cnt = (uint32_t*)(sc + o_cnt);
  uint32_t launches = 0;
  for (size_t done = 0; done < n_draw; done += chunk) {
    const size_t m = std::min(chunk, n_draw - done);
    artp::sample_states_kernel<<<grid_for(h, m, 128), 128, 0, s>>>(h->samp, nullptr, seed, first_sample + done, m, d_st, d_sf,
                                                                   nullptr);
    CU_TRY(h, cudaGetLastError());
    artp::Work w;
    w.s1 = nullptr; w.s2 = nullptr; w.s2f = d_sf; w.valid = d_val; w.item_base = 0; w.n_items = (uint32_t)m; w.steps = 0;
    w.edge_mode = 0;
    rc = run_items(h, w, s);
    if (rc) return rc;
    launches += h->stats.last_launches + 1;
    if (!h->samp.from_distribution) {   // rejected (outside-map) candidates carry NaN states
      artp::reject_nan_kernel<<<grid_for(h, m, 256), 256, 0, s>>>(d_st, m, d_val);
      launches += 1;
    }
    rc = compact_valid_impl(h, d_val, m, 0, d_idx, d_cnt, s);
    if (rc) return rc;
    gather_chunk_kernel<<<grid_for(h, m * 7, 256), 256, 0, s>>>(d_st, d_idx, d_cnt, d_count, capacity, d_states_out);
    add_count_kernel<<<1, 1, 0, s>>>(d_count, d_cnt);
    CU_TRY(h, cudaGetLastError());
    launches += 5;
    h->stats.kernel_launches += 3 + (h->samp.from_distribution ? 0 : 1);
    h->stats.poses_checked += m;
  }
  h->stats.last_launches = launches;
  return ARTP_OK;
}

int artp_sample_valid(artp_handle* hh, uint64_t seed, uint64_t first_sample, size_t n_draw, double* states, size_t capacity,
                      size_t* n_valid) {
  LOCK_HANDLE(h, hh);
  const size_t cap = std::min(capacity, n_draw);
  int rc = sampler_ready(h);
  if (rc) return rc;
  if (!n_valid || (cap && !states)) { h->err = "null buffer"; return ARTP_E_INVALID; }
  char* r[2];   // states | count
  if ((rc = host_call_begin(h, {cap * 7 * sizeof(double), sizeof(uint32_t)}, r))) return rc;
  rc = artp_sample_valid_device(hh, seed, first_sample, n_draw, (double*)r[0], cap, (uint32_t*)r[1], h->stream);
  if (rc) return rc;
  uint32_t cnt = 0;
  CU_TRY(h, cudaMemcpyAsync(&cnt, r[1], sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
  rc = host_call_end(h, true);
  if (rc == ARTP_E_CUDA) return rc;
  const size_t keep = std::min<size_t>(cnt, cap);
  if (keep) {   // the copy's size is the count: it follows the call's end (d_stage is still ours: the lock is held)
    CU_TRY(h, cudaMemcpyAsync(states, r[0], keep * 7 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(h, cudaStreamSynchronize(h->stream));
  }
  *n_valid = cnt;      // > capacity means the output was truncated to `capacity` states
  return rc;
}

// ---------------------------------------------------------------------------------------------------------------
// Start / goal repair: StartState / GoalStateRegion::sampleGoal (start.cpp:7-41, goal.cpp:11-41), and the goal's
// projection onto the map (planner.cpp:223-237, map.cpp:77-90)
// ---------------------------------------------------------------------------------------------------------------
// Argument checks shared by both forms; `radius` only when it is a host buffer.
static int ball_search_args(Handle* h, size_t n, uint32_t n_iter, const double* radius) {
  if (!h->has_map) { h->err = "no map set"; return ARTP_E_NOMAP; }
  if ((uint64_t)n >= (1ull << 32) || n * ((uint64_t)n_iter + 1) >= (1ull << 32)) {
    h->err = "n * (n_iter + 1) candidates must be < 2^32"; return ARTP_E_INVALID;
  }
  if (radius)
    for (size_t q = 0; q < n; ++q)
      if (!(radius[q] >= 0.0 && std::isfinite(radius[q]))) { h->err = "radius must be finite and >= 0"; return ARTP_E_INVALID; }
  return ARTP_OK;
}

int artp_find_valid_near_device(artp_handle* hh, const double* d_centres, size_t n, const double* d_radius, uint32_t n_iter,
                                const double* d_offsets, uint64_t seed, uint64_t first_draw, double* d_states_out,
                                int32_t* d_index, void* stream) {
  LOCK_HANDLE(h, hh);
  int rc = ball_search_args(h, n, n_iter, nullptr);
  if (rc) return rc;
  if (n == 0) return ARTP_OK;
  if (!d_centres || !d_radius || !d_states_out || !d_index) { h->err = "null buffer"; return ARTP_E_INVALID; }
  CU_TRY(h, cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  ChainScope cs(h, 0, s);
  if (cs.rc) return cs.rc;
  const uint64_t total = n * ((uint64_t)n_iter + 1);
  const size_t chunk = (size_t)std::min<uint64_t>(total, kSampleChunk);
  // scratch: candidate states f32 | verdicts | first valid candidate per query
  const size_t o_val = (chunk * 7 * sizeof(float) + 255) & ~(size_t)255, o_best = o_val + ((chunk + 255) & ~(size_t)255);
  if ((rc = grow(h, h->d_samp_scratch, h->samp_scratch_cap, o_best + n * sizeof(uint32_t)))) return rc;
  float* d_sf = (float*)h->d_samp_scratch;
  uint8_t* d_val = (uint8_t*)(h->d_samp_scratch + o_val);
  uint32_t* d_best = (uint32_t*)(h->d_samp_scratch + o_best);
  artp::BallSearch b{d_centres, d_radius, d_offsets, seed, first_draw, n_iter};
  CU_TRY(h, cudaMemsetAsync(d_best, 0xFF, n * sizeof(uint32_t), s));
  uint32_t launches = 0;
  for (uint64_t c0 = 0; c0 < total; c0 += chunk) {
    const size_t m = (size_t)std::min<uint64_t>(chunk, total - c0);
    artp::ball_candidates_kernel<<<grid_for(h, m, 128), 128, 0, s>>>(b, c0, m, d_sf);
    CU_TRY(h, cudaGetLastError());
    artp::Work w;
    w.s1 = nullptr; w.s2 = nullptr; w.s2f = d_sf; w.valid = d_val; w.item_base = 0; w.n_items = (uint32_t)m; w.steps = 0;
    w.edge_mode = 0;
    if ((rc = run_items(h, w, s))) return rc;
    launches += h->stats.last_launches + 2;
    artp::ball_first_valid_kernel<<<grid_for(h, m, 256), 256, 0, s>>>(d_val, c0, m, n_iter, d_best);
    CU_TRY(h, cudaGetLastError());
    h->stats.kernel_launches += 2;
    h->stats.poses_checked += m;
  }
  artp::ball_result_kernel<<<grid_for(h, n, 128), 128, 0, s>>>(b, n, d_best, d_states_out, d_index);
  CU_TRY(h, cudaGetLastError());
  h->stats.kernel_launches += 1;
  h->stats.last_launches = launches + 1;
  return ARTP_OK;
}

int artp_find_valid_near(artp_handle* hh, const double* centres, size_t n, const double* radius, uint32_t n_iter,
                         const double* offsets, uint64_t seed, uint64_t first_draw, double* states_out, int32_t* index) {
  LOCK_HANDLE(h, hh);
  if (n && (!centres || !radius || !states_out || !index)) { h->err = "null buffer"; return ARTP_E_INVALID; }
  int rc = ball_search_args(h, n, n_iter, radius);
  if (rc) return rc;
  if (n == 0) return ARTP_OK;
  const size_t sb = n * 7 * sizeof(double), ob = offsets ? n * (size_t)n_iter * 2 * sizeof(double) : 0;
  char* r[5];   // centres | radius | offsets | states | index
  if ((rc = host_call_begin(h, {sb, n * sizeof(double), ob, sb, n * sizeof(int32_t)}, r))) return rc;
  CU_TRY(h, cudaMemcpyAsync(r[0], centres, sb, cudaMemcpyHostToDevice, h->stream));
  CU_TRY(h, cudaMemcpyAsync(r[1], radius, n * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  if (ob) CU_TRY(h, cudaMemcpyAsync(r[2], offsets, ob, cudaMemcpyHostToDevice, h->stream));
  rc = artp_find_valid_near_device(hh, (const double*)r[0], n, (const double*)r[1], n_iter, offsets ? (const double*)r[2] : nullptr,
                                   seed, first_draw, (double*)r[3], (int32_t*)r[4], h->stream);
  if (rc) return rc;
  CU_TRY(h, cudaMemcpyAsync(states_out, r[3], sb, cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(h, cudaMemcpyAsync(index, r[4], n * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h, true);
}

int artp_ball_offsets(artp_handle* hh, uint64_t seed, uint64_t first_draw, size_t n, uint32_t n_iter, const double* radius,
                      double* offsets) {
  LOCK_HANDLE(h, hh);
  const size_t total = n * (size_t)n_iter;
  if (total == 0) return ARTP_OK;
  if (!radius || !offsets) { h->err = "null buffer"; return ARTP_E_INVALID; }
  if ((uint64_t)n >= (1ull << 32)) { h->err = "n must be < 2^32"; return ARTP_E_INVALID; }
  char* r[2];   // radius | offsets
  int rc = host_call_begin(h, {n * sizeof(double), total * 2 * sizeof(double)}, r);
  if (rc) return rc;
  CU_TRY(h, cudaMemcpyAsync(r[0], radius, n * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  artp::ball_offsets_kernel<<<grid_for(h, total, 256), 256, 0, h->stream>>>(seed, first_draw, n, n_iter, (const double*)r[0],
                                                                            (double*)r[1]);
  CU_TRY(h, cudaGetLastError());
  CU_TRY(h, cudaMemcpyAsync(offsets, r[1], total * 2 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  if ((rc = host_call_end(h))) return rc;
  h->stats.kernel_launches += 1;
  h->stats.last_launches = 1;
  return ARTP_OK;
}

int artp_pose_from_2d(artp_handle* hh, const double* states_in, size_t n, double* states_out, uint8_t* inside) {
  LOCK_HANDLE(h, hh);
  if (!h->has_map) { h->err = "no map set"; return ARTP_E_NOMAP; }
  if (h->win_rows != h->rows) { h->err = "not available on a map window (artp_set_map_window)"; return ARTP_E_INVALID; }
  if (!h->has_normals) {
    h->err = "no normal layers for this map (artp_estimate_normals or artp_set_sampler after artp_set_map)"; return ARTP_E_INVALID;
  }
  if (n == 0) return ARTP_OK;
  if (!states_in || !states_out) { h->err = "null buffer"; return ARTP_E_INVALID; }
  char* r[3];   // states in | states out | inside
  int rc = host_call_begin(h, {n * 7 * sizeof(double), n * 7 * sizeof(double), n}, r);
  if (rc) return rc;
  artp::SamplerDev m{};
  sampler_map_view(h, m);
  CU_TRY(h, cudaMemcpyAsync(r[0], states_in, n * 7 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  artp::pose_from_2d_kernel<<<grid_for(h, n, 128), 128, 0, h->stream>>>(m, (const double*)r[0], n, (double*)r[1], (uint8_t*)r[2]);
  CU_TRY(h, cudaGetLastError());
  CU_TRY(h, cudaMemcpyAsync(states_out, r[1], n * 7 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  if (inside) CU_TRY(h, cudaMemcpyAsync(inside, r[2], n, cudaMemcpyDeviceToHost, h->stream));
  if ((rc = host_call_end(h))) return rc;
  h->stats.kernel_launches += 1;
  h->stats.last_launches = 1;
  return ARTP_OK;
}

// cv::circle(kernel, (r, r), r, 255, FILLED) on a size x size zero image, r = size / 2 (utils.cpp:106-111): OpenCV's
// integer midpoint circle (imgproc/src/drawing.cpp, Circle()): for every step (dx, dy) of the octant walk the rows
// cy -+ dy get the span cx -+ dx and the rows cy -+ dx the span cx -+ dy, everything clipped to the image.
static artp::MorphKernel make_circular_kernel(int size) {
  artp::MorphKernel k;
  std::memset(&k, 0, sizeof(k));
  if (size <= 0) {   // empty element: cv::erode / cv::dilate fall back to the 3 x 3 box, anchor (1, 1)
    k.size = 3; k.anchor = 1;
    for (int r = 0; r < 3; ++r) { k.lo[r] = 0; k.hi[r] = 2; }
    return k;
  }
  k.size = size; k.anchor = size / 2;
  for (int r = 0; r < size; ++r) { k.lo[r] = 127; k.hi[r] = -1; }
  const int radius = size / 2, cx = radius, cy = radius;
  auto span = [&](int y, int x0, int x1) {
    if (y < 0 || y >= size) return;
    x0 = std::max(x0, 0); x1 = std::min(x1, size - 1);
    if (x0 > x1) return;
    k.lo[y] = (int8_t)std::min<int>(k.lo[y], x0); k.hi[y] = (int8_t)std::max<int>(k.hi[y], x1);
  };
  int err = 0, dx = radius, dy = 0, plus = 1, minus = (radius << 1) - 1;
  while (dx >= dy) {
    span(cy - dy, cx - dx, cx + dx); span(cy + dy, cx - dx, cx + dx);
    span(cy - dx, cx - dy, cx + dy); span(cy + dx, cx - dy, cx + dy);
    dy++; err += plus; plus += 2;
    const int mask = (err <= 0) - 1;
    err -= minus & mask; dx += mask; minus -= mask & 2;
  }
  return k;
}

int artp_debug_circular_kernel(int size, uint8_t* out) {   // test hook: the size x size element as 0 / 1 bytes (row-major)
  if (size > artp::kMaxMorph || !out) return ARTP_E_INVALID;
  const artp::MorphKernel k = make_circular_kernel(size);
  for (int r = 0; r < k.size; ++r) for (int c = 0; c < k.size; ++c) out[r * k.size + c] = (c >= k.lo[r] && c <= k.hi[r]) ? 1 : 0;
  return k.size;
}

// cv::dilate / cv::erode of a rows x cols layer with getCircularKernel(size), one launch on s.
static void launch_morph(bool dilate, const float* src, float* dst, int rows, int cols, int size, unsigned grid, cudaStream_t s) {
  const artp::MorphKernel k = make_circular_kernel(size);
  if (dilate) artp::morph_kernel<true><<<grid, 256, 0, s>>>(src, dst, rows, cols, k);
  else artp::morph_kernel<false><<<grid, 256, 0, s>>>(src, dst, rows, cols, k);
}

int artp_process_basic(artp_handle* hh, const float* elevation, const float* traversability, const float* observed, int rows,
                       int cols, double res, const artp_basic_params* bp, float* elevation_masked, float* traversability_thresholded) {
  LOCK_HANDLE(h, hh);
  if (!elevation || !traversability || !bp || !elevation_masked || rows < 1 || cols < 1 || !(res > 0)) {
    h->err = "bad arguments"; return ARTP_E_INVALID;
  }
  if (bp->unknown_space_untraversable && !observed) { h->err = "unknown_space_untraversable needs the observed layer"; return ARTP_E_INVALID; }
  // basic.cpp:65-74: cell counts of the structuring elements
  const int foothold = (int)std::ceil(bp->foothold_size / res), margin = (int)std::ceil(2 * bp->foothold_margin / res),
            hole = (int)std::floor(bp->foothold_margin_max_hole_size / res),
            search = (int)std::ceil(2 * bp->foothold_margin_max_drop_search_radius / res);
  if (std::max(std::max(foothold, margin), std::max(hole, search)) > artp::kMaxMorph) {
    h->err = "structuring element larger than 64 cells"; return ARTP_E_LIMIT;
  }
  const size_t n = (size_t)rows * cols, lb = n * sizeof(float);
  char* stage;
  int rc = host_call_begin(h, {9 * lb}, &stage);
  if (rc) return rc;
  h->has_basic_layers = false;
  if ((rc = grow(h, h->d_basic_keep, h->basic_keep_cap, 2 * n))) return rc;
  float* L = (float*)stage;   // 0 elev, 1 trav, 2 observed, 3 T0, 4 A, 5 B, 6 elev eroded, 7 elev dilated, 8 out
  cudaStream_t s = h->stream;
  CU_TRY(h, cudaMemcpyAsync(L, elevation, lb, cudaMemcpyHostToDevice, s));
  CU_TRY(h, cudaMemcpyAsync(L + n, traversability, lb, cudaMemcpyHostToDevice, s));
  if (observed) CU_TRY(h, cudaMemcpyAsync(L + 2 * n, observed, lb, cudaMemcpyHostToDevice, s));
  const unsigned grid = (unsigned)std::min<size_t>((n + 255) / 256, (size_t)h->sm_count * 16);
  auto morph = [&](bool dil, const float* src, float* dst, int size) { launch_morph(dil, src, dst, rows, cols, size, grid, s); };
  float *E = L, *T0 = L + 3 * n, *A = L + 4 * n, *B = L + 5 * n, *Elo = L + 6 * n, *Ehi = L + 7 * n, *O = L + 8 * n;
  artp::basic_threshold_kernel<<<grid, 256, 0, s>>>(L + n, L + 2 * n, bp->unknown_space_untraversable ? 1 : 0, bp->traversability_thres, n, T0);
  morph(true, T0, A, hole); morph(false, A, B, hole);                    // dilateAndErode: close holes (:72)
  morph(false, E, Elo, search);                                          // elevation - erode(elevation) (:75-77)
  morph(true, E, Ehi, margin);                                           // dilate(elevation) - elevation (:84)
  artp::basic_select_kernel<<<grid, 256, 0, s>>>(0, E, Elo, Ehi, T0, B, (float)bp->foothold_margin_max_drop, (float)bp->foothold_margin_min_step, n, A);
  morph(false, A, B, margin);                                            // erode by the safety margin (:90)
  artp::basic_select_kernel<<<grid, 256, 0, s>>>(1, E, Elo, Ehi, T0, B, (float)bp->foothold_margin_max_drop, (float)bp->foothold_margin_min_step, n, A);
  morph(false, A, B, foothold); morph(true, B, A, foothold);             // erodeAndDilate: remove small patches (:95)
  artp::basic_final_kernel<<<grid, 256, 0, s>>>(E, T0, A, n, B, O);
  CU_TRY(h, cudaGetLastError());
  CU_TRY(h, cudaMemcpyAsync(elevation_masked, O, lb, cudaMemcpyDeviceToHost, s));
  if (traversability_thresholded) CU_TRY(h, cudaMemcpyAsync(traversability_thresholded, B, lb, cudaMemcpyDeviceToHost, s));
  // kept for artp_set_sample_filter(h, NULL, NULL, ...)
  if (observed) CU_TRY(h, cudaMemcpyAsync(h->d_basic_keep, L + 2 * n, lb, cudaMemcpyDeviceToDevice, s));
  CU_TRY(h, cudaMemcpyAsync(h->d_basic_keep + n, B, lb, cudaMemcpyDeviceToDevice, s));
  if ((rc = host_call_end(h))) return rc;
  h->basic_rows = rows; h->basic_cols = cols;
  h->has_basic_layers = true;
  h->has_basic_observed = observed != nullptr;
  h->stats.kernel_launches += 11;
  h->stats.last_launches = 11;
  return ARTP_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// The sampler's distribution (artp_distribution.cuh): Basic::setTraversabilityFilter, then computeInverseSampleDensity ->
// applyBaseSampleDistribution -> applyMaxUnknownProbability -> computeCumulativeProbabilityDistribution
// (planner.cpp:39-58), the chain sampleGraph re-applies every recompute_density_after_n_samples vertices.
// ---------------------------------------------------------------------------------------------------------------
int artp_set_sample_filter(artp_handle* hh, const float* traversability_thresholded, const float* observed,
                           float* traversability_sample_filter) {
  LOCK_HANDLE(h, hh);
  if (!h->has_map) { h->err = "no map set"; return ARTP_E_NOMAP; }
  if (h->win_rows != h->rows) { h->err = "not available on a map window (artp_set_map_window)"; return ARTP_E_INVALID; }
  const int rows = h->rows, cols = h->cols;
  const bool basic_fits = h->has_basic_layers && h->basic_rows == rows && h->basic_cols == cols;
  if (!traversability_thresholded && !basic_fits) {
    h->err = "no traversability_thresholded layer: pass it, or run artp_process_basic on a map of this size first";
    return ARTP_E_INVALID;
  }
  const bool basic_observed = !observed && basic_fits && h->has_basic_observed;
  // basic.cpp:116-122, with the implicit double -> int conversions of the int size parameters
  const artp_params& p = h->p;
  const int reach = (int)(std::sqrt(p.reach_x * p.reach_x + p.reach_y * p.reach_y) / h->res);
  const int wall = (int)(std::min((p.torso_length - p.reach_x) * 0.5, (p.torso_width - p.reach_y) * 0.5) / h->res);
  if (std::max(reach, wall) > artp::kMaxMorph) { h->err = "structuring element larger than 64 cells"; return ARTP_E_LIMIT; }
  const size_t n = (size_t)rows * cols, lb = n * sizeof(float);
  char* r[3];   // caller's traversability_thresholded | dilated | closed
  int rc = host_call_begin(h, {lb, lb, lb}, r);
  if (rc) return rc;
  h->has_sample_filter = h->has_dist_observed = false;
  if ((rc = grow(h, h->d_dist_layers, h->dist_layers_cap, 2 * n))) return rc;
  cudaStream_t s = h->stream;
  float *filter = h->d_dist_layers, *obs = h->d_dist_layers + n;
  const float* thr = traversability_thresholded ? (const float*)r[0] : h->d_basic_keep + n;
  if (traversability_thresholded) CU_TRY(h, cudaMemcpyAsync(r[0], traversability_thresholded, lb, cudaMemcpyHostToDevice, s));
  if (observed) CU_TRY(h, cudaMemcpyAsync(obs, observed, lb, cudaMemcpyHostToDevice, s));
  if (basic_observed) CU_TRY(h, cudaMemcpyAsync(obs, h->d_basic_keep, lb, cudaMemcpyDeviceToDevice, s));
  const unsigned grid = grid_for(h, n, 256);
  launch_morph(true, thr, (float*)r[1], rows, cols, reach, grid, s);              // dilateAndErode: step over small obstacles
  launch_morph(false, (float*)r[1], (float*)r[2], rows, cols, reach, grid, s);
  launch_morph(false, (float*)r[2], filter, rows, cols, wall, grid, s);           // erode: keep away from walls
  CU_TRY(h, cudaGetLastError());
  if (traversability_sample_filter)
    CU_TRY(h, cudaMemcpyAsync(traversability_sample_filter, filter, lb, cudaMemcpyDeviceToHost, s));
  if ((rc = host_call_end(h))) return rc;
  h->has_sample_filter = true;
  h->has_dist_observed = observed || basic_observed;
  h->stats.kernel_launches += 3;
  h->stats.last_launches = 3;
  return ARTP_OK;
}

// getGaussianKernel(ksize, sigma, CV_32F) for sigma > 0: exp(-x^2 / (2 sigma^2)) at x = i - (ksize - 1) / 2, normalised
// by the double sum, then cast to float -- equal to OpenCV's coefficients (tests/test_sample_distribution_cpu.py).
static artp::GaussTaps gauss_taps(int ksize, double sigma) {
  artp::GaussTaps k;
  std::memset(&k, 0, sizeof(k));
  std::vector<double> v(ksize);
  const double scale2X = -0.5 / (sigma * sigma);
  double sum = 0.0;
  for (int i = 0; i < ksize; ++i) {
    const double x = i - (ksize - 1) * 0.5;
    v[i] = std::exp(scale2X * (x * x));
    sum += v[i];
  }
  const double inv = 1.0 / sum;
  k.half = ksize / 2;
  for (int t = 0; t <= k.half; ++t) k.w[t] = (float)(v[k.half + t] * inv);
  return k;
}

int artp_debug_gaussian_kernel(int ksize, double sigma, float* out) {   // test hook: the ksize coefficients
  if (ksize < 1 || ksize > artp::kMaxGaussTaps || !(ksize & 1) || !(sigma > 0) || !out) return ARTP_E_INVALID;
  const artp::GaussTaps k = gauss_taps(ksize, sigma);
  for (int i = 0; i < ksize; ++i) out[i] = k.w[std::abs(i - k.half)];
  return ksize;
}

// Argument checks shared by both forms; the blur's kernel size and sigma in cells (sample_density.cpp:33-35).
static int distribution_args(Handle* h, const artp_sample_distribution_params* dp, int* ksize, double* sigma) {
  if (!h->has_map) { h->err = "no map set"; return ARTP_E_NOMAP; }
  if (h->win_rows != h->rows) { h->err = "not available on a map window (artp_set_map_window)"; return ARTP_E_INVALID; }
  if (!dp) { h->err = "null distribution params"; return ARTP_E_INVALID; }
  *ksize = 0; *sigma = 0.0;
  if (dp->use_inverse_vertex_density) {
    if (!(dp->density_blur_radius > 0.0 && std::isfinite(dp->density_blur_radius))) {
      h->err = "density_blur_radius must be finite and > 0"; return ARTP_E_INVALID;
    }
    const double cells = 6 * dp->density_blur_radius / h->res;
    if (!(cells < artp::kMaxGaussTaps + 1)) { h->err = "Gaussian kernel larger than 1023 cells"; return ARTP_E_LIMIT; }
    int k = (int)cells;
    if (k % 2 == 0) k += 1;
    if (k > artp::kMaxGaussTaps) { h->err = "Gaussian kernel larger than 1023 cells"; return ARTP_E_LIMIT; }
    *ksize = k;
    *sigma = dp->density_blur_radius / h->res;
  }
  if (dp->use_max_prob_unknown_samples) {
    if (!(dp->max_prob_unknown_samples >= 0.0 && dp->max_prob_unknown_samples <= 1.0)) {
      h->err = "max_prob_unknown_samples must lie in [0, 1]"; return ARTP_E_INVALID;
    }
    if (!h->has_dist_observed) {
      h->err = "the unknown-space cap needs the observed layer (artp_set_sample_filter after artp_set_map)"; return ARTP_E_INVALID;
    }
  }
  return ARTP_OK;
}

// Scratch of one update: n_samples | blur pass | sample_probability | known row sums | unknown row sums | max bits, mult[2].
struct DistScratch { float *n_samples, *pass, *prob; double *known, *unknown; unsigned int* max_bits; float* mult; };
static int dist_scratch(Handle* h, DistScratch* d) {
  const size_t lb = ((size_t)h->rows * h->cols * sizeof(float) + 255) & ~(size_t)255, rb = ((size_t)h->rows * sizeof(double) + 255) & ~(size_t)255;
  int rc = grow(h, h->d_dist_scratch, h->dist_scratch_cap, 3 * lb + 2 * rb + 256);
  if (rc) return rc;
  char* b = h->d_dist_scratch;
  d->n_samples = (float*)b; d->pass = (float*)(b + lb); d->prob = (float*)(b + 2 * lb);
  d->known = (double*)(b + 3 * lb); d->unknown = (double*)(b + 3 * lb + rb);
  d->max_bits = (unsigned int*)(b + 3 * lb + 2 * rb); d->mult = (float*)(b + 3 * lb + 2 * rb + 64);
  return ARTP_OK;
}

// The chain on s into d->prob and the sampler's CDF layers; arguments checked by distribution_args.
static int update_distribution(Handle* h, const artp_sample_distribution_params* dp, int ksize, double sigma,
                               const double* d_states, size_t n, cudaStream_t s, DistScratch* d) {
  int rc;
  if ((rc = ensure_sampler_layers(h)) || (rc = dist_scratch(h, d))) return rc;
  const int rows = h->rows, cols = h->cols;
  const size_t ncell = (size_t)rows * cols;
  const unsigned grid = grid_for(h, ncell, 256);
  uint32_t launches = 0;
  const float* n_blur = nullptr;
  if (dp->use_inverse_vertex_density) {                                          // sample_density.cpp:21-42
    CU_TRY(h, cudaMemsetAsync(d->n_samples, 0, ncell * sizeof(float), s));
    CU_TRY(h, cudaMemsetAsync(d->max_bits, 0, sizeof(unsigned int), s));
    if (n) {
      artp::SamplerDev m{};
      sampler_map_view(h, m);
      artp::vertex_histogram_kernel<<<grid_for(h, n, 256), 256, 0, s>>>(m, d_states, n, d->n_samples);
      ++launches;
    }
    const artp::GaussTaps k = gauss_taps(ksize, sigma);
    artp::gauss_pass_kernel<0><<<grid, 256, 0, s>>>(d->n_samples, d->pass, rows, cols, k);
    artp::gauss_pass_kernel<1><<<grid, 256, 0, s>>>(d->pass, d->n_samples, rows, cols, k);
    artp::abs_max_kernel<<<grid, 256, 0, s>>>(d->n_samples, ncell, d->max_bits);
    launches += 3;
    n_blur = d->n_samples;
  }
  artp::combine_kernel<<<grid, 256, 0, s>>>(n_blur, d->max_bits, h->has_sample_filter ? h->d_dist_layers : nullptr, ncell, d->prob);
  ++launches;
  if (dp->use_max_prob_unknown_samples) {                                        // probability_distribution.cpp:50-91
    const float* obs = h->d_dist_layers + ncell;
    artp::cap_rows_kernel<<<(rows + 63) / 64, 64, 0, s>>>(d->prob, obs, rows, cols, d->known, d->unknown);
    artp::cap_mult_kernel<<<1, 32, 0, s>>>(d->known, d->unknown, rows, dp->max_prob_unknown_samples, d->mult);
    artp::cap_apply_kernel<<<grid, 256, 0, s>>>(d->prob, obs, d->mult, ncell);
    launches += 3;
  }
  CU_TRY(h, cudaGetLastError());
  if ((rc = launch_sample_cdf(h, d->prob, s))) return rc;
  launches += 2;
  h->has_device_cdf = true;
  h->has_sampler = false;          // the sampler must be (re)armed with artp_set_sampler
  h->stats.kernel_launches += launches;
  h->stats.last_launches = launches;
  return ARTP_OK;
}

int artp_update_sample_distribution_device(artp_handle* hh, const artp_sample_distribution_params* dp,
                                           const double* d_vertex_states, size_t n, void* stream) {
  LOCK_HANDLE(h, hh);
  int ksize;
  double sigma;
  int rc = distribution_args(h, dp, &ksize, &sigma);
  if (rc) return rc;
  if (n && !d_vertex_states) { h->err = "null buffer"; return ARTP_E_INVALID; }
  CU_TRY(h, cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  ChainScope cs(h, 0, s);
  if (cs.rc) return cs.rc;
  DistScratch d;
  return update_distribution(h, dp, ksize, sigma, d_vertex_states, n, s, &d);
}

int artp_update_sample_distribution(artp_handle* hh, const artp_sample_distribution_params* dp, const double* vertex_states,
                                    size_t n, float* sample_probability, float* cum_prob, float* cum_prob_rowwise) {
  LOCK_HANDLE(h, hh);
  int ksize;
  double sigma;
  int rc = distribution_args(h, dp, &ksize, &sigma);
  if (rc) return rc;
  if (n && !vertex_states) { h->err = "null buffer"; return ARTP_E_INVALID; }
  const size_t sb = n * 7 * sizeof(double), ncell = (size_t)h->rows * h->cols;
  char* r[1];
  if ((rc = host_call_begin(h, {sb}, r))) return rc;
  if (n) CU_TRY(h, cudaMemcpyAsync(r[0], vertex_states, sb, cudaMemcpyHostToDevice, h->stream));
  DistScratch d;
  if ((rc = update_distribution(h, dp, ksize, sigma, (const double*)r[0], n, h->stream, &d))) return rc;
  if (sample_probability)
    CU_TRY(h, cudaMemcpyAsync(sample_probability, d.prob, ncell * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  if (cum_prob)
    CU_TRY(h, cudaMemcpyAsync(cum_prob, h->d_samp_layers + 4 * ncell, ncell * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  if (cum_prob_rowwise)
    CU_TRY(h, cudaMemcpyAsync(cum_prob_rowwise, h->d_samp_layers + 5 * ncell, (size_t)h->rows * sizeof(float),
                              cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h);
}

static_assert(ARTP_COST_NET_LIGHT == artp_cnn::kNetLight && ARTP_COST_NET_FULL == artp_cnn::kNetFull,
              "the ABI's network numbers are the library's");

size_t artp_cost_weights_size(void) { return artp_cnn::blob_floats(ARTP_COST_NET_LIGHT); }

size_t artp_cost_weights_size_for(int network) { return artp_cnn::blob_floats(network); }

int artp_get_cost_network(artp_handle* hh, int* network) {
  LOCK_HANDLE(h, hh);
  if (!network) return ARTP_E_INVALID;
  *network = artp_cnn::network(h->cnn);
  if (*network < 0) { h->err = "motion-cost weights not set"; return ARTP_E_NOWEIGHTS; }
  return ARTP_OK;
}

int artp_set_cost_weights(artp_handle* hh, const float* blob, size_t n_floats) {
  LOCK_HANDLE(h, hh);
  if (!blob) return ARTP_E_INVALID;
  return artp_cnn::set_weights(h->cnn, blob, n_floats, h->stream, h->err);
}

int artp_update_features(artp_handle* hh) {
  LOCK_HANDLE(h, hh);
  if (!h->has_map) { h->err = "no map set"; return ARTP_E_NOMAP; }
  if (h->win_rows != h->rows) { h->err = "not available on a map window (artp_set_map_window)"; return ARTP_E_INVALID; }
  return artp_cnn::update_features(h->cnn, h->d_H[0], h->rows, h->cols, h->pitch, h->chk.Lx / h->rows, h->chk.cx, h->chk.cy,
                                   h->stream, h->cnn_mode & 1, h->err);
}

int artp_motion_cost_device(artp_handle* hh, const float* d_edges, size_t n, float* d_cost3, void* stream) {
  LOCK_HANDLE(h, hh);
  if (n && (!d_edges || !d_cost3)) { h->err = "null buffer"; return ARTP_E_INVALID; }
  int rc = artp_cnn::motion_cost(h->cnn, d_edges, n, d_cost3, (cudaStream_t)stream, h->err);
  if (rc == 0 && n) { h->stats.kernel_launches += 1; h->stats.last_launches = 1; }
  return rc;
}

int artp_motion_cost(artp_handle* hh, const float* edges, size_t n, float* cost3) {
  LOCK_HANDLE(h, hh);
  if (n == 0) return ARTP_OK;
  if (!edges || !cost3) { h->err = "null buffer"; return ARTP_E_INVALID; }
  char* r[2];   // edges | cost3
  int rc = host_call_begin(h, {n * 6 * sizeof(float), n * 3 * sizeof(float)}, r);
  if (rc) return rc;
  CU_TRY(h, cudaMemcpyAsync(r[0], edges, n * 6 * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  rc = artp_motion_cost_device(hh, (const float*)r[0], n, (float*)r[1], h->stream);
  if (rc) return rc;
  CU_TRY(h, cudaMemcpyAsync(cost3, r[1], n * 3 * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h);
}

int artp_combine_cost(artp_handle* hh, const float* cost3, size_t n, double* cost, uint8_t* feasible) {
  if (!hh || (n && (!cost3 || !cost || !feasible))) return ARTP_E_INVALID;
  Handle* h = reinterpret_cast<Handle*>(hh);
  const float we = h->p.cost_w_energy, wt = h->p.cost_w_time, wr = h->p.cost_w_risk;
  for (size_t i = 0; i < n; ++i) {
    const float ce = cost3[3 * i], ct = cost3[3 * i + 1], cr = cost3[3 * i + 2];
    // getCost: getEnergy/getTime/getRisk return double (motion_cost_objective.h:30-46), so the weighted sum is evaluated
    // in double on exact float products
    cost[i] = (double)ce * (double)we + (double)ct * (double)wt + (double)cr * (double)wr;
    feasible[i] = (double)cr <= (double)h->p.risk_threshold ? 1 : 0;   // isFeasible (getRisk returns double)
  }
  return ARTP_OK;
}

static int check_cost_net(Handle* h) {
  if (!artp_cnn::has_weights(h->cnn)) { h->err = "motion-cost weights not set"; return ARTP_E_NOWEIGHTS; }
  if (!artp_cnn::has_features(h->cnn)) {
    h->err = "features not computed (call artp_update_features after artp_set_map)";
    return ARTP_E_NOWEIGHTS;
  }
  return ARTP_OK;
}

// Touches no per-handle scratch (the head reads the feature map and weights only), so, like artp_motion_cost_device, it
// joins no scratch group.
int artp_motion_cost_split_device(artp_handle* hh, const double* d_s1, const double* d_s2, size_t n,
                                  const uint32_t* d_piece_off, size_t total_pieces, float* d_rows, float* d_cost3,
                                  double* d_cost, void* stream) {
  LOCK_HANDLE(h, hh);
  if (n == 0) return ARTP_OK;
  if (!d_s1 || !d_s2 || !d_piece_off || !d_rows || !d_cost3 || !d_cost) { h->err = "null buffer"; return ARTP_E_INVALID; }
  if (total_pieces < n || total_pieces > 0xFFFFFFFFull) {
    h->err = "total_pieces must lie in [n, 2^32) (every edge has at least one piece)";
    return ARTP_E_INVALID;
  }
  int rc = check_cost_net(h);
  if (rc) return rc;
  CU_TRY(h, cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  split_rows_kernel<<<(unsigned)std::min<size_t>((total_pieces + 255) / 256, (size_t)h->sm_count * 8), 256, 0, s>>>(
      d_s1, d_s2, (uint32_t)n, d_piece_off, total_pieces, d_rows);
  CU_TRY(h, cudaGetLastError());
  if ((rc = artp_cnn::motion_cost(h->cnn, d_rows, total_pieces, d_cost3, s, h->err))) return rc;
  split_reduce_kernel<<<(unsigned)std::min<size_t>((n + 255) / 256, (size_t)h->sm_count * 8), 256, 0, s>>>(
      d_cost3, d_piece_off, n, h->p.cost_w_energy, h->p.cost_w_time, h->p.cost_w_risk, h->p.risk_threshold, d_cost);
  CU_TRY(h, cudaGetLastError());
  h->stats.kernel_launches += 3;
  h->stats.last_launches = 3;
  return ARTP_OK;
}

int artp_motion_cost_split(artp_handle* hh, const double* s1, const double* s2, size_t n, double max_query_edge_length,
                           double* cost) {
  LOCK_HANDLE(h, hh);
  if (n == 0) return ARTP_OK;
  if (!s1 || !s2 || !cost) { h->err = "null buffer"; return ARTP_E_INVALID; }
  if (!(max_query_edge_length > 0.0)) { h->err = "max_query_edge_length must be > 0"; return ARTP_E_INVALID; }
  int rc = check_cost_net(h);
  if (rc) return rc;
  std::vector<uint32_t> off(n + 1);
  size_t total = 0;
  for (size_t e = 0; e < n; ++e) {
    off[e] = (uint32_t)total;
    // n_interp = (unsigned)(lateralDistance (utils.h:52-61) / max_query_edge_length), motion_cost_objective.cpp:40-45
    const double dx = s2[7 * e] - s1[7 * e], dy = s2[7 * e + 1] - s1[7 * e + 1];
    const double q = std::sqrt(dx * dx + dy * dy) / max_query_edge_length;
    if (!(q < 4294967296.0)) { h->err = "edge too long or not finite (n_interp must fit 32 bits)"; return ARTP_E_INVALID; }
    total += (size_t)(unsigned int)q + 1;
    if (total > 0xFFFFFFFFull) { h->err = "too many pieces (>= 2^32)"; return ARTP_E_INVALID; }
  }
  off[n] = (uint32_t)total;
  const size_t sb = n * 7 * sizeof(double);
  char* r[6];   // s1 | s2 | piece offsets | rows | cost3 | cost
  rc = host_call_begin(h, {sb, sb, (n + 1) * sizeof(uint32_t), total * 6 * sizeof(float), total * 3 * sizeof(float),
                           n * sizeof(double)}, r);
  if (rc) return rc;
  CU_TRY(h, cudaMemcpyAsync(r[0], s1, sb, cudaMemcpyHostToDevice, h->stream));
  CU_TRY(h, cudaMemcpyAsync(r[1], s2, sb, cudaMemcpyHostToDevice, h->stream));
  CU_TRY(h, cudaMemcpyAsync(r[2], off.data(), (n + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
  rc = artp_motion_cost_split_device(hh, (const double*)r[0], (const double*)r[1], n, (const uint32_t*)r[2], total,
                                     (float*)r[3], (float*)r[4], (double*)r[5], h->stream);
  if (rc) return rc;
  CU_TRY(h, cudaMemcpyAsync(cost, r[5], n * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h);   // `off` outlives its H2D copy: the call synchronises before it returns
}

int artp_get_features(artp_handle* hh, float* out, size_t n_floats, int* hf, int* wf) {
  LOCK_HANDLE(h, hh);
  if (!hf || !wf) return ARTP_E_INVALID;
  artp_cnn::feature_shape(h->cnn, hf, wf);
  if (!out) return ARTP_OK;
  return artp_cnn::copy_features(h->cnn, out, n_floats, h->err);
}

int artp_set_cnn_mode(artp_handle* hh, int mode) {
  if (!hh) return ARTP_E_INVALID;
  Handle* h = reinterpret_cast<Handle*>(hh);
  if (mode & ~1) { h->err = "unknown motion-cost network mode (bit 0 is the only mode bit)"; return ARTP_E_INVALID; }
  h->cnn_mode = mode;
  return ARTP_OK;
}

int artp_get_cnn_timing(artp_handle* hh, float* ms3) {
  if (!hh || !ms3) return ARTP_E_INVALID;
  artp_cnn::last_times(reinterpret_cast<Handle*>(hh)->cnn, ms3);
  return ARTP_OK;
}

}  // extern "C"
