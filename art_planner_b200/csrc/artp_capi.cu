// art_planner_b200/csrc/artp_capi.cu -- C ABI (include/artp.h) over the sm_90a kernels: the handle, errors, stats and
// timing, the map upload, the validity pipeline with the pose / motion / edge checks, compaction and bit packing. The
// sampler and the learned cost live in artp_sampling.cu and artp_cost.cu; artp_internal.h holds what the units share.
// Host side mirrors the reference's checker objects: artp_create ~ StateValidityChecker ctor,
// artp_set_map ~ setMap + updateHeightField (HeightMapBoxChecker::setHeightField,
// art_planner/src/validity_checker/height_map_box_checker.cpp:38-54), artp_check_* ~ isValid / checkMotion.
// No CPU fallback: every entry point fails with ARTP_E_CUDA if the device or the kernel image is unusable.
#include <cassert>
#include <climits>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <cudaTypedefs.h>
#include <type_traits>
#include <vector>

#include "artp_internal.h"
#include "artp_kernels.cuh"
#include "artp_tiles.cuh"

namespace artp_api {

constexpr int kMaxSlices = 9;   // H2D slices per host-fed round: at most 8 scheduled fractions and the remainder
// Dynamic shared memory caps of the per-map launch shapes, which artp_create gives the kernels as their attribute:
// the grouping stage's plane store (upload_map refuses a map above it; the latency-path kernels share the store), a
// box_tiles_warp_kernel CTA's tiles, and a reach_groups_kernel CTA's tiles (set_shapes).
constexpr int kMaxStoreSmem = 200 * 1024, kMaxTileSmem = 200 * 1024, kMaxGroupsSmem = 160 * 1024;

struct QueueCtr { uint32_t end, claim; };   // classify appends records up to end, the queue's box kernel claims from claim
// The three box queues of a round (Pipeline::d_ctr), or one host-fed slice's share of them (Pipeline::d_slices). One
// 32-byte sector each: the box kernels of consecutive slices claim from their records at the same time.
struct alignas(32) BoxQueues { QueueCtr big, reach, group; };
struct Counters { BoxQueues q; uint32_t defer; };   // a round's queues, and its boxes deferred to the grouping stage

// A kernel's launch for the current map: at most `grid` CTAs of `block` threads with `smem` bytes of dynamic shared memory.
struct Shape { int grid = 0, block = 0, smem = 0; };

// The validity pipeline of a handle: box queues, per-map launch shapes, and the streams and events of its rounds.
struct Pipeline {
  enum { kBig, kReach, kGroup };   // the record queues, in BoxQueues order
  Counters* d_ctr = nullptr;
  // classify -> [kBig] the big-tile queue (torso boxes, reach boxes of unusual size), [kReach] the one-warp-per-box
  // reach-box queue (zones with mergeable planes or not reduced by the tables), [kGroup] the 8-lane-group kernel's queue
  // (merge-free zones, with or without -inf)
  artp::BoxRec* recs[3] = {};
  uint32_t* d_defer = nullptr;     // deferred record list (bit 31: reach-box queue)
  size_t recs_cap = 0;             // entries of each record queue and of d_defer
  BoxQueues* d_slices = nullptr;   // per slice of a host-fed round: its share of the three queues
  unsigned long long* d_compact_state = nullptr;   // compaction: tile counter, then one status word per tile (compact_kernel)
  size_t compact_state_cap = 0;
  uint32_t compact_epoch = 0;      // epoch of the last compaction's tile statuses
  // stage B (artp_tiles.cuh): [0] big tiles (torso queue), [1] small tiles (reach-box queue)
  artp::TileCfg tile_cfg[2] = {};
  CUtensorMap tile_map[2][2];      // [cfg][layer]: 2-D tile maps over elevation / elevation_masked
  Shape tile[2];                   // stage B's two queues
  Shape groups;                    // the 8-lane-group kernel; grid 0: no 8-lane queue
  Shape grouping;                  // the plane-grouping stage, also the dynamic shared memory of the latency-path kernels
  int tcap = 0;                    // triangles of the grouping stage's plane store
  int tcap_override = 0;           // test hook (artp_debug_set_group_capacity)
  int mode = 0;                    // artp_set_mode
  uint8_t* h_small_out = nullptr;  // mapped pinned host bytes the latency-path kernel writes its verdicts to
  bool deferred_unread = false;    // the last round's deferred boxes are not yet counted in stats.poses_deferred
  // artp_create creates the streams (non-blocking) and ordering events (cudaEventDisableTiming) from these two arrays.
  cudaStream_t streams[4] = {};
  cudaStream_t& copy_stream = streams[0];    // H2D slices of the host-buffer API
  cudaStream_t& box_stream = streams[1];     // box stages of slice i, concurrent with the copy + classify of slice i + 1
  cudaStream_t& group_stream = streams[2];   // the 8-lane-group kernel, beside the other box kernels
  cudaStream_t& tile_stream = streams[3];    // device rounds: the big-tile kernel, at the greatest stream priority
  cudaEvent_t order_ev[2 * kMaxSlices + 3] = {};
  cudaEvent_t *const copy_ev = order_ev, *const slice_ev = order_ev + kMaxSlices;   // slice i: H2D landed, classify done
  cudaEvent_t& box_ev = order_ev[2 * kMaxSlices];   // a round's kernels on box_stream / group_stream / tile_stream done
  cudaEvent_t &group_ev = order_ev[2 * kMaxSlices + 1], &tile_ev = order_ev[2 * kMaxSlices + 2];
  // artp_set_timing: a timed round records ev[0] before classify and ev[i] after stage i of classify | big tiles |
  // reach-box warps | 8-lane groups | plane grouping
  int timing = 0;
  cudaEvent_t ev[6] = {};
  bool ev_valid = false;
  // Releases whatever artp_create and the calls created (the handle's device is current).
  ~Pipeline() {
    for (cudaStream_t s : streams) if (s) { cudaStreamSynchronize(s); cudaStreamDestroy(s); }
    for (cudaEvent_t e : order_ev) if (e) cudaEventDestroy(e);
    for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
    for (artp::BoxRec* r : recs) cudaFree(r);
    cudaFree(d_ctr); cudaFree(d_defer); cudaFree(d_slices); cudaFree(d_compact_state);
    if (h_small_out) cudaFreeHost(h_small_out);
  }
};

}  // namespace artp_api

using namespace artp_api;

namespace {

thread_local std::string g_create_error;

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
void code_scale_of(float lo, float hi, float& base, float& step) {
  base = lo <= hi ? lo : 0.0f;
  int e = -126;
  while (e < 127 && artp::code_dec(base, std::ldexp(1.0f, e), artp::kCodeMax) < hi) ++e;
  step = std::ldexp(1.0f, e);
}
void code_scale(const float* layer, size_t n, float& base, float& step) {
  float lo = HUGE_VALF, hi = -HUGE_VALF;
  for (size_t i = 0; i < n; ++i) {
    const float v = layer[i] * 1.0f + 0.0f;   // the stored height (reverse_columns_kernel)
    if (std::fabs(v) < HUGE_VALF) { lo = std::min(lo, v); hi = std::max(hi, v); }
  }
  code_scale_of(lo, hi, base, step);
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
    const unsigned long long key = plane_key(artp::nkey(pl[0]), artp::nkey(pl[2]), artp::dkey(pl[3]));
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
    const int kx0 = artp::nkey(pl[0] - e2), kx1 = artp::nkey(pl[0] + e2);
    const int kz0 = artp::nkey(pl[2] - e2), kz1 = artp::nkey(pl[2] + e2);
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

// Ordered compaction in one pass: a single-pass scan with decoupled look-back (Merrill & Garland 2016). Each CTA takes the
// next tile of kCompactTile items from a counter, so a tile only ever waits on tiles whose CTAs are already running. Warp w of
// a tile owns kCompactRounds consecutive runs of 32 items; a run's 32 flags are one ballot (one word of a bit-packed mask),
// which gives the in-tile ranks. The CTA publishes its tile's count (AGGREGATE), then warp 0 sums the statuses of the
// preceding tiles back to the nearest INCLUSIVE one and publishes the tile's inclusive prefix; the scatter then writes the
// indices in item order. Status word of a tile: epoch (bits 34-63) | flag (bits 32-33) | value (bits 0-31). A status of
// another epoch (an earlier call) reads as not yet published, so the states need no reset between calls. Word 0 of the
// state array is the tile counter; the CTA that draws the last tile sets it back to 0 and writes the count.
constexpr int kCompactThreads = 256, kCompactRounds = 16;
constexpr int kCompactTile = kCompactThreads * kCompactRounds;   // 4096 items
constexpr unsigned long long kTileAggregate = 1ull << 32, kTileInclusive = 2ull << 32, kTileFlags = 3ull << 32;
constexpr uint32_t kCompactEpochs = 1u << 30;
// BITS: the mask is bit-packed (item i = bit i&31 of word i>>5, artp_pack_valid_bits_device), else one byte per item.
template <bool BITS, typename IndexT>
__global__ void __launch_bounds__(kCompactThreads)
compact_kernel(const uint8_t* __restrict__ valid, size_t n, int64_t base, unsigned long long* __restrict__ state, uint32_t epoch,
               IndexT* __restrict__ out, uint32_t* __restrict__ count) {
  __shared__ uint32_t s_tile, s_before;
  __shared__ uint32_t wsum[kCompactThreads / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const size_t ntiles = (n + kCompactTile - 1) / kCompactTile;
  if (threadIdx.x == 0) {
    s_tile = (uint32_t)atomicAdd(state, 1ull);
    if (s_tile == ntiles - 1) *state = 0ull;   // every other CTA has drawn its tile: ready for the next call
  }
  __syncthreads();
  const uint32_t tile = s_tile;
  const size_t run0 = (size_t)tile * kCompactTile + (size_t)wid * 32 * kCompactRounds;   // first item of this warp's runs
  uint32_t bal[kCompactRounds];
  if (BITS) {
    const uint32_t* words = reinterpret_cast<const uint32_t*>(valid);
    const size_t wi = (run0 >> 5) + lane;
    uint32_t mine = 0;
    if (lane < kCompactRounds && wi < (n + 31) / 32) {
      mine = words[wi];
      if (n - 32 * wi < 32) mine &= (1u << (n - 32 * wi)) - 1u;   // bits past n are not items
    }
#pragma unroll
    for (int r = 0; r < kCompactRounds; ++r) bal[r] = __shfl_sync(0xffffffffu, mine, r);
  } else {
    uint8_t v[kCompactRounds];
#pragma unroll
    for (int r = 0; r < kCompactRounds; ++r) {
      const size_t i = run0 + 32 * r + lane;
      v[r] = i < n ? valid[i] : 0;
    }
#pragma unroll
    for (int r = 0; r < kCompactRounds; ++r) bal[r] = __ballot_sync(0xffffffffu, v[r] != 0);
  }
  uint32_t wtot = 0;
#pragma unroll
  for (int r = 0; r < kCompactRounds; ++r) wtot += __popc(bal[r]);
  if (lane == 0) wsum[wid] = wtot;
  __syncthreads();
  const unsigned long long tag = (unsigned long long)epoch << 34;
  volatile unsigned long long* st = state + 1;
  if (wid == 0) {
    uint32_t x = lane < kCompactThreads / 32 ? wsum[lane] : 0u;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane < kCompactThreads / 32) wsum[lane] = x;   // inclusive prefix over the warps
    const uint32_t agg = __shfl_sync(0xffffffffu, x, kCompactThreads / 32 - 1);
    uint32_t before = 0;
    if (tile == 0) {
      if (lane == 0) st[0] = tag | kTileInclusive | agg;
    } else {
      if (lane == 0) st[tile] = tag | kTileAggregate | agg;
      for (long long j = (long long)tile - 1;; j -= 32) {   // lane k reads tile j - k
        const long long t = j - lane;
        unsigned long long s;
        do {
          s = t >= 0 ? st[t] : (tag | kTileInclusive);
        } while (__any_sync(0xffffffffu, (s >> 34) != epoch || !(s & kTileFlags)));
        const unsigned inc = __ballot_sync(0xffffffffu, (s & kTileFlags) == kTileInclusive);
        const int stop = inc ? __ffs(inc) - 1 : 31;   // the nearest inclusive prefix ends the look-back
        uint32_t v = lane <= stop ? (uint32_t)s : 0u;
#pragma unroll
        for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        before += v;
        if (inc) break;
      }
      if (lane == 0) st[tile] = tag | kTileInclusive | (uint32_t)(before + agg);
    }
    if (lane == 0) {
      s_before = before;
      if (tile == ntiles - 1) *count = before + agg;
    }
  }
  __syncthreads();
  uint32_t pos = s_before + (wid ? wsum[wid - 1] : 0u);
  const unsigned lt = (1u << lane) - 1u;
#pragma unroll
  for (int r = 0; r < kCompactRounds; ++r) {
    if ((bal[r] >> lane) & 1u) out[pos + __popc(bal[r] & lt)] = (IndexT)(base + (int64_t)(run0 + 32 * r + lane));
    pos += __popc(bal[r]);
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

int ensure_queues(Handle* h, size_t n_items) {
  const size_t need = 5 * std::min(n_items, kChunkItems);
  if (h->pipe->recs_cap >= need) return ARTP_OK;
  const size_t cap = std::max<size_t>(need, 1u << 16);
  h->pipe->recs_cap = 0;   // the four buffers share it: set once all four have grown
  for (artp::BoxRec*& r : h->pipe->recs) { size_t had = 0; TRY(grow(h, r, had, cap)); }
  size_t had = 0;
  TRY(grow(h, h->pipe->d_defer, had, cap));
  h->pipe->recs_cap = cap;
  return ARTP_OK;
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

// Stage launchers shared by both rounds. Each launches its kernel over the items [lo, hi) of w (items); W is artp::Work,
// or artp::WhyWork for the explain form of the kernels (artp_box_verdicts).
template <class W>
constexpr bool kWhyOf = std::is_same_v<W, artp::WhyWork>;
template <class W>
W items(W w, size_t lo, size_t hi) {
  w.item_base = (uint32_t)lo;
  w.n_items = (uint32_t)hi;
  return w;
}
template <class W>
int launch_classify(Handle* h, const W& w, size_t lo, size_t hi, BoxQueues* q, cudaStream_t s) {
  const Pipeline& p = *h->pipe;
  return launch(h, artp::classify_items_kernel<kWhyOf<W>>, (unsigned)((hi - lo + artp::kClassifyItems - 1) / artp::kClassifyItems),
                artp::kClassifyItems, 0, s, h->chk, items(w, lo, hi), p.recs[p.kBig], p.recs[p.kReach],
                p.groups.grid ? p.recs[p.kGroup] : nullptr, &q->big.end, &q->reach.end, &q->group.end, p.mode == 1);
}

// Classify appends to the queues q, each box kernel takes its queue's entries: the big-tile queue and the two reach-box
// queues (one warp per box; 8-lane groups), which exist only for some box sizes. reach_cap caps both reach grids.
template <class W>
int launch_big_tile(Handle* h, const W& w, size_t lo, size_t hi, BoxQueues* q, cudaStream_t s) {
  Pipeline& p = *h->pipe;
  const int wpc = p.tile[0].block / 32;   // no more CTAs than there can be boxes: up to five big-tile boxes per item
  const unsigned grid = (unsigned)std::min<size_t>((size_t)p.tile[0].grid, (5 * (hi - lo) + wpc - 1) / wpc);
  return launch(h, artp::box_tiles_warp_kernel<kWhyOf<W>>, grid, p.tile[0].block, p.tile[0].smem, s, h->chk, p.tile_map[0][0],
                p.tile_map[0][1], p.tile_cfg[0], items(w, lo, hi), p.recs[p.kBig], &q->big.end, &q->big.claim, &p.d_ctr->defer,
                p.d_defer, 0u, p.mode == 1);
}
template <class W>
int launch_reach_warp(Handle* h, const W& w, size_t lo, size_t hi, BoxQueues* q, cudaStream_t s, unsigned reach_cap) {
  if (!h->chk.reach_tw) return ARTP_OK;
  Pipeline& p = *h->pipe;
  const int wpc = p.tile[1].block / 32;
  const unsigned grid = (unsigned)std::min<size_t>({(size_t)p.tile[1].grid, (4 * (hi - lo) + wpc - 1) / wpc, reach_cap});
  return launch(h, artp::box_tiles_warp_kernel<kWhyOf<W>>, grid, p.tile[1].block, p.tile[1].smem, s, h->chk, p.tile_map[1][1],
                p.tile_map[1][1], p.tile_cfg[1], items(w, lo, hi), p.recs[p.kReach], &q->reach.end, &q->reach.claim,
                &p.d_ctr->defer, p.d_defer, artp::kDeferReachBit, p.mode == 1);
}
template <class W>
int launch_reach_groups(Handle* h, const W& w, size_t lo, size_t hi, BoxQueues* q, cudaStream_t s, unsigned reach_cap) {
  const Pipeline& p = *h->pipe;
  if (!p.groups.grid) return ARTP_OK;
  const unsigned grid = (unsigned)std::min<size_t>({(size_t)p.groups.grid, (hi - lo + 7) / 8, reach_cap});
  return launch(h, artp::reach_groups_kernel<kWhyOf<W>>, grid, p.groups.block, p.groups.smem, s, h->chk, p.tile_map[1][1], p.tile_cfg[1],
                items(w, lo, hi), p.recs[p.kGroup], &q->group.end, &q->group.claim);
}

// The plane-grouping stage over every box the round [lo, hi) deferred.
template <class W>
int launch_grouping(Handle* h, const W& w, size_t lo, size_t hi, cudaStream_t s) {
  const Pipeline& p = *h->pipe;
  const unsigned grid = (unsigned)std::min<size_t>((size_t)p.grouping.grid, 5 * (hi - lo));
  return launch(h, artp::box_items_block_kernel<kWhyOf<W>>, grid, p.grouping.block, p.grouping.smem, s, h->chk, items(w, lo, hi),
                p.recs[p.kBig], p.recs[p.kReach], &p.d_ctr->defer, p.d_defer, p.tcap, h->d_err);
}

// Device round: the items [base, end) are on the device. Classify, the three box kernels, then the grouping stage. The box
// kernels only ever clear verdicts of different boxes, so the two reach kernels fork onto box_stream / group_stream after
// the classify stage (each kernel has a latency floor of 20-30 us), and the big-tile kernel onto tile_stream, whose greatest
// priority gets its CTAs onto the SMs before the 8-lane kernel fills them (on the default priority it started after the
// 8-lane kernel in about half of the steps and ended last). The grouping stage waits for tile_stream and box_stream only;
// group_stream joins s after it. With stage timing on, everything runs in order on s, and a timed round records the
// per-stage events.
template <class W>
int run_round_device(Handle* h, const W& w, cudaStream_t s, size_t base, size_t end, bool timed) {
  Pipeline& p = *h->pipe;
  CU_TRY(h, cudaMemsetAsync(p.d_ctr, 0, sizeof(Counters), s));
  if (timed) CU_TRY(h, cudaEventRecord(p.ev[0], s));
  BoxQueues* q = &p.d_ctr->q;
  TRY(launch_classify(h, w, base, end, q, s));
  if (timed) CU_TRY(h, cudaEventRecord(p.ev[1], s));
  const bool fork = !p.timing && h->chk.reach_tw;
  if (fork) {
    CU_TRY(h, cudaEventRecord(p.slice_ev[0], s));
    CU_TRY(h, cudaStreamWaitEvent(p.tile_stream, p.slice_ev[0], 0));
    CU_TRY(h, cudaStreamWaitEvent(p.box_stream, p.slice_ev[0], 0));
    if (p.groups.grid) CU_TRY(h, cudaStreamWaitEvent(p.group_stream, p.slice_ev[0], 0));
  }
  TRY(launch_big_tile(h, w, base, end, q, fork ? p.tile_stream : s));
  if (timed) CU_TRY(h, cudaEventRecord(p.ev[2], s));
  TRY(launch_reach_warp(h, w, base, end, q, fork ? p.box_stream : s, UINT_MAX));
  if (timed) CU_TRY(h, cudaEventRecord(p.ev[3], s));
  TRY(launch_reach_groups(h, w, base, end, q, fork ? p.group_stream : s, UINT_MAX));
  if (fork) {
    // The grouping stage reads the defer list, which only the two box_tiles_warp_kernel launches (tile_stream,
    // box_stream) write. reach_groups_kernel defers nothing, and it and the grouping stage only ever clear verdict bytes
    // of different boxes, so the grouping stage need not wait for it: group_stream joins s after the grouping launch.
    CU_TRY(h, cudaEventRecord(p.tile_ev, p.tile_stream));
    CU_TRY(h, cudaStreamWaitEvent(s, p.tile_ev, 0));
    CU_TRY(h, cudaEventRecord(p.box_ev, p.box_stream));
    CU_TRY(h, cudaStreamWaitEvent(s, p.box_ev, 0));
  }
  if (timed) CU_TRY(h, cudaEventRecord(p.ev[4], s));
  TRY(launch_grouping(h, w, base, end, s));
  if (timed) { CU_TRY(h, cudaEventRecord(p.ev[5], s)); p.ev_valid = true; }
  if (fork && p.groups.grid) {
    CU_TRY(h, cudaEventRecord(p.group_ev, p.group_stream));
    CU_TRY(h, cudaStreamWaitEvent(s, p.group_ev, 0));
  }
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
  Pipeline& p = *h->pipe;
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
  CU_TRY(h, cudaMemsetAsync(p.d_ctr, 0, sizeof(Counters), s));
  const unsigned reach_cap = (unsigned)(kPipeReachCtasPerSm * h->sm_count);
  for (int si = 0; si < ncut; ++si) {
    const size_t lo = cut[si], hi = cut[si + 1];
    CU_TRY(h, cudaMemcpyAsync(feed.dev + lo * feed.bytes_per_item, feed.host + lo * feed.bytes_per_item,
                              (hi - lo) * feed.bytes_per_item, cudaMemcpyHostToDevice, p.copy_stream));
    CU_TRY(h, cudaEventRecord(p.copy_ev[si], p.copy_stream));
    CU_TRY(h, cudaStreamWaitEvent(s, p.copy_ev[si], 0));
    TRY(launch_classify(h, w, lo, hi, &p.d_ctr->q, s));
    TRY(launch(h, close_slice_kernel, 1, 1, 0, s, &p.d_ctr->q, p.d_slices, si));
    CU_TRY(h, cudaEventRecord(p.slice_ev[si], s));
    CU_TRY(h, cudaStreamWaitEvent(p.box_stream, p.slice_ev[si], 0));
    if (p.groups.grid) CU_TRY(h, cudaStreamWaitEvent(p.group_stream, p.slice_ev[si], 0));
    // the big-tile queue (torso boxes: few) of this slice behind its reach-box queue: issued ahead of the reach kernels,
    // it made host-fed calls 2-4 % slower (H100 80GB HBM3, 400 W power limit)
    TRY(launch_reach_groups(h, w, lo, hi, p.d_slices + si, p.group_stream, reach_cap));
    TRY(launch_reach_warp(h, w, lo, hi, p.d_slices + si, p.box_stream, reach_cap));
    TRY(launch_big_tile(h, w, lo, hi, p.d_slices + si, p.box_stream));
  }
  if (p.groups.grid) {
    // the grouping stage (box_stream) runs last: the group kernels must not clear a verdict after it has been copied out
    CU_TRY(h, cudaEventRecord(p.group_ev, p.group_stream));
    CU_TRY(h, cudaStreamWaitEvent(p.box_stream, p.group_ev, 0));
  }
  TRY(launch_grouping(h, w, base, end, p.box_stream));
  CU_TRY(h, cudaEventRecord(p.box_ev, p.box_stream));
  CU_TRY(h, cudaStreamWaitEvent(s, p.box_ev, 0));
  return ARTP_OK;
}

// Launch the pipeline for a prepared Work (items 0 .. w.n_items = the whole call) on stream s, in rounds of kChunkItems
// work items (bounds the box queues), and count the items in stats.poses_checked. With a host feed, a round larger than
// one slice is piped; any other round (and every round while stage timing is on) has its states copied on s and runs as
// a device round.
// The explain form (W = artp::WhyWork) has no piped round: its host feed is copied round by round.
template <class W>
int run_items(Handle* h, W w, cudaStream_t s, const HostFeed* feed = nullptr) {
  const size_t n_total = w.n_items;
  TRY(ensure_queues(h, n_total));
  for (size_t base = 0; base < n_total; base += kChunkItems) {
    const size_t end = std::min(n_total, base + kChunkItems);
    if (!kWhyOf<W> && feed && feed->slice_items < end - base && !h->pipe->timing) {
      if constexpr (!kWhyOf<W>) TRY(run_round_piped(h, w, s, *feed, base, end));
    } else {
      if (feed)
        CU_TRY(h, cudaMemcpyAsync(feed->dev + base * feed->bytes_per_item, feed->host + base * feed->bytes_per_item,
                                  (end - base) * feed->bytes_per_item, cudaMemcpyHostToDevice, s));
      TRY(run_round_device(h, w, s, base, end, h->pipe->timing && end == n_total));
    }
  }
  h->pipe->deferred_unread = true;
  h->stats.poses_checked += n_total;
  return ARTP_OK;
}

int check_common(Handle* h, size_t n) {
  TRY(require_map(h));
  if (n >= (size_t)0xFFFFFFF0u) { h->err = "too many items for one call"; return ARTP_E_LIMIT; }
  return ARTP_OK;
}

// Latency path for n <= kSmallBatch host states (doubles): one launch, verdicts through mapped host memory.
int check_poses_small(Handle* h, const artp::SmallBatch& sb, size_t n, uint8_t* valid, int steps = -1) {
  Pipeline& p = *h->pipe;
  TRY(host_call_begin(h));
  uint8_t* d_out = nullptr;
  CU_TRY(h, cudaHostGetDevicePointer((void**)&d_out, p.h_small_out, 0));
  TRY(launch(h, artp::pose_small_kernel, (unsigned)n, 256, p.grouping.smem, h->stream, h->chk, sb, d_out, p.tcap, h->d_err,
      p.mode == 1, steps));
  const int rc = host_call_end(h, true);
  if (rc == ARTP_E_CUDA) return rc;
  if (steps < 0) {
    std::memcpy(valid, p.h_small_out, n);
  } else {   // n = edges * (steps + 1) state verdicts -> one flag per edge
    const size_t per = (size_t)steps + 1;
    for (size_t e = 0; e < n / per; ++e) {
      uint8_t ok = 1;
      for (size_t j = 0; j < per; ++j) ok &= p.h_small_out[e * per + j];
      valid[e] = ok;
    }
  }
  h->stats.poses_checked += n;
  p.ev_valid = false;
  return rc;
}

// The validity pipeline over n states on the device (T = double, or float: the caller has already applied the
// double -> float cast that Pose3FromSE3, utils.h:25-38, performs first) into d_valid, on s; with a host feed the states
// arrive from the host in slices.
template <typename T>
int check_states(Handle* h, const T* d_states, size_t n, uint8_t* d_valid, cudaStream_t s, const HostFeed* feed = nullptr) {
  artp::Work w;
  if constexpr (std::is_same_v<T, float>) w.s2f = d_states; else w.s2 = d_states;
  w.valid = d_valid;
  w.n_items = (uint32_t)n;
  return run_items(h, w, s, feed);
}

// The explain form of check_states: every box of each of the n states decided, the ARTP_BOX_* words into d_why, on s.
template <typename T>
int box_verdicts_on(Handle* h, const T* d_states, size_t n, uint16_t* d_why, cudaStream_t s) {
  // the explain form's kernels get artp_create's shared-memory limits at their first use, not at artp_create: a handle
  // that never explains never loads them
  const std::pair<const void*, int> caps[] = {{(const void*)artp::box_items_block_kernel<true>, kMaxStoreSmem},
                                              {(const void*)artp::box_tiles_warp_kernel<true>, kMaxTileSmem},
                                              {(const void*)artp::reach_groups_kernel<true>, kMaxGroupsSmem}};
  for (const auto& [k, bytes] : caps) CU_TRY(h, cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  artp::WhyWork w;
  if constexpr (std::is_same_v<T, float>) w.s2f = d_states; else w.s2 = d_states;
  w.why = d_why;
  w.n_items = (uint32_t)n;
  return run_items(h, w, s);
}

// artp_box_verdicts[_device]'s refusals before the null-buffer check: those of artp_check_poses, and a map window.
int box_verdict_args(Handle* h, size_t n) {
  TRY(check_common(h, n));
  return require_whole_map(h);
}

// The pose entry points. A float state gives the same verdict as the double one while the H2D stream is 28 B/pose
// instead of 56. With on_device, states and valid are device buffers and the call is asynchronous on stream; otherwise
// they are host buffers: up to kSmallBatch states take the latency path, more are fed to the device in slices.
template <typename T>
int check_poses(Handle* h, const T* states, size_t n, uint8_t* valid, bool on_device, cudaStream_t stream) {
  TRY(check_common(h, n));
  if (n == 0) return ARTP_OK;
  if (!states || !valid) return null_buffer(h);
  if (on_device) {
    CU_TRY(h, cudaSetDevice(h->device));
    ChainScope cs(h, 0, stream);
    if (cs.rc) return cs.rc;
    return check_states(h, states, n, valid, stream);
  }
  if (n <= (size_t)artp::kSmallBatch && !h->pipe->timing) {
    artp::SmallBatch sb;
    for (size_t i = 0; i < n * 7; ++i) (&sb.s[0][0])[i] = (double)states[i];   // exact; a float state is cast back in the kernel
    return check_poses_small(h, sb, n, valid);
  }
  char* r[2];
  TRY(host_call_begin(h, {n * 7 * sizeof(T), n}, r));
  const HostFeed feed = std::is_same_v<T, float>
                            ? HostFeed{(const char*)states, r[0], 7 * sizeof(T), 256 * 1024, {0.08f, 0.17f, 0.25f, 0.25f, 0.25f}}
                            : HostFeed{(const char*)states, r[0], 7 * sizeof(T), 128 * 1024, {0.06f, 0.14f, 0.20f, 0.20f, 0.20f, 0.20f}};
  TRY(check_states(h, (const T*)r[0], n, (uint8_t*)r[1], h->stream, &feed));
  CU_TRY(h, cudaMemcpyAsync(valid, r[1], n, cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h, true);
}

// Motions: n edges of n_steps interior states each, as n * (n_steps + 1) work items.
int motion_items(Handle* h, size_t n, int n_steps) {
  if (n_steps < 0) { h->err = "n_steps < 0"; return ARTP_E_INVALID; }
  return check_common(h, n * ((size_t)n_steps + 1));
}
int check_motions_on(Handle* h, const double* d_s1, const double* d_s2, size_t n, int n_steps, uint8_t* d_valid, cudaStream_t s) {
  TRY(launch(h, fill_u8_kernel, grid_for(h, n, 256, 8), 256, 0, s, d_valid, n, 1));
  const size_t items = n * ((size_t)n_steps + 1);
  artp::Work w;
  w.s1 = d_s1; w.s2 = d_s2; w.valid = d_valid; w.n_items = (uint32_t)items; w.steps = n_steps; w.edge_mode = 1;
  return run_items(h, w, s);
}

// valid_prefix[e] = number of leading 1s in item_valid[item_off[e] .. item_off[e+1])
__global__ void edge_prefix_kernel(const uint8_t* __restrict__ item_valid, const uint32_t* __restrict__ item_off, size_t n,
                                   int32_t* __restrict__ valid_prefix) {
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x) {
    const uint32_t o0 = item_off[e];
    valid_prefix[e] = (int32_t)artp::leading_valid(item_valid + o0, item_off[e + 1] - o0);
  }
}

// Edge e checks the items d_item_off[e] .. d_item_off[e+1] between d_s1[e] and d_s2[e] (interior states, or with
// `quotient` the segment states of the motion) and gets the number of leading valid ones in d_valid_prefix[e].
int check_items_prefix(Handle* h, const double* d_s1, const double* d_s2, size_t n, const uint32_t* d_item_off,
                       size_t total_items, uint8_t* d_item_valid, int32_t* d_valid_prefix, void* stream, int quotient) {
  TRY(check_common(h, total_items));
  if (n == 0) return ARTP_OK;
  if (!d_s1 || !d_s2 || !d_item_off || !d_valid_prefix || (total_items && !d_item_valid)) {
    return null_buffer(h);
  }
  if (n >= 0xFFFFFFFFull) { h->err = "too many edges"; return ARTP_E_INVALID; }
  CU_TRY(h, cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  ChainScope cs(h, 0, s);
  if (cs.rc) return cs.rc;
  if (total_items) {
    artp::Work w;
    w.s1 = d_s1; w.s2 = d_s2; w.valid = d_item_valid; w.n_items = (uint32_t)total_items;
    w.item_off = d_item_off; w.n_edges = (uint32_t)n; w.quotient = quotient;
    TRY(run_items(h, w, s));
  }
  return launch(h, edge_prefix_kernel, grid_for(h, n, 256, 8), 256, 0, s, d_item_valid, d_item_off, n, d_valid_prefix);
}

// check_items_prefix over host buffers: the n = off.size() - 1 edges (s1[e], s2[e]) with their item offsets `off`;
// valid_prefix[e] receives edge e's number of leading valid items.
int check_items_prefix_host(Handle* h, const double* s1, const double* s2, const std::vector<uint32_t>& off, int quotient,
                            int32_t* valid_prefix) {
  const size_t n = off.size() - 1, total = off[n], sb = n * 7 * sizeof(double);
  char* r[5];   // s1 | s2 | off | prefix | item flags
  TRY(host_call_begin(h, {sb, sb, (n + 1) * sizeof(uint32_t), n * sizeof(int32_t), total}, r));
  CU_TRY(h, cudaMemcpyAsync(r[0], s1, sb, cudaMemcpyHostToDevice, h->stream));
  CU_TRY(h, cudaMemcpyAsync(r[1], s2, sb, cudaMemcpyHostToDevice, h->stream));
  CU_TRY(h, cudaMemcpyAsync(r[2], off.data(), (n + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
  TRY(check_items_prefix(h, (const double*)r[0], (const double*)r[1], n, (const uint32_t*)r[2], total, (uint8_t*)r[4],
                         (int32_t*)r[3], h->stream, quotient));
  CU_TRY(h, cudaMemcpyAsync(valid_prefix, r[3], n * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h, true);   // `off` outlives its H2D copy: the call synchronises before it returns
}

int pack_valid_bits(Handle* h, const uint8_t* d_valid, size_t n, uint32_t* d_bits, cudaStream_t s) {
  if (n == 0) return ARTP_OK;
  if (!d_valid || !d_bits) return null_buffer(h);
  CU_TRY(h, cudaSetDevice(h->device));
  const size_t words = (n + 31) / 32;
  return launch(h, pack_bits_kernel, grid_for(h, words * 32, 256, 8), 256, 0, s, d_valid, n, d_bits);
}

// The elapsed times ev[from] -> ev[to] of each pair into ms, once the last timed round has ended.
int timed_round_ms(Handle* h, float* ms, std::initializer_list<std::pair<int, int>> pairs) {
  const Pipeline& p = *h->pipe;
  if (!ms) return ARTP_E_INVALID;
  if (!p.timing || !p.ev_valid) { h->err = "timing not enabled or no call recorded"; return ARTP_E_INVALID; }
  CU_TRY(h, cudaSetDevice(h->device));
  CU_TRY(h, cudaEventSynchronize(p.ev[5]));
  for (const auto& [from, to] : pairs) CU_TRY(h, cudaEventElapsedTime(ms++, p.ev[from], p.ev[to]));
  return ARTP_OK;
}

// out = the launch of `kernel` at block threads and smem bytes of dynamic shared memory, full grid. The kernel's
// shared-memory attribute is set once, in artp_create.
template <typename... P>
int fit_shape(Handle* h, void (*kernel)(P...), int block, int smem, Shape& out) {
  int per_sm = 0;
  CU_TRY(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, block, smem));
  out = {h->sm_count * std::max(per_sm, 1), block, smem};
  return ARTP_OK;
}

// The box kernels' launch shapes for the map just installed (h->d_H, pitch, cols, win_row0), from each box's zone bound
// span and the grouping stage's plane store (upload_map): occupancy grids, tile maps, chk's reach tile.
int set_shapes(Handle* h, const int span[2][2], int tcap, int store) {
  Pipeline& p = *h->pipe;
  TRY(fit_shape(h, artp::box_items_block_kernel<false>, artp::kBlockStageThreads, store, p.grouping));
  p.tcap = tcap;
  // Stage B tiles (artp_tiles.cuh): a zone spans at most ceil(2 r / s) + 3 vertices per axis; + 3 columns because the
  // tile starts at x0 & ~3; width rounded up to a multiple of 4 floats (16-byte rows).
  PFN_cuTensorMapEncodeTiled encode = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", (void**)&encode, cudaEnableDefault, &qres) != cudaSuccess || !encode) {
    h->err = "cuTensorMapEncodeTiled not available from the driver"; return ARTP_E_CUDA;
  }
  h->chk.reach_tw = 0; h->chk.reach_th = 0;
  for (int q = 0; q < 2; ++q) {          // 0: big tiles (torso box bound), 1: small tiles (reach box bound)
    const int tw = std::min((span[q][0] + 3 + 3 + 3) & ~3, 256), th = std::min(span[q][1] + 3, 256);
    artp::TileCfg tc;
    tc.tw = tw; tc.th = th; tc.bytes = (uint32_t)tw * th * 4; tc.stride = (tc.bytes + 127u) & ~127u;
    // big tiles: one slot per warp (three 8-warp CTAs per SM hide the copy latency better than a second 7 KB slot);
    // small tiles: two slots, the next box's tile is in flight while this one is decided
    tc.slots = (tc.stride > 2048) ? 1 : 2;
    int wpc = 8;
    while (wpc > 1 && (size_t)wpc * tc.slots * tc.stride + 128 > 72 * 1024) wpc >>= 1;
    if ((size_t)wpc * tc.slots * tc.stride + 128 > kMaxTileSmem) {
      if (q == 1) { p.tile[1] = Shape{}; continue; }   // no reach-box queue: everything takes the big-tile queue
      // boxes this large relative to the cells: tiles capped, oversized zones go to the grouping stage
      tc.tw = 64; tc.th = 64; tc.bytes = 64 * 64 * 4; tc.stride = tc.bytes; tc.slots = 1; wpc = 4;
    }
    const cuuint64_t gdim[2] = {(cuuint64_t)h->pitch, (cuuint64_t)h->cols};
    const cuuint64_t gstr[1] = {(cuuint64_t)h->pitch * sizeof(float)};
    const cuuint32_t box[2] = {(cuuint32_t)tc.tw, (cuuint32_t)tc.th};
    const cuuint32_t one[2] = {1, 1};
    for (int layer = 0; layer < 2; ++layer) {
      const CUresult cr = encode(&p.tile_map[q][layer], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, h->d_H[layer], gdim, gstr, box, one,
                                 CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                 CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (cr != CUDA_SUCCESS) { h->err = "cuTensorMapEncodeTiled failed (" + std::to_string((int)cr) + ")"; return ARTP_E_CUDA; }
    }
    tc.x_off = h->win_row0;
    p.tile_cfg[q] = tc;
    p.tile[q] = {0, wpc * 32, (int)((size_t)wpc * tc.slots * tc.stride + 128)};
    if (q == 1) { h->chk.reach_tw = tc.tw; h->chk.reach_th = tc.th; }
  }
  p.groups = Shape{};
  if (h->chk.reach_tw && p.tile_cfg[1].tw <= 127 && p.tile_cfg[1].th <= 255) {   // task packing: 7 + 8 bits of cell coordinates
    const int gsm = artp::kMaxTileWarps * 8 * (int)p.tile_cfg[1].stride + 128;
    if (gsm <= kMaxGroupsSmem && !std::getenv("ARTP_NO_GROUPS")) {   // ARTP_NO_GROUPS: every reach box takes the one-warp-per-box queue
      TRY(fit_shape(h, artp::reach_groups_kernel<false>, artp::kMaxTileWarps * 32, gsm, p.groups));
    }
  }
  for (Shape& t : p.tile)
    if (t.block) TRY(fit_shape(h, artp::box_tiles_warp_kernel<false>, t.block, t.smem, t));
  return ARTP_OK;
}

}  // namespace

// Sticky plane-grouping overflow (set by the device, see Handle::h_err): read and clear.
int artp_api::take_sticky_error(Handle* h) {
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

int artp_api::check_states_f32(Handle* h, const float* d_states, size_t n, uint8_t* d_valid, cudaStream_t s) {
  return check_states(h, d_states, n, d_valid, s);
}

int artp_api::box_verdicts_f32(Handle* h, const float* d_states, size_t n, uint16_t* d_why, cudaStream_t s) {
  return box_verdicts_on(h, d_states, n, d_why, s);
}

int artp_api::check_states_cta(Handle* h, const double* d_states, const uint32_t* d_count, const uint32_t* d_stop, size_t max_n,
                               uint8_t* d_valid, cudaStream_t s) {
  if (max_n == 0) return ARTP_OK;
  TRY(launch(h, artp::pose_states_kernel, (unsigned)max_n, 256, h->pipe->grouping.smem, s, h->chk, d_states, d_count, d_stop,
             d_valid, h->pipe->tcap, h->d_err));
  h->pipe->ev_valid = false;
  return ARTP_OK;
}

int artp_api::compact_valid(Handle* h, const uint8_t* d_valid, size_t n, int64_t base, void* d_indices, uint32_t* d_count,
                            cudaStream_t s, bool bits, bool u32) {
  Pipeline& p = *h->pipe;
  if (n == 0) { CU_TRY(h, cudaMemsetAsync(d_count, 0, sizeof(uint32_t), s)); return ARTP_OK; }
  ChainScope cs(h, 1, s);
  if (cs.rc) return cs.rc;
  const size_t nt = (n + kCompactTile - 1) / kCompactTile;
  if (p.compact_state_cap < nt + 1 || p.compact_epoch + 1 >= kCompactEpochs) {
    // a new array, or the epochs wrapped: clear it once (word 0, the tile counter, included)
    TRY(grow(h, p.d_compact_state, p.compact_state_cap, nt + 1));
    CU_TRY(h, cudaMemsetAsync(p.d_compact_state, 0, p.compact_state_cap * sizeof(unsigned long long), s));
    p.compact_epoch = 0;
  }
  const uint32_t epoch = ++p.compact_epoch;
  auto run = [&](auto kernel, auto* indices) {
    return launch(h, kernel, (unsigned)nt, kCompactThreads, 0, s, d_valid, n, base, p.d_compact_state, epoch, indices, d_count);
  };
  if (bits) return run(compact_kernel<true, int64_t>, (int64_t*)d_indices);
  if (u32) return run(compact_kernel<false, uint32_t>, (uint32_t*)d_indices);
  return run(compact_kernel<false, int64_t>, (int64_t*)d_indices);
}

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
  if ((e = cudaFuncGetAttributes(&fa, artp::box_tiles_warp_kernel<false>)) != cudaSuccess)
    return fail("no usable kernel image (built for sm_90a)", e);
  int prio_least = 0, prio_greatest = 0;
  if ((e = cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest)) != cudaSuccess) return fail("cudaDeviceGetStreamPriorityRange", e);
  if ((e = cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking)) != cudaSuccess) return fail("cudaStreamCreate", e);
  Pipeline& p = *(h->pipe = new Pipeline());
  for (cudaStream_t& st : p.streams) {
    e = &st == &p.tile_stream ? cudaStreamCreateWithPriority(&st, cudaStreamNonBlocking, prio_greatest)
                              : cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking);
    if (e != cudaSuccess) return fail("cudaStreamCreate", e);
  }
  for (cudaEvent_t& ev : p.order_ev)
    if ((e = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming)) != cudaSuccess) return fail("cudaEventCreate", e);
  for (cudaEvent_t& ev : h->chain_ev)
    if ((e = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming)) != cudaSuccess) return fail("cudaEventCreate", e);
  if ((e = cudaMalloc(&p.d_slices, kMaxSlices * sizeof(BoxQueues))) != cudaSuccess) return fail("cudaMalloc", e);
  if ((e = cudaMalloc(&p.d_ctr, sizeof(Counters))) != cudaSuccess) return fail("cudaMalloc", e);
  if ((e = cudaHostAlloc((void**)&p.h_small_out, 64, cudaHostAllocMapped)) != cudaSuccess) return fail("cudaHostAlloc", e);
  // A kernel's max-dynamic-shared-memory attribute belongs to the kernel in the device's context, so every handle on the
  // device shares it. Each kernel gets the most that any accepted map can ask of it, here and never per map: a handle
  // that set it to its own map's size would lower it under the launches of a handle holding a larger map.
  const std::pair<const void*, int> smem_caps[] = {
      {(const void*)artp::pose_small_kernel, kMaxStoreSmem}, {(const void*)artp::pose_states_kernel, kMaxStoreSmem},
      {(const void*)artp::box_items_block_kernel<false>, kMaxStoreSmem}, {(const void*)artp::box_tiles_warp_kernel<false>, kMaxTileSmem},
      {(const void*)artp::reach_groups_kernel<false>, kMaxGroupsSmem}};
  for (const auto& [k, bytes] : smem_caps)
    if ((e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes)) != cudaSuccess)
      return fail("cudaFuncSetAttribute", e);
  if ((e = cudaHostAlloc((void**)&h->h_err, 64, cudaHostAllocMapped)) != cudaSuccess) return fail("cudaHostAlloc", e);
  *h->h_err = 0;
  if ((e = cudaHostGetDevicePointer((void**)&h->d_err, h->h_err, 0)) != cudaSuccess) return fail("cudaHostGetDevicePointer", e);
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
  delete h->pipe;
  for (int k = 0; k < 2; ++k) for (int l = 0; l <= artp::kMaxLevel; ++l) { cudaFree(h->d_T[k][l]); cudaFree(h->d_C[k][l]); }
  cudaFree(h->d_H[0]); cudaFree(h->d_H[1]); cudaFree(h->d_stage); cudaFree(h->d_simplify);
  sampling_free(h);
  roadmap_free(h);
  planner_free(h);
  cost_net_free(h);
  if (h->h_err) cudaFreeHost(h->h_err);
  for (cudaEvent_t ev : h->chain_ev) if (ev) cudaEventDestroy(ev);
  delete h;
}

int artp_has_map(const artp_handle* hh) {
  if (!hh) return 0;
  Handle* h = reinterpret_cast<Handle*>(const_cast<artp_handle*>(hh));
  std::lock_guard<std::mutex> lock(h->mtx);
  return h->has_map ? 1 : 0;
}

int artp_set_mode(artp_handle* hh, int mode) {
  LOCK_HANDLE(h, hh);
  if (mode < 0 || mode > 1) return ARTP_E_INVALID;
  h->pipe->mode = mode;
  return ARTP_OK;
}

int artp_set_timing(artp_handle* hh, int enable) {
  LOCK_HANDLE(h, hh);
  CU_TRY(h, cudaSetDevice(h->device));
  if (enable && !h->pipe->ev[0]) for (cudaEvent_t& ev : h->pipe->ev) CU_TRY(h, cudaEventCreate(&ev));
  h->pipe->timing = enable ? 1 : 0;
  h->pipe->ev_valid = false;
  return ARTP_OK;
}

int artp_get_last_timing(artp_handle* hh, float* ms3) {
  LOCK_HANDLE(h, hh);
  return timed_round_ms(h, ms3, {{0, 1}, {1, 4}, {4, 5}});   // classify | box stages | plane grouping
}

int artp_get_last_stage_timing(artp_handle* hh, float* ms5) {
  LOCK_HANDLE(h, hh);
  return timed_round_ms(h, ms5, {{0, 1}, {1, 2}, {2, 3}, {3, 4}, {4, 5}});
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
  h->pipe->tcap_override = max_triangles;   // takes effect at the next artp_set_map
  return ARTP_OK;
}

int artp_debug_get_reach_queue(artp_handle* hh, void* recs, size_t cap, size_t* n) {
  LOCK_HANDLE(h, hh);
  if (!n || (cap && !recs)) return ARTP_E_INVALID;
  CU_TRY(h, cudaSetDevice(h->device));
  Counters ctr{};
  CU_TRY(h, cudaMemcpy(&ctr, h->pipe->d_ctr, sizeof(ctr), cudaMemcpyDeviceToHost));   // synchronises the device
  *n = ctr.q.reach.end;
  const size_t k = std::min(cap, (size_t)ctr.q.reach.end);
  if (k) CU_TRY(h, cudaMemcpy(recs, h->pipe->recs[h->pipe->kReach], k * sizeof(artp::BoxRec), cudaMemcpyDeviceToHost));
  return ARTP_OK;
}

int artp_get_stats(artp_handle* hh, artp_stats* out) {
  LOCK_HANDLE(h, hh);
  if (!out) return ARTP_E_INVALID;
  CU_TRY(h, cudaSetDevice(h->device));
  Counters ctr{};
  CU_TRY(h, cudaMemcpy(&ctr, h->pipe->d_ctr, sizeof(ctr), cudaMemcpyDeviceToHost));   // synchronises the device
  h->stats.last_deferred = ctr.defer;
  h->stats.last_queued_boxes = ctr.q.big.end + ctr.q.reach.end + ctr.q.group.end;
  h->stats.last_queued_warp_stage = ctr.q.big.end;
  h->stats.last_queued_reach_stage = ctr.q.reach.end;
  h->stats.last_reach_plane_stage = ctr.q.group.end;
  if (h->pipe->deferred_unread) { h->stats.poses_deferred += ctr.defer; h->pipe->deferred_unread = false; }
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
  LOCK_CALL(h, hh);
  h->planner_map = false;
  return upload_map(h, elevation, elevation_masked, false, rows, cols, res, cx, cy, row0, nrows);
}

}  // extern "C"

int artp_api::upload_map(Handle* h, const float* elevation, const float* elevation_masked, bool device_src, int rows, int cols,
                         double res, double cx, double cy, int row0, int nrows) {
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
  // Each box's zone, bounded by its half-diagonal r: at most ceil(2 r / s) + 3 vertices along an axis of cell size s. The
  // same bound sizes the range tables, the grouping stage's plane store and the tiles of stage B.
  int span[2][2], kmax[2], tcap = 0;
  for (int k = 0; k < 2; ++k) {
    const float* sd = h->chk.side[k];
    const double r = 0.5 * std::sqrt((double)sd[0] * sd[0] + (double)sd[1] * sd[1] + (double)sd[2] * sd[2]);
    span[k][0] = (int)std::ceil(2.0 * r * f.iW); span[k][1] = (int)std::ceil(2.0 * r * f.iD);
    const int nxm = std::min(rows, span[k][0] + 4), nzm = std::min(cols, span[k][1] + 4);
    tcap = std::max(tcap, 2 * (nxm - 1) * (nzm - 1));
    int kk = 0;
    while ((2 << kk) <= std::min(nxm, nzm) && kk < artp::kMaxLevel) ++kk;   // floor(log2(min dim bound))
    kmax[k] = kk;
  }
  if (h->pipe->tcap_override > 0) tcap = std::min(tcap, h->pipe->tcap_override);   // test hook: force the overflow path
  tcap = (tcap + 3) & ~3;
  const int store = tcap * 21 + 64;   // bytes of the grouping stage's plane store
  if (store > kMaxStoreSmem) {
    h->err = "box/map resolution combination exceeds the plane-grouping kernel's shared-memory store";
    return ARTP_E_LIMIT;
  }
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
  TRY(grow(h, h->d_stage, h->stage_cap, ncell * sizeof(float)));
  const float* src[2] = {elevation, elevation_masked};
  float cbase[2], cstep[2];
  if (device_src) {   // the finite range of each layer from the device: the only bytes that come back
    uint32_t* d_mm = (uint32_t*)h->d_stage;
    uint32_t mm[6];
    for (int k = 0; k < 2; ++k) TRY(finite_min_max(h, src[k], ncell, d_mm + 3 * k, h->stream));
    TRY(copy_async(h, mm, d_mm, sizeof(mm), cudaMemcpyDeviceToHost, h->stream));
    TRY(sync_stream(h, h->stream));
    for (int k = 0; k < 2; ++k)
      code_scale_of(mm[3 * k + 2] ? key_float(mm[3 * k]) : HUGE_VALF, mm[3 * k + 2] ? key_float(mm[3 * k + 1]) : -HUGE_VALF,
                    cbase[k], cstep[k]);
  } else {
    for (int k = 0; k < 2; ++k) code_scale(src[k], ncell, cbase[k], cstep[k]);
  }
  // plane tables (temporary): 4 slots per cell = load factor 0.5 for the 2 triangles of a cell
  size_t cap = 1;
  while (cap < 4 * ncell) cap <<= 1;
  PlaneSlot* d_tab = nullptr;
  unsigned char* d_merge = nullptr;   // [0, npad): mergeable cells; [npad, 3 npad): two byte-flag levels (ping-pong while building)
  CU_TRY(h, cudaMalloc(&d_tab, cap * sizeof(PlaneSlot)));
  if (cudaMalloc(&d_merge, 3 * npad) != cudaSuccess) { cudaFree(d_tab); h->err = "cudaMalloc (plane tables)"; return ARTP_E_CUDA; }
  for (int k = 0; k < 2; ++k) {
    if (!device_src) TRY(copy_async(h, h->d_stage, src[k], ncell * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    const unsigned g4 = (unsigned)h->sm_count * 4, g8 = (unsigned)h->sm_count * 8;
    TRY(launch(h, reverse_columns_kernel, g4, 256, 0, h->stream, device_src ? src[k] : (const float*)h->d_stage, h->d_H[k], nrows,
               cols, pitch));
    artp::Field fk = f;                     // local storage, global geometry: cell x of the window is global cell x + row0
    fk.H = h->d_H[k]; fk.pitch = pitch; fk.nx = nrows;
    TRY(launch(h, plane_table_clear_kernel, g8, 256, 0, h->stream, d_tab, cap));
    CU_TRY(h, cudaMemsetAsync(d_merge, 0, npad, h->stream));
    TRY(launch(h, plane_table_insert_kernel, g8, 256, 0, h->stream, fk, row0, d_tab, (uint32_t)(cap - 1)));
    TRY(launch(h, plane_table_query_kernel, g8, 256, 0, h->stream, fk, row0, d_tab, (uint32_t)(cap - 1), d_merge));
    for (int l = 1; l <= kmax[k]; ++l) {
      unsigned char* nf_prev = d_merge + npad * (size_t)(1 + ((l - 1) & 1));
      unsigned char* nf_cur = d_merge + npad * (size_t)(1 + (l & 1));
      TRY(launch(h, build_level_kernel, g4, 256, 0, h->stream, h->d_H[k], l > 1 ? h->d_T[k][l - 1] : nullptr,
          l > 1 ? nf_prev : nullptr, d_merge, h->d_T[k][l], nf_cur, nrows, cols, pitch, 1 << (l - 1)));
      TRY(launch(h, build_codes_kernel, g4, 256, 0, h->stream, h->d_T[k][l], nf_cur, h->d_C[k][l], npad, cbase[k], cstep[k]));
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
  TRY(set_shapes(h, span, tcap, store));
  h->has_map = true;
  sampling_forget_map(h);
  h->res = res;
  return ARTP_OK;
}

extern "C" {

int artp_check_poses(artp_handle* hh, const double* states, size_t n, uint8_t* valid) {
  LOCK_CALL(h, hh);
  return check_poses(h, states, n, valid, false, nullptr);
}
int artp_check_poses_f32(artp_handle* hh, const float* states, size_t n, uint8_t* valid) {
  LOCK_CALL(h, hh);
  return check_poses(h, states, n, valid, false, nullptr);
}
int artp_check_poses_device(artp_handle* hh, const double* d_states, size_t n, uint8_t* d_valid, void* stream) {
  LOCK_CALL(h, hh);
  return check_poses(h, d_states, n, d_valid, true, (cudaStream_t)stream);
}
int artp_check_poses_f32_device(artp_handle* hh, const float* d_states, size_t n, uint8_t* d_valid, void* stream) {
  LOCK_CALL(h, hh);
  return check_poses(h, d_states, n, d_valid, true, (cudaStream_t)stream);
}

int artp_box_verdicts(artp_handle* hh, const double* states, size_t n, uint16_t* why) {
  LOCK_CALL(h, hh);
  TRY(box_verdict_args(h, n));
  if (n == 0) return ARTP_OK;
  if (!states || !why) return null_buffer(h);
  const size_t sb = n * 7 * sizeof(double), wb = n * sizeof(uint16_t);
  char* r[2];   // states | words
  TRY(host_call_begin(h, {sb, wb}, r));
  TRY(copy_async(h, r[0], states, sb, cudaMemcpyHostToDevice, h->stream));
  TRY(box_verdicts_on(h, (const double*)r[0], n, (uint16_t*)r[1], h->stream));
  TRY(copy_async(h, why, r[1], wb, cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h, true);
}
int artp_box_verdicts_device(artp_handle* hh, const double* d_states, size_t n, uint16_t* d_why, void* stream) {
  LOCK_CALL(h, hh);
  TRY(box_verdict_args(h, n));
  if (n == 0) return ARTP_OK;
  if (!d_states || !d_why) return null_buffer(h);
  CU_TRY(h, cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  ChainScope cs(h, 0, s);
  if (cs.rc) return cs.rc;
  return box_verdicts_on(h, d_states, n, d_why, s);
}

int artp_check_motions_device(artp_handle* hh, const double* d_s1, const double* d_s2, size_t n, int n_steps,
                              uint8_t* d_valid, void* stream) {
  LOCK_CALL(h, hh);
  TRY(motion_items(h, n, n_steps));
  if (n == 0) return ARTP_OK;
  if (!d_s1 || !d_s2 || !d_valid) return null_buffer(h);
  CU_TRY(h, cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  ChainScope cs(h, 0, s);
  if (cs.rc) return cs.rc;
  return check_motions_on(h, d_s1, d_s2, n, n_steps, d_valid, s);
}

int artp_check_motions(artp_handle* hh, const double* s1, const double* s2, size_t n, int n_steps, uint8_t* valid) {
  LOCK_CALL(h, hh);
  TRY(require_map(h));
  if (n == 0) return ARTP_OK;
  if (!s1 || !s2 || !valid) return null_buffer(h);
  if (n_steps >= 0 && n * ((size_t)n_steps + 1) <= (size_t)artp::kSmallBatch && 2 * n <= (size_t)artp::kSmallBatch &&
      !h->pipe->timing) {
    // latency path (a single checkMotion call): one fused launch, interpolation on the device as in the pipeline
    artp::SmallBatch sb;
    for (size_t e = 0; e < n; ++e) {
      std::memcpy(sb.s[2 * e], s1 + 7 * e, 7 * sizeof(double));
      std::memcpy(sb.s[2 * e + 1], s2 + 7 * e, 7 * sizeof(double));
    }
    return check_poses_small(h, sb, n * ((size_t)n_steps + 1), valid, n_steps);
  }
  TRY(motion_items(h, n, n_steps));
  const size_t sb = n * 7 * sizeof(double);
  char* r[3];
  TRY(host_call_begin(h, {sb, sb, n}, r));
  CU_TRY(h, cudaMemcpyAsync(r[0], s1, sb, cudaMemcpyHostToDevice, h->stream));
  CU_TRY(h, cudaMemcpyAsync(r[1], s2, sb, cudaMemcpyHostToDevice, h->stream));
  TRY(check_motions_on(h, (const double*)r[0], (const double*)r[1], n, n_steps, (uint8_t*)r[2], h->stream));
  CU_TRY(h, cudaMemcpyAsync(valid, r[2], n, cudaMemcpyDeviceToHost, h->stream));
  return host_call_end(h, true);
}

int artp_check_edge_interiors_device(artp_handle* hh, const double* d_s1, const double* d_s2, size_t n,
                                     const uint32_t* d_item_off, size_t total_items, uint8_t* d_item_valid,
                                     int32_t* d_valid_prefix, void* stream) {
  LOCK_CALL(h, hh);
  return check_items_prefix(h, d_s1, d_s2, n, d_item_off, total_items, d_item_valid, d_valid_prefix, stream, 0);
}

int artp_check_edge_interiors(artp_handle* hh, const double* s1, const double* s2, size_t n, const int32_t* n_interp,
                              double max_lateral, int32_t* valid_prefix) {
  LOCK_CALL(h, hh);
  TRY(require_map(h));
  if (n == 0) return ARTP_OK;
  if (!s1 || !s2 || !valid_prefix) return null_buffer(h);
  if (!n_interp && !(max_lateral > 0.0)) { h->err = "n_interp == NULL needs max_lateral > 0"; return ARTP_E_INVALID; }
  std::vector<uint32_t> off(n + 1);
  size_t total = 0;
  for (size_t e = 0; e < n; ++e) {
    off[e] = (uint32_t)total;
    const long long ne = n_interp ? n_interp[e] : artp::lateral_count(s1 + 7 * e, s2 + 7 * e, max_lateral);
    if (ne < 0) { h->err = "n_interp < 0"; return ARTP_E_INVALID; }
    total += (size_t)ne;
    if (total >= 0xFFFFFFFFull) { h->err = "too many interior states (>= 2^32)"; return ARTP_E_INVALID; }
  }
  off[n] = (uint32_t)total;
  return check_items_prefix_host(h, s1, s2, off, 0, valid_prefix);
}

// SE3StateSpace::validSegmentCount on the host (artp::valid_segment_count).
int artp_valid_segment_count(const artp_se3_space* sp, const double* s1, const double* s2, size_t n, int32_t* nd) {
  if (!sp || (n && (!s1 || !s2 || !nd))) return ARTP_E_INVALID;
  artp::SegLen seg;
  if (!artp::segment_lengths(*sp, seg)) return ARTP_E_INVALID;
  for (size_t i = 0; i < n; ++i) nd[i] = (int32_t)artp::valid_segment_count(s1 + 7 * i, s2 + 7 * i, seg);
  return ARTP_OK;
}

int artp_check_motions_segments(artp_handle* hh, const double* s1, const double* s2, size_t n, const int32_t* nd,
                                const artp_se3_space* sp, uint8_t* valid, double* last_valid_t) {
  LOCK_CALL(h, hh);
  TRY(require_map(h));
  if (n == 0) return ARTP_OK;
  if (!s1 || !s2 || !valid || (!nd && !sp)) { h->err = "null buffer (nd == NULL needs the space parameters)"; return ARTP_E_INVALID; }
  artp::SegLen sl;
  if (!nd && !artp::segment_lengths(*sp, sl)) { h->err = "bad SE3 space parameters"; return ARTP_E_INVALID; }
  std::vector<int32_t> seg(n);
  std::vector<uint32_t> off(n + 1);
  size_t total = 0;
  for (size_t e = 0; e < n; ++e) {
    seg[e] = nd ? nd[e] : (int32_t)artp::segment_count(s1 + 7 * e, s2 + 7 * e, sl);
    if (seg[e] < 0) { h->err = "segment count < 0"; return ARTP_E_INVALID; }
    if (seg[e] < 1) seg[e] = 1;                 // a caller's nd = 0 (identical states): only s2 is checked
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

int artp_compact_valid_device(artp_handle* hh, const uint8_t* d_valid, size_t n, int64_t base, int64_t* d_indices,
                              uint32_t* d_count, void* stream) {
  LOCK_CALL(h, hh);
  if (!d_valid || !d_indices || !d_count) return null_buffer(h);
  CU_TRY(h, cudaSetDevice(h->device));
  return compact_valid(h, d_valid, n, base, d_indices, d_count, (cudaStream_t)stream);
}

int artp_compact_valid_u32_device(artp_handle* hh, const uint8_t* d_valid, size_t n, uint32_t base, uint32_t* d_indices,
                                  uint32_t* d_count, void* stream) {
  LOCK_CALL(h, hh);
  if (!d_valid || !d_indices || !d_count) return null_buffer(h);
  if (n + (size_t)base > 0xFFFFFFFFull) { h->err = "indices do not fit 32 bits"; return ARTP_E_INVALID; }
  CU_TRY(h, cudaSetDevice(h->device));
  return compact_valid(h, d_valid, n, (int64_t)base, d_indices, d_count, (cudaStream_t)stream, false, true);
}

// isValid for a shard + the bit-packed verdicts the multi-GPU exchange sends, in one call on one stream.
int artp_check_poses_bits_device(artp_handle* hh, const double* d_states, size_t n, uint8_t* d_valid, uint32_t* d_bits, void* stream) {
  LOCK_CALL(h, hh);
  TRY(check_poses(h, d_states, n, d_valid, true, (cudaStream_t)stream));
  return pack_valid_bits(h, d_valid, n, d_bits, (cudaStream_t)stream);
}

int artp_pack_valid_bits_device(artp_handle* hh, const uint8_t* d_valid, size_t n, uint32_t* d_bits, void* stream) {
  LOCK_CALL(h, hh);
  return pack_valid_bits(h, d_valid, n, d_bits, (cudaStream_t)stream);
}

int artp_compact_bits_device(artp_handle* hh, const uint32_t* d_bits, size_t n, int64_t base, int64_t* d_indices,
                             uint32_t* d_count, void* stream) {
  LOCK_CALL(h, hh);
  if (!d_bits || !d_indices || !d_count) return null_buffer(h);
  CU_TRY(h, cudaSetDevice(h->device));
  return compact_valid(h, reinterpret_cast<const uint8_t*>(d_bits), n, base, d_indices, d_count, (cudaStream_t)stream, true);
}

}  // extern "C"
