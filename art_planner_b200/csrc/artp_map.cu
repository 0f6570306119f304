// art_planner_b200/csrc/artp_map.cu -- the installed map of the C ABI (include/artp.h): artp_set_map and
// artp_set_map_window ~ setMap + updateHeightField (HeightMapBoxChecker::setHeightField,
// art_planner/src/validity_checker/height_map_box_checker.cpp:38-54), and artp_has_map. The unit owns the map's device
// buffers -- both column-reversed height layers and their range tables and compact codes -- and is the only one that
// writes what the others read of the map: Handle::map and the map fields of Handle::chk (artp_internal.h). The
// reductions over a layer (its finite range, whether it holds a non-finite cell) live here too.
#include <cmath>
#include <cstring>

#include "artp_internal.h"

namespace artp_api {

// The map's device buffers: each layer at Handle::map.pitch (pad columns never read) and its range-table and code levels
// 1 .. kmax, allocated at their first use and kept while the window's rows and columns stay the same.
struct MapStore {
  float* d_H[2] = {nullptr, nullptr};
  float2* d_T[2][artp::kMaxLevel + 1] = {};
  uint32_t* d_C[2][artp::kMaxLevel + 1] = {};    // compact conservative copies of d_T (Field::C)
  ~MapStore() {
    for (int k = 0; k < 2; ++k) {
      for (int l = 0; l <= artp::kMaxLevel; ++l) { cudaFree(d_T[k][l]); cudaFree(d_C[k][l]); }
      cudaFree(d_H[k]);
    }
  }
};

}  // namespace artp_api

using namespace artp_api;

namespace {

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

// ---------------------------------------------------------------------------------------------------------------
// Reductions over a layer
__device__ __forceinline__ uint32_t float_key(float f) {   // order-preserving: a < b <=> key(a) < key(b)
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// minCoeffOfFinites / maxCoeffOfFinites: min and max over the finite cells, -0 taken as +0 (the two compare equal).
__global__ void finite_min_max_kernel(const float* __restrict__ a, size_t n, uint32_t* __restrict__ out) {
  uint32_t lo = 0xFFFFFFFFu, hi = 0u, cnt = 0u;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float v = a[i] + 0.0f;
    if (fabsf(v) < CUDART_INF_F) { const uint32_t k = float_key(v); lo = min(lo, k); hi = max(hi, k); ++cnt; }
  }
  lo = __reduce_min_sync(0xFFFFFFFFu, lo);
  hi = __reduce_max_sync(0xFFFFFFFFu, hi);
  cnt = __reduce_add_sync(0xFFFFFFFFu, cnt);
  if ((threadIdx.x & 31) == 0 && cnt) { atomicMin(out, lo); atomicMax(out + 1, hi); atomicAdd(out + 2, cnt); }
}

// out[0] = 1 when a cell is NaN or +-inf, out[1] = 1 when a cell is +-inf (both zeroed first).
__global__ void nonfinite_any_kernel(const float* __restrict__ a, size_t n, uint32_t* __restrict__ out) {
  uint32_t nonfinite = 0u, inf = 0u;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float v = fabsf(a[i]);
    nonfinite |= !(v < CUDART_INF_F);
    inf |= v == CUDART_INF_F;
  }
  nonfinite = __reduce_or_sync(0xFFFFFFFFu, nonfinite);
  inf = __reduce_or_sync(0xFFFFFFFFu, inf);
  if ((threadIdx.x & 31) == 0) {
    if (nonfinite) atomicOr(out, 1u);
    if (inf) atomicOr(out + 1, 1u);
  }
}

MapStore& map_store(Handle* h) {
  if (!h->map_store) h->map_store = new MapStore();
  return *h->map_store;
}

}  // namespace

int artp_api::finite_min_max(Handle* h, const float* d_layer, size_t n, uint32_t* d_out, cudaStream_t s) {
  CU_TRY(h, cudaMemsetAsync(d_out, 0xFF, sizeof(uint32_t), s));
  CU_TRY(h, cudaMemsetAsync(d_out + 1, 0, 2 * sizeof(uint32_t), s));
  return launch(h, finite_min_max_kernel, grid_for(h, n, 256, 8), 256, 0, s, d_layer, n, d_out);
}

int artp_api::nonfinite_any(Handle* h, const float* d_layer, size_t n, uint32_t* d_out, cudaStream_t s) {
  CU_TRY(h, cudaMemsetAsync(d_out, 0, 2 * sizeof(uint32_t), s));
  return launch(h, nonfinite_any_kernel, grid_for(h, n, 256, 8), 256, 0, s, d_layer, n, d_out);
}

float artp_api::key_float(uint32_t key) {
  const uint32_t u = (key & 0x80000000u) ? (key & 0x7FFFFFFFu) : ~key;
  float f;
  std::memcpy(&f, &u, sizeof(f));
  return f;
}

void artp_api::map_free(Handle* h) {
  delete h->map_store;
  h->map_store = nullptr;
}

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
  int store = 0;
  TRY(plane_store(h, tcap, store));
  // upload (the previous map may still be in use by asynchronous calls on the caller's streams)
  CU_TRY(h, cudaDeviceSynchronize());
  h->chain_busy[0] = h->chain_busy[1] = false;
  MapStore& m = map_store(h);
  const int pitch = (nrows + 3) & ~3;
  const size_t npad = (size_t)pitch * cols;
  if (h->map.win_rows != nrows || h->map.cols != cols) {
    for (int k = 0; k < 2; ++k) {
      cudaFree(m.d_H[k]); m.d_H[k] = nullptr;
      for (int l = 0; l <= artp::kMaxLevel; ++l) {
        cudaFree(m.d_T[k][l]); cudaFree(m.d_C[k][l]);
        m.d_T[k][l] = nullptr; m.d_C[k][l] = nullptr;
      }
      CU_TRY(h, cudaMalloc(&m.d_H[k], npad * sizeof(float)));
    }
  }
  for (int k = 0; k < 2; ++k)
    for (int l = 1; l <= kmax[k]; ++l)
      if (!m.d_T[k][l]) {
        CU_TRY(h, cudaMalloc(&m.d_T[k][l], npad * sizeof(float2)));
        CU_TRY(h, cudaMalloc(&m.d_C[k][l], npad * sizeof(uint32_t)));
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
    TRY(launch(h, reverse_columns_kernel, g4, 256, 0, h->stream, device_src ? src[k] : (const float*)h->d_stage, m.d_H[k], nrows,
               cols, pitch));
    artp::Field fk = f;                     // local storage, global geometry: cell x of the window is global cell x + row0
    fk.H = m.d_H[k]; fk.pitch = pitch; fk.nx = nrows;
    TRY(launch(h, plane_table_clear_kernel, g8, 256, 0, h->stream, d_tab, cap));
    CU_TRY(h, cudaMemsetAsync(d_merge, 0, npad, h->stream));
    TRY(launch(h, plane_table_insert_kernel, g8, 256, 0, h->stream, fk, row0, d_tab, (uint32_t)(cap - 1)));
    TRY(launch(h, plane_table_query_kernel, g8, 256, 0, h->stream, fk, row0, d_tab, (uint32_t)(cap - 1), d_merge));
    for (int l = 1; l <= kmax[k]; ++l) {
      unsigned char* nf_prev = d_merge + npad * (size_t)(1 + ((l - 1) & 1));
      unsigned char* nf_cur = d_merge + npad * (size_t)(1 + (l & 1));
      TRY(launch(h, build_level_kernel, g4, 256, 0, h->stream, m.d_H[k], l > 1 ? m.d_T[k][l - 1] : nullptr,
          l > 1 ? nf_prev : nullptr, d_merge, m.d_T[k][l], nf_cur, nrows, cols, pitch, 1 << (l - 1)));
      TRY(launch(h, build_codes_kernel, g4, 256, 0, h->stream, m.d_T[k][l], nf_cur, m.d_C[k][l], npad, cbase[k], cstep[k]));
    }
  }
  CU_TRY(h, cudaStreamSynchronize(h->stream));
  cudaFree(d_tab); cudaFree(d_merge);
  MapView& v = h->map;
  v.rows = rows; v.cols = cols; v.pitch = pitch; v.win_row0 = row0; v.win_rows = nrows;
  v.H[0] = m.d_H[0]; v.H[1] = m.d_H[1];
  f.pitch = pitch;
  f.x_lo = row0; f.x_hi = row0 + nrows - 1;
  for (int k = 0; k < 2; ++k) {
    f.H = m.d_H[k] - row0;                  // indexed with GLOBAL vertex indices x in [x_lo, x_hi]
    f.kmax = kmax[k];
    f.cbase = cbase[k]; f.cstep = cstep[k];
    for (int l = 0; l <= artp::kMaxLevel; ++l) {
      f.T[l] = (l >= 1 && l <= kmax[k]) ? m.d_T[k][l] - row0 : nullptr;
      f.C[l] = (l >= 1 && l <= kmax[k]) ? m.d_C[k][l] - row0 : nullptr;
    }
    h->chk.f[k] = f;
  }
  h->chk.err_word = h->d_err;
  h->chk.Lx = Lx; h->chk.Ly = Ly; h->chk.cx = cx; h->chk.cy = cy;
  h->chk.cell_margin = 0.02f + 2e-6f * (float)std::max(rows, cols);
  TRY(set_shapes(h, span, tcap, store));
  v.has_map = true;
  sampling_forget_map(h);
  v.res = res;
  return ARTP_OK;
}

extern "C" {

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

int artp_has_map(const artp_handle* hh) {
  if (!hh) return 0;
  Handle* h = reinterpret_cast<Handle*>(const_cast<artp_handle*>(hh));
  std::lock_guard<std::mutex> lock(h->mtx);
  return h->map.has_map ? 1 : 0;
}

}  // extern "C"
