// art_planner_b200/csrc/artp_inpaint.cuh -- inpaintMatrix (art_planner/src/utils.cpp:13-63) on the device, bit for bit
// with OpenCV's cv::inpaint(radius 3, INPAINT_TELEA) as restated by oracle/inpaint_oracle.py.
//
// The image is the cols x rows image of the column-major layer: image row y = grid_map column j, image column x =
// grid_map row i, so image raster index y * W + x (W = rows) IS the layer's memory index.
//
// Exactness. OpenCV's march pops a stable priority queue in (T, push order). Computing a cell reads f, t and out only
// within Chebyshev distance 4 of it (radius 3, +1 for the image gradient), and the outer pass (icvCalcFMM with negated T)
// only touches the ring within 3 of the mask. So two holes further apart than 7 never read what the other writes, and the
// 8-connected components of the mask dilated by the 7 x 7 square ("interaction components") are independent marches: each
// run alone in its own (T, push order) pops its cells in the same relative order as the whole-image queue does. One warp
// marches one component; the components run in parallel.
//
//   inp_prep_kernel      8-bit conversion (fused multiply-add, like convertTo's SIMD path) and the NaN mask
//   inp_region_kernel    band / ring / interaction region, union-find seeds
//   inp_union_kernel     8-neighbour unions inside the region (atomicMin union-find)
//   inp_root_kernel      labels flattened to their roots; each root takes a component slot
//   inp_bbox_kernel      each component's bounding box and cell count (its heap's capacity)
//   inp_class_*_kernel   the order the warps take components in: largest size class first
//   inp_march_kernel     one warp per component: outer FMM, negation, TELEA march
//   inp_finish_kernel    back to float (two float operations), column / row 0 copies
//
// The cost server's preparation of the same raw layer (cost_query_server.py, _elvMapProcess) reuses the stages from
// region to march on an image of its own, with its own prep and finish (cm_prep_kernel, cm_finish_kernel). Stated once,
// all float32 round-to-nearest with no contraction (oracle/cost_map_oracle.py restates it):
//   1. E = layer[::-1, ::-1], rows x cols: E[r][c] = layer(rows-1-r, cols-1-c), the image the trunk reads.
//   2. No cell NaN or +-inf: the result is E itself.
//   3. Otherwise mn / mx = min / max over the finite cells, d = mx - mn, and on the finite cells
//      q = trunc(((E - mn) * 255) / d) (so the max cell can land at 254; 0 / 0 when mx == mn gives byte 0, so that map
//      comes back as mn everywhere); the mask is ~isfinite(E), and a masked cell holds 0. Both zeros are numpy's
//      astype(uint8) of NaN on x86-64. The march reads a masked cell before filling it only through the image gradient's
//      clamped reads at the border, so its byte matters only for components within two cells of the border.
//   4. TELEA with radius 3 on q in E's orientation (image row r, column c: raster index r * cols + c).
//   5. out = ((float)u * d) / 255 + mn on every cell, known cells too; no row / column 0 copies.
// The C ABI refuses (ARTP_E_INVALID, before any work) a +-inf cell and a layer without a finite cell, where the server's
// output is NaN, and a range whose d * 255 overflows, where it casts infinite quotients to 8 bits (undefined in numpy).
//
// The heap of a component is a binary min-heap on the 64-bit key (order-preserving T bits << 32 | push sequence) in global
// memory; the initial band's sequence is its raster index (Heap->Add pushes it in raster order, all at T = 0), later
// pushes count from N. All arithmetic uses explicit round-to-nearest intrinsics, so no contraction can change a bit.
#pragma once
#include <math_constants.h>

#include <cstdint>

namespace artp_inpaint {

enum : uint8_t { F_INS = 1, F_RING = 2, F_CHG = 4, F_BAND = 8, F_MASK = 16, F_REGION = 32 };
constexpr int kRange = 3;
constexpr int kWin = 2 * kRange + 1;             // 7 x 7 window, 49 offsets
constexpr int kWarps = 4;                        // warps per march CTA

struct Comp {   // one interaction component
  int root, y0, y1, x0, x1, count;
};

__device__ __forceinline__ uint32_t t_key(float t) {   // order-preserving, -0 folded to +0
  const uint32_t u = __float_as_uint(__fadd_rn(t, 0.0f));
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ uint8_t to_u8(float x, float a, float b) {   // saturate_cast<uchar>(fma(x, a, b))
  const float v = __fmaf_rn(x, a, b);
  if (!(fabsf(v) < 2147483648.0f)) return 0;           // cvRound's INT_MIN for non-finite / out of range
  const int r = __float2int_rn(v);
  return (uint8_t)min(255, max(0, r));
}

// min / max from finite_min_max's keys (artp_map.cu)
__device__ __forceinline__ float key_to_float(uint32_t key) {
  return __uint_as_float((key & 0x80000000u) ? (key & 0x7FFFFFFFu) : ~key);
}

struct Scale { float mn, alpha, beta, scale; };
__device__ __forceinline__ Scale scale_of(const uint32_t* mm) {
  Scale s;
  s.mn = key_to_float(mm[0]);
  const float mx = key_to_float(mm[1]);
  const float rg = __fsub_rn(mx, s.mn);
  s.alpha = __fdiv_rn(255.0f, rg);                                 // 255/(max-min), float
  s.beta = __fdiv_rn(__fmul_rn(-s.mn, 255.0f), rg);                // -min*255/(max-min), float
  s.scale = __fdiv_rn(rg, 255.0f);                                 // (max-min)/255
  return s;
}

__global__ void inp_prep_kernel(const float* __restrict__ layer, size_t n, const uint32_t* __restrict__ mm,
                                uint8_t* __restrict__ img, uint8_t* __restrict__ flag) {
  const Scale s = scale_of(mm);
  for (size_t c = blockIdx.x * (size_t)blockDim.x + threadIdx.x; c < n; c += (size_t)gridDim.x * blockDim.x) {
    const float v = layer[c];
    img[c] = to_u8(v, s.alpha, s.beta);
    flag[c] = isnan(v) ? F_MASK : 0;
  }
}

__global__ void inp_region_kernel(int H, int W, uint8_t* __restrict__ flag, float* __restrict__ t, int* __restrict__ label) {
  const size_t n = (size_t)H * W;
  for (size_t c = blockIdx.x * (size_t)blockDim.x + threadIdx.x; c < n; c += (size_t)gridDim.x * blockDim.x) {
    const int y = (int)(c / W), x = (int)(c % W);
    const uint8_t fc = flag[c];
    bool near = false;
    for (int dy = -kRange; dy <= kRange && !near; ++dy) {
      const int yy = y + dy;
      if (yy < 0 || yy >= H) continue;
      for (int dx = -kRange; dx <= kRange; ++dx) {
        const int xx = x + dx;
        if (xx >= 0 && xx < W && (flag[(size_t)yy * W + xx] & F_MASK)) { near = true; break; }
      }
    }
    uint8_t nf = fc & F_MASK;
    float tv = 1.0e6f;
    if (fc & F_MASK) nf |= F_INS | F_REGION;
    else if (near) {
      const bool band = (y > 0 && (flag[c - W] & F_MASK)) || (y + 1 < H && (flag[c + W] & F_MASK)) ||
                        (x > 0 && (flag[c - 1] & F_MASK)) || (x + 1 < W && (flag[c + 1] & F_MASK));
      nf |= F_REGION | (band ? F_BAND : F_RING);
      if (band) tv = 0.0f;
    }
    t[c] = tv;
    label[c] = near ? (int)c : -1;
    flag[c] = (uint8_t)(nf | (fc & F_MASK));
  }
}

__device__ __forceinline__ int uf_find(const int* L, int x) {
  int p = L[x];
  while (p != x) { x = p; p = L[x]; }
  return x;
}

__device__ void uf_union(int* L, int a, int b) {
  bool done = false;
  while (!done) {
    a = uf_find(L, a); b = uf_find(L, b);
    if (a < b) { const int old = atomicMin(&L[b], a); done = old == b; b = old; }
    else if (b < a) { const int old = atomicMin(&L[a], b); done = old == a; a = old; }
    else done = true;
  }
}

__global__ void inp_union_kernel(int H, int W, int* __restrict__ label) {
  const size_t n = (size_t)H * W;
  for (size_t c = blockIdx.x * (size_t)blockDim.x + threadIdx.x; c < n; c += (size_t)gridDim.x * blockDim.x) {
    if (label[c] < 0) continue;
    const int y = (int)(c / W), x = (int)(c % W);
    if (x + 1 < W && label[c + 1] >= 0) uf_union(label, (int)c, (int)c + 1);
    if (y + 1 < H) {
      const size_t d = c + W;
      if (label[d] >= 0) uf_union(label, (int)c, (int)d);
      if (x + 1 < W && label[d + 1] >= 0) uf_union(label, (int)c, (int)d + 1);
      if (x > 0 && label[d - 1] >= 0) uf_union(label, (int)c, (int)d - 1);
    }
  }
}

__global__ void inp_root_kernel(size_t n, int* __restrict__ label, int* __restrict__ slot_of, Comp* __restrict__ comps,
                                int* __restrict__ counters) {
  for (size_t c = blockIdx.x * (size_t)blockDim.x + threadIdx.x; c < n; c += (size_t)gridDim.x * blockDim.x) {
    if (label[c] < 0) continue;
    const int r = uf_find(label, (int)c);
    if (r == (int)c) {
      const int k = atomicAdd(&counters[0], 1);
      slot_of[c] = k;
      comps[k] = Comp{(int)c, 0x7FFFFFFF, -1, 0x7FFFFFFF, -1, 0};
    }
  }
}

__global__ void inp_flatten_kernel(size_t n, int* __restrict__ label) {
  for (size_t c = blockIdx.x * (size_t)blockDim.x + threadIdx.x; c < n; c += (size_t)gridDim.x * blockDim.x)
    if (label[c] >= 0) label[c] = uf_find(label, (int)c);
}

__global__ void inp_bbox_kernel(int H, int W, const int* __restrict__ label, const int* __restrict__ slot_of,
                                Comp* __restrict__ comps) {
  const size_t n = (size_t)H * W;
  for (size_t c = blockIdx.x * (size_t)blockDim.x + threadIdx.x; c < n; c += (size_t)gridDim.x * blockDim.x) {
    const int r = label[c];
    if (r < 0) continue;
    Comp* cp = comps + slot_of[r];
    const int y = (int)(c / W), x = (int)(c % W);
    atomicMin(&cp->y0, y); atomicMax(&cp->y1, y);
    atomicMin(&cp->x0, x); atomicMax(&cp->x1, x);
    atomicAdd(&cp->count, 1);
  }
}

// Hand components out largest first: order = component slots by descending power-of-two size class (counters[4 + c]
// counts class c, counters[36 + c] is its cursor). A giant component then starts at once instead of after the small ones.
__global__ void inp_class_count_kernel(const Comp* __restrict__ comps, int* __restrict__ counters) {
  const int n_comp = counters[0];
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n_comp; k += gridDim.x * blockDim.x)
    atomicAdd(&counters[4 + 31 - __clz(comps[k].count)], 1);
}

__global__ void inp_class_scatter_kernel(const Comp* __restrict__ comps, int* __restrict__ counters, int* __restrict__ order) {
  const int n_comp = counters[0];
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n_comp; k += gridDim.x * blockDim.x) {
    const int cls = 31 - __clz(comps[k].count);
    int start = 0;
    for (int c = cls + 1; c < 32; ++c) start += counters[4 + c];
    order[start + atomicAdd(&counters[36 + cls], 1)] = k;
  }
}

// ---- the march ---------------------------------------------------------------------------------------------------------

struct Grid {
  int H, W;
  uint8_t* img;
  uint8_t* flag;
  float* t;
  __device__ __forceinline__ bool in(int y, int x) const { return y >= 0 && y < H && x >= 0 && x < W; }
  __device__ __forceinline__ size_t at(int y, int x) const { return (size_t)y * W + x; }
  // the padded matrices' reads: outside the image t = 1e6 and f = KNOWN
  __device__ __forceinline__ float T(int y, int x) const { return in(y, x) ? t[at(y, x)] : 1.0e6f; }
  __device__ __forceinline__ bool inside(int y, int x, uint8_t bit) const { return in(y, x) && (flag[at(y, x)] & bit); }
  __device__ __forceinline__ float O(int y, int x) const { return (float)img[at(y, x)]; }
};

// FastMarching_solve: double arithmetic on two float T values, rounded to float
__device__ __forceinline__ float fm_solve(const Grid& g, int y1, int x1, int y2, int x2, uint8_t bit) {
  const double a11 = g.T(y1, x1), a22 = g.T(y2, x2), m12 = fmin(a11, a22);
  const bool k1 = !g.inside(y1, x1, bit), k2 = !g.inside(y2, x2, bit);
  double sol;
  if (k1) {
    if (k2) {
      const double d = __dsub_rn(a11, a22);
      if (fabs(d) >= 1.0) sol = __dadd_rn(1.0, m12);
      else sol = __dmul_rn(__dadd_rn(__dadd_rn(a11, a22), __dsqrt_rn(__dsub_rn(2.0, __dmul_rn(d, d)))), 0.5);
    } else {
      sol = __dadd_rn(1.0, a11);
    }
  } else if (k2) {
    sol = __dadd_rn(1.0, a22);
  } else {
    sol = __dadd_rn(1.0, m12);
  }
  return __double2float_rn(sol);
}

__device__ __forceinline__ float dist4(const Grid& g, int y, int x, uint8_t bit) {
  const float a = fminf(fm_solve(g, y - 1, x, y, x - 1, bit), fm_solve(g, y + 1, x, y, x - 1, bit));
  const float c = fminf(fm_solve(g, y - 1, x, y, x + 1, bit), fm_solve(g, y + 1, x, y, x + 1, bit));
  return fminf(a, c);
}

struct Heap {   // binary min-heap on (key, cell); lane 0 only
  unsigned long long* key;
  int* cell;
  int n = 0;
  __device__ void push(unsigned long long k, int c) {
    int i = n++;
    while (i > 0) {
      const int p = (i - 1) >> 1;
      const unsigned long long pk = key[p];
      if (pk <= k) break;
      key[i] = pk; cell[i] = cell[p];
      i = p;
    }
    key[i] = k; cell[i] = c;
  }
  __device__ int pop() {
    const int top = cell[0];
    const unsigned long long k = key[--n];
    const int c = cell[n];
    int i = 0;
    for (;;) {
      int ch = 2 * i + 1;
      if (ch >= n) break;
      unsigned long long ck = key[ch];
      if (ch + 1 < n && key[ch + 1] < ck) { ++ch; ck = key[ch]; }
      if (k <= ck) break;
      key[i] = ck; cell[i] = cell[ch];
      i = ch;
    }
    if (n > 0) { key[i] = k; cell[i] = c; }
    return top;
  }
};

// Push the component's band cells, in raster order, with T = 0 and their raster index as sequence.
__device__ void push_band(const Grid& g, const Comp& cp, const int* label, Heap& hp, int lane) {
  for (int y = cp.y0; y <= cp.y1; ++y)
    for (int x = cp.x0; x <= cp.x1; x += 32) {
      const int xx = x + lane;
      bool b = false;
      if (xx <= cp.x1) {
        const size_t c = g.at(y, xx);
        b = label[c] == cp.root && (g.flag[c] & F_BAND);
      }
      unsigned m = __ballot_sync(0xFFFFFFFFu, b);
      if (lane == 0)
        while (m) {
          const int l = __ffs(m) - 1; m &= m - 1;
          const size_t c = g.at(y, x + l);
          hp.push(((unsigned long long)t_key(0.0f) << 32) | (unsigned long long)c, (int)c);
        }
    }
  __syncwarp();
}

__global__ void __launch_bounds__(32 * kWarps)
inp_march_kernel(Grid g, const int* __restrict__ label, const Comp* __restrict__ comps, const int* __restrict__ order,
                 const int* counters_ro,
                 int* counters, unsigned long long* __restrict__ heap_key, int* __restrict__ heap_cell) {
  __shared__ float sh_w[kWarps][kWin * kWin], sh_o[kWarps][kWin * kWin], sh_jx[kWarps][kWin * kWin], sh_jy[kWarps][kWin * kWin];
  __shared__ uint8_t sh_ok[kWarps][kWin * kWin];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int n_comp = counters_ro[0];
  const uint32_t seq0 = (uint32_t)((size_t)g.H * g.W);
  for (;;) {
    int k = 0;
    if (lane == 0) k = atomicAdd(&counters[1], 1);
    k = __shfl_sync(0xFFFFFFFFu, k, 0);
    if (k >= n_comp) break;
    const Comp cp = comps[order[k]];
    long long base = 0;
    if (lane == 0) base = (long long)atomicAdd(reinterpret_cast<unsigned long long*>(counters + 2), (unsigned long long)cp.count);
    base = __shfl_sync(0xFFFFFFFFu, base, 0);
    Heap hp{heap_key + base, heap_cell + base, 0};
    uint32_t seq = seq0;

    // outer pass: icvCalcFMM over the ring, seeded with the band; then T = -T on every popped cell
    push_band(g, cp, label, hp, lane);
    if (lane == 0) {
      while (hp.n > 0) {
        const int c = hp.pop();
        g.flag[c] |= F_CHG;
        const int yy = c / g.W, xx = c % g.W;
        const int ny[4] = {yy - 1, yy, yy + 1, yy}, nx[4] = {xx, xx - 1, xx, xx + 1};
        for (int q = 0; q < 4; ++q) {
          const int y = ny[q], x = nx[q];
          if (!g.inside(y, x, F_RING)) continue;
          const float d = dist4(g, y, x, F_RING);
          const size_t cc = g.at(y, x);
          g.t[cc] = d;
          g.flag[cc] &= (uint8_t)~F_RING;
          hp.push(((unsigned long long)t_key(d) << 32) | seq++, (int)cc);
        }
      }
    }
    __syncwarp();
    for (int y = cp.y0; y <= cp.y1; ++y)
      for (int x = cp.x0 + lane; x <= cp.x1; x += 32) {
        const size_t c = g.at(y, x);
        if (label[c] == cp.root && (g.flag[c] & F_CHG)) { g.t[c] = -g.t[c]; g.flag[c] &= (uint8_t)~F_CHG; }
      }
    __syncwarp();

    // TELEA march
    seq = seq0;
    push_band(g, cp, label, hp, lane);
    for (;;) {
      int c = 0, live = 0;
      if (lane == 0 && hp.n > 0) { c = hp.pop(); live = 1; }
      live = __shfl_sync(0xFFFFFFFFu, live, 0);
      if (!live) break;
      c = __shfl_sync(0xFFFFFFFFu, c, 0);
      const int yy = c / g.W, xx = c % g.W;
      for (int q = 0; q < 4; ++q) {
        const int i = q == 0 ? yy - 1 : q == 2 ? yy + 1 : yy;
        const int j = q == 1 ? xx - 1 : q == 3 ? xx + 1 : xx;
        if (!g.inside(i, j, F_INS)) continue;   // warp-uniform
        const float d = dist4(g, i, j, F_INS);
        const size_t cij = g.at(i, j);
        __syncwarp();
        if (lane == 0) g.t[cij] = d;
        __syncwarp();
        const float tij = d;
        float gx, gy;
        if (!g.inside(i, j + 1, F_INS)) {
          gx = !g.inside(i, j - 1, F_INS) ? __fmul_rn(__fsub_rn(g.T(i, j + 1), g.T(i, j - 1)), 0.5f) : __fsub_rn(g.T(i, j + 1), tij);
        } else {
          gx = !g.inside(i, j - 1, F_INS) ? __fsub_rn(tij, g.T(i, j - 1)) : 0.0f;
        }
        if (!g.inside(i + 1, j, F_INS)) {
          gy = !g.inside(i - 1, j, F_INS) ? __fmul_rn(__fsub_rn(g.T(i + 1, j), g.T(i - 1, j)), 0.5f) : __fsub_rn(g.T(i + 1, j), tij);
        } else {
          gy = !g.inside(i - 1, j, F_INS) ? __fsub_rn(tij, g.T(i - 1, j)) : 0.0f;
        }
        // the window's terms, one offset per lane
        for (int p = lane; p < kWin * kWin; p += 32) {
          const int dy = p / kWin - kRange, dx = p % kWin - kRange;
          const int k2 = i + dy, l2 = j + dx;
          bool ok = g.in(k2, l2) && !(g.flag[g.at(k2, l2)] & F_INS) && dx * dx + dy * dy <= kRange * kRange;
          if (ok) {
            const int km = k2 + (k2 == 0), kp = k2 - (k2 == g.H - 1);
            const int lm = l2 + (l2 == 0), lp = l2 - (l2 == g.W - 1);
            const float ry = (float)(-dy), rx = (float)(-dx);
            const float vl = __fadd_rn(__fmul_rn(rx, rx), __fmul_rn(ry, ry));
            const float dst = __double2float_rn(__ddiv_rn(1.0, __dmul_rn((double)vl, __dsqrt_rn((double)vl))));
            const float lev = __double2float_rn(__ddiv_rn(1.0, (double)__fadd_rn(1.0f, fabsf(__fsub_rn(g.t[g.at(k2, l2)], tij)))));
            float dir = __fadd_rn(__fmul_rn(rx, gx), __fmul_rn(ry, gy));
            if ((double)fabsf(dir) <= 0.01) dir = 0.000001f;
            const float w = fabsf(__fmul_rn(__fmul_rn(dst, lev), dir));
            float gix, giy;
            if (!g.inside(k2, l2 + 1, F_INS)) {
              gix = !g.inside(k2, l2 - 1, F_INS) ? __fmul_rn(g.O(km, lp + 1) - g.O(km, lm - 1), 2.0f) : g.O(km, lp + 1) - g.O(km, lm);
            } else {
              gix = !g.inside(k2, l2 - 1, F_INS) ? g.O(km, lp) - g.O(km, lm - 1) : 0.0f;
            }
            if (!g.inside(k2 + 1, l2, F_INS)) {
              giy = !g.inside(k2 - 1, l2, F_INS) ? __fmul_rn(g.O(kp + 1, lm) - g.O(km - 1, lm), 2.0f) : g.O(kp + 1, lm) - g.O(km, lm);
            } else {
              giy = !g.inside(k2 - 1, l2, F_INS) ? g.O(kp, lm) - g.O(km - 1, lm) : 0.0f;
            }
            sh_w[wid][p] = w;
            sh_o[wid][p] = __fmul_rn(w, g.O(k2, l2));
            sh_jx[wid][p] = __fmul_rn(w, __fmul_rn(gix, rx));
            sh_jy[wid][p] = __fmul_rn(w, __fmul_rn(giy, ry));
          }
          sh_ok[wid][p] = ok;
        }
        __syncwarp();
        if (lane == 0) {   // the reference's k-major / l-minor order, in float
          float Ia = 0.0f, Jx = 0.0f, Jy = 0.0f, s = 1.0e-20f;
          for (int p = 0; p < kWin * kWin; ++p) {
            if (!sh_ok[wid][p]) continue;
            Ia = __fadd_rn(Ia, sh_o[wid][p]);
            Jx = __fsub_rn(Jx, sh_jx[wid][p]);
            Jy = __fsub_rn(Jy, sh_jy[wid][p]);
            s = __fadd_rn(s, sh_w[wid][p]);
          }
          const float den = __fadd_rn(__fsqrt_rn(__fadd_rn(__fmul_rn(Jx, Jx), __fmul_rn(Jy, Jy))), 1.0e-20f);
          const float sat = __fadd_rn(__fadd_rn(__fdiv_rn(Ia, s), __fdiv_rn(__fadd_rn(Jx, Jy), den)), 0.5f);
          g.img[cij] = to_u8(sat, 1.0f, 0.0f);
          g.flag[cij] &= (uint8_t)~F_INS;
          hp.push(((unsigned long long)t_key(d) << 32) | seq++, (int)cij);
        }
        __syncwarp();
      }
    }
  }
}

// back to float (two float operations) and the column / row 0 copies: out(i, j) = base(max(i, 1), max(j, 1))
__global__ void inp_finish_kernel(const uint8_t* __restrict__ img, int rows, int cols, const uint32_t* __restrict__ mm,
                                  float* __restrict__ out) {
  const Scale s = scale_of(mm);
  const size_t n = (size_t)rows * cols;
  for (size_t c = blockIdx.x * (size_t)blockDim.x + threadIdx.x; c < n; c += (size_t)gridDim.x * blockDim.x) {
    const int i = (int)(c % rows), j = (int)(c / rows);
    const size_t src = (size_t)max(j, 1) * rows + max(i, 1);
    out[c] = __fadd_rn(__fmul_rn((float)img[src], s.scale), s.mn);
  }
}

// ---- the cost server's preparation (steps 1-5 above) --------------------------------------------------------------------

// Steps 1 and 3: E's orientation, the truncating 8-bit conversion of the finite cells and the ~isfinite mask.
__global__ void cm_prep_kernel(const float* __restrict__ layer, int rows, int cols, const uint32_t* __restrict__ mm,
                               uint8_t* __restrict__ img, uint8_t* __restrict__ flag) {
  const float mn = key_to_float(mm[0]), d = __fsub_rn(key_to_float(mm[1]), mn);
  const size_t n = (size_t)rows * cols;
  for (size_t c = blockIdx.x * (size_t)blockDim.x + threadIdx.x; c < n; c += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(c / cols), x = (int)(c % cols);
    const float v = layer[(size_t)(rows - 1 - r) + (size_t)(cols - 1 - x) * rows];
    const bool known = fabsf(v) < CUDART_INF_F;
    const float q = __fdiv_rn(__fmul_rn(__fsub_rn(v, mn), 255.0f), d);   // NaN when d = 0: byte 0
    img[c] = known && q >= 0.0f ? (uint8_t)__float2int_rz(q) : 0;
    flag[c] = known ? 0 : F_MASK;
  }
}

// Step 5 (img: the marched image) or step 2 (img null: the layer itself), written as the layer P with
// E'[r][c] = P(rows-1-r, cols-1-c): out[i + j * rows] = P(i, j), or with reverse_cols out[i + (cols-1-j) * rows], the
// heightfield layout whose E[r][c] the trunk's SRC_MAP read takes from out[c * rows + rows-1-r] (pitch = rows).
__global__ void cm_finish_kernel(const uint8_t* __restrict__ img, const float* __restrict__ layer, int rows, int cols,
                                 const uint32_t* __restrict__ mm, bool reverse_cols, float* __restrict__ out) {
  const float mn = key_to_float(mm[0]), d = __fsub_rn(key_to_float(mm[1]), mn);
  const size_t n = (size_t)rows * cols;
  for (size_t c = blockIdx.x * (size_t)blockDim.x + threadIdx.x; c < n; c += (size_t)gridDim.x * blockDim.x) {
    const int i = (int)(c % rows), j = (int)(c / rows);
    const float v = img ? __fadd_rn(__fdiv_rn(__fmul_rn((float)img[(size_t)(rows - 1 - i) * cols + (cols - 1 - j)], d), 255.0f), mn)
                        : layer[c];
    out[(size_t)(reverse_cols ? cols - 1 - j : j) * rows + i] = v;
  }
}

}  // namespace artp_inpaint
