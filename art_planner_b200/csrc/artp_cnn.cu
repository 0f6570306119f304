// art_planner_b200/csrc/artp_cnn.cu -- the learned motion-cost network on sm_90a, and the unit of the C ABI that owns it:
// its weights, features, mode and timing, and the trunk and head launches the other units run through it.
//
// Reference: art_planner_motion_cost/src/art_planner_motion_cost/predictor/network_light.py
//   CNNpart :78-110  conv3x3(1->24)+BN, conv3x3(24->24)+BN+LReLU(0.3), maxpool 2/2, conv3x3(24->48)+BN+LReLU,
//                    conv3x3(48->48)+BN+LReLU, maxpool 3/1, conv3x3(48->48)+BN+LReLU, conv15x15(48->48)+BN+LReLU
//   FCpart  :113-165 and CostQuery.__call__ (cost_query.py:39-69), server centring (cost_query_server.py:160-161)
// and the full-width network.py (same file but for the widths: 32 where light has 24, 64 where it has 48, out0 80->64,
// out1 64->32 x 3). The weight blob's length picks the network (kNets); every kernel below is instantiated for both.
// The tensor-core path and its fp32 CUDA-core cross-check (artp_set_cnn_mode bit 0) both run 8 trunk kernels;
// artp_set_cost_weights runs 17 folding kernels.
//
// Numerics: the reference evaluates in fp16; parity here is against the fp32 evaluation of the same module to 1e-4
// relative, so everything accumulates in fp32 and the 15x15 convolution -- 83.6 % of the FLOPs, implicit GEMM
// M = output pixels, N = 48, K = 225 taps x 48 channels -- runs on the tensor cores (wgmma) with an error-compensated
// fp16 split (a = a_hi + a_lo, w = w_hi + w_lo; D += a_hi*w_hi + a_hi*w_lo + a_lo*w_hi, fp32 accumulate in
// registers), which keeps ~22 mantissa bits per product.
//
// Tensor-core kernel (conv_wgmma_kernel<KS,...>, described for the 15x15 layer): one CTA per 16(y) x 8(x) output tile
// (M = 128 = two warpgroups of m64 wgmma, N = 48).
//   * The whole input halo brick [30 y][24 x][64 ch] (hi and lo, 92 KB each) is TMA-loaded ONCE into 128B-swizzled
//     shared memory; pixels are 128-byte rows, image rows are 24 pixels = 3 swizzle atoms apart, so every one of the
//     225 taps is just a shifted view of the same brick. The A fragments are read from it with ldmatrix at the shifted
//     pixel rows (swizzle applied in the address), so no per-tap activation traffic leaves shared memory.
//   * Weights [tap][48][64] fp16 hi/lo stream through a 3-stage TMA ring (12 KB per tap) and are the wgmma B operand
//     straight from shared memory (K-major, 128B swizzle descriptors).
//   * Warp 8 = TMA producer; warps 0..7 = two MMA warpgroups, which also run the epilogue (+bias -> LeakyReLU -> fp32
//     NHWC feature map) from their register accumulators.
// Layers 2..5 (3x3) use the same kernel with an 18 x 16-pixel brick and 9 taps, writing either fp32 NHWC (before a
// max-pool) or directly the next layer's fp16 hi/lo NHWC-64 input; layer 1 (Cin = 1) stays on CUDA cores.
// A complete fp32 CUDA-core path (conv3x3_kernel, conv15_reference_kernel) is kept as the in-library cross-check.
// This translation unit is compiled WITHOUT -fmad=false (no bit-exactness requirement here).
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>
#include <string>

#include "artp_internal.h"

namespace artp_cnn {

// The widths that tell the two architectures apart: c1 = init_conv1/2, c3 = init_conv3..5 and init_flatten (the
// feature channels), nh = out0_conv1, b = out1_conv1..3 (the out2 convs read b and give 1 each).
struct NetDims { int c1, c3, nh, b[3]; };
constexpr NetDims kNets[2] = {{24, 48, 48, {24, 24, 36}},    // ARTP_COST_NET_LIGHT: network_light.py
                              {32, 64, 64, {32, 32, 32}}};   // ARTP_COST_NET_FULL: network.py

struct LayerDef { int cout, cin, k; bool bn; };
// Layer l of the blob order: init_conv1..5, init_flatten, tar0_conv1, out0_conv1, out1_conv1..3, out2_conv1..3.
static LayerDef layer_def(int net, int l) {
  const NetDims& d = kNets[net];
  if (l == 0) return {d.c1, 1, 3, true};
  if (l == 1) return {d.c1, d.c1, 3, true};
  if (l == 2) return {d.c3, d.c1, 3, true};
  if (l <= 4) return {d.c3, d.c3, 3, true};
  if (l == 5) return {d.c3, d.c3, 15, true};
  if (l == 6) return {16, 10, 1, true};
  if (l == 7) return {d.nh, d.c3 + 16, 1, true};
  if (l <= 10) return {d.b[l - 8], d.nh, 1, true};
  return {1, d.b[l - 11], 1, false};
}
static const float kBnEps = 1e-5f;
// Trunk layers whose output the tensor-core path stores as an fp16 hi/lo split (directly, or after a max-pool), in the
// bit order of the overflow flag the split kernels raise.
static const char* const kSplitLayerNames[5] = {"init_conv1", "init_conv2", "init_conv3", "init_conv4", "init_conv5"};

static size_t blob_floats(int net) {
  if (net != ARTP_COST_NET_LIGHT && net != ARTP_COST_NET_FULL) return 0;
  size_t n = 0;
  for (int i = 0; i < 14; ++i) {
    const LayerDef l = layer_def(net, i);
    n += (size_t)l.cout * l.cin * l.k * l.k + (l.bn ? 4 * l.cout : l.cout);
  }
  return n;
}

// ------------------------------------------------------------------------------------------------
// fp32 direct 3x3 convolution, NHWC, BN folded, optional LeakyReLU(0.3). One thread per output pixel, all COUT
// accumulators in registers; input tile and weight slice staged in shared memory per chunk of CK input channels.
// SRC_MAP: the input is the heightfield layer as artp_set_map stores it (H[x + z*pitch] = layer(x, nz-1-z));
// the network input E[r][c] = layer(rows-1-r, cols-1-c) = H[(rows-1-r) + c*pitch] (cost_query_server.py:74).
// ------------------------------------------------------------------------------------------------
template <int CIN, int COUT, int CK, bool ACT, bool SRC_MAP>
__global__ void __launch_bounds__(256) conv3x3_kernel(const float* __restrict__ in, int H, int W, int in_pitch,
                                                      const float* __restrict__ wf /*[9][CIN][COUT]*/,
                                                      const float* __restrict__ bias, float* __restrict__ out) {
  constexpr int T = 16;
  __shared__ float tile[(T + 2) * (T + 2) * CK];
  __shared__ __align__(16) float wsm[9 * CK * COUT];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int ox0 = blockIdx.x * T, oy0 = blockIdx.y * T;
  const int OH = H - 2, OW = W - 2;
  float acc[COUT];
#pragma unroll
  for (int i = 0; i < COUT; ++i) acc[i] = 0.0f;
  for (int c0 = 0; c0 < CIN; c0 += CK) {
    for (int i = threadIdx.x; i < (T + 2) * (T + 2) * CK; i += 256) {
      const int ci = i % CK, p = i / CK, px = p % (T + 2), py = p / (T + 2);
      const int iy = oy0 + py, ix = ox0 + px;
      float v = 0.0f;
      if (iy < H && ix < W) {
        if (SRC_MAP) v = __ldg(in + (size_t)ix * in_pitch + (H - 1 - iy));   // E[iy][ix], rows = H (x), cols = W (y)
        else v = __ldg(in + ((size_t)iy * W + ix) * CIN + c0 + ci);
      }
      tile[i] = v;
    }
    for (int i = threadIdx.x; i < 9 * CK * COUT; i += 256) {
      const int co = i % COUT, r = i / COUT, ci = r % CK, tap = r / CK;
      wsm[i] = __ldg(wf + ((size_t)tap * CIN + c0 + ci) * COUT + co);
    }
    __syncthreads();
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int ky = tap / 3, kx = tap % 3;
      const float* tp = tile + ((ty + ky) * (T + 2) + tx + kx) * CK;
#pragma unroll
      for (int ci = 0; ci < CK; ++ci) {
        const float v = tp[ci];
        const float4* wp = reinterpret_cast<const float4*>(wsm + (tap * CK + ci) * COUT);
#pragma unroll
        for (int q = 0; q < COUT / 4; ++q) {
          const float4 w4 = wp[q];
          acc[4 * q + 0] = fmaf(v, w4.x, acc[4 * q + 0]);
          acc[4 * q + 1] = fmaf(v, w4.y, acc[4 * q + 1]);
          acc[4 * q + 2] = fmaf(v, w4.z, acc[4 * q + 2]);
          acc[4 * q + 3] = fmaf(v, w4.w, acc[4 * q + 3]);
        }
      }
    }
    __syncthreads();
  }
  const int oy = oy0 + ty, ox = ox0 + tx;
  if (oy < OH && ox < OW) {
    float* op = out + ((size_t)oy * OW + ox) * COUT;
#pragma unroll
    for (int co = 0; co < COUT; ++co) {
      float v = acc[co] + __ldg(bias + co);
      if (ACT) v = v > 0.0f ? v : 0.3f * v;
      op[co] = v;
    }
  }
}

// max pooling, NHWC fp32: K x K window, stride S (2/2 and 3/1 in the reference).
__global__ void maxpool_kernel(const float* __restrict__ in, int H, int W, int C, int K, int S, float* __restrict__ out,
                               int OH, int OW) {
  const size_t total = (size_t)OH * OW * C;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const size_t p = i / C;
    const int ox = (int)(p % OW), oy = (int)(p / OW);
    float m = -INFINITY;
    for (int dy = 0; dy < K; ++dy)
      for (int dx = 0; dx < K; ++dx) m = fmaxf(m, in[((size_t)(oy * S + dy) * W + ox * S + dx) * C + c]);
    out[i] = m;
  }
}

// Fold BN into conv weights: wf[tap][cin][cout] = w[cout][cin][tap] * gamma/sqrt(var+eps); bias = beta - mean*scale.
__global__ void fold_conv_kernel(const float* __restrict__ w, const float* __restrict__ bn /*gamma,beta,mean,var*/, int cout,
                                 int cin, int kk, float* __restrict__ wf, float* __restrict__ bias) {
  const int total = cout * cin * kk;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int co = i % cout, r = i / cout, ci = r % cin, tap = r / cin;
    const float s = bn[co] / sqrtf(bn[3 * cout + co] + kBnEps);
    wf[i] = w[((size_t)co * cin + ci) * kk + tap] * s;
  }
  for (int co = blockIdx.x * blockDim.x + threadIdx.x; co < cout; co += gridDim.x * blockDim.x) {
    const float s = bn[co] / sqrtf(bn[3 * cout + co] + kBnEps);
    bias[co] = bn[cout + co] - bn[2 * cout + co] * s;
  }
}

// ------------------------------------------------------------------------------------------------
// wgmma / TMA / mbarrier primitives (inline PTX, sm_90a)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t"
      "}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// K-major, 128B-swizzled shared-memory matrix descriptor of the B operand (sm_90 GMMA layout): 128-byte rows, 8-row
// swizzle atoms 1024 B apart (SBO); the start address advances by 32 B per K = 16 step inside the atom.
__device__ __forceinline__ uint64_t make_desc_b(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);     // start address, bits [0,14)
  d |= (uint64_t)1 << 16;                      // leading byte offset (unused for swizzled K-major), bits [16,30)
  d |= (uint64_t)(1024 >> 4) << 32;            // stride byte offset, bits [32,46)
  d |= (uint64_t)1 << 62;                      // layout type SWIZZLE_128B, bits [62,64)
  return d;
}

// D[64 x N] += A[64 x 16] (registers, the mma.m16n8k16 A fragment per warp) * B[16 x N] (shared memory, K-major),
// fp16 inputs, fp32 accumulators (thread holds N/2 of them).
template <int N>
__device__ __forceinline__ void wgmma_rs(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t bdesc);
template <>
__device__ __forceinline__ void wgmma_rs<48>(float (&d)[24], const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %29, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, "
      "{%24, %25, %26, %27}, %28, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(1)
      : "memory");
}
template <>
__device__ __forceinline__ void wgmma_rs<32>(float (&d)[16], const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "{%16, %17, %18, %19}, %20, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(1)
      : "memory");
}
template <>
__device__ __forceinline__ void wgmma_rs<64>(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(1)
      : "memory");
}

constexpr int kTileY = 16, kTileX = 8;           // output tile: M = 128 pixels = two warpgroups of 8 image rows x 8
constexpr int kConvThreads = 288;                // warps 0..7 = two MMA warpgroups (+ epilogue), warp 8 = TMA producer
constexpr int kMaxSmem = 227 * 1024;             // dynamic shared memory one block may use on sm_90

template <int KS, int NOUT>
struct ConvCfg {
  static constexpr int kBrickY = kTileY + KS - 1;
  static constexpr int kBrickX = ((kTileX + KS - 1) + 7) & ~7;   // row pitch = whole swizzle atoms (8 pixels = 1024 B)
  static constexpr int kBrickBytes = kBrickY * kBrickX * 128;    // per split term
  static constexpr int kWStageBytes = 2 * NOUT * 128;            // hi + lo weight tile of one tap
  static constexpr int kFixed = 2 * kBrickBytes + 1024 /*align slack*/ + 256 /*barriers*/;
  // A three-deep weight ring where it fits. The full network's 15x15 layer (two 92 KB bricks, 16 KB per tap at N = 64)
  // would need 234 752 B with three stages, over the limit, so it runs with two (DESIGN.md section 4.3).
  static constexpr int kWStages = kFixed + 3 * kWStageBytes <= kMaxSmem ? 3 : 2;
  static constexpr int kSmem = kFixed + kWStages * kWStageBytes;
  static_assert(kSmem <= kMaxSmem, "conv tile does not fit the 227 KB of shared memory a block may use");
};

// Implicit-GEMM convolution on wgmma (see the file header). KS x KS taps, KSTEPS x 16 input channels multiplied per
// tap (channels are stored padded to 64 = one 128-byte swizzle row per pixel), NOUT = wgmma N, NMAIN fp32 accumulators
// for the a_hi*w_hi products (tap t -> t % NMAIN) + 1 for the two correction terms.
// SPLIT_OUT: write the activation as fp16 hi/lo NHWC-64 (the next layer's TMA source) instead of fp32 NHWC; an
// activation beyond the fp16 range sets `split_bit` in *overflow.
// inv_scale[n]: the power of two that undoes output channel n's weight scale (fold_tc_kernel).
template <int KS, int KSTEPS, int NOUT, int NMAIN, bool SPLIT_OUT>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_wgmma_kernel(const __grid_constant__ CUtensorMap map_ahi, const __grid_constant__ CUtensorMap map_alo,
                  const __grid_constant__ CUtensorMap map_whi, const __grid_constant__ CUtensorMap map_wlo,
                  const float* __restrict__ bias, const float* __restrict__ inv_scale, float* __restrict__ out,
                  __half* __restrict__ out_hi, __half* __restrict__ out_lo, int OH, int OW, int cout,
                  unsigned* __restrict__ overflow, unsigned split_bit) {
  using Cfg = ConvCfg<KS, NOUT>;
  constexpr int kTaps = KS * KS, kNA = NOUT / 2, kWStages = Cfg::kWStages;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  unsigned char* a_hi = smem;
  unsigned char* a_lo = smem + Cfg::kBrickBytes;
  unsigned char* w_st = smem + 2 * Cfg::kBrickBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(w_st + kWStages * Cfg::kWStageBytes);
  uint64_t* bar_brick = bars;                 // TMA -> MMA: activations landed
  uint64_t* bar_full = bars + 1;              // [kWStages] TMA -> MMA: weight tap landed
  uint64_t* bar_empty = bars + 1 + kWStages;  // [kWStages] MMA -> TMA: stage consumed (one arrival per MMA warp)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int x0 = blockIdx.x * kTileX, y0 = blockIdx.y * kTileY;

  if (threadIdx.x == 0) {
    mbar_init(bar_brick, 1);
    for (int s = 0; s < kWStages; ++s) { mbar_init(bar_full + s, 1); mbar_init(bar_empty + s, 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      // activations: one box [64 ch][kBrickX x][kBrickY y] per split term (out-of-range pixels are zero-filled by TMA)
      mbar_expect_tx(bar_brick, 2 * Cfg::kBrickBytes);
      tma_load_3d(a_hi, &map_ahi, bar_brick, 0, x0, y0);
      tma_load_3d(a_lo, &map_alo, bar_brick, 0, x0, y0);
      // weights: ring over the taps
      for (int t = 0; t < kTaps; ++t) {
        const int s = t % kWStages, round = t / kWStages;
        if (round > 0) mbar_wait(bar_empty + s, (round - 1) & 1);
        mbar_expect_tx(bar_full + s, Cfg::kWStageBytes);
        tma_load_2d(w_st + s * Cfg::kWStageBytes, &map_whi, bar_full + s, 0, t * NOUT);
        tma_load_2d(w_st + s * Cfg::kWStageBytes + NOUT * 128, &map_wlo, bar_full + s, 0, t * NOUT);
      }
    }
    return;   // the MMA warps wait for every stage this warp filled, so the CTA outlives its copies
  }

  // Warpgroup g owns output pixels m = 64g .. 64g+63 (m = yl*8 + xl); warp q of it the 16 rows 16q .. 16q+15, i.e. image
  // rows yl = 8g + 2q (+1). ldmatrix.x4 lane l addresses row (l & 7) of 8x8 matrix l >> 3: matrices 0/1 = rows 0-7 / 8-15
  // at channels 0-7 of the K step, matrices 2/3 the same rows at channels 8-15.
  const int g = warp >> 2, q = warp & 3;
  const int mi = lane >> 3;
  const int yl = 8 * g + 2 * q + (mi & 1), xl = lane & 7, kc = mi >> 1;
  const uint32_t ahi = smem_u32(a_hi), alo = smem_u32(a_lo);
  float acc[NMAIN][kNA], corr[kNA];
#pragma unroll
  for (int i = 0; i < kNA; ++i) {
    corr[i] = 0.0f;
#pragma unroll
    for (int a = 0; a < NMAIN; ++a) acc[a][i] = 0.0f;
  }
  mbar_wait(bar_brick, 0);
  for (int t0 = 0; t0 < kTaps; t0 += NMAIN) {
#pragma unroll
    for (int u = 0; u < NMAIN; ++u) {
      const int t = t0 + u;
      if (t < kTaps) {
        const int s = t % kWStages;
        mbar_wait(bar_full + s, (t / kWStages) & 1);
        // every tap is a shifted view of the brick: pixel (yl + ky, xl + kx); the 128B swizzle permutes the 16-byte
        // chunks of a pixel row by (row index & 7), the brick being 1024-byte aligned
        const uint32_t p = (uint32_t)((yl + t / KS) * Cfg::kBrickX + xl + t % KS);
        uint32_t ah[KSTEPS][4], al[KSTEPS][4];
#pragma unroll
        for (int j = 0; j < KSTEPS; ++j) {
          const uint32_t off = p * 128u + ((((uint32_t)(2 * j + kc)) ^ (p & 7u)) << 4);
          ldsm_x4(ahi + off, ah[j]);
          ldsm_x4(alo + off, al[j]);
        }
        const uint32_t whi = smem_u32(w_st + s * Cfg::kWStageBytes), wlo = whi + NOUT * 128;
        wgmma_fence();
        // The tensor core truncates when it adds into the fp32 accumulator, so a single accumulator would take
        // thousands of biased roundings in the 15x15 layer. Spread them: the a_hi*w_hi products go round-robin to NMAIN
        // accumulators, both small correction terms to one more; the epilogue sums them in fp32 round-to-nearest.
#pragma unroll
        for (int j = 0; j < KSTEPS; ++j) {   // KSTEPS x 16 channels; pad channels beyond are never multiplied
          wgmma_rs<NOUT>(acc[u], ah[j], make_desc_b(whi + j * 32));
          wgmma_rs<NOUT>(corr, ah[j], make_desc_b(wlo + j * 32));
          wgmma_rs<NOUT>(corr, al[j], make_desc_b(whi + j * 32));
        }
        wgmma_commit();
        wgmma_wait_all();
        if (lane == 0) mbar_arrive(bar_empty + s);   // frees the weight stage for the producer
      }
    }
  }

  // epilogue: accumulator element i of lane l sits at row 16q + l/4 + 8*((i/2)&1), column 8*(i/4) + 2*(l&3) + (i&1)
  float v[kNA];
#pragma unroll
  for (int i = 0; i < kNA; ++i) {
    float sum = 0.0f;
#pragma unroll
    for (int a = 0; a < NMAIN; ++a) sum += acc[a][i];
    v[i] = sum + corr[i];
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int oy = y0 + 8 * g + 2 * q + h, ox = x0 + (lane >> 2);
    if (oy >= OH || ox >= OW) continue;
    const size_t pix = (size_t)oy * OW + ox;
#pragma unroll
    for (int c8 = 0; c8 < NOUT / 8; ++c8) {
      const int n = 8 * c8 + 2 * (lane & 3);
      float f[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float x = 0.0f;
        if (n + e < cout) {
          x = v[4 * c8 + 2 * h + e] * __ldg(inv_scale + n + e) + __ldg(bias + n + e);
          x = x > 0.0f ? x : 0.3f * x;
        }
        f[e] = x;
      }
      if (SPLIT_OUT) {
        const __half h0 = __float2half_rn(f[0]), h1 = __float2half_rn(f[1]);
        if (__hisinf(h0) | __hisinf(h1)) atomicOr(overflow, split_bit);
        reinterpret_cast<__half2*>(out_hi + pix * 64)[n / 2] = __halves2half2(h0, h1);
        reinterpret_cast<__half2*>(out_lo + pix * 64)[n / 2] =
            __halves2half2(__float2half_rn(f[0] - __half2float(h0)), __float2half_rn(f[1] - __half2float(h1)));
      } else {
        float* op = out + pix * cout;
        if (n < cout) op[n] = f[0];
        if (n + 1 < cout) op[n + 1] = f[1];
      }
    }
    if (SPLIT_OUT) {   // pad channels of the next layer's input
      for (int n = NOUT + 2 * (lane & 3); n < 64; n += 8) {
        reinterpret_cast<__half2*>(out_hi + pix * 64)[n / 2] = __float2half2_rn(0.0f);
        reinterpret_cast<__half2*>(out_lo + pix * 64)[n / 2] = __float2half2_rn(0.0f);
      }
    }
  }
}

// First layer (Cin = 1, no activation after its BN) on CUDA cores, reading the map layer directly and writing the
// fp16 hi/lo NHWC-64 input of the second layer. One thread per (pixel, group of 8 output channels): the eight threads of
// a pixel write its two 128-byte rows as sixteen 16-byte stores; channels C1..63 are zero. An output beyond the fp16
// range sets bit 0 of *overflow.
template <int C1>
__global__ void __launch_bounds__(256) conv1_split_kernel(const float* __restrict__ layer, int H, int W, int pitch,
                                                          const float* __restrict__ wf /*[9][1][C1]*/, const float* __restrict__ bias,
                                                          __half* __restrict__ hi, __half* __restrict__ lo,
                                                          unsigned* __restrict__ overflow) {
  static_assert(C1 % 8 == 0 && C1 <= 64, "C1 output channels fill whole 8-channel groups of a 64-channel pixel row");
  __shared__ float sw[9 * C1 + C1];
  for (int i = threadIdx.x; i < 9 * C1 + C1; i += blockDim.x) sw[i] = i < 9 * C1 ? wf[i] : bias[i - 9 * C1];
  __syncthreads();
  const int OH = H - 2, OW = W - 2;
  const size_t total = (size_t)OH * OW * 8;
  // consecutive pixels take consecutive image rows (oy): the map layer is contiguous along that axis
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int v4 = (int)(i & 7);
    const size_t p = i >> 3;
    const int oy = (int)(p % OH), ox = (int)(p / OH);
    const size_t pix = (size_t)oy * OW + ox;
    __half2 hh[4], ll[4];
    if (v4 < C1 / 8) {
      float in[9];
#pragma unroll
      for (int t = 0; t < 9; ++t) in[t] = __ldg(layer + (size_t)(ox + t % 3) * pitch + (H - 1 - (oy + t / 3)));   // E[r][c]
#pragma unroll
      for (int e2 = 0; e2 < 4; ++e2) {
        float f[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int n = 8 * v4 + 2 * e2 + e;
          float a = sw[9 * C1 + n];
#pragma unroll
          for (int t = 0; t < 9; ++t) a = fmaf(in[t], sw[t * C1 + n], a);
          f[e] = a;
        }
        const __half h0 = __float2half_rn(f[0]), h1 = __float2half_rn(f[1]);
        if (__hisinf(h0) | __hisinf(h1)) atomicOr(overflow, 1u);
        hh[e2] = __halves2half2(h0, h1);
        ll[e2] = __halves2half2(__float2half_rn(f[0] - __half2float(h0)), __float2half_rn(f[1] - __half2float(h1)));
      }
    } else {
#pragma unroll
      for (int e2 = 0; e2 < 4; ++e2) { hh[e2] = __float2half2_rn(0.0f); ll[e2] = __float2half2_rn(0.0f); }
    }
    reinterpret_cast<uint4*>(hi + pix * 64)[v4] = *reinterpret_cast<uint4*>(hh);
    reinterpret_cast<uint4*>(lo + pix * 64)[v4] = *reinterpret_cast<uint4*>(ll);
  }
}

// max pooling (K x K, stride S) of an fp32 NHWC [H][W][C] activation (C a multiple of 8) into fp16 hi/lo NHWC-64.
// One thread per (pixel, 8 channels): two 16-byte loads per tap, one 16-byte store per output array. An output beyond
// the fp16 range sets `split_bit` in *overflow.
__global__ void maxpool_split_kernel(const float* __restrict__ in, int H, int W, int C, int K, int S, __half* __restrict__ hi,
                                     __half* __restrict__ lo, int OH, int OW, unsigned* __restrict__ overflow,
                                     unsigned split_bit) {
  const size_t total = (size_t)OH * OW * 8;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int v8 = (int)(i & 7);
    const size_t p = i >> 3;
    const int ox = (int)(p % OW), oy = (int)(p / OW);
    float m[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) m[e] = 0.0f;
    if (8 * v8 < C) {
#pragma unroll
      for (int e = 0; e < 8; ++e) m[e] = -INFINITY;
      for (int dy = 0; dy < K; ++dy)
        for (int dx = 0; dx < K; ++dx) {
          const float4* q = reinterpret_cast<const float4*>(in + ((size_t)(oy * S + dy) * W + ox * S + dx) * C + 8 * v8);
          const float4 a = __ldg(q), b = __ldg(q + 1);
          m[0] = fmaxf(m[0], a.x); m[1] = fmaxf(m[1], a.y); m[2] = fmaxf(m[2], a.z); m[3] = fmaxf(m[3], a.w);
          m[4] = fmaxf(m[4], b.x); m[5] = fmaxf(m[5], b.y); m[6] = fmaxf(m[6], b.z); m[7] = fmaxf(m[7], b.w);
        }
    }
    __half2 hh[4], ll[4];
#pragma unroll
    for (int e2 = 0; e2 < 4; ++e2) {
      const __half h0 = __float2half_rn(m[2 * e2]), h1 = __float2half_rn(m[2 * e2 + 1]);
      if (__hisinf(h0) | __hisinf(h1)) atomicOr(overflow, split_bit);
      hh[e2] = __halves2half2(h0, h1);
      ll[e2] = __halves2half2(__float2half_rn(m[2 * e2] - __half2float(h0)), __float2half_rn(m[2 * e2 + 1] - __half2float(h1)));
    }
    reinterpret_cast<uint4*>(hi + p * 64)[v8] = *reinterpret_cast<uint4*>(hh);
    reinterpret_cast<uint4*>(lo + p * 64)[v8] = *reinterpret_cast<uint4*>(ll);
  }
}

// Weight scale of a tensor-core layer, one block per output channel n: the power of two 2^k that brings the channel's
// largest folded |w| into [2^14, 2^15), so that w_hi stays below the fp16 maximum (65504) and w_lo above the fp16
// subnormals wherever the weight matters; inv_scale[n] = 2^-k, which undoes it exactly in the epilogue.
__global__ void __launch_bounds__(256) tc_scale_kernel(const float* __restrict__ w /*[cout][cin][taps]*/,
                                                       const float* __restrict__ bn, int cout, int cin, int taps,
                                                       float* __restrict__ inv_scale) {
  __shared__ float red[256];
  const int n = blockIdx.x;
  const float s = bn[n] / sqrtf(bn[3 * cout + n] + kBnEps);
  float m = 0.0f;
  for (int i = threadIdx.x; i < cin * taps; i += blockDim.x) m = fmaxf(m, fabsf(w[(size_t)n * cin * taps + i] * s));
  red[threadIdx.x] = m;
  __syncthreads();
  for (int k = blockDim.x / 2; k > 0; k >>= 1) {
    if (threadIdx.x < k) red[threadIdx.x] = fmaxf(red[threadIdx.x], red[threadIdx.x + k]);
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    int e = 0;
    frexpf(red[0], &e);                          // max|w| < 2^e (e = 0 for an all-zero channel)
    const int k = min(max(15 - e, -100), 100);   // both 2^k and 2^-k stay normal fp32 numbers
    inv_scale[n] = ldexpf(1.0f, -k);
  }
}

// Tensor-core weights of one layer: [taps][NOUT][64] fp16 hi/lo (K-major rows of 128 B; pad rows / channels zero),
// BN scale and the channel's power-of-two weight scale folded; bias = beta - mean*scale.
__global__ void fold_tc_kernel(const float* __restrict__ w /*[cout][cin][taps]*/, const float* __restrict__ bn, int cout, int cin,
                               int taps, int nout, const float* __restrict__ inv_scale, __half* __restrict__ whi,
                               __half* __restrict__ wlo, float* __restrict__ bias) {
  const int total = taps * nout * 64;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int c = i & 63, r = i >> 6, n = r % nout, tap = r / nout;
    float v = 0.0f;
    if (c < cin && n < cout) {
      const float s = bn[n] / sqrtf(bn[3 * cout + n] + kBnEps);
      v = w[((size_t)n * cin + c) * taps + tap] * s * (1.0f / inv_scale[n]);
    }
    const __half h = __float2half_rn(v);
    whi[i] = h;
    wlo[i] = __float2half_rn(v - __half2float(h));
  }
  for (int n = blockIdx.x * blockDim.x + threadIdx.x; n < cout; n += gridDim.x * blockDim.x) {
    const float s = bn[n] / sqrtf(bn[3 * cout + n] + kBnEps);
    bias[n] = bn[cout + n] - bn[2 * cout + n] * s;
  }
}

// Reference implementation of the 15x15 layer on CUDA cores (fp32, C channels in and out), used by the self-check
// entry point only.
template <int C>
__global__ void conv15_reference_kernel(const float* __restrict__ in /*[H][W][C]*/, int H, int W,
                                        const float* __restrict__ wf /*[225][C][C]*/, const float* __restrict__ bias,
                                        float* __restrict__ out) {
  const int OH = H - 14, OW = W - 14;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= OH * OW * C) return;
  const int n = i % C, p = i / C, ox = p % OW, oy = p / OW;
  float acc = 0.0f;
  for (int ky = 0; ky < 15; ++ky)
    for (int kx = 0; kx < 15; ++kx) {
      const float* ip = in + ((size_t)(oy + ky) * W + ox + kx) * C;
      const float* wp = wf + (size_t)(ky * 15 + kx) * C * C + n;
      for (int c = 0; c < C; ++c) acc = fmaf(ip[c], wp[c * C], acc);
    }
  const float f = acc + bias[n];
  out[i] = f > 0.0f ? f : 0.3f * f;
}

// ------------------------------------------------------------------------------------------------
// Query head: CostQuery.__call__ + FCpart, one thread per query, folded weights in shared memory.
// ------------------------------------------------------------------------------------------------
// folded head weights (CF feature channels, out0 width NH, out1 widths B1..B3; light: 48, 48, 24/24/36): tar0
// [10][16]+b[16], out0 [CF+16][NH]+b[NH], o11 [NH][B1]+b, o12 [NH][B2]+b, o13 [NH][B3]+b, o21 [B1]+b[1], o22 [B2]+b[1],
// o23 [B3]+b[1]
__host__ __device__ constexpr int head_floats(int cf, int nh, int b1, int b2, int b3) {
  return 10 * 16 + 16 + (cf + 16) * nh + nh + (nh + 1) * (b1 + b2 + b3) + (b1 + b2 + b3) + 3;
}

// The widths are template parameters so that x / h stay in registers, fully unrolled, for either network.
template <int CF, int NH, int B1, int B2, int B3>
__global__ void __launch_bounds__(128) head_kernel(const float* __restrict__ feats /*[Hf][Wf][CF]*/, int Hf, int Wf,
                                                    const float* __restrict__ hw, const float* __restrict__ edges, size_t n,
                                                    float* __restrict__ cost3, double res, double Lx, double Ly, double cx,
                                                    double cy) {
  constexpr int kIn = CF + 16, kHeadFloats = head_floats(CF, NH, B1, B2, B3);
  extern __shared__ float sw[];
  for (int i = threadIdx.x; i < kHeadFloats; i += blockDim.x) sw[i] = hw[i];
  __syncthreads();
  const size_t q = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (q >= n) return;
  const float* e = edges + 6 * q;
  // float64 arithmetic on the float32 request values, like the numpy/torch float64 path of the server
  double tx = (double)e[0] - cx, ty = (double)e[1] - cy, tyaw = (double)e[2];
  const double sx = (double)e[3] - cx, sy = (double)e[4] - cy, syaw = (double)e[5];
  tx -= sx; ty -= sy; tyaw -= syaw;
  const double feat_res = res * 2.0;
  const int row_bias = (int)((Lx / res - 48.0) / 2.0 * 0.5), col_bias = (int)((Ly / res - 48.0) / 2.0 * 0.5);
  double rr = sx / feat_res + row_bias, cc = sy / feat_res + col_bias;
  rr = fmin(fmax(rr, 1.0), (double)(Hf - 2));
  cc = fmin(fmax(cc, 1.0), (double)(Wf - 2));
  const int row = (int)rr, col = (int)cc;   // .long() truncation
  float x[kIn];
  {
    const float4* fp = reinterpret_cast<const float4*>(feats + ((size_t)row * Wf + col) * CF);
#pragma unroll
    for (int i = 0; i < CF / 4; ++i) { const float4 v = __ldg(fp + i); x[4 * i] = v.x; x[4 * i + 1] = v.y; x[4 * i + 2] = v.z; x[4 * i + 3] = v.w; }
  }
  const float dx = (float)tx, dy = (float)ty;
  float ang = (float)tyaw;
  const float PI = 3.14159265358979323846f;
  if (ang > PI) ang -= 2.0f * PI;
  if (ang < -PI) ang += 2.0f * PI;
  const float sya = (float)syaw;
  const float info[10] = {dx, dy, sqrtf(dx * dx + dy * dy), atan2f(dy, dx), ang, cosf(ang), sinf(ang), sya, cosf(sya), sinf(sya)};
  const float* w = sw;
  // tar0: 10 -> 16 (BN folded, no activation)
#pragma unroll
  for (int o = 0; o < 16; ++o) {
    float a = w[160 + o];
#pragma unroll
    for (int i = 0; i < 10; ++i) a = fmaf(info[i], w[i * 16 + o], a);
    x[CF + o] = a;
  }
  w += 176;
  float h[NH];
#pragma unroll
  for (int o = 0; o < NH; ++o) h[o] = w[kIn * NH + o];
  for (int i = 0; i < kIn; ++i) {
    const float v = x[i];
#pragma unroll
    for (int o = 0; o < NH; ++o) h[o] = fmaf(v, w[i * NH + o], h[o]);
  }
#pragma unroll
  for (int o = 0; o < NH; ++o) h[o] = h[o] > 0.0f ? h[o] : 0.3f * h[o];
  w += kIn * NH + NH;
  float outv[3];
  const int widths[3] = {B1, B2, B3};
  const float* w2 = w + NH * (B1 + B2 + B3) + (B1 + B2 + B3);
  for (int b = 0; b < 3; ++b) {
    const int nb = widths[b];
    float acc2 = 0.0f;
    for (int o = 0; o < nb; ++o) {
      float a = w[NH * nb + o];
      for (int i = 0; i < NH; ++i) a = fmaf(h[i], w[i * nb + o], a);
      a = a > 0.0f ? a : 0.3f * a;
      acc2 = fmaf(a, w2[o], acc2);
    }
    acc2 += w2[nb];
    outv[b] = acc2;
    w += NH * nb + nb;
    w2 += nb + 1;
  }
  cost3[3 * q + 0] = fmaxf(outv[0], 0.0f);                        // power  (ReLU)
  cost3[3 * q + 1] = fmaxf(outv[1], 0.0f);                        // time   (ReLU)
  cost3[3 * q + 2] = 1.0f - 1.0f / (1.0f + expf(-outv[2]));       // 1 - sigmoid
}

// Fold the head's 1x1 convs (+BN) into [Cin][Cout] matrices + bias, in head_kernel's order.
struct HeadDims { int cin[8], cout[8]; };   // blob layers 6..13
__global__ void fold_head_kernel(const float* __restrict__ blob, const size_t* __restrict__ offs, HeadDims d,
                                 float* __restrict__ hw) {
  // offs[l] = offset of layer l (6..13) in the blob; single block
  const int* cin = d.cin;
  const int* cout = d.cout;
  int o = 0;
  for (int l = 0; l < 8; ++l) {
    const float* w = blob + offs[l];
    const float* bn = w + (size_t)cout[l] * cin[l];
    const bool has_bn = l < 5;
    for (int i = threadIdx.x; i < cin[l] * cout[l]; i += blockDim.x) {
      const int co = i % cout[l], ci = i / cout[l];
      const float s = has_bn ? bn[co] / sqrtf(bn[3 * cout[l] + co] + kBnEps) : 1.0f;
      hw[o + i] = w[(size_t)co * cin[l] + ci] * s;
    }
    for (int co = threadIdx.x; co < cout[l]; co += blockDim.x) {
      float b;
      if (has_bn) { const float s = bn[co] / sqrtf(bn[3 * cout[l] + co] + kBnEps); b = bn[cout[l] + co] - bn[2 * cout[l] + co] * s; }
      else b = bn[co];   // conv bias
      hw[o + cin[l] * cout[l] + co] = b;
    }
    o += cin[l] * cout[l] + cout[l];
  }
}

// ------------------------------------------------------------------------------------------------
// host state
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// One tensor-core layer: weights (hi/lo), bias, and its launch geometry.
struct TcLayer { __half *whi = nullptr, *wlo = nullptr; float* inv_scale = nullptr; int nout = 0; };

// The trunk's activations: h* / l* = fp16 hi / lo NHWC-64, f* = fp32 NHWC, feat = the feature map; overflow = the fp16
// range overflow of the tensor-core path's activation splits, bit i = output of trunk layer i (kSplitLayerNames).
struct Acts {
  __half *h1, *l1, *hp2, *lp2, *h3, *l3, *hp4, *lp4, *h5, *l5;
  float *f1, *f2, *fp2, *f3, *f4, *fp4, *f5, *feat;
  unsigned* overflow;
};

}  // namespace artp_cnn

using namespace artp_api;
using namespace artp_cnn;

namespace artp_api {

struct CostNet {
  int mode = 0;   // artp_set_cnn_mode
  bool has_weights = false, has_features = false;
  // The loaded network (-1: none yet). The weights, the activations, the tensor maps and the kernel attributes are laid
  // out for it.
  int net = -1;
  LayerDef layers[14];
  size_t layer_off[14];
  // The weights, one scratch group (carve): the blob, the head's layer offsets in it, the folded head, and per trunk
  // layer l the folded fp32 weights [k*k][cin][cout] (layer 0 always, 1..5 for the CUDA-core path) and bias, and for
  // l = 1..5 the tensor-core weights.
  char* d_w = nullptr;
  size_t w_cap = 0;
  float* d_blob = nullptr;
  size_t* d_offs = nullptr;
  float* d_head = nullptr;
  float* d_wf[6] = {};
  float* d_bias[6] = {};
  TcLayer tc[6];
  // The activations, another scratch group, laid out for the map of rows x cols.
  char* d_act = nullptr;
  size_t act_cap = 0;
  Acts a{};
  int rows = 0, cols = 0;
  int Hf = 0, Wf = 0;
  double res = 0, Lx = 0, Ly = 0, cx = 0, cy = 0;
  EncodeTiledFn encode = nullptr;
  // Per tensor-core layer: activation hi/lo, weight hi/lo. Valid while the map size and the network stay, which is also
  // while the regions they address stay where they are.
  CUtensorMap maps[6][4];
  bool maps_valid = false;
  bool attrs_set = false;
  float last_ms[3] = {0, 0, 0};
  cudaEvent_t ev[4] = {};
  unsigned* h_overflow = nullptr;   // pinned
};

}  // namespace artp_api

namespace {

// A handle without the state reads as one without weights.
const CostNet& view(const Handle* h) {
  static const CostNet none{};
  return h->cost_net ? *h->cost_net : none;
}
CostNet& state(Handle* h) {
  if (!h->cost_net) h->cost_net = new CostNet();
  return *h->cost_net;
}

// wgmma N of tensor-core layer l (1..5): Cout rounded up to a multiple of 16 (light init_conv2: 24 -> 32)
int tc_nout(const LayerDef& l) { return (l.cout + 15) / 16 * 16; }

int head_floats(int net) {
  const NetDims& d = kNets[net];
  return artp_cnn::head_floats(d.c3, d.nh, d.b[0], d.b[1], d.b[2]);
}

int set_weights(Handle* h, const float* blob, size_t n) {
  int net = -1;
  for (int k : {ARTP_COST_NET_LIGHT, ARTP_COST_NET_FULL}) if (n == blob_floats(k)) net = k;
  if (net < 0) { h->err = "weight blob has the wrong number of floats (neither network_light nor network)"; return ARTP_E_INVALID; }
  CU_TRY(h, cudaSetDevice(h->device));
  CostNet& c = state(h);
  cudaStream_t st = h->stream;
  if (c.net != net) {
    // Another architecture: the features, tensor maps and kernel attributes of the old one go.
    c.maps_valid = false;
    c.attrs_set = false;
    c.has_weights = c.has_features = false;
    c.net = net;
    for (int l = 0; l < 14; ++l) c.layers[l] = layer_def(net, l);
  }
  const LayerDef* L = c.layers;
  auto wf = [&](int l) { return (size_t)L[l].k * L[l].k * L[l].cin * L[l].cout * sizeof(float); };
  auto tc = [&](int l) { return (size_t)L[l].k * L[l].k * tc_nout(L[l]) * 64 * sizeof(__half); };
  auto ch = [&](int l) { return L[l].cout * sizeof(float); };
  char* r[30];   // blob | offsets | head | wf[0..5] | bias[0..5] | whi[1..5] | wlo[1..5] | inv_scale[1..5]
  TRY(carve(h, c.d_w, c.w_cap,
            {n * sizeof(float), 8 * sizeof(size_t), head_floats(net) * sizeof(float), wf(0), wf(1), wf(2), wf(3), wf(4),
             wf(5), ch(0), ch(1), ch(2), ch(3), ch(4), ch(5), tc(1), tc(2), tc(3), tc(4), tc(5), tc(1), tc(2), tc(3), tc(4),
             tc(5), ch(1), ch(2), ch(3), ch(4), ch(5)},
            r));
  c.d_blob = (float*)r[0];
  c.d_offs = (size_t*)r[1];
  c.d_head = (float*)r[2];
  for (int l = 0; l < 6; ++l) { c.d_wf[l] = (float*)r[3 + l]; c.d_bias[l] = (float*)r[9 + l]; }
  for (int l = 1; l < 6; ++l) c.tc[l] = {(__half*)r[14 + l], (__half*)r[19 + l], (float*)r[24 + l], tc_nout(L[l])};
  size_t off = 0;
  for (int l = 0; l < 14; ++l) {
    c.layer_off[l] = off;
    off += (size_t)L[l].cout * L[l].cin * L[l].k * L[l].k + (L[l].bn ? 4 * L[l].cout : L[l].cout);
  }
  TRY(copy_async(h, c.d_blob, blob, n * sizeof(float), cudaMemcpyHostToDevice, st));
  TRY(copy_async(h, c.d_offs, c.layer_off + 6, 8 * sizeof(size_t), cudaMemcpyHostToDevice, st));
  for (int l = 0; l < 6; ++l) {
    const int kk = L[l].k * L[l].k;
    const float* w = c.d_blob + c.layer_off[l];
    const float* bn = w + (size_t)L[l].cout * L[l].cin * kk;
    // fp32 folded weights (first layer + the CUDA-core path) and biases
    TRY(launch(h, fold_conv_kernel, 256, 256, 0, st, w, bn, L[l].cout, L[l].cin, kk, c.d_wf[l], c.d_bias[l]));
    if (l >= 1) {
      TRY(launch(h, tc_scale_kernel, L[l].cout, 256, 0, st, w, bn, L[l].cout, L[l].cin, kk, c.tc[l].inv_scale));
      TRY(launch(h, fold_tc_kernel, 256, 256, 0, st, w, bn, L[l].cout, L[l].cin, kk, c.tc[l].nout,
                 c.tc[l].inv_scale, c.tc[l].whi, c.tc[l].wlo, c.d_bias[l]));
    }
  }
  HeadDims hd;
  for (int l = 0; l < 8; ++l) { hd.cin[l] = L[6 + l].cin; hd.cout[l] = L[6 + l].cout; }
  TRY(launch(h, fold_head_kernel, 1, 256, 0, st, c.d_blob, c.d_offs, hd, c.d_head));
  TRY(sync_stream(h, st));
  c.has_weights = true;
  c.has_features = false;
  return ARTP_OK;
}

int get_encoder(Handle* h, CostNet& c) {
  if (c.encode) return ARTP_OK;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn) {
    h->err = "cuTensorMapEncodeTiled not available from the driver";
    return ARTP_E_CUDA;
  }
  c.encode = reinterpret_cast<EncodeTiledFn>(fn);
  return ARTP_OK;
}

// maps[0..1]: activations hi/lo [H][W][64] fp16, box (64, brick_x, brick_y); maps[2..3]: weights [taps*nout][64], box (64, nout)
int encode_layer_maps(Handle* h, CostNet& c, CUtensorMap* maps, __half* ahi, __half* alo, int H, int W, int brick_x,
                      int brick_y, __half* whi, __half* wlo, int taps, int nout) {
  TRY(get_encoder(h, c));
  const cuuint64_t adim[3] = {64, (cuuint64_t)W, (cuuint64_t)H};
  const cuuint64_t astr[2] = {128, (cuuint64_t)W * 128};
  const cuuint32_t abox[3] = {64, (cuuint32_t)brick_x, (cuuint32_t)brick_y};
  const cuuint32_t one3[3] = {1, 1, 1};
  const cuuint64_t wdim[2] = {64, (cuuint64_t)taps * nout};
  const cuuint64_t wstr[1] = {128};
  const cuuint32_t wbox[2] = {64, (cuuint32_t)nout};
  void* ptrs[4] = {ahi, alo, whi, wlo};
  for (int i = 0; i < 4; ++i) {
    CUresult r;
    if (i < 2)
      r = c.encode(&maps[i], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, ptrs[i], adim, astr, abox, one3, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    else
      r = c.encode(&maps[i], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, ptrs[i], wdim, wstr, wbox, one3, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { h->err = "cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")"; return ARTP_E_CUDA; }
  }
  return ARTP_OK;
}

template <int KS, int KSTEPS, int NOUT, int NMAIN, bool SPLIT>
int launch_tc(Handle* h, CostNet& c, int layer, __half* ahi, __half* alo, int H, int W, float* out, __half* ohi, __half* olo,
              cudaStream_t st) {
  using Cfg = ConvCfg<KS, NOUT>;
  CUtensorMap* maps = c.maps[layer];
  if (!c.maps_valid)
    TRY(encode_layer_maps(h, c, maps, ahi, alo, H, W, Cfg::kBrickX, Cfg::kBrickY, c.tc[layer].whi, c.tc[layer].wlo, KS * KS, NOUT));
  auto kern = conv_wgmma_kernel<KS, KSTEPS, NOUT, NMAIN, SPLIT>;
  if (!c.attrs_set) CU_TRY(h, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmem));
  const int OH = H - KS + 1, OW = W - KS + 1;
  const dim3 grid((OW + kTileX - 1) / kTileX, (OH + kTileY - 1) / kTileY);
  return launch(h, kern, grid, kConvThreads, Cfg::kSmem, st, maps[0], maps[1], maps[2], maps[3], c.d_bias[layer],
                c.tc[layer].inv_scale, out, ohi, olo, OH, OW, c.layers[layer].cout, c.a.overflow, 1u << layer);
}

// Extents of every trunk activation for a rows x cols map.
struct TrunkDims {
  int H0, W0, H1, W1, H2, W2, HP2, WP2, H3, W3, H4, W4, HP4, WP4, H5, W5, H6, W6;
  TrunkDims(int rows, int cols) : H0(rows), W0(cols) {
    H1 = H0 - 2; W1 = W0 - 2; H2 = H1 - 2; W2 = W1 - 2; HP2 = H2 / 2; WP2 = W2 / 2;
    H3 = HP2 - 2; W3 = WP2 - 2; H4 = H3 - 2; W4 = W3 - 2; HP4 = H4 - 2; WP4 = W4 - 2;
    H5 = HP4 - 2; W5 = WP4 - 2; H6 = H5 - 14; W6 = W5 - 14;
  }
};

// The trunk's launches for one network: C1 channels after init_conv1/2, C3 after init_conv3..5 and init_flatten. Events
// ev[0..3] bracket the 3x3 stack and the 15x15 layer.
template <int NET>
int run_trunk(Handle* h, CostNet& c, const float* d_layer, int pitch, const TrunkDims& d, cudaStream_t st) {
  constexpr int C1 = kNets[NET].c1, C3 = kNets[NET].c3;
  constexpr int K2 = (C1 + 15) / 16, N2 = 16 * K2, K4 = C3 / 16;   // wgmma K steps / N of init_conv2 and the C3 layers
  static_assert(C3 % 16 == 0, "C3 channels are whole K = 16 steps");
  auto grid2 = [](int oh, int ow) { return dim3((ow + 15) / 16, (oh + 15) / 16); };
  const unsigned g1 = h->sm_count * 8;
  const Acts& a = c.a;
  CU_TRY(h, cudaEventRecord(c.ev[0], st));
  if (c.mode & 1) {   // the fp32 CUDA-core path
    TRY(launch(h, conv3x3_kernel<1, C1, 1, false, true>, grid2(d.H1, d.W1), 256, 0, st, d_layer, d.H0, d.W0, pitch,
               c.d_wf[0], c.d_bias[0], a.f1));
    TRY(launch(h, conv3x3_kernel<C1, C1, 8, true, false>, grid2(d.H2, d.W2), 256, 0, st, a.f1, d.H1, d.W1, 0,
               c.d_wf[1], c.d_bias[1], a.f2));
    TRY(launch(h, maxpool_kernel, g1, 256, 0, st, a.f2, d.H2, d.W2, C1, 2, 2, a.fp2, d.HP2, d.WP2));
    TRY(launch(h, conv3x3_kernel<C1, C3, 8, true, false>, grid2(d.H3, d.W3), 256, 0, st, a.fp2, d.HP2, d.WP2, 0,
               c.d_wf[2], c.d_bias[2], a.f3));
    TRY(launch(h, conv3x3_kernel<C3, C3, 8, true, false>, grid2(d.H4, d.W4), 256, 0, st, a.f3, d.H3, d.W3, 0,
               c.d_wf[3], c.d_bias[3], a.f4));
    TRY(launch(h, maxpool_kernel, g1, 256, 0, st, a.f4, d.H4, d.W4, C3, 3, 1, a.fp4, d.HP4, d.WP4));
    TRY(launch(h, conv3x3_kernel<C3, C3, 8, true, false>, grid2(d.H5, d.W5), 256, 0, st, a.fp4, d.HP4, d.WP4, 0,
               c.d_wf[4], c.d_bias[4], a.f5));
    CU_TRY(h, cudaEventRecord(c.ev[1], st));
    CU_TRY(h, cudaEventRecord(c.ev[2], st));
    TRY(launch(h, conv15_reference_kernel<C3>, (d.H6 * d.W6 * C3 + 255) / 256, 256, 0, st, a.f5, d.H5, d.W5,
               c.d_wf[5], c.d_bias[5], a.feat));
  } else {
    TRY(launch(h, conv1_split_kernel<C1>, g1, 256, 0, st, d_layer, d.H0, d.W0, pitch, c.d_wf[0],
               c.d_bias[0], a.h1, a.l1, a.overflow));
    TRY((launch_tc<3, K2, N2, 1, false>(h, c, 1, a.h1, a.l1, d.H1, d.W1, a.f2, nullptr, nullptr, st)));
    TRY(launch(h, maxpool_split_kernel, g1, 256, 0, st, a.f2, d.H2, d.W2, C1, 2, 2, a.hp2, a.lp2, d.HP2, d.WP2,
               a.overflow, 1u << 1));
    TRY((launch_tc<3, K2, C3, 1, true>(h, c, 2, a.hp2, a.lp2, d.HP2, d.WP2, nullptr, a.h3, a.l3, st)));
    TRY((launch_tc<3, K4, C3, 1, false>(h, c, 3, a.h3, a.l3, d.H3, d.W3, a.f4, nullptr, nullptr, st)));
    TRY(launch(h, maxpool_split_kernel, g1, 256, 0, st, a.f4, d.H4, d.W4, C3, 3, 1, a.hp4, a.lp4, d.HP4, d.WP4,
               a.overflow, 1u << 3));
    TRY((launch_tc<3, K4, C3, 1, true>(h, c, 4, a.hp4, a.lp4, d.HP4, d.WP4, nullptr, a.h5, a.l5, st)));
    CU_TRY(h, cudaEventRecord(c.ev[1], st));
    CU_TRY(h, cudaEventRecord(c.ev[2], st));
    TRY((launch_tc<15, K4, C3, 2, false>(h, c, 5, a.h5, a.l5, d.H5, d.W5, a.feat, nullptr, nullptr, st)));
    c.maps_valid = true;
    c.attrs_set = true;
  }
  return ARTP_OK;
}

}  // namespace

int artp_api::cost_network(const Handle* h) {
  const CostNet& c = view(h);
  return c.has_weights ? c.net : -1;
}

int artp_api::check_cost_weights(Handle* h) {
  if (cost_network(h) < 0) { h->err = "motion-cost weights not set"; return ARTP_E_NOWEIGHTS; }
  return ARTP_OK;
}

int artp_api::check_cost_net(Handle* h) {
  TRY(check_cost_weights(h));
  if (!view(h).has_features) {
    h->err = "features not computed (call artp_update_features after artp_set_map)";
    return ARTP_E_NOWEIGHTS;
  }
  return ARTP_OK;
}

// CostPredictor.updateFeatures (predictor.py:28-36): the CNN trunk over the layer, one synchronisation of st.
int artp_api::update_features(Handle* h, const float* d_layer, int rows, int cols, int pitch, double res, double cx,
                              double cy, cudaStream_t st) {
  if (rows < 64 || cols < 64) { h->err = "map too small for the motion-cost network (needs >= 64 x 64 cells)"; return ARTP_E_INVALID; }
  CU_TRY(h, cudaSetDevice(h->device));
  CostNet& c = *h->cost_net;
  c.has_features = false;
  const TrunkDims d(rows, cols);
  const size_t c1 = c.layers[0].cout, c3 = c.layers[2].cout;
  auto split = [](int hh, int ww) { return (size_t)hh * ww * 64 * sizeof(__half); };
  auto f32 = [](int hh, int ww, size_t ch) { return (size_t)hh * ww * ch * sizeof(float); };
  char* r[19];   // the members of Acts in order
  TRY(carve(h, c.d_act, c.act_cap,
            {split(d.H1, d.W1), split(d.H1, d.W1), split(d.HP2, d.WP2), split(d.HP2, d.WP2), split(d.H3, d.W3),
             split(d.H3, d.W3), split(d.HP4, d.WP4), split(d.HP4, d.WP4), split(d.H5, d.W5), split(d.H5, d.W5),
             f32(d.H1, d.W1, c1), f32(d.H2, d.W2, c1), f32(d.HP2, d.WP2, c1), f32(d.H3, d.W3, c3), f32(d.H4, d.W4, c3),
             f32(d.HP4, d.WP4, c3), f32(d.H5, d.W5, c3), f32(d.H6, d.W6, c3), sizeof(unsigned)},
            r));
  c.a = {(__half*)r[0], (__half*)r[1], (__half*)r[2], (__half*)r[3], (__half*)r[4], (__half*)r[5], (__half*)r[6],
         (__half*)r[7], (__half*)r[8], (__half*)r[9], (float*)r[10], (float*)r[11], (float*)r[12], (float*)r[13],
         (float*)r[14], (float*)r[15], (float*)r[16], (float*)r[17], (unsigned*)r[18]};
  if (rows != c.rows || cols != c.cols) {
    c.rows = rows; c.cols = cols;
    c.maps_valid = false;
  }
  if (!c.ev[0]) for (auto& e : c.ev) CU_TRY(h, cudaEventCreate(&e));
  if (!c.h_overflow) CU_TRY(h, cudaMallocHost(&c.h_overflow, sizeof(unsigned)));
  CU_TRY(h, cudaMemsetAsync(c.a.overflow, 0, sizeof(unsigned), st));
  TRY(c.net == ARTP_COST_NET_FULL ? run_trunk<ARTP_COST_NET_FULL>(h, c, d_layer, pitch, d, st)
                                  : run_trunk<ARTP_COST_NET_LIGHT>(h, c, d_layer, pitch, d, st));
  CU_TRY(h, cudaEventRecord(c.ev[3], st));
  TRY(copy_async(h, c.h_overflow, c.a.overflow, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
  TRY(sync_stream(h, st));
  if (*c.h_overflow) {
    // The tensor-core path holds activations as fp16 hi + lo: beyond 65504 the split has no representation, and the
    // features would silently be inf / NaN. The CUDA-core path (artp_set_cnn_mode bit 0) has fp32 range throughout.
    int l = 0;
    while (!(*c.h_overflow & (1u << l))) ++l;
    h->err = std::string("motion-cost trunk: an activation of ") + kSplitLayerNames[l] +
             " exceeds the fp16 range (65504) of the tensor-core path's hi/lo split; the elevation or weight scale is out "
             "of range for it (the CUDA-core path, artp_set_cnn_mode bit 0, has fp32 range)";
    return ARTP_E_LIMIT;
  }
  cudaEventElapsedTime(&c.last_ms[0], c.ev[0], c.ev[1]);   // layers 1..5
  cudaEventElapsedTime(&c.last_ms[1], c.ev[2], c.ev[3]);   // 15x15 layer
  cudaEventElapsedTime(&c.last_ms[2], c.ev[0], c.ev[3]);   // whole trunk
  c.Hf = d.H6; c.Wf = d.W6;
  c.res = res; c.Lx = rows * res; c.Ly = cols * res; c.cx = cx; c.cy = cy;
  c.has_features = true;
  return ARTP_OK;
}

int artp_api::map_features(Handle* h) {
  // The resolution as artp_set_map received it: the head's row / column bias truncates (rows * res) / res like the
  // reference, and Lx / rows may differ from res in the last bit, which moves that truncation (e.g. 116 rows at 0.04).
  return update_features(h, h->map.H[0], h->map.rows, h->map.cols, h->map.pitch, h->map.res, h->chk.cx, h->chk.cy,
                         h->stream);
}

int artp_api::cost_head(Handle* h, const float* d_edges, size_t n, float* d_cost3, cudaStream_t st) {
  if (n == 0) return ARTP_OK;
  CU_TRY(h, cudaSetDevice(h->device));
  const CostNet& c = *h->cost_net;
  // One thread per query. Small batches (config 4: 4096 queries) use one-warp CTAs so that the batch spreads over the
  // SMs (128 CTAs instead of 32: 39 -> ~10 us); big batches amortise the 29 KB weight load over 128 queries per CTA.
  const int bt = n <= (size_t)h->sm_count * 128 ? 32 : 128;
  const unsigned grid = (unsigned)((n + bt - 1) / bt);
  const size_t smem = head_floats(c.net) * sizeof(float);   // 30 KB light, 46.8 KB full: under the 48 KB default
  constexpr NetDims L = kNets[ARTP_COST_NET_LIGHT], F = kNets[ARTP_COST_NET_FULL];
  auto kern = c.net == ARTP_COST_NET_FULL ? head_kernel<F.c3, F.nh, F.b[0], F.b[1], F.b[2]>
                                          : head_kernel<L.c3, L.nh, L.b[0], L.b[1], L.b[2]>;
  return launch(h, kern, grid, bt, smem, st, c.a.feat, c.Hf, c.Wf, c.d_head, d_edges, n, d_cost3,
                c.res, c.Lx, c.Ly, c.cx, c.cy);
}

void artp_api::cost_net_free(Handle* h) {
  CostNet* c = h->cost_net;
  if (!c) return;
  cudaFree(c->d_w);
  cudaFree(c->d_act);
  for (cudaEvent_t e : c->ev) if (e) cudaEventDestroy(e);
  cudaFreeHost(c->h_overflow);
  delete c;
}

extern "C" {

size_t artp_cost_weights_size(void) { return blob_floats(ARTP_COST_NET_LIGHT); }

size_t artp_cost_weights_size_for(int network) { return blob_floats(network); }

int artp_get_cost_network(artp_handle* hh, int* network) {
  LOCK_HANDLE(h, hh);
  if (!network) return ARTP_E_INVALID;
  *network = cost_network(h);
  return check_cost_weights(h);
}

int artp_set_cost_weights(artp_handle* hh, const float* blob, size_t n_floats) {
  LOCK_CALL(h, hh);
  if (!blob) return ARTP_E_INVALID;
  return set_weights(h, blob, n_floats);
}

int artp_update_features(artp_handle* hh) {
  LOCK_CALL(h, hh);
  TRY(require_whole_map(h));
  TRY(check_cost_weights(h));
  return map_features(h);
}

int artp_get_features(artp_handle* hh, float* out, size_t n_floats, int* hf, int* wf) {
  LOCK_HANDLE(h, hh);
  if (!hf || !wf) return ARTP_E_INVALID;
  const CostNet& c = view(h);
  *hf = c.Hf;
  *wf = c.Wf;
  if (!out) return ARTP_OK;
  TRY(check_cost_net(h));
  if (n_floats != (size_t)c.Hf * c.Wf * c.layers[5].cout) { h->err = "feature buffer size mismatch"; return ARTP_E_INVALID; }
  CU_TRY(h, cudaMemcpy(out, c.a.feat, n_floats * sizeof(float), cudaMemcpyDeviceToHost));
  return ARTP_OK;
}

int artp_set_cnn_mode(artp_handle* hh, int mode) {
  LOCK_HANDLE(h, hh);
  if (mode & ~1) { h->err = "unknown motion-cost network mode (bit 0 is the only mode bit)"; return ARTP_E_INVALID; }
  state(h).mode = mode;
  return ARTP_OK;
}

int artp_get_cnn_timing(artp_handle* hh, float* ms3) {
  LOCK_HANDLE(h, hh);
  if (!ms3) return ARTP_E_INVALID;
  const CostNet& c = view(h);
  for (int i = 0; i < 3; ++i) ms3[i] = c.last_ms[i];
  return ARTP_OK;
}

}  // extern "C"
