// Flow colour coding (RAFT/utils/flow_viz.py: flow_to_image :109-132, flow_uv_to_colors :70-106, make_colorwheel
// :20-67) for a batch of B flows [B,H,W,2] fp32 -> uint8 [B,H,W,3], each image normalised by its own maximum radius.
//
// max kernel: grid (parts, B); each CTA takes the maximum of r = sqrt(u*u + v*v) over kPart pixels of one image and
// stores it to workspace[b * parts + part] as the float's bit pattern (r >= +0, so unsigned order is float order; a
// non-finite u or v stores kBad, above every float, as the reference raises IndexError there). A maximum is exact in
// any order. colour kernel: grid (tiles, B); each CTA reduces its image's partials first (from L2), then colours
// kTile pixels. An image with a non-finite value is left unwritten and its maximum reported as NaN.
// HBM traffic per pixel: 8 B read by the max pass, 8 B read + 3 B written by the colour pass, 19 B in all.
//
// Arithmetic is numpy's under NEP 50 with no contraction: float32 for the radius, the normalisation, the angle and
// the wheel coordinate fk; float64 from f = fk - k0 on (float32 minus int32 promotes).
#include "common.h"

namespace fgt {
namespace flowviz {

constexpr int kThreads = 256;
constexpr int kMaxPix = 16;                          // pixels per thread, max pass
constexpr int kColPix = 8;                           // pixels per thread, colour pass
constexpr long long kPart = kThreads * kMaxPix;      // pixels per max CTA
constexpr long long kTile = kThreads * kColPix;      // pixels per colour CTA
constexpr unsigned kBad = 0x7fc00000u;               // NaN bits: marks a non-finite input
constexpr int kCols = 55;                            // RY + YG + GC + CB + BM + MR

// make_colorwheel: floor(255 * i / n) of each ramp, as integers (exact: no quotient of these is within an ulp of an
// integer it does not equal)
struct Wheel {
  unsigned char c[kCols][3];
};
constexpr Wheel make_wheel() {
  Wheel w{};
  const int n[6] = {15, 6, 4, 11, 13, 6};
  int k = 0;
  for (int i = 0; i < n[0]; ++i, ++k) w.c[k][0] = 255, w.c[k][1] = 255 * i / n[0], w.c[k][2] = 0;          // RY
  for (int i = 0; i < n[1]; ++i, ++k) w.c[k][0] = 255 - 255 * i / n[1], w.c[k][1] = 255, w.c[k][2] = 0;    // YG
  for (int i = 0; i < n[2]; ++i, ++k) w.c[k][0] = 0, w.c[k][1] = 255, w.c[k][2] = 255 * i / n[2];          // GC
  for (int i = 0; i < n[3]; ++i, ++k) w.c[k][0] = 0, w.c[k][1] = 255 - 255 * i / n[3], w.c[k][2] = 255;    // CB
  for (int i = 0; i < n[4]; ++i, ++k) w.c[k][0] = 255 * i / n[4], w.c[k][1] = 0, w.c[k][2] = 255;          // BM
  for (int i = 0; i < n[5]; ++i, ++k) w.c[k][0] = 255, w.c[k][1] = 0, w.c[k][2] = 255 - 255 * i / n[5];    // MR
  return w;
}
__constant__ Wheel c_wheel = make_wheel();

__device__ __forceinline__ unsigned radius_bits(float2 f) {
  if (!isfinite(f.x) || !isfinite(f.y)) return kBad;
  return __float_as_uint(__fsqrt_rn(__fadd_rn(__fmul_rn(f.x, f.x), __fmul_rn(f.y, f.y))));
}

__device__ __forceinline__ unsigned block_max(unsigned v, unsigned* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  v = 0;
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) v = max(v, red[w]);
  return v;
}

__global__ void __launch_bounds__(kThreads) flow_max_kernel(const float2* __restrict__ flow, long long hw,
                                                            unsigned* __restrict__ part) {
  __shared__ unsigned red[kThreads / 32];
  const float2* img = flow + static_cast<long long>(blockIdx.y) * hw;
  const long long p0 = static_cast<long long>(blockIdx.x) * kPart + threadIdx.x;
  unsigned m = 0;
#pragma unroll
  for (int k = 0; k < kMaxPix; ++k) {
    const long long p = p0 + static_cast<long long>(k) * kThreads;
    if (p < hw) m = max(m, radius_bits(__ldg(img + p)));
  }
  m = block_max(m, red);
  if (threadIdx.x == 0) part[static_cast<long long>(blockIdx.y) * gridDim.x + blockIdx.x] = m;
}

// flow_uv_to_colors for one pixel of the normalised flow (un, vn); writes the three channels in RGB or BGR order.
// w: the wheel divided by 255.0 in float64, [kCols][3]
__device__ __forceinline__ void colour(float un, float vn, int bgr, const double* w, unsigned char* o) {
  const float rad = __fsqrt_rn(__fadd_rn(__fmul_rn(un, un), __fmul_rn(vn, vn)));
  // -v and -u are sign flips, so (+-0) selects between wheel entries 0 and 54 exactly as numpy does
  const float a = __fdiv_rn(atan2f(-vn, -un), 3.14159265358979323846f);
  const float fk = __fmul_rn(__fdiv_rn(__fadd_rn(a, 1.0f), 2.0f), static_cast<float>(kCols - 1));
  const int k0 = static_cast<int>(floorf(fk));
  const int k1 = k0 + 1 == kCols ? 0 : k0 + 1;
  const double f = __dsub_rn(static_cast<double>(fk), static_cast<double>(k0));
  const double g = __dsub_rn(1.0, f);
  const double r = static_cast<double>(rad);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const double c0 = w[3 * k0 + i], c1 = w[3 * k1 + i];
    double col = __dadd_rn(__dmul_rn(g, c0), __dmul_rn(f, c1));
    col = rad <= 1.0f ? __dsub_rn(1.0, __dmul_rn(r, __dsub_rn(1.0, col))) : __dmul_rn(col, 0.75);
    o[bgr ? 2 - i : i] = static_cast<unsigned char>(floor(__dmul_rn(255.0, col)));
  }
}

__global__ void __launch_bounds__(kThreads) flow_colour_kernel(const float2* __restrict__ flow, long long hw, int parts,
                                                               const unsigned* __restrict__ part, int bgr,
                                                               unsigned char* __restrict__ out,
                                                               float* __restrict__ maxima) {
  __shared__ unsigned red[kThreads / 32];
  __shared__ double wheel[kCols * 3];   // tmp[k] / 255.0 (:97-98), once per CTA instead of six divisions per pixel
  for (int i = threadIdx.x; i < kCols * 3; i += kThreads) wheel[i] = __ddiv_rn(c_wheel.c[i / 3][i % 3], 255.0);
  const int b = blockIdx.y;
  unsigned m = 0;
  for (int i = threadIdx.x; i < parts; i += kThreads) m = max(m, part[static_cast<long long>(b) * parts + i]);
  m = block_max(m, red);                            // (its barrier also publishes `wheel`)
  const float rmax = __uint_as_float(m);
  if (blockIdx.x == 0 && threadIdx.x == 0 && maxima) maxima[b] = rmax;
  if (m == kBad) return;
  const float d = __fadd_rn(rmax, 1e-5f);           // rad_max + epsilon (float32 + Python float stays float32)
  const float2* img = flow + static_cast<long long>(b) * hw;
  unsigned char* dst = out + static_cast<long long>(b) * hw * 3;
  const long long p0 = static_cast<long long>(blockIdx.x) * kTile + threadIdx.x;
  // every load is issued before the first is used, so the thread waits for global memory once
  float2 f[kColPix];
#pragma unroll
  for (int k = 0; k < kColPix; ++k) {
    const long long p = p0 + static_cast<long long>(k) * kThreads;
    f[k] = p < hw ? __ldg(img + p) : make_float2(0.f, 0.f);
  }
#pragma unroll
  for (int k = 0; k < kColPix; ++k) {
    const long long p = p0 + static_cast<long long>(k) * kThreads;
    if (p < hw) colour(__fdiv_rn(f[k].x, d), __fdiv_rn(f[k].y, d), bgr, wheel, dst + 3 * p);
  }
}

inline int parts_of(long long hw) { return static_cast<int>((hw + kPart - 1) / kPart); }

}  // namespace flowviz
}  // namespace fgt

using namespace fgt::flowviz;

static int flowviz_check(int B, int H, int W) {
  FGT_REQUIRE(B >= 1 && H >= 1 && W >= 1, FGT_ERR_ARG, "flow_to_image: empty batch or image (B=%d H=%d W=%d)", B, H,
              W);
  FGT_REQUIRE(B <= 65535, FGT_ERR_ARG, "flow_to_image: B = %d exceeds 65535 images per call", B);
  const long long hw = static_cast<long long>(H) * W;
  FGT_REQUIRE((hw + kTile - 1) / kTile <= 0x7fffffffLL, FGT_ERR_ARG, "flow_to_image: %dx%d is too large", H, W);
  return FGT_OK;
}

extern "C" long long fgt_flow_to_image_workspace(int B, int H, int W) {
  const int rc = flowviz_check(B, H, W);
  if (rc != FGT_OK) return rc;
  return static_cast<long long>(B) * parts_of(static_cast<long long>(H) * W) * static_cast<long long>(sizeof(unsigned));
}

extern "C" int fgt_flow_to_image(const float* flow, int B, int H, int W, int bgr, void* workspace,
                                 long long workspace_bytes, unsigned char* out, float* maxima, fgt_stream_t stream) {
  FGT_REQUIRE(flow && workspace && out, FGT_ERR_ARG, "flow_to_image: null pointer");
  const int rc = flowviz_check(B, H, W);
  if (rc != FGT_OK) return rc;
  FGT_REQUIRE(reinterpret_cast<uintptr_t>(flow) % 8 == 0, FGT_ERR_ARG, "flow_to_image: flow is not 8-byte aligned");
  const long long need = fgt_flow_to_image_workspace(B, H, W);
  FGT_REQUIRE(workspace_bytes >= need, FGT_ERR_ARG, "flow_to_image: workspace of %lld bytes, %lld needed",
              workspace_bytes, need);
  const long long hw = static_cast<long long>(H) * W;
  const int parts = parts_of(hw);
  const float2* f2 = reinterpret_cast<const float2*>(flow);
  unsigned* ws = static_cast<unsigned*>(workspace);
  FGT_LAUNCH(flow_max_kernel, dim3(parts, B), dim3(kThreads), 0, stream, f2, hw, ws);
  FGT_LAUNCH(flow_colour_kernel, dim3(static_cast<unsigned>((hw + kTile - 1) / kTile), B), dim3(kThreads), 0, stream,
             f2, hw, parts, static_cast<const unsigned*>(ws), bgr ? 1 : 0, out, maxima);
  return FGT_OK;
}
