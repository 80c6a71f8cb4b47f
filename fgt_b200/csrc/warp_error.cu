// Flow warping error (E_warp) of a clip: the reference's image_warp and the forward half of fbConsistencyCheck
// (FGT/models/utils/fbConsistencyCheck.py), with grid_sample's align_corners=True convention, composed in float64
// (definition: oracle/warp_error_oracle.py).
//
// tile kernel: one CTA per (pair t, 32x32 pixel tile), 32x8 threads, four rows per thread. For each pixel it samples
// the backward flow B_t at x + F_t(x), evaluates the occlusion test, samples the C channels of frame t+1 at the same
// position and accumulates, in float64, (sum M*err, sum M, sum M*hole*err, sum M*hole) with err = sum_c (I_t - W_t)^2.
// The CTA writes those four doubles to the workspace, reduced over its warps in a fixed order. reduce kernel: one warp
// per pair sums its tiles in a fixed order, so a pair's sums depend on nothing but its own inputs and are the same bit
// for bit from run to run.
//
// The float32 arithmetic is spelled out with __f*_rn intrinsics, so nothing is contracted except where the reference
// itself fuses: ATen's vectorised CPU grid sampler (AVX2 / AVX-512 builds, which the reference's numbers come from)
// adds its four bilinear terms as nw_v*nw followed by three fused multiply-adds.
// Bytes per pixel and pair: F_t and the 2-channel B_t sample (8 + 8, the B corners mostly from L1/L2), frame t and
// frame t+1 (2 C element sizes), the hole (1, with masks), plus the optional maps (4 C + 1 written).
#include "common.h"

namespace fgt {
namespace warp_error {

constexpr int kTX = 32, kTY = 32, kRowsPerThread = 4;
constexpr int kThreads = kTX * kTY / kRowsPerThread;     // 256: 32 x 8
constexpr int kWarps = kThreads / 32;
static_assert(kThreads == 256, "one thread per entry of the uint8 quotient table");

struct Geometry {
  int H, W, C;
  float sx, sy;        // (W - 1) / 2, (H - 1) / 2: exact in float32
  double step_x, step_y;   // np.linspace's step 2 / (n - 1)
};

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// np.linspace(-1, 1, n)[i] cast to float32: i * step + (-1) in float64, the last point exactly 1
__device__ __forceinline__ float linspace32(int i, int n, double step) {
  return i == n - 1 ? 1.f : __double2float_rn(__dadd_rn(__dmul_rn(static_cast<double>(i), step), -1.0));
}

// Bilinear sample position of pixel (x, y) moved by (fx, fy): corner offsets (or -1 outside the image) and weights
struct Sample {
  long long off[4];    // nw, ne, sw, se pixel offsets within the plane, -1 = zero padding
  float wt[4];
};

__device__ __forceinline__ Sample locate(int x, int y, float fx, float fy, const Geometry& g) {
  const float gx = linspace32(x, g.W, g.step_x), gy = linspace32(y, g.H, g.step_y);
  // image_warp: grid + flow / ((n - 1) / 2); grid_sample (align_corners): (g + 1) * (n - 1) / 2
  const float ix = __fmul_rn(__fadd_rn(__fadd_rn(gx, __fdiv_rn(fx, g.sx)), 1.f), g.sx);
  const float iy = __fmul_rn(__fadd_rn(__fadd_rn(gy, __fdiv_rn(fy, g.sy)), 1.f), g.sy);
  const float x0 = floorf(ix), y0 = floorf(iy);
  const float w = __fsub_rn(ix, x0), e = __fsub_rn(1.f, w);
  const float n = __fsub_rn(iy, y0), s = __fsub_rn(1.f, n);
  Sample r;
  r.wt[0] = __fmul_rn(s, e);
  r.wt[1] = __fmul_rn(s, w);
  r.wt[2] = __fmul_rn(n, e);
  r.wt[3] = __fmul_rn(n, w);
  // in-bounds tests on the float corners (false for NaN), before any conversion to int
  const bool xw = x0 >= 0.f && x0 < static_cast<float>(g.W), xe = x0 >= -1.f && x0 < static_cast<float>(g.W - 1);
  const bool yn = y0 >= 0.f && y0 < static_cast<float>(g.H), ys = y0 >= -1.f && y0 < static_cast<float>(g.H - 1);
  const long long xi = (xw || xe) ? static_cast<long long>(x0) : 0, yi = (yn || ys) ? static_cast<long long>(y0) : 0;
  r.off[0] = xw && yn ? yi * g.W + xi : -1;
  r.off[1] = xe && yn ? yi * g.W + xi + 1 : -1;
  r.off[2] = xw && ys ? (yi + 1) * g.W + xi : -1;
  r.off[3] = xe && ys ? (yi + 1) * g.W + xi + 1 : -1;
  return r;
}

// ATen's CPU bilinear sum: nw_v*nw, then fused ne, sw, se terms; a corner outside the image contributes 0 * weight
__device__ __forceinline__ float blend(const float v[4], const float wt[4]) {
  float o = __fmul_rn(v[0], wt[0]);
  o = __fmaf_rn(v[1], wt[1], o);
  o = __fmaf_rn(v[2], wt[2], o);
  return __fmaf_rn(v[3], wt[3], o);
}

// I = float32(V) / 255, the division correctly rounded; uint8 values through a table of the 256 quotients
template <typename T>
__device__ __forceinline__ float unit(const T* p, const float* lut) {
  if constexpr (sizeof(T) == 1) return lut[__ldg(p)];
  else return __fdiv_rn(__ldg(p), 255.f);
}

// ws[(t * tiles + tile) * 4 + k] = (sum M*err, sum M, sum M*hole*err, sum M*hole) of the tile
template <typename T>
__global__ void __launch_bounds__(kThreads) warp_error_tile_kernel(const T* __restrict__ frames,
                                                                   const unsigned char* __restrict__ masks,
                                                                   const float* __restrict__ flow_f,
                                                                   const float* __restrict__ flow_b, Geometry g,
                                                                   double* __restrict__ ws, float* __restrict__ warped,
                                                                   unsigned char* __restrict__ valid) {
  __shared__ float lut[sizeof(T) == 1 ? 256 : 1];
  if (sizeof(T) == 1) {
    lut[threadIdx.x] = __fdiv_rn(static_cast<float>(threadIdx.x), 255.f);
    __syncthreads();
  }
  const int t = blockIdx.z, H = g.H, W = g.W, C = g.C;
  const long long plane = static_cast<long long>(H) * W;
  const float* fx_p = flow_f + 2 * t * plane;
  const float* fy_p = fx_p + plane;
  const float* bx_p = flow_b + 2 * t * plane;
  const float* by_p = bx_p + plane;
  const T* cur = frames + t * plane * C;
  const T* nxt = cur + plane * C;
  const int x = blockIdx.x * kTX + (threadIdx.x & 31);
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
  for (int k = 0; k < kRowsPerThread; ++k) {
    const int y = blockIdx.y * kTY + (threadIdx.x >> 5) + k * (kThreads / 32);
    if (x >= W || y >= H) continue;
    const long long px = static_cast<long long>(y) * W + x;
    const float fx = __ldg(fx_p + px), fy = __ldg(fy_p + px);
    const Sample sm = locate(x, y, fx, fy, g);
    float vx[4], vy[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      vx[q] = sm.off[q] >= 0 ? __ldg(bx_p + sm.off[q]) : 0.f;
      vy[q] = sm.off[q] >= 0 ? __ldg(by_p + sm.off[q]) : 0.f;
    }
    const float bx = blend(vx, sm.wt), by = blend(vy, sm.wt);
    // fbConsistencyCheck: |F + B(x+F)|^2 > alpha1 * (|F|^2 + |B(x+F)|^2) + alpha2 marks an occlusion
    const float dx = __fadd_rn(fx, bx), dy = __fadd_rn(fy, by);
    const float len_d = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
    const float mag = __fadd_rn(__fadd_rn(__fmul_rn(fx, fx), __fmul_rn(fy, fy)),
                                __fadd_rn(__fmul_rn(bx, bx), __fmul_rn(by, by)));
    const bool ok = !(len_d > __fadd_rn(__fmul_rn(0.01f, mag), 0.5f));
    double err = 0.0;
    for (int c = 0; c < C; ++c) {
      float v[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) v[q] = sm.off[q] >= 0 ? unit(nxt + sm.off[q] * C + c, lut) : 0.f;
      const float wv = blend(v, sm.wt);
      const double d = static_cast<double>(unit(cur + px * C + c, lut)) - static_cast<double>(wv);
      err = __dadd_rn(err, __dmul_rn(d, d));
      if (warped) warped[(t * plane + px) * C + c] = wv;
    }
    if (valid) valid[t * plane + px] = ok ? 1 : 0;
    if (ok) {
      acc[0] += err;
      acc[1] += 1.0;
      if (masks && masks[t * plane + px] != 0) {
        acc[2] += err;
        acc[3] += 1.0;
      }
    }
  }
  __shared__ double red[kWarps][4];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const double s = warp_sum(acc[k]);
    if (lane == 0) red[wid][k] = s;
  }
  __syncthreads();
  if (threadIdx.x < 4) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) s += red[w][threadIdx.x];
    const long long tile = static_cast<long long>(blockIdx.y) * gridDim.x + blockIdx.x;
    ws[(static_cast<long long>(t) * gridDim.x * gridDim.y + tile) * 4 + threadIdx.x] = s;
  }
}

// one warp per pair: out[t][k] = the fixed-order sum of its tiles' partials
__global__ void warp_error_reduce_kernel(const double* __restrict__ ws, int P, long long tiles, double* __restrict__ out) {
  const int t = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31;
  if (t >= P) return;
  const double* p = ws + t * tiles * 4;
  double s[4] = {0.0, 0.0, 0.0, 0.0};
  for (long long i = lane; i < tiles; i += 32)
#pragma unroll
    for (int k = 0; k < 4; ++k) s[k] += p[4 * i + k];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const double v = warp_sum(s[k]);
    if (lane == 0) out[4LL * t + k] = v;
  }
}

inline long long tiles_of(int H, int W) {
  return static_cast<long long>((W + kTX - 1) / kTX) * ((H + kTY - 1) / kTY);
}

template <typename T>
int launch_tiles(const void* frames, const unsigned char* masks, const float* flow_f, const float* flow_b, int P,
                 const Geometry& g, double* ws, float* warped, unsigned char* valid, fgt_stream_t s) {
  const dim3 grid((g.W + kTX - 1) / kTX, (g.H + kTY - 1) / kTY, P);
  FGT_LAUNCH(warp_error_tile_kernel<T>, grid, dim3(kThreads), 0, s, static_cast<const T*>(frames), masks, flow_f,
             flow_b, g, ws, warped, valid);
  return FGT_OK;
}

}  // namespace warp_error
}  // namespace fgt

using namespace fgt::warp_error;

static int warp_error_check(int N, int H, int W, int C) {
  FGT_REQUIRE(N >= 2, FGT_ERR_ARG, "warp_error: %d frames (at least 2, one pair, needed)", N);
  FGT_REQUIRE(H >= 2 && W >= 2, FGT_ERR_ARG, "warp_error: frames of %dx%d (at least 2x2 needed)", H, W);
  FGT_REQUIRE(C == 1 || C == 3, FGT_ERR_ARG, "warp_error: %d channels (1 or 3 supported)", C);
  FGT_REQUIRE(N - 1 <= 65535, FGT_ERR_ARG, "warp_error: %d pairs exceed 65535 per call", N - 1);
  return FGT_OK;
}

extern "C" long long fgt_warp_error_workspace(int N, int H, int W, int C) {
  const int rc = warp_error_check(N, H, W, C);
  if (rc != FGT_OK) return rc;
  return static_cast<long long>(N - 1) * tiles_of(H, W) * 4 * static_cast<long long>(sizeof(double));
}

extern "C" int fgt_warp_error(const void* frames, int frame_dtype, const unsigned char* masks, const float* flow_f,
                              const float* flow_b, int N, int H, int W, int C, void* workspace,
                              long long workspace_bytes, double* out, float* warped, unsigned char* valid,
                              fgt_stream_t stream) {
  FGT_REQUIRE(frames && flow_f && flow_b && workspace && out, FGT_ERR_ARG, "warp_error: null pointer");
  int rc = warp_error_check(N, H, W, C);
  if (rc != FGT_OK) return rc;
  FGT_REQUIRE(frame_dtype == FGT_METRIC_U8 || frame_dtype == FGT_METRIC_F32, FGT_ERR_ARG,
              "warp_error: unsupported frame dtype code %d (FGT_METRIC_U8 or FGT_METRIC_F32)", frame_dtype);
  const long long need = fgt_warp_error_workspace(N, H, W, C);
  FGT_REQUIRE(workspace_bytes >= need, FGT_ERR_ARG, "warp_error: workspace of %lld bytes, %lld needed",
              workspace_bytes, need);
  Geometry g;
  g.H = H;
  g.W = W;
  g.C = C;
  g.sx = static_cast<float>((W - 1.0) / 2.0);
  g.sy = static_cast<float>((H - 1.0) / 2.0);
  g.step_x = 2.0 / (W - 1);
  g.step_y = 2.0 / (H - 1);
  double* ws = static_cast<double*>(workspace);
  const int P = N - 1;
  rc = frame_dtype == FGT_METRIC_F32
           ? launch_tiles<float>(frames, masks, flow_f, flow_b, P, g, ws, warped, valid, stream)
           : launch_tiles<uint8_t>(frames, masks, flow_f, flow_b, P, g, ws, warped, valid, stream);
  if (rc != FGT_OK) return rc;
  constexpr int kReduceWarps = 4;
  FGT_LAUNCH(warp_error_reduce_kernel, dim3((P + kReduceWarps - 1) / kReduceWarps), dim3(32 * kReduceWarps), 0,
             stream, ws, P, tiles_of(H, W), out);
  return FGT_OK;
}
