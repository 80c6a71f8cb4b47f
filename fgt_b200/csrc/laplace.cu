// Batched region fill = discrete Laplace solve inside hole masks (tool/utils/region_fill.py:7-138,
// called per flow channel by diffusion(), tool/video_inpainting.py:44-52). The reference assembles a sparse
// matrix per image and calls scipy's direct solver; here all B images are solved together, matrix-free,
// with conjugate gradients in fp64 (the system — diagonal = number of in-image 4-neighbours, -1 towards
// neighbours inside the mask — is symmetric positive definite whenever the mask does not cover the image).
// HBM-bound: one iteration = two kernels streaming ~5 fp64 arrays over the masked pixels.
//
// Per-iteration scalars never need resetting: iteration k accumulates <p,Ap> into pap[k*B + b] and the new
// <r,r> into rr[(k+1)*B + b] of zero-initialised arrays, and reads the ones finished by earlier kernels.
#include "common.h"

namespace fgt {

constexpr int kLapThreads = 256;
constexpr int kLapPerThread = 8;  // pixels per thread -> few blocks -> few same-address double atomics

__device__ __forceinline__ double block_sum(double v, double* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double s = 0.0;
  if (warp == 0) {
    s = lane < (kLapThreads >> 5) ? red[lane] : 0.0;
    for (int o = 4; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  }
  __syncthreads();
  return s;  // valid in thread 0
}

// x = 0, r = p = b with b(p) = sum of the image values of p's in-image neighbours outside the mask
// (formRightSide, region_fill.py:69-112); rr[0] = <r,r>.
__global__ void lap_init_kernel(const double* __restrict__ img, const unsigned char* __restrict__ mask, int H, int W,
                                double* __restrict__ x, double* __restrict__ r, double* __restrict__ p,
                                double* __restrict__ rr) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ double red[kLapThreads / 32];
  const int b = blockIdx.y;
  const long long base = static_cast<long long>(b) * H * W;
  double acc = 0.0;
  for (int j = 0; j < kLapPerThread; ++j) {
    const int i = (blockIdx.x * kLapPerThread + j) * kLapThreads + threadIdx.x;
    if (i >= H * W) break;
    double bv = 0.0;
    if (mask[base + i]) {
      const int y = i / W, xx = i - y * W;
      if (y > 0 && !mask[base + i - W]) bv += img[base + i - W];
      if (y < H - 1 && !mask[base + i + W]) bv += img[base + i + W];
      if (xx > 0 && !mask[base + i - 1]) bv += img[base + i - 1];
      if (xx < W - 1 && !mask[base + i + 1]) bv += img[base + i + 1];
    }
    x[base + i] = 0.0;
    r[base + i] = bv;
    p[base + i] = bv;
    acc += bv * bv;
  }
  const double s = block_sum(acc, red);
  if (threadIdx.x == 0 && s != 0.0) atomicAdd(&rr[b], s);
}

// p_new = r + beta * p_old (beta = rr[k] / rr[k-1], 0 at k = 0), Ap = A p_new, pap[k] += <p_new, Ap>.
// Neighbours' p_new are recomputed from r and p_old (ping-pong buffers: p_old is read-only here).
__global__ void lap_dir_kernel(const unsigned char* __restrict__ mask, int B, int H, int W,
                               const double* __restrict__ r, const double* __restrict__ p_old,
                               double* __restrict__ p_new, double* __restrict__ ap, const double* __restrict__ rr,
                               double* __restrict__ pap, int k) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ double red[kLapThreads / 32];
  const int b = blockIdx.y;
  const long long base = static_cast<long long>(b) * H * W;
  double beta = 0.0;
  if (k > 0) {
    const double den = rr[static_cast<long long>(k - 1) * B + b];
    beta = den > 0.0 ? rr[static_cast<long long>(k) * B + b] / den : 0.0;
  }
  double acc = 0.0;
  for (int j = 0; j < kLapPerThread; ++j) {
    const int i = (blockIdx.x * kLapPerThread + j) * kLapThreads + threadIdx.x;
    if (i >= H * W) break;
    if (!mask[base + i]) continue;
    const int y = i / W, xx = i - y * W;
    const double pc = r[base + i] + beta * p_old[base + i];
    double a = 0.0;
    int cnt = 0;
    if (y > 0) { ++cnt; if (mask[base + i - W]) a -= r[base + i - W] + beta * p_old[base + i - W]; }
    if (y < H - 1) { ++cnt; if (mask[base + i + W]) a -= r[base + i + W] + beta * p_old[base + i + W]; }
    if (xx > 0) { ++cnt; if (mask[base + i - 1]) a -= r[base + i - 1] + beta * p_old[base + i - 1]; }
    if (xx < W - 1) { ++cnt; if (mask[base + i + 1]) a -= r[base + i + 1] + beta * p_old[base + i + 1]; }
    a += static_cast<double>(cnt) * pc;
    p_new[base + i] = pc;
    ap[base + i] = a;
    acc += pc * a;
  }
  const double s = block_sum(acc, red);
  if (threadIdx.x == 0 && s != 0.0) atomicAdd(&pap[static_cast<long long>(k) * B + b], s);
}

// alpha = rr[k] / pap[k]; x += alpha p; r -= alpha Ap; rr[k+1] += <r,r>.
__global__ void lap_update_kernel(const unsigned char* __restrict__ mask, int B, int H, int W,
                                  const double* __restrict__ p, const double* __restrict__ ap, double* __restrict__ x,
                                  double* __restrict__ r, double* __restrict__ rr, const double* __restrict__ pap,
                                  int k) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ double red[kLapThreads / 32];
  const int b = blockIdx.y;
  const long long base = static_cast<long long>(b) * H * W;
  const double den = pap[static_cast<long long>(k) * B + b];
  const double alpha = den > 0.0 ? rr[static_cast<long long>(k) * B + b] / den : 0.0;
  double acc = 0.0;
  for (int j = 0; j < kLapPerThread; ++j) {
    const int i = (blockIdx.x * kLapPerThread + j) * kLapThreads + threadIdx.x;
    if (i >= H * W) break;
    if (!mask[base + i]) continue;
    x[base + i] += alpha * p[base + i];
    const double rn = r[base + i] - alpha * ap[base + i];
    r[base + i] = rn;
    acc += rn * rn;
  }
  const double s = block_sum(acc, red);
  if (threadIdx.x == 0 && s != 0.0) atomicAdd(&rr[static_cast<long long>(k + 1) * B + b], s);
}

// out = x inside the mask, the input image outside (region_fill.py:15-16).
__global__ void lap_finish_kernel(const double* __restrict__ img, const unsigned char* __restrict__ mask, long long total,
                                  const double* __restrict__ x, double* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    out[i] = mask[i] ? x[i] : img[i];
}

}  // namespace fgt

using namespace fgt;

static dim3 lap_grid(int B, int H, int W) {
  const int per_block = kLapThreads * kLapPerThread;
  return dim3((H * W + per_block - 1) / per_block, B);
}

extern "C" int fgt_regionfill_init(const double* img, const unsigned char* mask, int B, int H, int W, double* x,
                                   double* r, double* p, double* rr, fgt_stream_t stream) {
  FGT_REQUIRE(img && mask && x && r && p && rr && B >= 1 && H >= 1 && W >= 1, FGT_ERR_ARG, "regionfill_init: bad argument");
  FGT_LAUNCH(lap_init_kernel, lap_grid(B, H, W), dim3(kLapThreads), 0, stream, img, mask, H, W, x, r, p, rr);
  return FGT_OK;
}

extern "C" int fgt_regionfill_iters(const unsigned char* mask, int B, int H, int W, double* x, double* r, double* p0,
                                    double* p1, double* ap, double* rr, double* pap, int k0, int iters,
                                    fgt_stream_t stream) {
  FGT_REQUIRE(mask && x && r && p0 && p1 && ap && rr && pap && B >= 1 && k0 >= 0 && iters >= 1, FGT_ERR_ARG,
              "regionfill_iters: bad argument");
  const dim3 grid = lap_grid(B, H, W);
  for (int k = k0; k < k0 + iters; ++k) {
    double* p_old = (k & 1) ? p1 : p0;  // iteration k reads the direction written by iteration k-1
    double* p_new = (k & 1) ? p0 : p1;
    FGT_LAUNCH(lap_dir_kernel, grid, dim3(kLapThreads), 0, stream, mask, B, H, W, static_cast<const double*>(r),
               static_cast<const double*>(p_old), p_new, ap, static_cast<const double*>(rr), pap, k);
    FGT_LAUNCH(lap_update_kernel, grid, dim3(kLapThreads), 0, stream, mask, B, H, W, static_cast<const double*>(p_new),
               static_cast<const double*>(ap), x, r, rr, static_cast<const double*>(pap), k);
  }
  return FGT_OK;
}

extern "C" int fgt_regionfill_finish(const double* img, const unsigned char* mask, long long total, const double* x,
                                     double* out, fgt_stream_t stream) {
  FGT_REQUIRE(img && mask && x && out && total >= 1, FGT_ERR_ARG, "regionfill_finish: bad argument");
  FGT_LAUNCH(lap_finish_kernel, dim3(grid_stride(total, 256)), dim3(256), 0, stream, img, mask, total, x, out);
  return FGT_OK;
}
