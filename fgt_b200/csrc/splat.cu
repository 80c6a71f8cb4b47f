// Forward flow splatting: LAFC/models/utils/flow_warp.py:4-94 (`flow_prop` / `warp` / `sample_one` /
// `get_gaussian_weights`) — every source pixel is scattered to the four integer neighbours of its flow target
// with Gaussian weights exp(-d^2), and the accumulated features are divided by the accumulated weight where it is
// positive. (Dead code in the reference — no caller — but named by the north star; SURVEY §8 row a10.)
// The reference repeats the flow over the channels and runs four put_(accumulate=True) passes per tensor; here one
// thread per source pixel computes the four targets and weights once and issues the atomics for all channels, the
// weight sum is accumulated once per pixel instead of once per channel, and a second kernel normalises.
// Note the reference's naming: flow channel 0 ("y") shifts the COLUMN index, channel 1 ("x") the ROW index
// (flow_warp.py:24-25,60-61,72-77). HBM-bound scatter; float atomics => summation order differs from the reference's
// sequential put_ (tolerance 1e-5 relative in the tests).
#include "common.h"

namespace fgt {

// Targets and weights of one source pixel (i, j) with flow (y: column shift, x: row shift): q = 0..3 are
// (x1,y1), (x1,y2), (x2,y1), (x2,y2) of flow_warp.py:37-40. __host__ __device__ so that the index / weight logic can be
// exercised without a GPU (fgt_flow_splat_targets_host).
__host__ __device__ inline void splat_targets(float x, float y, int i, int j, int H, int W, int backward, int* ti,
                                              int* tj, float* wt, bool* ok) {
  const float x1 = floorf(x), y1 = floorf(y);
  for (int q = 0; q < 4; ++q) {
    const float xs = x1 + static_cast<float>(q >> 1), ys = y1 + static_cast<float>(q & 1);
    const float dx = x - xs, dy = y - ys;
    wt[q] = expf(-(dx * dx + dy * dy));              // sigma = 1 (flow_warp.py:88-93)
    const long long sx = static_cast<long long>(xs), sy = static_cast<long long>(ys);
    const long long r = backward ? i - sx : i + sx;
    const long long c = backward ? j - sy : j + sy;
    ok[q] = r >= 0 && r < H && c >= 0 && c < W;      // flow_warp.py:66
    ti[q] = static_cast<int>(r);
    tj[q] = static_cast<int>(c);
  }
}

__global__ void splat_kernel(const float* __restrict__ feat, const float* __restrict__ flow, int B, int C, int H, int W,
                             int backward, float* __restrict__ acc, float* __restrict__ wsum) {
  pdl_launch_dependents();
  pdl_wait();
  const long long HW = static_cast<long long>(H) * W;
  const long long total = static_cast<long long>(B) * HW;
  for (long long g = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; g < total;
       g += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int b = static_cast<int>(g / HW);
    const long long p = g - b * HW;
    const int i = static_cast<int>(p / W), j = static_cast<int>(p - static_cast<long long>(i) * W);
    int ti[4], tj[4];
    float wt[4];
    bool ok[4];
    splat_targets(flow[(b * 2LL + 1) * HW + p], flow[(b * 2LL + 0) * HW + p], i, j, H, W, backward, ti, tj, wt, ok);
#pragma unroll
    for (int q = 0; q < 4; ++q)
      if (ok[q]) atomicAdd(&wsum[b * HW + static_cast<long long>(ti[q]) * W + tj[q]], wt[q]);
    for (int ch = 0; ch < C; ++ch) {
      const float f = feat[(static_cast<long long>(b) * C + ch) * HW + p];
      float* dst = acc + (static_cast<long long>(b) * C + ch) * HW;
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (ok[q]) atomicAdd(&dst[static_cast<long long>(ti[q]) * W + tj[q]], f * wt[q]);
    }
  }
}

// acc /= wsum where wsum > 0 (flow_warp.py:44-45), in place.
__global__ void splat_norm_kernel(float* __restrict__ acc, const float* __restrict__ wsum, int B, int C, long long HW) {
  pdl_launch_dependents();
  pdl_wait();
  const long long total = static_cast<long long>(B) * C * HW;
  for (long long g = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; g < total;
       g += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long bc = g / HW;
    const float o = wsum[(bc / C) * HW + (g - bc * HW)];
    if (o > 0.f) acc[g] = acc[g] / o;
  }
}

}  // namespace fgt

using namespace fgt;

extern "C" int fgt_flow_splat(const float* feat, const float* flow, int B, int C, int H, int W, int backward, float* out,
                              float* wsum, fgt_stream_t stream) {
  FGT_REQUIRE(feat && flow && out && wsum && B >= 1 && C >= 1 && H >= 1 && W >= 1, FGT_ERR_ARG,
              "flow_splat: bad argument");
  const long long HW = static_cast<long long>(H) * W;
  FGT_CUDA(cudaMemsetAsync(out, 0, sizeof(float) * B * C * HW, stream));
  FGT_CUDA(cudaMemsetAsync(wsum, 0, sizeof(float) * B * HW, stream));
  FGT_LAUNCH(splat_kernel, dim3(grid_stride(B * HW, 256)), dim3(256), 0, stream, feat, flow, B, C, H, W, backward, out,
             wsum);
  FGT_LAUNCH(splat_norm_kernel, dim3(grid_stride(B * C * HW, 256)), dim3(256), 0, stream, out,
             static_cast<const float*>(wsum), B, C, HW);
  return FGT_OK;
}

// HOST-ONLY test hook: the per-pixel target / weight computation the kernel runs (same __host__ __device__ function).
extern "C" int fgt_flow_splat_targets_host(float x, float y, int i, int j, int H, int W, int backward, int* ti_host,
                                           int* tj_host, float* wt_host, int* ok_host) {
  FGT_REQUIRE(ti_host && tj_host && wt_host && ok_host, FGT_ERR_ARG, "flow_splat_targets_host: bad argument");
  bool ok[4];
  splat_targets(x, y, i, j, H, W, backward, ti_host, tj_host, wt_host, ok);
  for (int q = 0; q < 4; ++q) ok_host[q] = ok[q];
  return FGT_OK;
}
