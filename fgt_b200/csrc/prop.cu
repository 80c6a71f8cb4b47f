// Flow-guided gradient propagation on the GPU (tool/get_flowNN_gradient.py:11-534, Nonlocal=False):
// per-frame neighbour chaining with round-trip consistency, ordered bilinear gathers of the image
// gradients, confidence-weighted fusion. HBM-bound gather kernels over dense [N,H,W] state; frames
// are processed by successive launches (the reference's sequential frame dependence), pixels in
// parallel. Arithmetic reproduces the reference's types and operation order (float32 positions,
// float64 chaining/consistency, cv2.remap's 1/32-pixel fixed-point bilinear) with explicit
// round-to-nearest intrinsics so that no FMA contraction changes a rounding or a threshold test.
#include "common.h"

namespace fgt {

// cv2.remap(INTER_LINEAR, BORDER_CONSTANT=0) of channel `c` (stride `cs`) of a row-major float image.
__device__ __forceinline__ float remap_q32(const float* __restrict__ img, int H, int W, int cs, int c, float x,
                                           float y) {
  const int sx = __float2int_rn(__fmul_rn(x, 32.f));
  const int sy = __float2int_rn(__fmul_rn(y, 32.f));
  const int ix = sx >> 5, iy = sy >> 5;
  const float fx = __fdiv_rn(static_cast<float>(sx & 31), 32.f);
  const float fy = __fdiv_rn(static_cast<float>(sy & 31), 32.f);
  auto tap = [&](int yy, int xx) -> float {
    return (yy >= 0 && yy < H && xx >= 0 && xx < W) ? img[(static_cast<long long>(yy) * W + xx) * cs + c] : 0.f;
  };
  const float w00 = __fmul_rn(__fsub_rn(1.f, fy), __fsub_rn(1.f, fx));
  const float w01 = __fmul_rn(__fsub_rn(1.f, fy), fx);
  const float w10 = __fmul_rn(fy, __fsub_rn(1.f, fx));
  const float w11 = __fmul_rn(fy, fx);
  float acc = __fmul_rn(tap(iy, ix), w00);
  acc = __fadd_rn(acc, __fmul_rn(tap(iy, ix + 1), w01));
  acc = __fadd_rn(acc, __fmul_rn(tap(iy + 1, ix), w10));
  acc = __fadd_rn(acc, __fmul_rn(tap(iy + 1, ix + 1), w11));
  return acc;
}

__device__ __forceinline__ double hypot_rn(double a, double b) {
  return sqrt(__dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b)));
}

// One frame of one pass. slot 0 / dir -1: backward-flow neighbours ("Forward Pass", :76-235);
// slot 1 / dir +1: forward-flow neighbours ("Backward Pass", :241-370). State of frame tn = t+dir was
// finalised by the previous launch.
__global__ void prop_step_kernel(const uint8_t* __restrict__ mask, const float* __restrict__ step,
                                 const float* __restrict__ back, int H, int W, int t, int tn, double thres,
                                 double* __restrict__ nn_y, double* __restrict__ nn_x, int* __restrict__ nn_t,
                                 uint8_t* __restrict__ have, double* __restrict__ cuv) {
  pdl_launch_dependents();
  pdl_wait();
  const int HW = H * W;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += gridDim.x * blockDim.x) {
    if (!mask[static_cast<long long>(t) * HW + p]) continue;
    const int y = p / W, x = p - y * W;
    const float ny = __fadd_rn(static_cast<float>(y), step[2 * p + 1]);
    const float nx = __fadd_rn(static_cast<float>(x), step[2 * p]);
    const int iy = __float2int_rn(ny), ix = __float2int_rn(nx);  // np.round: half to even
    const float ry = __fadd_rn(ny, remap_q32(back, H, W, 2, 1, nx, ny));
    const float rx = __fadd_rn(nx, remap_q32(back, H, W, 2, 0, nx, ny));
    const double diff = hypot_rn(__dsub_rn(static_cast<double>(ry), static_cast<double>(y)),
                                 __dsub_rn(static_cast<double>(rx), static_cast<double>(x)));
    if (!(diff < thres)) continue;
    if (!(iy >= 0 && iy < H - 1 && ix >= 0 && ix < W - 1)) continue;
    const double ua = fabs(static_cast<double>(__fsub_rn(rx, static_cast<float>(x))));
    const double va = fabs(static_cast<double>(__fsub_rn(ry, static_cast<float>(y))));
    const long long q = static_cast<long long>(tn) * HW + static_cast<long long>(iy) * W + ix;  // neighbour cell
    const long long o = static_cast<long long>(t) * HW + p;
    if (!mask[q]) {  // case 1: neighbour is a known pixel
      nn_y[o] = static_cast<double>(ny);
      nn_x[o] = static_cast<double>(nx);
      nn_t[o] = tn;
      have[o] = 1;
      cuv[2 * o] = ua;
      cuv[2 * o + 1] = va;
    } else if (have[q] == 1) {  // case 2: chain through a hole pixel that already has a neighbour
      const double ty = __dadd_rn(nn_y[q], __dsub_rn(static_cast<double>(ny), static_cast<double>(iy)));
      const double tx = __dadd_rn(nn_x[q], __dsub_rn(static_cast<double>(nx), static_cast<double>(ix)));
      const long long tyi = __double2ll_rn(ty), txi = __double2ll_rn(tx);
      if (tyi >= 0 && tyi < H - 1 && txi >= 0 && txi < W - 1) {
        nn_y[o] = ty;
        nn_x[o] = tx;
        nn_t[o] = nn_t[q];
        have[o] = 1;
        cuv[2 * o] = fmax(ua, fabs(cuv[2 * q]));
        cuv[2 * o + 1] = fmax(va, fabs(cuv[2 * q + 1]));
      }
    }
  }
}

// Ordered in-place interpolation (:378-435): every hole pixel whose neighbour lives in source frame s
// gathers the 3-channel gradients of frame s (already final) at its neighbour position.
__global__ void prop_gather_kernel(const uint8_t* __restrict__ mask, const double* __restrict__ nn_y,
                                   const double* __restrict__ nn_x, const int* __restrict__ nn_t, int N, int H,
                                   int W, int s, float* __restrict__ gx, float* __restrict__ gy) {
  pdl_launch_dependents();
  pdl_wait();
  const long long HW = static_cast<long long>(H) * W;
  const long long total = HW * N;
  const float* sx = gx + s * HW * 3;
  const float* sy = gy + s * HW * 3;
  for (long long o = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; o < total;
       o += static_cast<long long>(gridDim.x) * blockDim.x) {
    if (!mask[o] || nn_t[o] != s) continue;
    const float px = static_cast<float>(nn_x[o]), py = static_cast<float>(nn_y[o]);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      gx[o * 3 + c] = remap_q32(sx, H, W, 3, c, px, py);
      gy[o * 3 + c] = remap_q32(sy, H, W, 3, c, px, py);
    }
  }
}

// Confidence-weighted fusion of the two candidates (:440-532) + mask of pixels still to fill.
__global__ void prop_fuse_kernel(const uint8_t* __restrict__ mask, const uint8_t* __restrict__ have0,
                                 const uint8_t* __restrict__ have1, const double* __restrict__ cuv0,
                                 const double* __restrict__ cuv1, long long total, double alpha,
                                 const float* __restrict__ gxb, const float* __restrict__ gyb,
                                 const float* __restrict__ gxf, const float* __restrict__ gyf,
                                 float* __restrict__ gx, float* __restrict__ gy, uint8_t* __restrict__ tofill) {
  pdl_launch_dependents();
  pdl_wait();
  for (long long o = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; o < total;
       o += static_cast<long long>(gridDim.x) * blockDim.x) {
    const bool m = mask[o] != 0;
    const bool h0 = m && have0[o] == 1, h1 = m && have1[o] == 1;
    tofill[o] = (m && !h0 && !h1) ? 1 : 0;
    if (!h0 && !h1) continue;
    const double c0 = h0 ? exp(-hypot_rn(cuv0[2 * o], cuv0[2 * o + 1]) / alpha) : 0.0;
    const double c1 = h1 ? exp(-hypot_rn(cuv1[2 * o], cuv1[2 * o + 1]) / alpha) : 0.0;
    const double den = __dadd_rn(c0, c1);
    double w0, w1;
    if (den == 0.0) {
      const double cnt = (h0 ? 1.0 : 0.0) + (h1 ? 1.0 : 0.0);
      w0 = (h0 ? 1.0 : 0.0) / cnt;
      w1 = (h1 ? 1.0 : 0.0) / cnt;
    } else {
      w0 = c0 / den;
      w1 = c1 / den;
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      gx[o * 3 + c] = static_cast<float>(__dadd_rn(__dmul_rn(static_cast<double>(gxb[o * 3 + c]), w0),
                                                   __dmul_rn(static_cast<double>(gxf[o * 3 + c]), w1)));
      gy[o * 3 + c] = static_cast<float>(__dadd_rn(__dmul_rn(static_cast<double>(gyb[o * 3 + c]), w0),
                                                   __dmul_rn(static_cast<double>(gyf[o * 3 + c]), w1)));
    }
  }
}

}  // namespace fgt

using namespace fgt;

extern "C" int fgt_prop_step(const uint8_t* mask, const float* flow_step, const float* flow_back, int H, int W, int t,
                             int tn, double thres, double* nn_y, double* nn_x, int* nn_t, uint8_t* have, double* cuv,
                             fgt_stream_t stream) {
  FGT_REQUIRE(mask && flow_step && flow_back && nn_y && nn_x && nn_t && have && cuv, FGT_ERR_ARG, "prop_step: null");
  FGT_LAUNCH(prop_step_kernel, dim3(grid_stride(static_cast<long long>(H) * W, 256)), dim3(256), 0, stream, mask,
             flow_step, flow_back, H, W, t, tn, thres, nn_y, nn_x, nn_t, have, cuv);
  return FGT_OK;
}

extern "C" int fgt_prop_gather(const uint8_t* mask, const double* nn_y, const double* nn_x, const int* nn_t, int N,
                               int H, int W, int s, float* gx, float* gy, fgt_stream_t stream) {
  FGT_REQUIRE(mask && nn_y && nn_x && nn_t && gx && gy, FGT_ERR_ARG, "prop_gather: null");
  FGT_LAUNCH(prop_gather_kernel, dim3(grid_stride(static_cast<long long>(N) * H * W, 256)), dim3(256), 0, stream, mask,
             nn_y, nn_x, nn_t, N, H, W, s, gx, gy);
  return FGT_OK;
}

extern "C" int fgt_prop_fuse(const uint8_t* mask, const uint8_t* have0, const uint8_t* have1, const double* cuv0,
                             const double* cuv1, int N, int H, int W, double alpha, const float* gx_bn,
                             const float* gy_bn, const float* gx_fn, const float* gy_fn, float* gx, float* gy,
                             uint8_t* tofill, fgt_stream_t stream) {
  FGT_REQUIRE(mask && have0 && have1 && cuv0 && cuv1 && gx && gy && tofill, FGT_ERR_ARG, "prop_fuse: null");
  const long long total = static_cast<long long>(N) * H * W;
  FGT_LAUNCH(prop_fuse_kernel, dim3(grid_stride(total, 256)), dim3(256), 0, stream, mask, have0, have1, cuv0, cuv1,
             total, alpha, gx_bn, gy_bn, gx_fn, gy_fn, gx, gy, tofill);
  return FGT_OK;
}
