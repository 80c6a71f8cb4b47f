// The tensor glue of FGT's validation (FGT/networks/network.py:258-352, Network._validate) on the device:
//   fgt_valid_flow_scale : resized flows [B,H,W,2] in place: u = u / pre_w * w, v = v / pre_h * h  (read_flows :431-432)
//   fgt_valid_inputs     : frames uint8 [t,H,W,3], masks uint8 [t,H,W] (0 / 1) -> frames [t,3,H,W] = x / 127.5 - 1
//                          (:296), masked [t,3,H,W] = frames * (1 - mask) (:306), masks [t,1,H,W] float (:291)
//   fgt_valid_norm_flows : out[i] = flows[i] / fmax[plane of i] (norm_flows :80-84; fmax from fgt_plane_max)
//   fgt_valid_score      : comp = out * m + frames * (1 - m) (:310), then clip((x + 1) / 2 * 255, 0, 255) as uint8 of
//                          comp and of the frames, NHWC [t,H,W,3] (metrics_calc :357-361)
// Every float operation is the IEEE single-precision operation the reference performs, in its order (explicit _rn
// intrinsics: no FMA contraction), so the outputs are bit-identical given the same inputs. HBM-bound streaming
// kernels: thread = pixel (all channels), grid-stride.
#include "common.h"

namespace fgt {
namespace valid {

__global__ void flow_scale_kernel(float2* __restrict__ flow, long long pixels, float pre_w, float w, float pre_h,
                                  float h) {
  pdl_launch_dependents();
  pdl_wait();
  for (long long g = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; g < pixels;
       g += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float2 f = flow[g];
    flow[g] = make_float2(__fmul_rn(__fdiv_rn(f.x, pre_w), w), __fmul_rn(__fdiv_rn(f.y, pre_h), h));
  }
}

__global__ void inputs_kernel(const unsigned char* __restrict__ frames, const unsigned char* __restrict__ masks,
                              long long total, long long HW, float* __restrict__ out_frames,
                              float* __restrict__ out_masked, float* __restrict__ out_masks) {
  pdl_launch_dependents();
  pdl_wait();
  for (long long g = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; g < total;
       g += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long j = g / HW, p = g - j * HW;
    const float m = masks[g] ? 1.0f : 0.0f;
    const float keep = __fsub_rn(1.0f, m);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float f = __fsub_rn(__fdiv_rn(static_cast<float>(frames[g * 3 + c]), 127.5f), 1.0f);
      out_frames[(j * 3 + c) * HW + p] = f;
      out_masked[(j * 3 + c) * HW + p] = __fmul_rn(f, keep);
    }
    out_masks[g] = m;
  }
}

__global__ void norm_flows_kernel(const float* __restrict__ flows, const float* __restrict__ fmax, long long total,
                                  long long plane, float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  for (long long g = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; g < total;
       g += static_cast<long long>(gridDim.x) * blockDim.x)
    out[g] = __fdiv_rn(flows[g], fmax[g / plane]);
}

// numpy's float32 clip to [0, 255] then astype(uint8): truncation; NaN (the reference's would be undefined) gives 0
__device__ __forceinline__ unsigned char to_u8(float x) {
  const float v = __fmul_rn(__fdiv_rn(__fadd_rn(x, 1.0f), 2.0f), 255.0f);
  return static_cast<unsigned char>(static_cast<int>(fminf(fmaxf(v, 0.0f), 255.0f)));
}

__global__ void score_kernel(const float* __restrict__ filled, const float* __restrict__ frames,
                             const float* __restrict__ masks, long long total, long long HW,
                             unsigned char* __restrict__ comp_u8, unsigned char* __restrict__ frames_u8) {
  pdl_launch_dependents();
  pdl_wait();
  for (long long g = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; g < total;
       g += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long j = g / HW, p = g - j * HW;
    const float m = masks[g];
    const float keep = __fsub_rn(1.0f, m);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const long long i = (j * 3 + c) * HW + p;
      const float f = frames[i];
      comp_u8[g * 3 + c] = to_u8(__fadd_rn(__fmul_rn(filled[i], m), __fmul_rn(f, keep)));
      frames_u8[g * 3 + c] = to_u8(f);
    }
  }
}

}  // namespace valid
}  // namespace fgt

using namespace fgt;
using namespace fgt::valid;

extern "C" int fgt_valid_flow_scale(float* flow, long long pixels, float pre_w, float w, float pre_h, float h,
                                    fgt_stream_t stream) {
  FGT_REQUIRE(flow && pixels >= 1, FGT_ERR_ARG, "valid_flow_scale: bad argument");
  FGT_REQUIRE(reinterpret_cast<uintptr_t>(flow) % 8 == 0, FGT_ERR_ARG, "valid_flow_scale: flow is not 8-byte aligned");
  FGT_LAUNCH(flow_scale_kernel, dim3(grid_stride(pixels, 256)), dim3(256), 0, stream, reinterpret_cast<float2*>(flow),
             pixels, pre_w, w, pre_h, h);
  return FGT_OK;
}

extern "C" int fgt_valid_inputs(const unsigned char* frames, const unsigned char* masks, int t, int H, int W,
                                float* out_frames, float* out_masked, float* out_masks, fgt_stream_t stream) {
  FGT_REQUIRE(frames && masks && out_frames && out_masked && out_masks && t >= 1 && H >= 1 && W >= 1, FGT_ERR_ARG,
              "valid_inputs: bad argument");
  const long long HW = static_cast<long long>(H) * W;
  FGT_LAUNCH(inputs_kernel, dim3(grid_stride(t * HW, 256)), dim3(256), 0, stream, frames, masks, t * HW, HW,
             out_frames, out_masked, out_masks);
  return FGT_OK;
}

extern "C" int fgt_valid_norm_flows(const float* flows, const float* fmax, int planes, long long plane_size, float* out,
                                    fgt_stream_t stream) {
  FGT_REQUIRE(flows && fmax && out && planes >= 1 && plane_size >= 1, FGT_ERR_ARG, "valid_norm_flows: bad argument");
  const long long total = planes * plane_size;
  FGT_LAUNCH(norm_flows_kernel, dim3(grid_stride(total, 256)), dim3(256), 0, stream, flows, fmax, total, plane_size,
             out);
  return FGT_OK;
}

extern "C" int fgt_valid_score(const float* filled, const float* frames, const float* masks, int t, int H, int W,
                               unsigned char* comp_u8, unsigned char* frames_u8, fgt_stream_t stream) {
  FGT_REQUIRE(filled && frames && masks && comp_u8 && frames_u8 && t >= 1 && H >= 1 && W >= 1, FGT_ERR_ARG,
              "valid_score: bad argument");
  const long long HW = static_cast<long long>(H) * W;
  FGT_LAUNCH(score_kernel, dim3(grid_stride(t * HW, 256)), dim3(256), 0, stream, filled, frames, masks, t * HW, HW,
             comp_u8, frames_u8);
  return FGT_OK;
}
