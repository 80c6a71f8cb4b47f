// The FGT stage's window loop around Model.forward (tool/video_inpainting.py:686-745), device-resident:
//   fgt_plane_max      : per (frame, channel) maximum of the completed flows          (norm_flows :402-407)
//   fgt_window_gather  : one window's model inputs from the clip tensors               (:719-722 + :695,:706-707)
//                        masked = (frame*2 - 1) * (1 - mask), flow / flow_max, mask, frames picked by id
//   fgt_window_compose : model output -> uint8-valued composite, merged into the clip  (:725-741)
//                        comp = u8((out+1)/2*255) * mask + u8(frame*255) * (1 - mask);
//                        first visit: stored, later visits: 0.5 * previous + 0.5 * comp
//   fgt_comp_to_u8     : final astype(np.uint8)                                         (:745)
// The reference does all of this on the host with one .cpu() round trip per window and per frame (:726-733).
// Every float operation is the IEEE single-precision operation the reference performs, in the same order
// (explicit _rn intrinsics: no FMA contraction), so given the same model output the composite is bit-identical.
// HBM-bound streaming kernels: thread = pixel (all channels), grid-stride.
#include "common.h"

namespace fgt {

// torch.max's maximum, in any reduction order: a NaN anywhere gives NaN (fmaxf would drop it); +0 ranks above -0
// (torch's own sign of a zero maximum depends on its reduction order).
__device__ __forceinline__ float max_nan(float a, float b) {
  if (isnan(a) || isnan(b)) return __int_as_float(0x7fffffff);
  return (a > b || (a == b && !signbit(a))) ? a : b;
}

__global__ void plane_max_kernel(const float* __restrict__ x, long long plane, float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[8];
  const float* p = x + static_cast<long long>(blockIdx.x) * plane;
  float m = -INFINITY;
  for (long long i = threadIdx.x; i < plane; i += blockDim.x) m = max_nan(m, p[i]);
  for (int o = 16; o > 0; o >>= 1) m = max_nan(m, __shfl_down_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x < 32) {
    m = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : -INFINITY;
    for (int o = 4; o > 0; o >>= 1) m = max_nan(m, __shfl_down_sync(0xffffffffu, m, o));
    if (threadIdx.x == 0) out[blockIdx.x] = m;
  }
}

// frames [N,3,H,W] in [0,1], masks [N,H,W] uint8, flows [N,2,H,W], fmax [N,2]; ids [t] frame ids of the window.
// out_frames [t,3,H,W], out_flows [t,2,H,W], out_masks [t,1,H,W] (float).
__global__ void window_gather_kernel(const float* __restrict__ frames, const unsigned char* __restrict__ masks,
                                     const float* __restrict__ flows, const float* __restrict__ fmax,
                                     const int* __restrict__ ids, int t, long long HW, float* __restrict__ out_frames,
                                     float* __restrict__ out_flows, float* __restrict__ out_masks) {
  pdl_launch_dependents();
  pdl_wait();
  const long long total = static_cast<long long>(t) * HW;
  for (long long g = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; g < total;
       g += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int j = static_cast<int>(g / HW);
    const long long p = g - j * HW;
    const int id = ids[j];
    const float m = masks[id * HW + p] ? 1.0f : 0.0f;
    const float keep = __fsub_rn(1.0f, m);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float normed = __fsub_rn(__fmul_rn(frames[(id * 3LL + c) * HW + p], 2.0f), 1.0f);   // frames * 2 - 1 (:695)
      out_frames[(j * 3LL + c) * HW + p] = __fmul_rn(normed, keep);                              // * (1 - mask) (:721)
    }
#pragma unroll
    for (int c = 0; c < 2; ++c)
      out_flows[(j * 2LL + c) * HW + p] = __fdiv_rn(flows[(id * 2LL + c) * HW + p], fmax[id * 2 + c]);
    out_masks[j * HW + p] = m;
  }
}

__device__ __forceinline__ float as_u8(float v) {   // numpy float32 -> uint8 for in-range values: truncation
  return static_cast<float>(static_cast<unsigned char>(static_cast<int>(v)));
}

// filled [t,3,H,W] (model output in [-1,1]); the first k window frames are composed into comp [N,H,W,3] (float,
// uint8-valued until averaged). first[i] != 0: frame ids[i] has not been visited before.
__global__ void window_compose_kernel(const float* __restrict__ filled, const float* __restrict__ frames,
                                      const unsigned char* __restrict__ masks, const int* __restrict__ ids,
                                      const unsigned char* __restrict__ first, int k, long long HW,
                                      float* __restrict__ comp) {
  pdl_launch_dependents();
  pdl_wait();
  const long long total = static_cast<long long>(k) * HW;
  for (long long g = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; g < total;
       g += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int j = static_cast<int>(g / HW);
    const long long p = g - j * HW;
    const int id = ids[j];
    const float m = masks[id * HW + p] ? 1.0f : 0.0f;
    const float keep = __fsub_rn(1.0f, m);
    const bool fresh = first[j] != 0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float o = filled[(j * 3LL + c) * HW + p];
      const float a = as_u8(__fmul_rn(__fmul_rn(__fadd_rn(o, 1.0f), 0.5f), 255.0f));    // ((out + 1) / 2) * 255 (:725-726)
      const float b = as_u8(__fmul_rn(frames[(id * 3LL + c) * HW + p], 255.0f));          // frame * 255 (:729)
      const float v = __fadd_rn(__fmul_rn(a, m), __fmul_rn(b, keep));                     // (:731-733)
      float* dst = comp + (id * HW + p) * 3 + c;
      *dst = fresh ? v : __fadd_rn(__fmul_rn(*dst, 0.5f), __fmul_rn(v, 0.5f));            // (:734-741)
    }
  }
}

__global__ void comp_to_u8_kernel(const float* __restrict__ comp, long long total, unsigned char* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  for (long long g = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; g < total;
       g += static_cast<long long>(gridDim.x) * blockDim.x)
    out[g] = static_cast<unsigned char>(static_cast<int>(comp[g]));
}

}  // namespace fgt

using namespace fgt;

extern "C" int fgt_plane_max(const float* x, int planes, long long plane_size, float* out, fgt_stream_t stream) {
  FGT_REQUIRE(x && out && planes >= 1 && plane_size >= 1, FGT_ERR_ARG, "plane_max: bad argument");
  FGT_LAUNCH(plane_max_kernel, dim3(planes), dim3(256), 0, stream, x, plane_size, out);
  return FGT_OK;
}

extern "C" int fgt_window_gather(const float* frames, const unsigned char* masks, const float* flows, const float* fmax,
                                 const int* ids, int t, int H, int W, float* out_frames, float* out_flows,
                                 float* out_masks, fgt_stream_t stream) {
  FGT_REQUIRE(frames && masks && flows && fmax && ids && out_frames && out_flows && out_masks && t >= 1 && H >= 1 && W >= 1,
              FGT_ERR_ARG, "window_gather: bad argument");
  const long long HW = static_cast<long long>(H) * W;
  FGT_LAUNCH(window_gather_kernel, dim3(grid_stride(t * HW, 256)), dim3(256), 0, stream, frames, masks, flows, fmax,
             ids, t, HW, out_frames, out_flows, out_masks);
  return FGT_OK;
}

extern "C" int fgt_window_compose(const float* filled, const float* frames, const unsigned char* masks, const int* ids,
                                  const unsigned char* first, int k, int H, int W, float* comp, fgt_stream_t stream) {
  FGT_REQUIRE(filled && frames && masks && ids && first && comp && k >= 1 && H >= 1 && W >= 1, FGT_ERR_ARG,
              "window_compose: bad argument");
  const long long HW = static_cast<long long>(H) * W;
  FGT_LAUNCH(window_compose_kernel, dim3(grid_stride(k * HW, 256)), dim3(256), 0, stream, filled, frames, masks, ids,
             first, k, HW, comp);
  return FGT_OK;
}

extern "C" int fgt_comp_to_u8(const float* comp, long long total, unsigned char* out, fgt_stream_t stream) {
  FGT_REQUIRE(comp && out && total >= 1, FGT_ERR_ARG, "comp_to_u8: bad argument");
  FGT_LAUNCH(comp_to_u8_kernel, dim3(grid_stride(total, 256)), dim3(256), 0, stream, comp, total, out);
  return FGT_OK;
}
