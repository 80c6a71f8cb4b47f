// Device-side versions of the driver's mask / resize glue (SURVEY 8f rank 3; tool/video_inpainting.py:264-268, 546-561,
// 637): scipy.ndimage.binary_dilation (default cross structuring element, `iterations` repeats), binary_fill_holes,
// cv2.resize INTER_NEAREST on uint8 masks and INTER_LINEAR on float32 images (= F.interpolate bilinear with
// align_corners=False). Byte / index work: bit-exact for the masks; the bilinear kernel performs OpenCV's float32
// operations in OpenCV's order (explicit _rn intrinsics, no FMA contraction), so it is bit-identical to cv2.resize on
// the driver's two-channel flows. HBM-bound helpers: one thread per output element, coalesced along x.
#include "common.h"
#include "ptx.cuh"

namespace fgt {

// One pass of binary dilation with the 3x3 cross (scipy's generate_binary_structure(2, 1)), border value 0.
__global__ void dilate_cross_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int B, int H, int W) {
  const long long total = static_cast<long long>(B) * H * W;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(i % W);
    const int y = static_cast<int>((i / W) % H);
    uint8_t v = in[i];
    if (!v) {
      if (x > 0 && in[i - 1]) v = 1;
      else if (x + 1 < W && in[i + 1]) v = 1;
      else if (y > 0 && in[i - W]) v = 1;
      else if (y + 1 < H && in[i + W]) v = 1;
    }
    out[i] = v ? 1 : 0;
  }
}

// binary_fill_holes: the complement of the background component(s) touching the image border (4-connectivity, the
// default structure). reach = background pixels known to be connected to the border; one pass = for every row a
// left-to-right and right-to-left propagation, then for every column a top-down and bottom-up propagation. Sweeps
// travel whole runs at once, so convex-ish holes settle in 2-3 passes; `changed` reports whether another pass is needed.
__global__ void fill_rows_kernel(const uint8_t* __restrict__ fg, uint8_t* __restrict__ reach, int B, int H, int W,
                                 int* __restrict__ changed) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;  // (image, row)
  if (r >= B * H) return;
  const int y = r % H;
  const long long base = static_cast<long long>(r) * W;
  bool ch = false;
  uint8_t prev = 0;
  for (int x = 0; x < W; ++x) {
    const long long i = base + x;
    uint8_t v = reach[i];
    if (!fg[i]) {
      const bool border = (x == 0) || (y == 0) || (y == H - 1) || (x == W - 1);
      if (!v && (prev || border)) { v = 1; reach[i] = 1; ch = true; }
    } else {
      v = 0;
    }
    prev = v;
  }
  prev = 0;
  for (int x = W - 1; x >= 0; --x) {
    const long long i = base + x;
    uint8_t v = reach[i];
    if (!fg[i]) {
      if (!v && prev) { v = 1; reach[i] = 1; ch = true; }
    } else {
      v = 0;
    }
    prev = v;
  }
  if (ch) *changed = 1;
}

__global__ void fill_cols_kernel(const uint8_t* __restrict__ fg, uint8_t* __restrict__ reach, int B, int H, int W,
                                 int* __restrict__ changed) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;  // (image, column): adjacent threads = adjacent columns
  if (c >= B * W) return;
  const int b = c / W, x = c - b * W;
  const long long base = static_cast<long long>(b) * H * W + x;
  bool ch = false;
  uint8_t prev = 0;
  for (int y = 0; y < H; ++y) {
    const long long i = base + static_cast<long long>(y) * W;
    uint8_t v = reach[i];
    if (!fg[i]) {
      if (!v && prev) { v = 1; reach[i] = 1; ch = true; }
    } else {
      v = 0;
    }
    prev = v;
  }
  prev = 0;
  for (int y = H - 1; y >= 0; --y) {
    const long long i = base + static_cast<long long>(y) * W;
    uint8_t v = reach[i];
    if (!fg[i]) {
      if (!v && prev) { v = 1; reach[i] = 1; ch = true; }
    } else {
      v = 0;
    }
    prev = v;
  }
  if (ch) *changed = 1;
}

__global__ void fill_finish_kernel(const uint8_t* __restrict__ reach, uint8_t* __restrict__ out, long long total) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    out[i] = reach[i] ? 0 : 1;  // everything not reachable from the border: the objects and their holes
}

// cv2.resize(..., interpolation=INTER_NEAREST) on uint8 [B,H,W(,C)]: sx = min(floor(dx * W / OW), W - 1).
__global__ void resize_nearest_u8_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int B, int H, int W,
                                         int C, int OH, int OW) {
  // OpenCV computes the step as 1 / (dst / src) in double (resize.cpp: inv_scale = dsize / ssize; ifx = 1 / inv_scale)
  const double fx = 1.0 / (static_cast<double>(OW) / W), fy = 1.0 / (static_cast<double>(OH) / H);
  const long long total = static_cast<long long>(B) * OH * OW * C;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % C);
    const long long t = i / C;
    const int dx = static_cast<int>(t % OW);
    const int dy = static_cast<int>((t / OW) % OH);
    const long long b = t / (static_cast<long long>(OW) * OH);
    const int sx = min(static_cast<int>(floor(dx * fx)), W - 1);
    const int sy = min(static_cast<int>(floor(dy * fy)), H - 1);
    out[i] = in[((b * H + sy) * W + sx) * C + c];
  }
}

// cv2.resize INTER_LINEAR on float32 [B,H,W,C] (channels last), as OpenCV's resizeGeneric_ computes it: source
// coordinate fp32((d + 0.5) * scale - 0.5) in double, s = floor, f = coordinate - s. Along x the weight collapses onto
// the edge sample (s < 0 -> (0, f = 0); s >= W-1 -> (W-1, f = 0)); along y f is kept and only the two rows are clamped
// to [0, H-1] (so an edge row is r * (1 - f) + r * f). Each row is a0 * left + a1 * right, then (1 - fy) * r0 + fy * r1,
// every product and sum rounded to float32 (no FMA). When H = 2 OH and W = 2 OW exactly, cv2 switches to INTER_AREA:
// (0 + (((a + b) + c) + d)) * 0.25 of the 2x2 block, a b the upper row. cv2 hands C = 1, 3 and 4 to IPP, whose arithmetic
// differs; the driver resizes flows (C = 2). With `nchw` (planes instead of interleaved channels) the arithmetic is
// ATen's CPU kernel as built with FMA (UpSample.h, align_corners = False): fp32 fma(scale, d + 0.5, -0.5), negative
// -> 0, s = trunc, the second tap clamped; rows fma(a0, left, a1 * right), then fma(1 - fy, r0, fy * r1). That is
// F.interpolate on the CPU bit for bit except on small images, where ATen takes a scalar path (within 1e-7 relative).
__global__ void resize_bilinear_f32_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int H, int W,
                                           int C, int OH, int OW, int nchw, float out_scale_c0, float out_scale_c1) {
  const double sxs = 1.0 / (static_cast<double>(OW) / W), sys = 1.0 / (static_cast<double>(OH) / H);
  const bool area2 = !nchw && W == 2 * OW && H == 2 * OH;
  const long long total = static_cast<long long>(B) * OH * OW * C;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    int c, dx, dy;
    long long b;
    if (nchw) {
      dx = static_cast<int>(i % OW);
      dy = static_cast<int>((i / OW) % OH);
      c = static_cast<int>((i / (static_cast<long long>(OW) * OH)) % C);
      b = i / (static_cast<long long>(OW) * OH * C);
    } else {
      c = static_cast<int>(i % C);
      const long long t = i / C;
      dx = static_cast<int>(t % OW);
      dy = static_cast<int>((t / OW) % OH);
      b = t / (static_cast<long long>(OW) * OH);
    }
    auto at = [&](int y, int x) -> float {
      return nchw ? in[((b * C + c) * H + y) * W + x] : in[((b * H + y) * W + x) * C + c];
    };
    float v;
    if (area2) {
      const int x0 = 2 * dx, y0 = 2 * dy;
      v = __fadd_rn(__fadd_rn(__fadd_rn(at(y0, x0), at(y0, x0 + 1)), at(y0 + 1, x0)), at(y0 + 1, x0 + 1));
      v = __fmul_rn(__fadd_rn(0.f, v), 0.25f);
    } else {
      float fx, fy;
      int sx, sy, sy0, sy1;
      if (nchw) {
        const float scx = static_cast<float>(W) / OW, scy = static_cast<float>(H) / OH;
        fx = fmaxf(__fmaf_rn(scx, __fadd_rn(static_cast<float>(dx), 0.5f), -0.5f), 0.f);
        fy = fmaxf(__fmaf_rn(scy, __fadd_rn(static_cast<float>(dy), 0.5f), -0.5f), 0.f);
        sx = min(static_cast<int>(fx), W - 1);
        sy0 = min(static_cast<int>(fy), H - 1);
        fx = __fsub_rn(fx, static_cast<float>(sx));
        fy = __fsub_rn(fy, static_cast<float>(sy0));
        sy1 = min(sy0 + 1, H - 1);
      } else {
        fx = static_cast<float>(__dsub_rn(__dmul_rn(dx + 0.5, sxs), 0.5));
        sx = static_cast<int>(floorf(fx));
        fx = __fsub_rn(fx, static_cast<float>(sx));
        if (sx < 0) { sx = 0; fx = 0.f; }
        if (sx >= W - 1) { sx = W - 1; fx = 0.f; }
        fy = static_cast<float>(__dsub_rn(__dmul_rn(dy + 0.5, sys), 0.5));
        sy = static_cast<int>(floorf(fy));
        fy = __fsub_rn(fy, static_cast<float>(sy));
        sy0 = min(max(sy, 0), H - 1);
        sy1 = min(max(sy + 1, 0), H - 1);
      }
      const int sx1 = min(sx + 1, W - 1);
      const float a0 = __fsub_rn(1.f, fx), a1 = fx, b0 = __fsub_rn(1.f, fy);
      if (nchw) {   // ATen's CPU kernel as built with FMA: fma(a0, left, a1 * right), likewise vertically
        const float r0 = __fmaf_rn(at(sy0, sx), a0, __fmul_rn(at(sy0, sx1), a1));
        const float r1 = __fmaf_rn(at(sy1, sx), a0, __fmul_rn(at(sy1, sx1), a1));
        v = __fmaf_rn(r0, b0, __fmul_rn(r1, fy));
      } else {
        const float r0 = __fadd_rn(__fmul_rn(at(sy0, sx), a0), __fmul_rn(at(sy0, sx1), a1));
        const float r1 = __fadd_rn(__fmul_rn(at(sy1, sx), a0), __fmul_rn(at(sy1, sx1), a1));
        v = __fadd_rn(__fmul_rn(r0, b0), __fmul_rn(r1, fy));
      }
    }
    if (c == 0) v = __fmul_rn(v, out_scale_c0);
    else if (c == 1) v = __fmul_rn(v, out_scale_c1);
    out[i] = v;
  }
}

}  // namespace fgt

using namespace fgt;

extern "C" int fgt_binary_dilate(const unsigned char* in, int B, int H, int W, int iterations, unsigned char* tmp,
                                 unsigned char* out, fgt_stream_t stream) {
  FGT_REQUIRE(in && tmp && out && B >= 1 && H >= 1 && W >= 1 && iterations >= 1, FGT_ERR_ARG, "binary_dilate: bad argument");
  FGT_REQUIRE(in != out && in != tmp && tmp != out, FGT_ERR_ARG, "binary_dilate: buffers must not alias");
  const long long total = static_cast<long long>(B) * H * W;
  // ping-pong so that the last pass lands in `out`
  const unsigned char* src = in;
  for (int it = 0; it < iterations; ++it) {
    unsigned char* dst = ((iterations - 1 - it) % 2 == 0) ? out : tmp;
    FGT_LAUNCH(dilate_cross_kernel, dim3(grid_stride(total, 256)), dim3(256), 0, stream, src, dst, B, H, W);
    src = dst;
  }
  return FGT_OK;
}

extern "C" int fgt_fill_holes_init(const unsigned char* fg, int B, int H, int W, unsigned char* reach, fgt_stream_t stream) {
  FGT_REQUIRE(fg && reach && B >= 1 && H >= 1 && W >= 1, FGT_ERR_ARG, "fill_holes: bad argument");
  FGT_CUDA(cudaMemsetAsync(reach, 0, static_cast<size_t>(B) * H * W, stream));
  return FGT_OK;
}

extern "C" int fgt_fill_holes_pass(const unsigned char* fg, int B, int H, int W, unsigned char* reach, int* changed,
                                   int passes, fgt_stream_t stream) {
  FGT_REQUIRE(fg && reach && changed && passes >= 1, FGT_ERR_ARG, "fill_holes: bad argument");
  FGT_CUDA(cudaMemsetAsync(changed, 0, sizeof(int), stream));
  for (int p = 0; p < passes; ++p) {
    FGT_LAUNCH(fill_rows_kernel, dim3((B * H + 63) / 64), dim3(64), 0, stream, fg, reach, B, H, W, changed);
    FGT_LAUNCH(fill_cols_kernel, dim3((B * W + 63) / 64), dim3(64), 0, stream, fg, reach, B, H, W, changed);
  }
  return FGT_OK;
}

extern "C" int fgt_fill_holes_finish(const unsigned char* reach, int B, int H, int W, unsigned char* out, fgt_stream_t stream) {
  FGT_REQUIRE(reach && out, FGT_ERR_ARG, "fill_holes: bad argument");
  const long long total = static_cast<long long>(B) * H * W;
  FGT_LAUNCH(fill_finish_kernel, dim3(grid_stride(total, 256)), dim3(256), 0, stream, reach, out, total);
  return FGT_OK;
}

extern "C" int fgt_resize_nearest_u8(const unsigned char* in, int B, int H, int W, int C, int OH, int OW, unsigned char* out,
                                     fgt_stream_t stream) {
  FGT_REQUIRE(in && out && B >= 1 && H >= 1 && W >= 1 && C >= 1 && OH >= 1 && OW >= 1, FGT_ERR_ARG, "resize_nearest: bad argument");
  const long long total = static_cast<long long>(B) * OH * OW * C;
  FGT_LAUNCH(resize_nearest_u8_kernel, dim3(grid_stride(total, 256)), dim3(256), 0, stream, in, out, B, H, W, C, OH,
             OW);
  return FGT_OK;
}

extern "C" int fgt_resize_bilinear_f32(const float* in, int B, int H, int W, int C, int OH, int OW, int nchw, float scale_c0,
                                       float scale_c1, float* out, fgt_stream_t stream) {
  FGT_REQUIRE(in && out && B >= 1 && H >= 1 && W >= 1 && C >= 1 && OH >= 1 && OW >= 1, FGT_ERR_ARG, "resize_bilinear: bad argument");
  const long long total = static_cast<long long>(B) * OH * OW * C;
  FGT_LAUNCH(resize_bilinear_f32_kernel, dim3(grid_stride(total, 256)), dim3(256), 0, stream, in, out, B, H, W, C, OH,
             OW, nchw, scale_c0, scale_c1);
  return FGT_OK;
}
