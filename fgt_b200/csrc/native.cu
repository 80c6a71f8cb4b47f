// Native-resolution output: the pipeline's working-resolution result `comp` [B,cH,cW,3] upscaled to the frames' size
// H x W and pasted into the original frames inside a feathered band around the mask. The definition, written once, is
// oracle/native_oracle.py; every step is integer arithmetic, so the kernels equal it bit for bit:
//   c   = number of pixels of D (the hole, cross-dilated r + 2k times by fgt_binary_dilate) in the (2k+1)^2 window
//         around the pixel, the edge replicated outside the image, A = (2k+1)^2;
//   up  = cv2 INTER_LINEAR fixed-point bilinear of comp (11-bit weights; horizontal pass exact, vertical pass rounded
//         as cv2's vectorised 8U code: (((b0*(S0>>4))>>16) + ((b1*(S1>>4))>>16) + 2) >> 2);
//   out = (c*up + (A-c)*frame + A/2) / A per channel.
// count_rows / count_cols: the two separable box sums of c (one thread per pixel, coalesced along x). composite: one
// thread per output pixel, all three channels; c = 0 copies the frame pixel without touching comp, c = A writes up
// without reading the frame. HBM-bound: 3 B of frame in, 3 B out and 2 B of c per pixel; comp is tiny and read-only.
#include "common.h"

namespace fgt {
namespace native {

constexpr int kMaxHalf = 127;  // A = (2k+1)^2 must fit the uint16 count; the u8 row sums hold up to 2k+1 = 255

// cv2.resize INTER_LINEAR: source coordinate float32((d + 0.5) * scale - 0.5), scale = 1 / (dst / src) in double as
// cv2 computes it; i = floor, f = x - i; clamped to the edge with f = 0; 11-bit weights round-half-even of 2048*(1-f)
// and 2048*f. Explicit _rn intrinsics: no contraction into FMA, so the numbers are numpy's.
__device__ __forceinline__ void axis_tap(int d, double scale, int src, int& i0, int& i1, int& w0, int& w1) {
  const float x = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn(static_cast<double>(d), 0.5), scale), 0.5));
  int i = static_cast<int>(floorf(x));
  float f = __fsub_rn(x, static_cast<float>(i));
  if (i < 0) { i = 0; f = 0.f; }
  if (i >= src - 1) { i = src - 1; f = 0.f; }
  i0 = i;
  i1 = min(i + 1, src - 1);
  w0 = __float2int_rn(__fmul_rn(2048.f, __fsub_rn(1.f, f)));
  w1 = __float2int_rn(__fmul_rn(2048.f, f));
}

// rs[m,y,x] = sum of D[m,y,clamp(x-k..x+k)]: positions outside the image count as the edge pixel
__global__ void count_rows_kernel(const uint8_t* __restrict__ D, uint8_t* __restrict__ rs, long long total, int W, int k) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(i % W);
    const uint8_t* row = D + (i - x);
    int s = 0;
    for (int d = -k; d <= k; ++d) s += row[min(max(x + d, 0), W - 1)] != 0;
    rs[i] = static_cast<uint8_t>(s);
  }
}

// c[m,y,x] = sum of rs[m,clamp(y-k..y+k),x]
__global__ void count_cols_kernel(const uint8_t* __restrict__ rs, uint16_t* __restrict__ c, long long total, int H, int W,
                                  int k) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long hw = static_cast<long long>(H) * W;
    const long long yx = i % hw;
    const int y = static_cast<int>(yx / W);
    const uint8_t* col = rs + (i - static_cast<long long>(y) * W);
    int s = 0;
    for (int d = -k; d <= k; ++d) s += col[static_cast<long long>(min(max(y + d, 0), H - 1)) * W];
    c[i] = static_cast<uint16_t>(s);
  }
}

__global__ void composite_kernel(const uint8_t* __restrict__ comp, int cH, int cW, const uint8_t* __restrict__ frames,
                                 int B, int H, int W, const uint16_t* __restrict__ c, long long c_stride, int A,
                                 uint8_t* __restrict__ out) {
  const double sx = 1.0 / (static_cast<double>(W) / cW), sy = 1.0 / (static_cast<double>(H) / cH);
  const long long hw = static_cast<long long>(H) * W, total = hw * B;
  for (long long p = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; p < total;
       p += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long b = p / hw, yx = p - b * hw;
    const int n = c[b * c_stride + yx];
    const uint8_t* fr = frames + 3 * p;
    uint8_t* o = out + 3 * p;
    if (n == 0) {
      o[0] = fr[0]; o[1] = fr[1]; o[2] = fr[2];
      continue;
    }
    const int y = static_cast<int>(yx / W), x = static_cast<int>(yx - static_cast<long long>(y) * W);
    int x0, x1, a0, a1, y0, y1, b0, b1;
    axis_tap(x, sx, cW, x0, x1, a0, a1);
    axis_tap(y, sy, cH, y0, y1, b0, b1);
    const uint8_t* r0 = comp + (b * cH + y0) * cW * 3;
    const uint8_t* r1 = comp + (b * cH + y1) * cW * 3;
    const int keep = A - n;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const int s0 = a0 * __ldg(r0 + 3 * x0 + ch) + a1 * __ldg(r0 + 3 * x1 + ch);
      const int s1 = a0 * __ldg(r1 + 3 * x0 + ch) + a1 * __ldg(r1 + 3 * x1 + ch);
      int up = (((b0 * (s0 >> 4)) >> 16) + ((b1 * (s1 >> 4)) >> 16) + 2) >> 2;
      up = min(max(up, 0), 255);
      o[ch] = static_cast<uint8_t>(keep == 0 ? up : (n * up + keep * fr[ch] + A / 2) / A);
    }
  }
}

// Workspace: the uint16 counts of n_masks masks, then the uint8 row sums they are built from.
inline long long counts_bytes(int n_masks, int H, int W) { return 2LL * n_masks * H * W; }

}  // namespace native
}  // namespace fgt

using namespace fgt::native;

static int native_check(int n_masks, int H, int W, int k) {
  FGT_REQUIRE(n_masks >= 1 && H >= 1 && W >= 1, FGT_ERR_ARG, "native: empty size (%d masks of %dx%d)", n_masks, H, W);
  FGT_REQUIRE(k >= 1 && k <= kMaxHalf, FGT_ERR_ARG,
              "native: window half-width k = %d outside [1, %d]: A = (2k+1)^2 must fit the uint16 count", k, kMaxHalf);
  return FGT_OK;
}

extern "C" long long fgt_native_workspace(int n_masks, int H, int W, int k) {
  const int rc = native_check(n_masks, H, W, k);
  if (rc != FGT_OK) return rc;
  return counts_bytes(n_masks, H, W) + static_cast<long long>(n_masks) * H * W;
}

extern "C" int fgt_native_count(const unsigned char* dilated, int n_masks, int H, int W, int k, void* workspace,
                                long long workspace_bytes, fgt_stream_t stream) {
  FGT_REQUIRE(dilated && workspace, FGT_ERR_ARG, "native_count: null pointer");
  int rc = native_check(n_masks, H, W, k);
  if (rc != FGT_OK) return rc;
  const long long need = fgt_native_workspace(n_masks, H, W, k);
  FGT_REQUIRE(workspace_bytes >= need, FGT_ERR_ARG, "native_count: workspace of %lld bytes, %lld needed", workspace_bytes,
              need);
  const long long total = static_cast<long long>(n_masks) * H * W;
  uint16_t* c = static_cast<uint16_t*>(workspace);
  uint8_t* rs = static_cast<uint8_t*>(workspace) + counts_bytes(n_masks, H, W);
  FGT_LAUNCH(count_rows_kernel, dim3(fgt::grid_stride(total, 256)), dim3(256), 0, stream, dilated, rs, total, W, k);
  FGT_LAUNCH(count_cols_kernel, dim3(fgt::grid_stride(total, 256)), dim3(256), 0, stream, rs, c, total, H, W, k);
  return FGT_OK;
}

extern "C" int fgt_native_composite(const unsigned char* comp, int B, int cH, int cW, const unsigned char* frames, int H,
                                    int W, int C, int shared_mask, int k, const void* workspace,
                                    long long workspace_bytes, unsigned char* out, fgt_stream_t stream) {
  FGT_REQUIRE(comp && frames && workspace && out, FGT_ERR_ARG, "native_composite: null pointer");
  FGT_REQUIRE(frames != out && comp != out, FGT_ERR_ARG, "native_composite: out must not alias the inputs");
  FGT_REQUIRE(B >= 1 && cH >= 1 && cW >= 1, FGT_ERR_ARG, "native_composite: empty size (%d comp frames of %dx%d)", B, cH, cW);
  FGT_REQUIRE(C == 3, FGT_ERR_ARG, "native_composite: frames and comp must have 3 channels (got %d)", C);
  int rc = native_check(shared_mask ? 1 : B, H, W, k);
  if (rc != FGT_OK) return rc;
  const double s = fmax(static_cast<double>(H) / cH, static_cast<double>(W) / cW);
  FGT_REQUIRE(static_cast<int>(ceil(s)) == k, FGT_ERR_ARG,
              "native_composite: comp %dx%d is not the working size the counts were built for (frames %dx%d need "
              "k = %d, counts have k = %d)", cH, cW, H, W, static_cast<int>(ceil(s)), k);
  const long long need = fgt_native_workspace(shared_mask ? 1 : B, H, W, k);
  FGT_REQUIRE(workspace_bytes >= need, FGT_ERR_ARG, "native_composite: workspace of %lld bytes, %lld needed",
              workspace_bytes, need);
  const long long total = static_cast<long long>(B) * H * W;
  FGT_LAUNCH(composite_kernel, dim3(fgt::grid_stride(total, 256)), dim3(256), 0, stream, comp, cH, cW, frames, B, H, W,
             static_cast<const uint16_t*>(workspace), shared_mask ? 0LL : static_cast<long long>(H) * W,
             (2 * k + 1) * (2 * k + 1), out);
  return FGT_OK;
}
