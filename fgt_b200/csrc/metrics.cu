// Quality metrics of result frames against ground truth (FGT/metrics: psnr.py, ssim.py, calculate_metrics' L1 / L2),
// batched over N frames x C channels, all arithmetic in float64.
//
// tile kernel: one CTA per (frame, channel, 32x32 tile of SSIM's valid positions). It stages the 42x42 input patch
// (the tile plus the 5-pixel halo of the 11-tap window) in shared memory as float (uint8 and float32 values are exact
// there), runs the separable Gaussian over the five quantities a, b, a^2, b^2, ab in float64 (rows into shared memory,
// then columns in registers), evaluates the SSIM map and sums it. In the same pass it sums (a - b)^2 and |a - b| over
// the input pixels the tile owns (tiles partition the frame). The filtered images never leave the SM; the CTA writes
// three doubles to the workspace. reduce kernel: one warp per frame sums its tiles in a fixed order, so a frame's
// values depend on nothing but its own pixels.
// fp64 work per valid position and channel: 5 x 11 FMAs along rows (times 42/32 for the halo rows), 5 x 11 along
// columns and ~20 for the map, about 275 FLOPs.
#include "common.h"

namespace fgt {
namespace metrics {

constexpr int kTX = 32, kTY = 32;             // valid positions per tile
constexpr int kR = 5, kTaps = 2 * kR + 1;     // 11-tap window
constexpr int kIX = kTX + 2 * kR, kIY = kTY + 2 * kR;
constexpr int kSA = kIX + 1;                  // odd float stride: rows of the input patch hit distinct banks
constexpr int kSH = kTX + 1;                  // odd double stride for the row-filtered planes
constexpr int kP = 8;                         // outputs per thread along a row (row pass) / a column (column pass)
constexpr int kThreads = 128;
constexpr size_t kSmem = 2 * sizeof(float) * kIY * kSA + 5 * sizeof(double) * kIY * kSH;
static_assert(kTX * kTY / kP == kThreads, "column pass: one strip per thread");

struct Gauss {
  double g[kTaps];
};

template <typename T>
__device__ __forceinline__ float load_px(const T* p) { return static_cast<float>(__ldg(p)); }

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ws[((n * C + c) * tiles + tile) * 3 + {0, 1, 2}] = (sum of the SSIM map, sum d^2, sum |d|)
template <typename TA, typename TB>
__global__ void __launch_bounds__(kThreads) metrics_tile_kernel(const TA* __restrict__ a, const TB* __restrict__ b,
                                                                int H, int W, int C, Gauss gw, double* __restrict__ ws) {
  extern __shared__ __align__(16) unsigned char smem[];
  float* sa = reinterpret_cast<float*>(smem);
  float* sb = sa + kIY * kSA;
  double* sh = reinterpret_cast<double*>(sb + kIY * kSA);   // 5 planes [kIY][kSH]
  const int tid = threadIdx.x;
  const int ntx = gridDim.x, nty = gridDim.y;
  const int n = blockIdx.z / C, c = blockIdx.z - n * C;
  const int x0 = blockIdx.x * kTX, y0 = blockIdx.y * kTY;   // first input column / row of the patch
  const long long frame = static_cast<long long>(n) * H * W;
  // owned input pixels: [x0 + 5, x0 + 37) inside, widened to the frame's edge by the first and last tile
  const int ox0 = blockIdx.x == 0 ? 0 : x0 + kR, ox1 = blockIdx.x == ntx - 1 ? W : x0 + kR + kTX;
  const int oy0 = blockIdx.y == 0 ? 0 : y0 + kR, oy1 = blockIdx.y == nty - 1 ? H : y0 + kR + kTY;

  // every load of the patch is issued before the first is used, so the CTA waits for global memory once
  constexpr int kLoads = (kIY * kIX + kThreads - 1) / kThreads;
  float va[kLoads], vb[kLoads];
#pragma unroll
  for (int k = 0; k < kLoads; ++k) {
    const int i = tid + k * kThreads, r = i / kIX, y = y0 + r, x = x0 + i - r * kIX;
    va[k] = vb[k] = 0.f;
    if (i < kIY * kIX && y < H && x < W) {
      const long long off = (frame + static_cast<long long>(y) * W + x) * C + c;
      va[k] = load_px(a + off);
      vb[k] = load_px(b + off);
    }
  }
  double sq = 0.0, ab = 0.0;
#pragma unroll
  for (int k = 0; k < kLoads; ++k) {
    const int i = tid + k * kThreads, r = i / kIX, q = i - r * kIX, y = y0 + r, x = x0 + q;
    if (i < kIY * kIX) {
      if (y >= oy0 && y < oy1 && x >= ox0 && x < ox1) {
        const double d = static_cast<double>(va[k]) - static_cast<double>(vb[k]);
        sq = fma(d, d, sq);
        ab += fabs(d);
      }
      sa[r * kSA + q] = va[k];
      sb[r * kSA + q] = vb[k];
    }
  }
  __syncthreads();

  // row pass: (row r, 8 consecutive columns) per item, lanes along rows
  for (int i = tid; i < kIY * (kTX / kP); i += kThreads) {
    const int r = i % kIY, x = (i / kIY) * kP;
    double acc[5][kP];
#pragma unroll
    for (int q = 0; q < 5; ++q)
#pragma unroll
      for (int o = 0; o < kP; ++o) acc[q][o] = 0.0;
    const float* ra = sa + r * kSA + x;
    const float* rb = sb + r * kSA + x;
#pragma unroll
    for (int j = 0; j < kP + 2 * kR; ++j) {
      const double va = ra[j], vb = rb[j];
      const double v[5] = {va, vb, va * va, vb * vb, va * vb};
#pragma unroll
      for (int o = 0; o < kP; ++o) {
        const int k = j - o;
        if (k >= 0 && k < kTaps) {
#pragma unroll
          for (int q = 0; q < 5; ++q) acc[q][o] = fma(gw.g[k], v[q], acc[q][o]);
        }
      }
    }
#pragma unroll
    for (int q = 0; q < 5; ++q)
#pragma unroll
      for (int o = 0; o < kP; ++o) sh[(q * kIY + r) * kSH + x + o] = acc[q][o];
  }
  __syncthreads();

  // column pass + map: (column x, 8 consecutive rows) per thread, lanes along x
  const int x = tid % kTX, ys = (tid / kTX) * kP;
  double acc[5][kP];
#pragma unroll
  for (int q = 0; q < 5; ++q)
#pragma unroll
    for (int o = 0; o < kP; ++o) acc[q][o] = 0.0;
#pragma unroll
  for (int j = 0; j < kP + 2 * kR; ++j) {
    double v[5];
#pragma unroll
    for (int q = 0; q < 5; ++q) v[q] = sh[(q * kIY + ys + j) * kSH + x];
#pragma unroll
    for (int o = 0; o < kP; ++o) {
      const int k = j - o;
      if (k >= 0 && k < kTaps) {
#pragma unroll
        for (int q = 0; q < 5; ++q) acc[q][o] = fma(gw.g[k], v[q], acc[q][o]);
      }
    }
  }
  // ssim.py's map with numpy's operation order and no contraction: equal inputs give exactly 1
  const double C1 = (0.01 * 255) * (0.01 * 255), C2 = (0.03 * 255) * (0.03 * 255);
  const int vx = x0 + x, vH = H - 2 * kR, vW = W - 2 * kR;
  double ss = 0.0;
#pragma unroll
  for (int o = 0; o < kP; ++o) {
    if (vx < vW && y0 + ys + o < vH) {
      const double mu1 = acc[0][o], mu2 = acc[1][o];
      const double mu1_sq = __dmul_rn(mu1, mu1), mu2_sq = __dmul_rn(mu2, mu2), mu1_mu2 = __dmul_rn(mu1, mu2);
      const double s1 = __dsub_rn(acc[2][o], mu1_sq), s2 = __dsub_rn(acc[3][o], mu2_sq);
      const double s12 = __dsub_rn(acc[4][o], mu1_mu2);
      const double num = __dmul_rn(__dadd_rn(__dmul_rn(2.0, mu1_mu2), C1), __dadd_rn(__dmul_rn(2.0, s12), C2));
      const double den = __dmul_rn(__dadd_rn(__dadd_rn(mu1_sq, mu2_sq), C1), __dadd_rn(__dadd_rn(s1, s2), C2));
      ss += __ddiv_rn(num, den);
    }
  }

  __shared__ double red[kThreads / 32][3];
  ss = warp_sum(ss);
  sq = warp_sum(sq);
  ab = warp_sum(ab);
  if ((tid & 31) == 0) {
    red[tid >> 5][0] = ss;
    red[tid >> 5][1] = sq;
    red[tid >> 5][2] = ab;
  }
  __syncthreads();
  if (tid < 3) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) s += red[w][tid];
    const long long tile = static_cast<long long>(blockIdx.y) * ntx + blockIdx.x;
    ws[(static_cast<long long>(blockIdx.z) * ntx * nty + tile) * 3 + tid] = s;
  }
}

// one warp per frame: out[n] = (l1, l2, psnr, ssim), ssim_c[n][c] (optional)
__global__ void metrics_reduce_kernel(const double* __restrict__ ws, int N, int H, int W, int C, int tiles,
                                      double* __restrict__ out, double* __restrict__ ssim_c) {
  const int n = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31;
  if (n >= N) return;
  double sq = 0.0, ab = 0.0, sc[3] = {0.0, 0.0, 0.0};
  for (int c = 0; c < C; ++c) {
    const double* p = ws + (static_cast<long long>(n) * C + c) * tiles * 3;
    double s = 0.0;
    for (int t = lane; t < tiles; t += 32) {
      s += p[3 * t];
      sq += p[3 * t + 1];
      ab += p[3 * t + 2];
    }
    sc[c] = warp_sum(s);
  }
  sq = warp_sum(sq);
  ab = warp_sum(ab);
  if (lane != 0) return;
  const double count = static_cast<double>(H) * W * C;
  const double positions = static_cast<double>(H - 2 * kR) * (W - 2 * kR);
  const double mse = sq / count;
  double ssim = 0.0;
  for (int c = 0; c < C; ++c) {
    sc[c] /= positions;
    if (ssim_c) ssim_c[static_cast<long long>(n) * C + c] = sc[c];
  }
  ssim = C == 1 ? sc[0] : ((sc[0] + sc[1]) + sc[2]) / 3.0;   // np.array(ssims).mean()
  double* o = out + 4LL * n;
  o[0] = ab / count;
  o[1] = sqrt(sq) / count;
  o[2] = mse == 0.0 ? 100.0 : 20.0 * log10(255.0 / sqrt(mse));
  o[3] = ssim;
}

// cv2.getGaussianKernel(11, 1.5) in float64: exp(-x^2 / (2 sigma^2)) normalised by its sum
inline Gauss gaussian() {
  Gauss g;
  const double sigma = 1.5, scale2x = -0.5 / (sigma * sigma);
  double sum = 0.0;
  for (int i = 0; i < kTaps; ++i) {
    const double x = i - (kTaps - 1) * 0.5;
    g.g[i] = exp(scale2x * x * x);
    sum += g.g[i];
  }
  sum = 1.0 / sum;
  for (int i = 0; i < kTaps; ++i) g.g[i] *= sum;
  return g;
}

template <typename TA, typename TB>
int launch_tiles(const void* a, const void* b, int N, int H, int W, int C, double* ws, fgt_stream_t s) {
  auto kern = metrics_tile_kernel<TA, TB>;
  if (const int rc = allow_dynamic_smem(kern, kSmem, "metrics_tile_kernel")) return rc;
  const dim3 grid((W - 2 * kR + kTX - 1) / kTX, (H - 2 * kR + kTY - 1) / kTY, N * C);
  return launch("metrics_tile_kernel", kern, grid, dim3(kThreads), kSmem, s, static_cast<const TA*>(a),
                static_cast<const TB*>(b), H, W, C, gaussian(), ws);
}

inline long long tiles_of(int H, int W) {
  return static_cast<long long>((W - 2 * kR + kTX - 1) / kTX) * ((H - 2 * kR + kTY - 1) / kTY);
}

}  // namespace metrics
}  // namespace fgt

using namespace fgt::metrics;

static int metrics_check(int N, int H, int W, int C) {
  FGT_REQUIRE(N >= 1, FGT_ERR_ARG, "metrics: no frames (N = %d)", N);
  FGT_REQUIRE(H >= kTaps && W >= kTaps, FGT_ERR_ARG,
              "metrics: frames of %dx%d are smaller than the 11x11 SSIM window", H, W);
  FGT_REQUIRE(C == 1 || C == 3, FGT_ERR_ARG, "metrics: %d channels (1 or 3 supported)", C);
  FGT_REQUIRE(static_cast<long long>(N) * C <= 65535, FGT_ERR_ARG,
              "metrics: N * C = %lld exceeds 65535 planes per call", static_cast<long long>(N) * C);
  return FGT_OK;
}

extern "C" long long fgt_metrics_workspace(int N, int H, int W, int C) {
  const int rc = metrics_check(N, H, W, C);
  if (rc != FGT_OK) return rc;
  return static_cast<long long>(N) * C * tiles_of(H, W) * 3 * static_cast<long long>(sizeof(double));
}

extern "C" int fgt_metrics(const void* a, int a_dtype, const void* b, int b_dtype, int N, int H, int W, int C,
                           void* workspace, long long workspace_bytes, double* out, double* ssim_c,
                           fgt_stream_t stream) {
  FGT_REQUIRE(a && b && workspace && out, FGT_ERR_ARG, "metrics: null pointer");
  int rc = metrics_check(N, H, W, C);
  if (rc != FGT_OK) return rc;
  const bool ok_a = a_dtype == FGT_METRIC_U8 || a_dtype == FGT_METRIC_F32;
  const bool ok_b = b_dtype == FGT_METRIC_U8 || b_dtype == FGT_METRIC_F32;
  FGT_REQUIRE(ok_a && ok_b, FGT_ERR_ARG, "metrics: unsupported dtype codes %d / %d (FGT_METRIC_U8 or FGT_METRIC_F32)",
              a_dtype, b_dtype);
  const long long need = fgt_metrics_workspace(N, H, W, C);
  FGT_REQUIRE(workspace_bytes >= need, FGT_ERR_ARG, "metrics: workspace of %lld bytes, %lld needed", workspace_bytes,
              need);
  double* ws = static_cast<double*>(workspace);
  const bool fa = a_dtype == FGT_METRIC_F32, fb = b_dtype == FGT_METRIC_F32;
  if (fa && fb) rc = launch_tiles<float, float>(a, b, N, H, W, C, ws, stream);
  else if (fa) rc = launch_tiles<float, uint8_t>(a, b, N, H, W, C, ws, stream);
  else if (fb) rc = launch_tiles<uint8_t, float>(a, b, N, H, W, C, ws, stream);
  else rc = launch_tiles<uint8_t, uint8_t>(a, b, N, H, W, C, ws, stream);
  if (rc != FGT_OK) return rc;
  constexpr int kWarps = 4;
  FGT_LAUNCH(metrics_reduce_kernel, dim3((N + kWarps - 1) / kWarps), dim3(32 * kWarps), 0, stream, ws, N, H, W, C,
             static_cast<int>(tiles_of(H, W)), out, ssim_c);
  return FGT_OK;
}
