// HBM-bound kernels of the RAFT path (RAFT/corr.py, RAFT/raft.py, RAFT/extractor.py): instance-norm
// statistics + normalise/ReLU/residual, correlation-pyramid pooling, the 9x9x4 bilinear correlation
// lookup (warp per pixel-level, patch staged in shared memory, shuffle-free coalesced rows),
// coordinate update and convex 8x upsampling. Tensor-core work (encoders, all-pairs correlation,
// update block) goes through gemm_tc.cu.
#include "common.h"
#include "ptx.cuh"

namespace fgt {

// ------------------------------------------------------------------------------------------
// per-(image, channel) sum and sum of squares of an NHWC fp32 tensor (nn.InstanceNorm2d statistics,
// RAFT/extractor.py:29-33,131-132). Block = 256 threads covering `C` channels x row slices; fp32
// partials over <=64 rows, double atomics across blocks.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(512) chan_stats_kernel(const float* __restrict__ x, int HW, int C,
                                                         int rows_per_block, double* __restrict__ stats) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red_s[512], red_q[512];
  const int img = blockIdx.y;
  const int r0 = blockIdx.x * rows_per_block;
  const int r1 = min(r0 + rows_per_block, HW);
  const float* base = x + static_cast<long long>(img) * HW * C;
  const int rstep = blockDim.x / C;       // row slots per block; thread t: channel t % C, slot t / C
  const int c = threadIdx.x % C;
  const int slot = threadIdx.x / C;
  float s = 0.f, q = 0.f;
  if (slot < rstep) {
    int r = r0 + slot;
    // eight independent loads in flight per thread (one at a time is latency bound)
    for (; r + 7 * rstep < r1; r += 8 * rstep) {
      float v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = __ldg(base + static_cast<long long>(r + j * rstep) * C + c);
#pragma unroll
      for (int j = 0; j < 8; ++j) { s += v[j]; q += v[j] * v[j]; }
    }
    for (; r < r1; r += rstep) {
      const float v = __ldg(base + static_cast<long long>(r) * C + c);
      s += v;
      q += v * v;
    }
  }
  red_s[threadIdx.x] = s;
  red_q[threadIdx.x] = q;
  __syncthreads();
  // one pair of atomics per (block, channel): same-address double atomics serialise at ~25 ns each,
  // which dominated the first version (4 row slots x 405 blocks per address)
  if (threadIdx.x < C) {
    double ds = 0.0, dq = 0.0;
    for (int j = 0; j < rstep; ++j) {
      ds += static_cast<double>(red_s[j * C + c]);
      dq += static_cast<double>(red_q[j * C + c]);
    }
    atomicAdd(&stats[(static_cast<long long>(img) * C + c) * 2], ds);
    atomicAdd(&stats[(static_cast<long long>(img) * C + c) * 2 + 1], dq);
  }
}

// y = (x - mean) * rstd ; optional ReLU ; optional residual: y = relu(y + res). fp32 and/or 16-bit out: split-bf16,
// or single-plane fp16 rows when plane == 0 (mixed-precision RAFT: the fp32 copy then holds the same fp16 values, the
// residual operand of a later block being an fp16 tensor under autocast).
// grid.y = image; per-channel scale / shift are derived once per block from the double statistics.
__global__ void instnorm_act_kernel(const float* __restrict__ x, const double* __restrict__ stats, int HW, int C,
                                    float eps, int relu, const float* __restrict__ res, float* __restrict__ out,
                                    __nv_bfloat16* __restrict__ hi, long long plane) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float sc[256], sh[256];
  const int img = blockIdx.y;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const double su = stats[(static_cast<long long>(img) * C + c) * 2];
    const double sq = stats[(static_cast<long long>(img) * C + c) * 2 + 1];
    const double mean = su / HW;
    const double var = fmax(sq / HW - mean * mean, 0.0);  // biased variance, like InstanceNorm2d
    const float rstd = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
    sc[c] = rstd;
    sh[c] = static_cast<float>(mean);
  }
  __syncthreads();
  const int C4 = C / 4;
  const long long total = static_cast<long long>(HW) * C4;
  const long long img_off = static_cast<long long>(img) * HW * C;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % C4) * 4;
    const long long off = img_off + (i / C4) * C + c;
    const float4 v = __ldg(reinterpret_cast<const float4*>(x + off));
    float o[4] = {(v.x - sh[c]) * sc[c], (v.y - sh[c + 1]) * sc[c + 1], (v.z - sh[c + 2]) * sc[c + 2],
                  (v.w - sh[c + 3]) * sc[c + 3]};
    if (relu) {
#pragma unroll
      for (int j = 0; j < 4; ++j) o[j] = fmaxf(o[j], 0.f);
    }
    const bool f16 = hi && plane == 0;
    if (res) {
      if (f16) {  // relu(norm(x)) is an fp16 tensor before the residual add (extractor.py:55-56)
#pragma unroll
        for (int j = 0; j < 4; ++j) o[j] = round_f16(o[j]);
      }
      const float4 r = __ldg(reinterpret_cast<const float4*>(res + off));
      o[0] = fmaxf(o[0] + r.x, 0.f); o[1] = fmaxf(o[1] + r.y, 0.f);
      o[2] = fmaxf(o[2] + r.z, 0.f); o[3] = fmaxf(o[3] + r.w, 0.f);
    }
    if (f16) {
#pragma unroll
      for (int j = 0; j < 4; ++j) o[j] = round_f16(o[j]);
    }
    if (out) *reinterpret_cast<float4*>(out + off) = make_float4(o[0], o[1], o[2], o[3]);
    if (hi) store16x4(hi + off, plane, o[0], o[1], o[2], o[3]);
  }
}

// ------------------------------------------------------------------------------------------
// 2x2 average pooling of the last two dims of [rows, h, w] (F.avg_pool2d(corr, 2, stride=2), corr.py:25-27)
// ------------------------------------------------------------------------------------------
__global__ void avgpool2_kernel(const float* __restrict__ in, long long rows, int h, int w, float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int oh = h / 2, ow = w / 2;
  const long long total = rows * oh * ow;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(i % ow);
    const int y = static_cast<int>((i / ow) % oh);
    const long long r = i / (static_cast<long long>(ow) * oh);
    const float* p = in + (r * h + 2 * y) * w + 2 * x;
    out[i] = ((p[0] + p[1]) + (p[w] + p[w + 1])) * 0.25f;
  }
}

// ------------------------------------------------------------------------------------------
// Correlation lookup (CorrBlock.__call__, corr.py:29-50 + bilinear_sampler, utils/utils.py:57-71):
// for every source pixel and pyramid level, a (2r+1)^2 window of bilinear samples around
// coords/2^level with zero padding and align_corners=True pixel coordinates. All window points share
// the fractional offset, so a (2r+2)^2 patch is staged once per (pixel, level) in shared memory.
// Window index a (first) offsets x, b (second) offsets y — the reference's meshgrid(dy, dx) stacking.
// Output: split-bf16 [n_pix, out_pitch], channel = level*(2r+1)^2 + a*(2r+1) + b; single-plane fp16 when plane == 0.
// ------------------------------------------------------------------------------------------
struct LookupLevels {
  const float* ptr[4];
  int h[4], w[4];
};

__global__ void corr_lookup_kernel(LookupLevels lv, int levels, int radius, const float* __restrict__ coords,
                                   int n_pix, int out_pitch, __nv_bfloat16* __restrict__ hi, long long plane) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float patch_smem[];
  const int warps_per_block = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int win = 2 * radius + 1, pw = win + 1;
  float* patch = patch_smem + warp * pw * pw;
  const long long n_items = static_cast<long long>(n_pix) * levels;
  for (long long item = static_cast<long long>(blockIdx.x) * warps_per_block + warp; item < n_items;
       item += static_cast<long long>(gridDim.x) * warps_per_block) {
    const int l = static_cast<int>(item % levels);
    const int p = static_cast<int>(item / levels);
    const float inv = 1.f / static_cast<float>(1 << l);
    float cx = coords[2 * p] * inv, cy = coords[2 * p + 1] * inv;
    cx = fminf(fmaxf(cx, -1.0e6f), 1.0e6f);
    cy = fminf(fmaxf(cy, -1.0e6f), 1.0e6f);
    const float fx0 = floorf(cx), fy0 = floorf(cy);
    const float fx = cx - fx0, fy = cy - fy0;
    const int x0 = static_cast<int>(fx0) - radius, y0 = static_cast<int>(fy0) - radius;
    const int h = lv.h[l], w = lv.w[l];
    const float* src = lv.ptr[l] + static_cast<long long>(p) * h * w;
    for (int e = lane; e < pw * pw; e += 32) {
      const int py = e / pw, px = e - py * pw;
      const int y = y0 + py, x = x0 + px;
      patch[e] = (y >= 0 && y < h && x >= 0 && x < w) ? __ldg(src + y * w + x) : 0.f;
    }
    __syncwarp();
    const float w00 = (1.f - fx) * (1.f - fy), w01 = fx * (1.f - fy), w10 = (1.f - fx) * fy, w11 = fx * fy;
    for (int o = lane; o < win * win; o += 32) {
      const int a = o / win, b = o - a * win;  // a -> x offset, b -> y offset
      const float v = w00 * patch[b * pw + a] + w01 * patch[b * pw + a + 1] + w10 * patch[(b + 1) * pw + a] +
                      w11 * patch[(b + 1) * pw + a + 1];
      store16(hi + static_cast<long long>(p) * out_pitch + l * win * win + o, plane, v);
    }
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------
// coords1 += delta (raft.py:132); emits flow = coords1 - coords0 (coords0 = pixel grid, raft.py:64-71)
// as NCHW fp32 (input of the 7x7 flow conv) and as the last two channels of the GRU input buffer x.
// x_plane == 0: x is single-plane fp16 (mixed precision), the flow channels are stored as fp16. delta_f16: delta is
// the flow head's output, an fp16 tensor under autocast, so it is rounded to fp16 before the fp32 add (raft.py:132).
// ------------------------------------------------------------------------------------------
__global__ void flow_update_kernel(float* __restrict__ coords, const float* __restrict__ delta, int delta_f16, int n_img,
                                   int h, int w, float* __restrict__ flow_nchw, __nv_bfloat16* __restrict__ x_hi,
                                   long long x_plane, int x_pitch, int x_chan) {
  pdl_launch_dependents();
  pdl_wait();
  const int n = h * w;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < n_img * n; p += gridDim.x * blockDim.x) {
    const int img = p / n, q = p - img * n;
    float cx = coords[2 * p], cy = coords[2 * p + 1];
    if (delta) {
      const float dx = delta[2 * p], dy = delta[2 * p + 1];
      cx += delta_f16 ? round_f16(dx) : dx;
      cy += delta_f16 ? round_f16(dy) : dy;
      coords[2 * p] = cx;
      coords[2 * p + 1] = cy;
    }
    const float fx = cx - static_cast<float>(q % w), fy = cy - static_cast<float>(q / w);
    flow_nchw[static_cast<long long>(img) * 2 * n + q] = fx;
    flow_nchw[static_cast<long long>(img) * 2 * n + n + q] = fy;
    if (x_hi) {
      __nv_bfloat16* xh = x_hi + static_cast<long long>(p) * x_pitch + x_chan;
      store16(xh, x_plane, fx);
      store16(xh + 1, x_plane, fy);
    }
  }
}

// ------------------------------------------------------------------------------------------
// fp16 -> split-bf16, exactly: an fp16 value has 11 significant bits, bf16 hi takes the top 8 and the residual (at most
// 4 bits, far above bf16's smallest normal) is exact in bf16 lo. Mixed-precision RAFT stores the feature net's output as
// fp16, as autocast does, and the 3-term correlation GEMM then computes the reference's fp32 correlation of those values
// (fmap.float(), raft.py:103-104). 8 elements per thread, 16-byte accesses.
// ------------------------------------------------------------------------------------------
__global__ void f16_to_split_kernel(const __half* __restrict__ src, long long n8, __nv_bfloat16* __restrict__ hi,
                                    long long plane) {
  pdl_launch_dependents();
  pdl_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n8;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(src) + i);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    float f[8];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float2 f2 = __half22float2(*reinterpret_cast<const __half2*>(&w[t]));
      f[2 * t] = f2.x;
      f[2 * t + 1] = f2.y;
    }
    store16x8(hi + 8 * i, plane, f);
  }
}

// ------------------------------------------------------------------------------------------
// Convex 8x upsampling (RAFT.upsample_flow, raft.py:73-84): softmax over the 9 mask logits of every
// fine pixel, weighted sum of the 3x3 neighbourhood of 8*flow (zero padded).
// mask: [n_img*h*w, 576] fp32 with channel = k*64 + i*8 + j; flow: [n_img, 2, h, w]; out: [n_img, 2, 8h, 8w] fp32.
// ------------------------------------------------------------------------------------------
__global__ void convex_upsample_kernel(const float* __restrict__ mask, const float* __restrict__ flow_all, int n_img,
                                       int h, int w, float* __restrict__ out_all) {
  pdl_launch_dependents();
  pdl_wait();
  const int n = h * w;
  const long long total = static_cast<long long>(n_img) * n * 64;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int sub = static_cast<int>(i & 63);
    const int pg = static_cast<int>(i >> 6);
    const int img = pg / n, p = pg - img * n;
    const int y = p / w, x = p - y * w;
    const float* flow_nchw = flow_all + static_cast<long long>(img) * 2 * n;
    float* out = out_all + static_cast<long long>(img) * 128 * n;
    const float* m = mask + static_cast<long long>(pg) * 576 + sub;
    float logit[9], mx = -INFINITY;
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      logit[k] = m[k * 64];
      mx = fmaxf(mx, logit[k]);
    }
    float den = 0.f, ax = 0.f, ay = 0.f;
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const float e = expf(logit[k] - mx);
      den += e;
      const int yy = y + k / 3 - 1, xx = x + k % 3 - 1;
      if (yy >= 0 && yy < h && xx >= 0 && xx < w) {
        ax += e * 8.f * flow_nchw[yy * w + xx];
        ay += e * 8.f * flow_nchw[n + yy * w + xx];
      }
    }
    const int oy = 8 * y + (sub >> 3), ox = 8 * x + (sub & 7);
    const long long HW = static_cast<long long>(64) * n;
    out[static_cast<long long>(oy) * (8 * w) + ox] = ax / den;
    out[HW + static_cast<long long>(oy) * (8 * w) + ox] = ay / den;
  }
}

// ------------------------------------------------------------------------------------------
// upflow8 (RAFT/utils/utils.py:80-82), the small model's upsampling: 8 * F.interpolate(flow, (8h, 8w), bilinear,
// align_corners=True). Source index and weights follow ATen's upsample_bilinear2d: scale = (in - 1) / (out - 1) in fp32
// (0 for a 1-pixel side), src = scale * dst, i0 = (int)src, i1 = i0 + (i0 < in - 1), lambda = src - i0.
// One thread per output pixel of one image, both flow channels; flow [n,2,h,w] -> out [n,2,8h,8w] fp32.
// ------------------------------------------------------------------------------------------
__global__ void upflow8_kernel(const float* __restrict__ flow, int n_img, int h, int w, float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int H = 8 * h, W = 8 * w;
  const float sy = static_cast<float>(h - 1) / static_cast<float>(H - 1);
  const float sx = static_cast<float>(w - 1) / static_cast<float>(W - 1);
  const long long total = static_cast<long long>(n_img) * H * W;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int ox = static_cast<int>(i % W);
    const int oy = static_cast<int>((i / W) % H);
    const int img = static_cast<int>(i / (static_cast<long long>(W) * H));
    const float fy = sy * static_cast<float>(oy), fx = sx * static_cast<float>(ox);
    const int y0 = static_cast<int>(fy), x0 = static_cast<int>(fx);
    const int y1 = y0 + (y0 < h - 1 ? 1 : 0), x1 = x0 + (x0 < w - 1 ? 1 : 0);
    const float ly = fy - static_cast<float>(y0), lx = fx - static_cast<float>(x0);
    const float hy = 1.f - ly, hx = 1.f - lx;
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const float* f = flow + (static_cast<long long>(img) * 2 + c) * h * w;
      const float v = hy * (hx * __ldg(f + y0 * w + x0) + lx * __ldg(f + y0 * w + x1)) +
                      ly * (hx * __ldg(f + y1 * w + x0) + lx * __ldg(f + y1 * w + x1));
      out[(static_cast<long long>(img) * 2 + c) * H * W + static_cast<long long>(oy) * W + ox] = 8.f * v;
    }
  }
}

}  // namespace fgt

using namespace fgt;

extern "C" int fgt_chan_stats(const float* x, int n, int HW, int C, double* stats, fgt_stream_t stream) {
  FGT_REQUIRE(x && stats && C >= 1 && C <= 256, FGT_ERR_ARG, "chan_stats: C=%d", C);
  FGT_CUDA(cudaMemsetAsync(stats, 0, sizeof(double) * 2 * n * C, stream));
  // about two blocks per SM over all images; each block reduces its rows in shared memory first
  int blocks_x = (2 * num_sms() + n - 1) / n;
  const int rstep = 512 / C;
  int rows_per_block = (HW + blocks_x - 1) / blocks_x;
  rows_per_block = ((rows_per_block + rstep - 1) / rstep) * rstep;
  if (rows_per_block < 8 * rstep) rows_per_block = 8 * rstep;
  dim3 grid((HW + rows_per_block - 1) / rows_per_block, n);
  FGT_LAUNCH(chan_stats_kernel, dim3(grid), dim3(512), 0, stream, x, HW, C, rows_per_block, stats);
  return FGT_OK;
}

extern "C" int fgt_instnorm_act(const float* x, const double* stats, int n, int HW, int C, float eps, int relu,
                                const float* res, float* out, void* out_hi, long long out_plane,
                                fgt_stream_t stream) {
  FGT_REQUIRE(x && stats && C % 4 == 0 && (out || out_hi), FGT_ERR_ARG, "instnorm_act: C=%d", C);
  FGT_REQUIRE(C <= 256, FGT_ERR_ARG, "instnorm_act: C=%d > 256", C);
  if (const int rc = check_act16("instnorm_act", out_hi, out_plane, 4, true)) return rc;
  const long long total = static_cast<long long>(HW) * (C / 4);
  const dim3 grid(grid_stride(total, 256), n);
  FGT_LAUNCH(instnorm_act_kernel, dim3(grid), dim3(256), 0, stream, x, stats, HW, C, eps, relu, res, out,
             reinterpret_cast<__nv_bfloat16*>(out_hi), out_plane);
  return FGT_OK;
}

extern "C" int fgt_avgpool2(const float* in, long long rows, int h, int w, float* out, fgt_stream_t stream) {
  FGT_REQUIRE(in && out && h >= 2 && w >= 2, FGT_ERR_ARG, "avgpool2: %dx%d", h, w);
  const long long total = rows * (h / 2) * (w / 2);
  FGT_LAUNCH(avgpool2_kernel, dim3(grid_stride(total, 256)), dim3(256), 0, stream, in, rows, h, w, out);
  return FGT_OK;
}

extern "C" int fgt_corr_lookup(const float* const* level_ptrs_host, const int* level_h_host, const int* level_w_host,
                               int levels, int radius, const float* coords, int n_pix, int out_pitch, void* out_hi,
                               long long out_plane, fgt_stream_t stream) {
  FGT_REQUIRE(levels >= 1 && levels <= 4 && radius >= 1 && radius <= 7, FGT_ERR_ARG, "corr_lookup: levels=%d r=%d",
              levels, radius);
  const int win = 2 * radius + 1;
  FGT_REQUIRE(out_pitch >= levels * win * win, FGT_ERR_ARG, "corr_lookup: out_pitch=%d", out_pitch);
  if (const int rc = check_act16("corr_lookup", out_hi, out_plane, 1, true)) return rc;
  LookupLevels lv;
  for (int i = 0; i < 4; ++i) {
    lv.ptr[i] = i < levels ? level_ptrs_host[i] : nullptr;
    lv.h[i] = i < levels ? level_h_host[i] : 0;
    lv.w[i] = i < levels ? level_w_host[i] : 0;
  }
  const int block = 256;
  const size_t smem = (block / 32) * (win + 1) * (win + 1) * sizeof(float);
  const long long items = static_cast<long long>(n_pix) * levels;
  FGT_LAUNCH(corr_lookup_kernel, dim3(grid_stride(items * 32, block)), dim3(block), smem, stream, lv, levels, radius,
             coords, n_pix, out_pitch, reinterpret_cast<__nv_bfloat16*>(out_hi), out_plane);
  return FGT_OK;
}

extern "C" int fgt_raft_flow_update(float* coords, const float* delta, int delta_f16, int n, int h, int w,
                                    float* flow_nchw, void* x_hi, long long x_plane, int x_pitch, int x_chan,
                                    fgt_stream_t stream) {
  FGT_REQUIRE(coords && flow_nchw && n >= 1, FGT_ERR_ARG, "raft_flow_update: null argument");
  FGT_REQUIRE(delta_f16 == 0 || delta_f16 == 1, FGT_ERR_ARG, "raft_flow_update: delta_f16=%d (0 or 1)", delta_f16);
  if (const int rc = check_act16("raft_flow_update", x_hi, x_plane, 1, true)) return rc;
  FGT_LAUNCH(flow_update_kernel, dim3(grid_stride(static_cast<long long>(n) * h * w, 256)), dim3(256), 0, stream,
             coords, delta, delta_f16, n, h, w, flow_nchw, reinterpret_cast<__nv_bfloat16*>(x_hi), x_plane, x_pitch,
             x_chan);
  return FGT_OK;
}

extern "C" int fgt_f16_to_split(const void* src, long long n, void* out_hi, long long out_plane, fgt_stream_t stream) {
  FGT_REQUIRE(src && out_hi && n >= 0 && n % 8 == 0 && out_plane >= n && (reinterpret_cast<uintptr_t>(src) & 15) == 0,
              FGT_ERR_ARG, "f16_to_split: n=%lld plane=%lld (multiples of 8, 16-byte aligned buffers)", n, out_plane);
  if (const int rc = check_act16("f16_to_split", out_hi, out_plane, 8, false)) return rc;
  if (n == 0) return FGT_OK;
  FGT_LAUNCH(f16_to_split_kernel, dim3(grid_stride(n / 8, 256)), dim3(256), 0, stream,
             reinterpret_cast<const __half*>(src), n / 8, reinterpret_cast<__nv_bfloat16*>(out_hi), out_plane);
  return FGT_OK;
}

extern "C" int fgt_convex_upsample(const float* mask, const float* flow_nchw, int n, int h, int w, float* out,
                                   fgt_stream_t stream) {
  FGT_REQUIRE(mask && flow_nchw && out && n >= 1, FGT_ERR_ARG, "convex_upsample: null argument");
  const long long total = static_cast<long long>(n) * h * w * 64;
  FGT_LAUNCH(convex_upsample_kernel, dim3(grid_stride(total, 256)), dim3(256), 0, stream, mask, flow_nchw, n, h, w,
             out);
  return FGT_OK;
}

extern "C" int fgt_upflow8(const float* flow_nchw, int n, int h, int w, float* out, fgt_stream_t stream) {
  FGT_REQUIRE(flow_nchw && out && n >= 1 && h >= 1 && w >= 1, FGT_ERR_ARG, "upflow8: n=%d h=%d w=%d", n, h, w);
  const long long total = static_cast<long long>(n) * 64 * h * w;
  FGT_LAUNCH(upflow8_kernel, dim3(grid_stride(total, 256)), dim3(256), 0, stream, flow_nchw, n, h, w, out);
  return FGT_OK;
}
