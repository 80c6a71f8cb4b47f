// Operand preparation of the flow-guided spatial window attention (SWMHSA, attention_flow.py:130-154) in ONE launch:
// everything between the flow gate and the Q|K / V projections that is not a contraction.
//
//   window rows  : token (frame, window, position) -> LayerNorm statistics over [x ; f'] (768 channels: the shared
//                  input of q_norm and k_norm, whose affines are folded into the projection weights) and over x alone
//                  (512 channels: v_norm), written as split-bf16 rows in window-major order (the reference's
//                  window_partition, :132-133,150-151); rows of the zero-padded grid are written as zeros.
//   pooled rows  : global token (frame, gy, gx) = depthwise gd x gd / stride gd convolution (+bias) of [x ; f'] (keys,
//                  global_extract_k, :135) and of x (values, global_extract_v, :145) over the zero-padded token grid,
//                  then the same two LayerNorms, written after the window rows of the frame (:140,152).
//
// One warp per window row; one block per pooled token (its gd*gd source tokens are spread over the block's 8 warps and
// the partial sums combined through shared memory in a fixed order, so a pooled token costs two dependent load rounds
// instead of sixteen). x and f' are read once per use (they were read four times by the separate dwpool / rownorm
// launches this replaces), statistics by warp shuffles, two-pass variance in registers. HBM-bound by design.
#include "common.h"
#include "ptx.cuh"

namespace fgt {

constexpr int kMaxVec = 6;  // float4 per lane: up to 768 channels per row (FGT: 512 + 256)
constexpr int kMaxVecV = 4; // value rows: up to 512 channels

// LayerNorm (no affine) of the first `nvec` float4 of val[] per lane (channels 4*(lane + 32 i)), stored 16-bit.
template <int NV>
__device__ __forceinline__ void swin_norm_store(const float4 (&val)[kMaxVec], int nvec, int C, float eps,
                                           __nv_bfloat16* __restrict__ hi, long long plane, int lane) {
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i)
    if (lane + 32 * i < nvec) sum += (val[i].x + val[i].y) + (val[i].z + val[i].w);
  const float mean = warp_sum(sum) / static_cast<float>(C);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i)
    if (lane + 32 * i < nvec) {
      const float a = val[i].x - mean, b = val[i].y - mean, c = val[i].z - mean, d = val[i].w - mean;
      sq += (a * a + b * b) + (c * c + d * d);
    }
  const float rstd = rsqrtf(warp_sum(sq) / static_cast<float>(C) + eps);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int v = lane + 32 * i;
    if (v < nvec)
      store16x4(hi + v * 4, plane, (val[i].x - mean) * rstd, (val[i].y - mean) * rstd, (val[i].z - mean) * rstd,
                (val[i].w - mean) * rstd);
  }
}

__device__ __forceinline__ void swin_zero_row(__nv_bfloat16* __restrict__ hi, long long plane, int nvec, int lane) {
  for (int v = lane; v < nvec; v += 32) zero16x4(hi + v * 4, plane);
}

struct SwinPrepArgs {
  const float* x;   // [bt*h*w, d]
  const float* fp;  // [bt*h*w, df]   re-weighted flow tokens f'
  int d, df, bt, h, w;
  const int* win_map;  // [bt * nl] -> token index or -1 (padding / dummy window)
  int nl, R;           // window rows per frame, rows per frame in the destination (window rows + padded pooled rows)
  int gd, gh, gw;      // pooling kernel = stride, pooled grid
  const float *gk_w, *gk_b, *gv_w, *gv_b;  // depthwise weights TAP-MAJOR [gd*gd, C] (coalesced float4 per tap), biases [C]
  __nv_bfloat16* qkn; long long qkn_plane;  // [bt*R, d+df] split
  __nv_bfloat16* vn; long long vn_plane;    // [bt*R, d] split
  float eps;
};

__global__ void __launch_bounds__(256, 2) swin_prep_kernel(const SwinPrepArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float4 part_k[8][kMaxVec * 32];   // per-warp partial sums of a pooled token (keys: d + df channels), 24 KB
  __shared__ float4 part_v[8][kMaxVecV * 32];  // (values: d channels), 16 KB
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int C = a.d + a.df;
  const int nvx = a.d / 4, nvc = C / 4;
  const int G = a.gh * a.gw;
  const int n_pool = a.bt * G;
  float4 kq[kMaxVec], vv[kMaxVec];
  if (static_cast<int>(blockIdx.x) < n_pool) {
    // ---------------------------------------------------------------- pooled (global) token: one block, taps over warps
    const int gi = blockIdx.x;
    const int f = gi / G, g = gi - f * G;
    const int gy = g / a.gw, gx = g - gy * a.gw;
    const long long drow = static_cast<long long>(f) * a.R + a.nl + g;
    const int kk = a.gd * a.gd;
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) {
      kq[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      vv[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    for (int tap = warp; tap < kk; tap += 8) {
      const int ky = tap / a.gd, kx = tap - ky * a.gd;
      const int y = gy * a.gd + ky, xx = gx * a.gd + kx;
      if (y >= a.h || xx >= a.w) continue;  // positions of the zero padding contribute nothing
      const long long tok = (static_cast<long long>(f) * a.h + y) * a.w + xx;
      const float4* xr = reinterpret_cast<const float4*>(a.x + tok * a.d);
      const float4* fr = reinterpret_cast<const float4*>(a.fp + tok * a.df);
      const float4* wkr = reinterpret_cast<const float4*>(a.gk_w + static_cast<long long>(tap) * C);
      const float4* wvr = reinterpret_cast<const float4*>(a.gv_w + static_cast<long long>(tap) * a.d);
#pragma unroll
      for (int i = 0; i < kMaxVec; ++i) {
        const int v = lane + 32 * i;
        if (v < nvc) {
          const float4 in = (v < nvx) ? __ldg(xr + v) : __ldg(fr + (v - nvx));
          const float4 wk = __ldg(wkr + v);
          kq[i].x = fmaf(wk.x, in.x, kq[i].x);
          kq[i].y = fmaf(wk.y, in.y, kq[i].y);
          kq[i].z = fmaf(wk.z, in.z, kq[i].z);
          kq[i].w = fmaf(wk.w, in.w, kq[i].w);
          if (v < nvx) {
            const float4 wv = __ldg(wvr + v);
            vv[i].x = fmaf(wv.x, in.x, vv[i].x);
            vv[i].y = fmaf(wv.y, in.y, vv[i].y);
            vv[i].z = fmaf(wv.z, in.z, vv[i].z);
            vv[i].w = fmaf(wv.w, in.w, vv[i].w);
          }
        }
      }
    }
#pragma unroll
    for (int i = 0; i < kMaxVec; ++i) {
      const int v = lane + 32 * i;
      if (v < nvc) part_k[warp][v] = kq[i];
      if (v < nvx) part_v[warp][v] = vv[i];
    }
    __syncthreads();
    if (warp == 0) {        // keys: bias + the 8 partial sums in warp order (fixed order: deterministic), LayerNorm, store
#pragma unroll
      for (int i = 0; i < kMaxVec; ++i) {
        const int v = lane + 32 * i;
        if (v < nvc) {
          float4 acc = __ldg(reinterpret_cast<const float4*>(a.gk_b) + v);
#pragma unroll
          for (int w = 0; w < 8; ++w) {
            const float4 q = part_k[w][v];
            acc.x += q.x; acc.y += q.y; acc.z += q.z; acc.w += q.w;
          }
          kq[i] = acc;
        }
      }
      swin_norm_store<kMaxVec>(kq, nvc, C, a.eps, a.qkn + drow * C, a.qkn_plane, lane);
    } else if (warp == 1) {  // values
#pragma unroll
      for (int i = 0; i < kMaxVec; ++i) {
        const int v = lane + 32 * i;
        if (v < nvx) {
          float4 acc = __ldg(reinterpret_cast<const float4*>(a.gv_b) + v);
#pragma unroll
          for (int w = 0; w < 8; ++w) {
            const float4 q = part_v[w][v];
            acc.x += q.x; acc.y += q.y; acc.z += q.z; acc.w += q.w;
          }
          vv[i] = acc;
        }
      }
      swin_norm_store<kMaxVec>(vv, nvx, a.d, a.eps, a.vn + drow * a.d, a.vn_plane, lane);
    }
    return;
  }
  // ------------------------------------------------------------------ window rows: one warp per row
  const long long n_win = static_cast<long long>(a.bt) * a.nl;
  const long long it = (static_cast<long long>(blockIdx.x) - n_pool) * 8 + warp;
  if (it >= n_win) return;
  const long long f = it / a.nl;
  const long long drow = f * a.R + (it - f * a.nl);
  const int src = a.win_map[it];
  if (src < 0) {
    swin_zero_row(a.qkn + drow * C, a.qkn_plane, nvc, lane);
    swin_zero_row(a.vn + drow * a.d, a.vn_plane, nvx, lane);
    return;
  }
  const float4* xr = reinterpret_cast<const float4*>(a.x + static_cast<long long>(src) * a.d);
  const float4* fr = reinterpret_cast<const float4*>(a.fp + static_cast<long long>(src) * a.df);
#pragma unroll
  for (int i = 0; i < kMaxVec; ++i) {
    const int v = lane + 32 * i;
    if (v < nvx) {
      kq[i] = __ldg(xr + v);
      vv[i] = kq[i];
    } else if (v < nvc) {
      kq[i] = __ldg(fr + (v - nvx));
    }
  }
  swin_norm_store<kMaxVec>(kq, nvc, C, a.eps, a.qkn + drow * C, a.qkn_plane, lane);
  swin_norm_store<kMaxVec>(vv, nvx, a.d, a.eps, a.vn + drow * a.d, a.vn_plane, lane);
}

}  // namespace fgt

extern "C" int fgt_swin_prep(const float* x, const float* fp, int d, int df, int bt, int h, int w, const int* win_map,
                             int nl, int R, int gd, int gh, int gw, const float* gk_w, const float* gk_b,
                             const float* gv_w, const float* gv_b, void* qkn_hi, long long qkn_plane, void* vn_hi,
                             long long vn_plane, float eps, fgt_stream_t stream) {
  FGT_REQUIRE(x && fp && win_map && gk_w && gk_b && gv_w && gv_b && qkn_hi && vn_hi, FGT_ERR_ARG, "swin_prep: null argument");
  FGT_REQUIRE(d % 4 == 0 && df % 4 == 0 && d >= 4 && df >= 4 && d + df <= 128 * fgt::kMaxVec && d <= 128 * fgt::kMaxVecV,
              FGT_ERR_ARG, "swin_prep: d=%d df=%d (d <= 512, d + df <= 768)", d, df);
  FGT_REQUIRE(bt >= 1 && h >= 1 && w >= 1 && nl >= 1 && gd >= 1 && gh >= 1 && gw >= 1 && R >= nl + gh * gw, FGT_ERR_ARG,
              "swin_prep: geometry bt=%d h=%d w=%d nl=%d R=%d gd=%d gh=%d gw=%d", bt, h, w, nl, R, gd, gh, gw);
  if (const int rc = fgt::check_act16("swin_prep: qkn", qkn_hi, qkn_plane, 4, true)) return rc;
  if (const int rc = fgt::check_act16("swin_prep: vn", vn_hi, vn_plane, 4, true)) return rc;
  FGT_REQUIRE((qkn_plane == 0) == (vn_plane == 0), FGT_ERR_ARG,
              "swin_prep: qkn and vn are both split-bf16 (plane > 0) or both single-plane fp16 (plane 0), got %lld / %lld",
              qkn_plane, vn_plane);
  fgt::SwinPrepArgs a;
  a.x = x; a.fp = fp; a.d = d; a.df = df; a.bt = bt; a.h = h; a.w = w; a.win_map = win_map; a.nl = nl; a.R = R;
  a.gd = gd; a.gh = gh; a.gw = gw; a.gk_w = gk_w; a.gk_b = gk_b; a.gv_w = gv_w; a.gv_b = gv_b;
  a.qkn = reinterpret_cast<__nv_bfloat16*>(qkn_hi); a.qkn_plane = qkn_plane;
  a.vn = reinterpret_cast<__nv_bfloat16*>(vn_hi); a.vn_plane = vn_plane; a.eps = eps;
  // blocks [0, bt*G): one pooled token each (its gd*gd source tokens spread over the 8 warps, combined in shared memory);
  // the following blocks: 8 window rows each (one warp per row)
  const int block = 256;
  const long long blocks = static_cast<long long>(bt) * gh * gw + (static_cast<long long>(bt) * nl + 7) / 8;
  FGT_LAUNCH(fgt::swin_prep_kernel, dim3(static_cast<unsigned>(blocks)), dim3(block), 0, stream, a);
  return FGT_OK;
}
