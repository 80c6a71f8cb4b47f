// HBM-bound helper kernels around the tensor-core engine (coalesced, vectorised, warp-shuffle
// reductions): layout packing, LayerNorm statistics, depthwise pooling / positional conv,
// fold / unfold of the fusion FFN, nearest upsampling. No tensor cores here on purpose.
#include "common.h"
#include "ptx.cuh"

namespace fgt {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ void store_split4(__nv_bfloat16* hi, __nv_bfloat16* lo, float a, float b, float c,
                                             float d) {
  __nv_bfloat16 h0, l0, h1, l1, h2, l2, h3, l3;
  split_bf16(a, h0, l0);
  split_bf16(b, h1, l1);
  split_bf16(c, h2, l2);
  split_bf16(d, h3, l3);
  *reinterpret_cast<uint2*>(hi) = make_uint2(pack_bf16x2(h0, h1), pack_bf16x2(h2, h3));
  *reinterpret_cast<uint2*>(lo) = make_uint2(pack_bf16x2(l0, l1), pack_bf16x2(l2, l3));
}

// Four consecutive 16-bit outputs: split-bf16 with the lo plane `plane` elements after hi, or single-plane fp16 rows
// (the A operand of a 1-term layer, mixed precision) when plane == 0.
__device__ __forceinline__ void store16x4(__nv_bfloat16* hi, long long plane, float a, float b, float c, float d) {
  if (plane == 0) *reinterpret_cast<uint2*>(hi) = make_uint2(pack_f16x2(a, b), pack_f16x2(c, d));
  else store_split4(hi, hi + plane, a, b, c, d);
}

// ------------------------------------------------------------------------------------------
// pack: NCHW fp32 (two sources concatenated on C) -> NHWC split-bf16 with channel padding and
// optional replication padding (ReplicationPad2d of the flow encoder, model.py:207).
// ------------------------------------------------------------------------------------------
__global__ void pack_nchw_kernel(const float* __restrict__ s0, int c0, const float* __restrict__ s1, int c1, int n,
                                 int H, int W, int pad, int cpad, __nv_bfloat16* __restrict__ hi, long long plane) {
  pdl_launch_dependents();
  pdl_wait();
  const int Wp = W + 2 * pad, Hp = H + 2 * pad;
  const long long total = static_cast<long long>(n) * Hp * Wp;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(i % Wp);
    const int y = static_cast<int>((i / Wp) % Hp);
    const int b = static_cast<int>(i / (static_cast<long long>(Wp) * Hp));
    const int sx = min(max(x - pad, 0), W - 1), sy = min(max(y - pad, 0), H - 1);
    for (int c = 0; c < cpad; ++c) {
      float v = 0.f;
      if (c < c0) v = s0[((static_cast<long long>(b) * c0 + c) * H + sy) * W + sx];
      else if (c < c0 + c1) v = s1[((static_cast<long long>(b) * c1 + (c - c0)) * H + sy) * W + sx];
      __nv_bfloat16 h, l;
      split_bf16(v, h, l);
      hi[i * cpad + c] = h;
      hi[plane + i * cpad + c] = l;
    }
  }
}

// ------------------------------------------------------------------------------------------
// im2col for the tiny-channel first layers (4->64 3x3 s2, 2->64 5x5 after ReplicationPad2d(2),
// model.py:34,207-208): gathers the k x k neighbourhood of NCHW fp32 inputs (two sources concatenated
// on C) into one 64-channel NHWC split row per output pixel, channel = (ky*k + kx)*cin + c. The
// convolution then is a single K=64 GEMM instead of k*k zero-padded 64-channel taps.
// ------------------------------------------------------------------------------------------
__global__ void im2col_nchw_kernel(const float* __restrict__ s0, int c0, const float* __restrict__ s1, int c1,
                                   int n, int H, int W, int k, int stride, int pad, int replicate, int OH, int OW,
                                   int cpad, float scale, float shift, __nv_bfloat16* __restrict__ hi,
                                   long long plane) {
  pdl_launch_dependents();
  pdl_wait();
  // one block = one output row (b, oy). The k input rows the row needs (all cin channels, padded to the width the
  // taps reach: Wp = (OW-1)*stride + k) are staged in shared memory first — coalesced global reads, bounds /
  // replication handled once per staged element — so the gather itself is 8 shared-memory loads per 16-byte store.
  extern __shared__ float srow[];  // [k][cin][Wp]
  const int cin = c0 + c1;
  const int Wp = (OW - 1) * stride + k;
  const int b = blockIdx.x / OH, oy = blockIdx.x - b * OH;
  const int tid = threadIdx.y * blockDim.x + threadIdx.x, nthr = blockDim.x * blockDim.y;
  const long long HWl = static_cast<long long>(H) * W;
  // staged row rc = ky*cin + c: one warp per row, lanes along x (no per-element integer division — the first version of
  // this loop spent 4x the instructions of the gather on idx / row_elems, r / Wp)
  const int lane = tid & 31, wrp = tid >> 5, nwarp = nthr >> 5;
  for (int rc = wrp; rc < k * cin; rc += nwarp) {
    const int ky = rc / cin, c = rc - ky * cin;
    int y = oy * stride + ky - pad;
    const bool y_ok = replicate || (y >= 0 && y < H);
    y = min(max(y, 0), H - 1);
    const float* src = (c < c0) ? s0 + (static_cast<long long>(b) * c0 + c) * HWl + static_cast<long long>(y) * W
                                : s1 + (static_cast<long long>(b) * c1 + (c - c0)) * HWl + static_cast<long long>(y) * W;
    float* dst = srow + rc * Wp;
    for (int xx = lane; xx < Wp; xx += 32) {
      int x = xx - pad;
      const bool ok = y_ok && (replicate || (x >= 0 && x < W));
      x = min(max(x, 0), W - 1);
      dst[xx] = ok ? fmaf(__ldg(src + x), scale, shift) : 0.f;
    }
  }
  // this thread's 8 output channels: ch = (ky*k + kx)*cin + c  ->  offset of (ky, c, kx) in the staged rows
  const int g = threadIdx.x;
  int off[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int ch = g * 8 + j;
    if (ch < k * k * cin) {
      const int tap = ch / cin, c = ch - tap * cin;
      const int ky = tap / k, kx = tap - ky * k;
      off[j] = (ky * cin + c) * Wp + kx;
    } else {
      off[j] = -1;
    }
  }
  __syncthreads();
  for (int ox = threadIdx.y; ox < OW; ox += blockDim.y) {
    const int x0 = ox * stride;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = off[j] >= 0 ? srow[off[j] + x0] : 0.f;
    const long long o = ((static_cast<long long>(b) * OH + oy) * OW + ox) * cpad + g * 8;
    if (plane == 0) {  // single-plane fp16 rows (input of a 1-term layer)
      *reinterpret_cast<uint4*>(hi + o) = make_uint4(pack_f16x2(v[0], v[1]), pack_f16x2(v[2], v[3]),
                                                     pack_f16x2(v[4], v[5]), pack_f16x2(v[6], v[7]));
    } else {
      uint32_t hw[4], lw[4];
#pragma unroll
      for (int t = 0; t < 4; ++t) split_bf16x2(v[2 * t], v[2 * t + 1], hw[t], lw[t]);
      *reinterpret_cast<uint4*>(hi + o) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
      *reinterpret_cast<uint4*>(hi + plane + o) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
    }
  }
}

// ------------------------------------------------------------------------------------------
// rownorm: per-row LayerNorm statistics (no affine: gamma/beta are folded into the consuming
// Linear) over the concatenation of up to two fp32 sources; optional gather map (dest row ->
// source row, <0 = write zeros: the reference's zero padding happens before/after LN in a way that
// makes padded rows exactly the LN bias, attention_flow.py:122-143, attention_base.py:87-92).
// One warp per destination row; two-pass mean / variance in registers.
// ------------------------------------------------------------------------------------------
constexpr int kNormMaxVec = 8;  // up to 8 float4 per lane -> C <= 1024
constexpr int kNormMaxDst = 8;  // destinations of one normalised row: the local buffer and/or NVLink peers

// Destination buffers of the normalised rows. More than one = the exchange step of frame-sharded TMHSA
// fused into the LayerNorm: every rank stores its rows straight into all peers' K/V-input buffers
// (P2P stores over NVLink), so no separate all-gather and no re-ordering copy is needed.
struct NormDests {
  __nv_bfloat16* hi[kNormMaxDst];
  int n;
};

__global__ void __launch_bounds__(256, 4) rownorm_kernel(const float* __restrict__ a, int ca, int lda, const float* __restrict__ b, int cb,
                               int ldb, const int* __restrict__ gather, int rows_per_batch, long long total_rows,
                               int dst_batch_rows, int dst_row0, const float* __restrict__ gamma,
                               const float* __restrict__ beta, const NormDests dst, long long plane, float eps) {
  pdl_launch_dependents();
  pdl_wait();
  const int C = ca + cb;
  const int lane = threadIdx.x & 31;
  const long long warp_id = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const int nvec = C / 4;
  for (long long d = warp_id; d < total_rows; d += nwarps) {
    // 32-bit division when the row count allows it (always, in this model): the 64-bit one is ~80 instructions per row
    const long long bidx = (total_rows <= 0x7fffffffLL) ? static_cast<long long>(static_cast<int>(d) / rows_per_batch)
                                                        : d / rows_per_batch;
    const long long drow = bidx * dst_batch_rows + dst_row0 + (d - bidx * rows_per_batch);
    const long long ooff = drow * C;
    long long src = d;
    if (gather) src = gather[d];
    if (src < 0) {
      for (int q = 0; q < dst.n; ++q) {
        for (int v = lane; v < nvec; v += 32) {
          *reinterpret_cast<uint2*>(dst.hi[q] + ooff + v * 4) = make_uint2(0u, 0u);
          if (plane) *reinterpret_cast<uint2*>(dst.hi[q] + ooff + plane + v * 4) = make_uint2(0u, 0u);
        }
      }
      continue;
    }
    float4 val[kNormMaxVec];
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < kNormMaxVec; ++i) {
      const int v = lane + 32 * i;
      if (v < nvec) {
        const int c = v * 4;
        val[i] = (c < ca) ? __ldg(reinterpret_cast<const float4*>(a + src * lda + c))
                          : __ldg(reinterpret_cast<const float4*>(b + src * ldb + (c - ca)));
        sum += (val[i].x + val[i].y) + (val[i].z + val[i].w);
      }
    }
    const float mean = warp_sum(sum) / static_cast<float>(C);
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < kNormMaxVec; ++i) {
      if (lane + 32 * i < nvec) {
        const float dx = val[i].x - mean, dy = val[i].y - mean, dz = val[i].z - mean, dw = val[i].w - mean;
        sq += (dx * dx + dy * dy) + (dz * dz + dw * dw);
      }
    }
    const float rstd = rsqrtf(warp_sum(sq) / static_cast<float>(C) + eps);
#pragma unroll
    for (int i = 0; i < kNormMaxVec; ++i) {
      const int v = lane + 32 * i;
      if (v < nvec) {
        float4 o = make_float4((val[i].x - mean) * rstd, (val[i].y - mean) * rstd, (val[i].z - mean) * rstd,
                               (val[i].w - mean) * rstd);
        if (gamma) {
          const float4 gm = __ldg(reinterpret_cast<const float4*>(gamma + v * 4));
          const float4 bt = __ldg(reinterpret_cast<const float4*>(beta + v * 4));
          o.x = o.x * gm.x + bt.x; o.y = o.y * gm.y + bt.y; o.z = o.z * gm.z + bt.z; o.w = o.w * gm.w + bt.w;
        }
        if (plane == 0) {  // single-plane fp16 rows (mixed precision)
          const uint2 hv = make_uint2(pack_f16x2(o.x, o.y), pack_f16x2(o.z, o.w));
          for (int q = 0; q < dst.n; ++q) *reinterpret_cast<uint2*>(dst.hi[q] + ooff + v * 4) = hv;
          continue;
        }
        uint32_t h0, l0, h1, l1;
        split_bf16x2(o.x, o.y, h0, l0);
        split_bf16x2(o.z, o.w, h1, l1);
        for (int q = 0; q < dst.n; ++q) {
          *reinterpret_cast<uint2*>(dst.hi[q] + ooff + v * 4) = make_uint2(h0, h1);
          *reinterpret_cast<uint2*>(dst.hi[q] + ooff + plane + v * 4) = make_uint2(l0, l1);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// dwpool: depthwise k x k / stride k convolution (+bias) over the zero-padded token grid of the
// channel concatenation [a ; b] -> fp32 pooled tokens (global_extract_k / global_extract_v,
// attention_flow.py:44-48,135,145).
// ------------------------------------------------------------------------------------------
__global__ void dwpool_kernel(const float* __restrict__ a, int ca, const float* __restrict__ b, int cb, int bt,
                              int h, int w, int k, int gh, int gw, const float* __restrict__ wt,
                              const float* __restrict__ bias, float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int C = ca + cb;
  const long long total = static_cast<long long>(bt) * gh * gw * C;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % C);
    const long long t = i / C;
    const int gx = static_cast<int>(t % gw);
    const int gy = static_cast<int>((t / gw) % gh);
    const int f = static_cast<int>(t / (static_cast<long long>(gw) * gh));
    float acc = bias[c];
    for (int ky = 0; ky < k; ++ky) {
      const int y = gy * k + ky;
      if (y >= h) break;
      for (int kx = 0; kx < k; ++kx) {
        const int x = gx * k + kx;
        if (x >= w) break;
        const long long tok = (static_cast<long long>(f) * h + y) * w + x;
        const float v = (c < ca) ? a[tok * ca + c] : b[tok * cb + (c - ca)];
        acc += wt[(c * k + ky) * k + kx] * v;
      }
    }
    out[i] = acc;
  }
}

// ------------------------------------------------------------------------------------------
// dwconv3x3 + identity on the token grid (AddPosEmb, model.py:75-88); writes fp32 and split.
// ------------------------------------------------------------------------------------------
__global__ void dwconv3_res_kernel(const float* __restrict__ x, int bt, int h, int w, int C,
                                   const float* __restrict__ wt, const float* __restrict__ bias,
                                   float* __restrict__ out, __nv_bfloat16* __restrict__ hi, long long plane) {
  pdl_launch_dependents();
  pdl_wait();
  // one block = one token row (frame, py); one thread = 4 consecutive channels, striding over the row's tokens: float4
  // loads of the 3x3 neighbourhood (coalesced along c), weights and bias of the thread's channels held in registers
  const int C4 = C / 4;
  const long long f = blockIdx.x / h;
  const int py = blockIdx.x - static_cast<int>(f) * h;
  for (int cq = threadIdx.x; cq < C4; cq += blockDim.x) {
   const int c = cq * 4;
   float wreg[4][9];
#pragma unroll
   for (int i = 0; i < 4; ++i)
#pragma unroll
     for (int tap = 0; tap < 9; ++tap) wreg[i][tap] = __ldg(wt + (c + i) * 9 + tap);
   const float4 b4 = __ldg(reinterpret_cast<const float4*>(bias + c));
   const int seg = (w + gridDim.y - 1) / gridDim.y;
   const int px_end = min(w, static_cast<int>(blockIdx.y + 1) * seg);
   for (int px = blockIdx.y * seg + threadIdx.y; px < px_end; px += blockDim.y) {
    const long long t = (f * h + py) * w + px;
    float4 acc = b4;
    float4 centre = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int y = py + ky - 1;
      if (y < 0 || y >= h) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int xx = px + kx - 1;
        if (xx < 0 || xx >= w) continue;
        const float4 v = __ldg(reinterpret_cast<const float4*>(x + ((f * h + y) * w + xx) * C + c));
        if (ky == 1 && kx == 1) centre = v;
        const int tap = ky * 3 + kx;
        acc.x += wreg[0][tap] * v.x;
        acc.y += wreg[1][tap] * v.y;
        acc.z += wreg[2][tap] * v.z;
        acc.w += wreg[3][tap] * v.w;
      }
    }
    const float4 v = make_float4(acc.x + centre.x, acc.y + centre.y, acc.z + centre.z, acc.w + centre.w);
    const long long o = t * C + c;
    *reinterpret_cast<float4*>(out + o) = v;
    if (hi) store16x4(hi + o, plane, v.x, v.y, v.z, v.w);
   }
  }
}

// ------------------------------------------------------------------------------------------
// fold: overlap-add of per-token patches back to the feature map (nn.Fold, ffn_base.py:57-75 /
// model.py:103-109). The hidden vector of a token is stored position-major: index p*C + c with
// p = ky*kw + kx (the Linear's output rows are permuted accordingly at weight-pack time), so
// both the gather here and the scatter in unfold are coalesced along c.
//   img[b,y,x,c] = scale(y,x) * sum_{patches covering (y,x)} hid[b, token, p, c]   (+ add[b,y,x,c])
// scale = 1/coverage-count when `normalize` (FusionFeedForward) else 1 (Vec2Patch).
// ------------------------------------------------------------------------------------------
// Sum of the patch entries covering pixel (y, x) of frame b, for kernels with ceil(k / stride) <= 3 (the model's 7x7 /
// stride 3): the <= 3x3 candidate loads are issued together (predicated) and added in the order of the general loops
// below (ty, tx descending) — the looped form keeps ONE load in flight per warp (each add waits for its load), which
// bounded both fold kernels at ~2.8-3.4 TB/s.
__device__ __forceinline__ float4 fold_gather3(const float* __restrict__ hid, int b, int th, int tw, int hidden, int C,
                                               int c, int kh, int kw, int st, int pd, int y, int x, int ty_hi,
                                               int tx_hi, int& cnt) {
  float4 v[3][3];
  bool ok[3][3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const int ty = ty_hi - i, ky = y + pd - st * ty;
    const bool oky = ty >= 0 && ky < kh;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const int tx = tx_hi - j, kx = x + pd - st * tx;
      ok[i][j] = oky && tx >= 0 && kx < kw;
      // candidates outside the coverage load a fixed valid address instead (an L1 hit, result unused): unconditional
      // loads are what lets the compiler issue all nine before the first add
      const float* src = ok[i][j] ? hid + ((static_cast<long long>(b) * th + ty) * tw + tx) * hidden + (ky * kw + kx) * C + c
                                  : hid + c;
      v[i][j] = __ldg(reinterpret_cast<const float4*>(src));
    }
  }
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  cnt = 0;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      if (ok[i][j]) {
        acc.x += v[i][j].x; acc.y += v[i][j].y; acc.z += v[i][j].z; acc.w += v[i][j].w;
        ++cnt;
      }
  return acc;
}

__global__ void fold_kernel(const float* __restrict__ hid, int bt, int th, int tw, int C, int kh, int kw, int st,
                            int pd, int OH, int OW, int normalize, const float* __restrict__ add,
                            float* __restrict__ out, __nv_bfloat16* __restrict__ hi, long long plane) {
  pdl_launch_dependents();
  pdl_wait();
  // one block = one output row (b, y); threadIdx.x = float4 channel group, threadIdx.y strides over x.
  // The contributing token rows are block-uniform; no per-element integer divisions by runtime values.
  const int C4 = C / 4;
  const int hidden = kh * kw * C;
  const int b = blockIdx.x / OH, y = blockIdx.x - b * OH;
  const int c = threadIdx.x * 4;
  if (threadIdx.x >= C4) return;
  const int ty_hi = min((y + pd) / st, th - 1);
  const bool cov3 = (kh + st - 1) / st <= 3 && (kw + st - 1) / st <= 3;
  for (int x = threadIdx.y; x < OW; x += blockDim.y) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    int cnt = 0;
    const int tx_hi = min((x + pd) / st, tw - 1);
    if (cov3) acc = fold_gather3(hid, b, th, tw, hidden, C, c, kh, kw, st, pd, y, x, ty_hi, tx_hi, cnt);
    else for (int ty = ty_hi; ty >= 0; --ty) {
      const int ky = y + pd - st * ty;
      if (ky >= kh) break;
      for (int tx = tx_hi; tx >= 0; --tx) {
        const int kx = x + pd - st * tx;
        if (kx >= kw) break;
        const float4 v = __ldg(reinterpret_cast<const float4*>(
            hid + ((static_cast<long long>(b) * th + ty) * tw + tx) * hidden + (ky * kw + kx) * C + c));
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        ++cnt;
      }
    }
    if (normalize) {
      const float sc = 1.f / static_cast<float>(cnt);
      acc.x *= sc; acc.y *= sc; acc.z *= sc; acc.w *= sc;
    }
    const long long o = ((static_cast<long long>(b) * OH + y) * OW + x) * C + c;
    if (add) {
      const float4 a4 = __ldg(reinterpret_cast<const float4*>(add + o));
      acc.x += a4.x; acc.y += a4.y; acc.z += a4.z; acc.w += a4.w;
    }
    if (out) *reinterpret_cast<float4*>(out + o) = acc;
    if (hi) store16x4(hi + o, plane, acc.x, acc.y, acc.z, acc.w);
  }
}

// unfold (+ReLU): feature map -> per-token patches, split-bf16 (nn.Unfold + ReLU, ffn_base.py:57-75,40).
// One block = one token; threadIdx.x = float4 channel group, threadIdx.y strides over the kh*kw positions.
__global__ void unfold_kernel(const float* __restrict__ img, int bt, int th, int tw, int C, int kh, int kw, int st,
                              int pd, int OH, int OW, int relu, __nv_bfloat16* __restrict__ hi, long long plane) {
  pdl_launch_dependents();
  pdl_wait();
  const int C4 = C / 4;
  if (threadIdx.x >= C4) return;
  const int P = kh * kw;
  const int tok = blockIdx.x;
  const int b = tok / (th * tw);
  const int rem = tok - b * th * tw;
  const int ty = rem / tw, tx = rem - ty * tw;
  const int c = threadIdx.x * 4;
  int ky = threadIdx.y / kw, kx = threadIdx.y - ky * kw;  // advanced incrementally below
  const int dky = blockDim.y / kw, dkx = blockDim.y - dky * kw;
  for (int pidx = threadIdx.y; pidx < P; pidx += blockDim.y) {
    const int y = ty * st + ky - pd, x = tx * st + kx - pd;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (y >= 0 && y < OH && x >= 0 && x < OW)
      v = __ldg(reinterpret_cast<const float4*>(img + ((static_cast<long long>(b) * OH + y) * OW + x) * C + c));
    if (relu) {
      v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
    }
    const long long o = (static_cast<long long>(tok) * P + pidx) * C + c;
    store_split4(hi + o, hi + plane + o, v.x, v.y, v.z, v.w);
    ky += dky;
    kx += dkx;
    if (kx >= kw) { kx -= kw; ++ky; }
  }
}

// fold -> (divide by coverage) -> unfold -> ReLU of the fusion FFN (ffn_base.py:57-75) WITHOUT the image round trip:
// every entry of a token's hidden patch belongs to exactly one pixel of the folded feature map, and the unfolded value
// at that entry is the (normalised) sum over all entries that map to the same pixel. One block = one image row (b, y):
// for each pixel the <= 9 covering (token, patch position) entries are summed in the same order as fold_kernel
// (bit-identical to fgt_fold + fgt_unfold), scaled, rectified, split once and written back to those same entries.
// Pixels that no patch covers do not exist for kernel >= stride; entries whose pixel lies in the padding ring are
// zeros (nn.Unfold pads with zeros) and are written by the second loop.
__global__ void fold_unfold_kernel(const float* __restrict__ hid, int bt, int th, int tw, int C, int kh, int kw, int st,
                                   int pd, int OH, int OW, int relu, __nv_bfloat16* __restrict__ hi, long long plane) {
  pdl_launch_dependents();
  pdl_wait();
  const int C4 = C / 4;
  if (threadIdx.x >= C4) return;
  const int hidden = kh * kw * C;
  const int c = threadIdx.x * 4;
  // rows y in [-pd, OH + pd): the padded rows only produce zeros. blockIdx.y splits the row into gridDim.y segments
  // (more blocks in flight: the kernel is latency-bound with one block per row)
  const int HP = OH + 2 * pd;
  const int b = blockIdx.x / HP, y = blockIdx.x - b * HP - pd;
  const bool y_in = y >= 0 && y < OH;
  const int ty_hi = min((y + pd) / st, th - 1);
  const bool cov3 = (kh + st - 1) / st <= 3 && (kw + st - 1) / st <= 3;
  const int seg = (OW + 2 * pd + gridDim.y - 1) / gridDim.y;
  const int x_lo = static_cast<int>(blockIdx.y) * seg - pd, x_hi = min(x_lo + seg, OW + pd);
  for (int x = x_lo + static_cast<int>(threadIdx.y); x < x_hi; x += blockDim.y) {
    const bool in = y_in && x >= 0 && x < OW;
    const int tx_hi = min((x + pd) / st, tw - 1);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    int cnt = 0;
    if (in) {
      if (cov3) acc = fold_gather3(hid, b, th, tw, hidden, C, c, kh, kw, st, pd, y, x, ty_hi, tx_hi, cnt);
      else for (int ty = ty_hi; ty >= 0; --ty) {
        const int ky = y + pd - st * ty;
        if (ky >= kh) break;
        for (int tx = tx_hi; tx >= 0; --tx) {
          const int kx = x + pd - st * tx;
          if (kx >= kw) break;
          const float4 v = __ldg(reinterpret_cast<const float4*>(
              hid + ((static_cast<long long>(b) * th + ty) * tw + tx) * hidden + (ky * kw + kx) * C + c));
          acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
          ++cnt;
        }
      }
      const float sc = 1.f / static_cast<float>(cnt);
      acc.x *= sc; acc.y *= sc; acc.z *= sc; acc.w *= sc;
      if (relu) {
        acc.x = fmaxf(acc.x, 0.f); acc.y = fmaxf(acc.y, 0.f); acc.z = fmaxf(acc.z, 0.f); acc.w = fmaxf(acc.w, 0.f);
      }
    }
    uint32_t h0, l0 = 0u, h1, l1 = 0u;
    if (plane == 0) {  // single-plane fp16 patches (mixed precision)
      h0 = pack_f16x2(acc.x, acc.y);
      h1 = pack_f16x2(acc.z, acc.w);
    } else {
      split_bf16x2(acc.x, acc.y, h0, l0);
      split_bf16x2(acc.z, acc.w, h1, l1);
    }
    for (int ty = ty_hi; ty >= 0; --ty) {
      const int ky = y + pd - st * ty;
      if (ky >= kh) break;
      if (ky < 0) continue;
      for (int tx = tx_hi; tx >= 0; --tx) {
        const int kx = x + pd - st * tx;
        if (kx >= kw) break;
        if (kx < 0) continue;
        const long long o = ((static_cast<long long>(b) * th + ty) * tw + tx) * hidden + (ky * kw + kx) * C + c;
        *reinterpret_cast<uint2*>(hi + o) = make_uint2(h0, h1);
        if (plane) *reinterpret_cast<uint2*>(hi + plane + o) = make_uint2(l0, l1);
      }
    }
  }
}

// nearest x2 upsampling of an NHWC split tensor (F.interpolate(scale_factor=2), network_blocks_2d.py:58-60); with both
// plane offsets 0, of a single-plane fp16 tensor (mixed-precision LAFC). A bit copy of 8 16-bit elements per thread.
__global__ void upsample2x_kernel(const __nv_bfloat16* __restrict__ in, long long in_plane, int n, int H, int W,
                                  int C, __nv_bfloat16* __restrict__ out, long long out_plane) {
  pdl_launch_dependents();
  pdl_wait();
  const int C8 = C / 8;
  const int planes = in_plane == 0 ? 1 : 2;
  const long long total = planes * static_cast<long long>(n) * (2 * H) * (2 * W) * C8;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % C8) * 8;
    long long r = i / C8;
    const int x = static_cast<int>(r % (2 * W));
    r /= (2 * W);
    const int y = static_cast<int>(r % (2 * H));
    r /= (2 * H);
    const int b = static_cast<int>(r % n);
    const int pl = static_cast<int>(r / n);
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(
        in + pl * in_plane + ((static_cast<long long>(b) * H + (y >> 1)) * W + (x >> 1)) * C + c));
    *reinterpret_cast<uint4*>(out + pl * out_plane + ((static_cast<long long>(b) * 2 * H + y) * 2 * W + x) * C + c) = v;
  }
}

// 16-bit output of the CUDA-core producers: split-bf16 (lo plane `plane` elements after hi, plane > 0) or single-plane
// fp16 (plane == 0); both are stored 4 elements (8 bytes) at a time.
static bool out16_ok(const void* hi, long long plane) {
  return hi == nullptr || (plane >= 0 && plane % 4 == 0 && (reinterpret_cast<uintptr_t>(hi) & 7) == 0);
}

static int grid_for(long long work_items, int block) {
  long long g = (work_items + block - 1) / block;
  const long long cap = static_cast<long long>(num_sms()) * 16;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return static_cast<int>(g);
}

// ------------------------------------------------------------------------------------------
// tapsum: second half of a k x k convolution with a handful of output channels (FGT decoder's final
// 64->3 conv, RAFT's flow head 256->2), computed "taps as N": a 1x1 GEMM first produces
// Y[p, tap*cout + c] = <W[c,:,tap], in[p,:]> for every input pixel p (the A tile is read ONCE instead of
// once per tap, which is what bounds a tiny-N implicit GEMM), then
//   out[n, y, x, c] = act(bias[c] + sum_tap Y[tap*cout + c][(n, y + ty - py, x + tx - px)])   (zero outside).
// Y is column-planar ([column][pixel], the GEMM's strided-store epilogue writes it coalesced), so every one
// of the k*k*cout reads of a warp is one contiguous 128-byte run of pixels.
// ------------------------------------------------------------------------------------------
constexpr int kTapsumMaxC = 4;

__global__ void tapsum_kernel(const float* __restrict__ Y, int H, int W, int cout, int kx, int ky, int px, int py,
                              long long ycol, const float* __restrict__ bias, int act, float* __restrict__ out,
                              long long os_n, long long os_y, long long os_x, long long os_c) {
  pdl_launch_dependents();
  pdl_wait();
  const int x = blockIdx.x * 32 + threadIdx.x;
  const int y = blockIdx.y * 8 + threadIdx.y;
  const int n = blockIdx.z;
  if (x >= W || y >= H) return;
  float acc[kTapsumMaxC];
#pragma unroll
  for (int c = 0; c < kTapsumMaxC; ++c) acc[c] = (c < cout && bias) ? __ldg(bias + c) : 0.f;
  for (int ty = 0; ty < ky; ++ty) {
    const int yy = y + ty - py;
    if (yy < 0 || yy >= H) continue;
    for (int tx = 0; tx < kx; ++tx) {
      const int xx = x + tx - px;
      if (xx < 0 || xx >= W) continue;
      const float* col = Y + (ty * kx + tx) * cout * ycol + (static_cast<long long>(n) * H + yy) * W + xx;
#pragma unroll
      for (int c = 0; c < kTapsumMaxC; ++c)
        if (c < cout) acc[c] += __ldg(col + c * ycol);
    }
  }
  float* o = out + n * os_n + y * os_y + x * os_x;
#pragma unroll
  for (int c = 0; c < kTapsumMaxC; ++c) {
    if (c < cout) {
      float v = acc[c];
      if (act == FGT_ACT_TANH) v = tanhf(v);
      else if (act == FGT_ACT_RELU) v = fmaxf(v, 0.f);
      else if (act == FGT_ACT_SIGMOID) v = 1.f / (1.f + expf(-v));
      else if (act == FGT_ACT_LEAKY02) v = v > 0.f ? v : 0.2f * v;
      o[c * os_c] = v;
    }
  }
}

}  // namespace fgt

using namespace fgt;

extern "C" int fgt_pack_nchw(const float* src0, int c0, const float* src1, int c1, int n, int H, int W, int pad,
                             int cpad, void* out_hi, long long out_plane, fgt_stream_t stream) {
  FGT_REQUIRE(src0 && c0 >= 1 && c0 + c1 <= cpad && cpad % 8 == 0 && (c1 == 0 || src1), FGT_ERR_ARG,
              "pack_nchw: c0=%d c1=%d cpad=%d", c0, c1, cpad);
  const long long total = static_cast<long long>(n) * (H + 2 * pad) * (W + 2 * pad);
  launch_k(pack_nchw_kernel, dim3(grid_for(total, 256)), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream), 
      src0, c0, src1, c1, n, H, W, pad, cpad, reinterpret_cast<__nv_bfloat16*>(out_hi), out_plane);
  FGT_CUDA(cudaGetLastError());
  return FGT_OK;
}

extern "C" int fgt_im2col_nchw(const float* src0, int c0, const float* src1, int c1, int n, int H, int W, int k,
                               int stride, int pad, int replicate, int OH, int OW, int cpad, float scale, float shift,
                               void* out_hi, long long out_plane, fgt_stream_t stream) {
  FGT_REQUIRE(src0 && c0 >= 1 && (c1 == 0 || src1) && cpad % 8 == 0 && k * k * (c0 + c1) <= cpad && k >= 1 &&
                  stride >= 1,
              FGT_ERR_ARG, "im2col_nchw: k=%d cin=%d cpad=%d", k, c0 + c1, cpad);
  FGT_REQUIRE(cpad <= 256, FGT_ERR_ARG, "im2col_nchw: cpad=%d > 256", cpad);
  const dim3 blk(cpad / 8, 256 / (cpad / 8));
  const size_t smem = static_cast<size_t>(k) * (c0 + c1) * ((OW - 1) * stride + k) * sizeof(float);
  constexpr size_t kIm2colSmemMax = 160 * 1024;
  FGT_REQUIRE(smem <= kIm2colSmemMax, FGT_ERR_ARG, "im2col_nchw: %zu bytes of staged input rows exceed %zu", smem, kIm2colSmemMax);
  static bool attr_set = false;
  if (!attr_set) {
    FGT_CUDA(cudaFuncSetAttribute(im2col_nchw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kIm2colSmemMax)));
    attr_set = true;
  }
  launch_k(im2col_nchw_kernel, dim3(n * OH), dim3(blk), smem, reinterpret_cast<cudaStream_t>(stream), 
      src0, c0, src1, c1, n, H, W, k, stride, pad, replicate, OH, OW, cpad, scale, shift,
      reinterpret_cast<__nv_bfloat16*>(out_hi), out_plane);
  FGT_CUDA(cudaGetLastError());
  return FGT_OK;
}

extern "C" int fgt_rownorm(const float* a, int ca, int lda, const float* b, int cb, int ldb, const int* gather,
                           int rows_per_batch, long long total_rows, int dst_batch_rows, int dst_row0,
                           const float* gamma, const float* beta, void* out_hi, long long out_plane, float eps,
                           fgt_stream_t stream) {
  void* one[1] = {out_hi};
  return fgt_rownorm_bcast(a, ca, lda, b, cb, ldb, gather, rows_per_batch, total_rows, dst_batch_rows, dst_row0,
                           gamma, beta, one, 1, out_plane, eps, stream);
}

extern "C" int fgt_rownorm_bcast(const float* a, int ca, int lda, const float* b, int cb, int ldb, const int* gather,
                                 int rows_per_batch, long long total_rows, int dst_batch_rows, int dst_row0,
                                 const float* gamma, const float* beta, void* const* out_his_host, int n_out,
                                 long long out_plane, float eps, fgt_stream_t stream) {
  const int C = ca + cb;
  FGT_REQUIRE(out_his_host && n_out >= 1 && n_out <= kNormMaxDst, FGT_ERR_ARG, "rownorm: n_out=%d", n_out);
  NormDests dst;
  for (int q = 0; q < kNormMaxDst; ++q)
    dst.hi[q] = q < n_out ? reinterpret_cast<__nv_bfloat16*>(out_his_host[q]) : nullptr;
  dst.n = n_out;
  for (int q = 0; q < n_out; ++q) {
    FGT_REQUIRE(dst.hi[q], FGT_ERR_ARG, "rownorm: destination %d is NULL", q);
    FGT_REQUIRE(out16_ok(dst.hi[q], out_plane), FGT_ERR_ARG,
                "rownorm: destination %d misaligned or plane offset %lld not a non-negative multiple of 4", q, out_plane);
  }
  FGT_REQUIRE(out_plane != 0 || n_out == 1, FGT_ERR_ARG,
              "rownorm: single-plane fp16 output (out_plane = 0) takes one destination, got %d", n_out);
  FGT_REQUIRE(a && ca % 4 == 0 && cb % 4 == 0 && C <= 128 * kNormMaxVec && lda % 4 == 0 && (cb == 0 || (b && ldb % 4 == 0)),
              FGT_ERR_ARG, "rownorm: ca=%d cb=%d lda=%d ldb=%d", ca, cb, lda, ldb);
  FGT_REQUIRE(rows_per_batch >= 1 && total_rows >= 1, FGT_ERR_ARG, "rownorm: rows");
  FGT_REQUIRE((gamma == nullptr) == (beta == nullptr), FGT_ERR_ARG, "rownorm: gamma and beta go together");
  const int block = 256;
  launch_k(rownorm_kernel, dim3(grid_for(total_rows * 32, block)), dim3(block), 0, reinterpret_cast<cudaStream_t>(stream), 
      a, ca, lda, b, cb, ldb, gather, rows_per_batch, total_rows, dst_batch_rows, dst_row0, gamma, beta, dst,
      out_plane, eps);
  FGT_CUDA(cudaGetLastError());
  return FGT_OK;
}

extern "C" int fgt_dwpool(const float* a, int ca, const float* b, int cb, int bt, int h, int w, int k, int gh,
                          int gw, const float* weight, const float* bias, float* out, fgt_stream_t stream) {
  FGT_REQUIRE(a && weight && bias && out && k >= 1 && gh >= 1 && gw >= 1, FGT_ERR_ARG, "dwpool: bad argument");
  const long long total = static_cast<long long>(bt) * gh * gw * (ca + cb);
  launch_k(dwpool_kernel, dim3(grid_for(total, 256)), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream), a, ca, b, cb, bt, h, w, k,
                                                                                        gh, gw, weight, bias, out);
  FGT_CUDA(cudaGetLastError());
  return FGT_OK;
}

extern "C" int fgt_dwconv3x3_res(const float* x, int bt, int h, int w, int C, const float* weight, const float* bias,
                                 float* out, void* out_hi, long long out_plane, fgt_stream_t stream) {
  FGT_REQUIRE(x && weight && bias && out, FGT_ERR_ARG, "dwconv3x3_res: null argument");
  FGT_REQUIRE(C % 4 == 0, FGT_ERR_ARG, "dwconv3x3_res: C=%d must be a multiple of 4", C);
  FGT_REQUIRE(out16_ok(out_hi, out_plane), FGT_ERR_ARG,
              "dwconv3x3_res: 16-bit output misaligned or plane offset %lld not a non-negative multiple of 4", out_plane);
  const int tx = (C / 4) < 128 ? (C / 4 + 31) / 32 * 32 : 128;   // threads along channels (x), tokens of the row along y
  launch_k(dwconv3_res_kernel, dim3(bt * h, w >= 16 ? 4 : 1), dim3(tx, 256 / tx > 0 ? 256 / tx : 1), 0, reinterpret_cast<cudaStream_t>(stream), 
      x, bt, h, w, C, weight, bias, out, reinterpret_cast<__nv_bfloat16*>(out_hi), out_plane);
  FGT_CUDA(cudaGetLastError());
  return FGT_OK;
}

extern "C" int fgt_fold(const float* hid, int bt, int th, int tw, int C, int kh, int kw, int stride, int pad, int OH,
                        int OW, int normalize, const float* add, float* out, void* out_hi, long long out_plane,
                        fgt_stream_t stream) {
  FGT_REQUIRE(hid && C % 4 == 0 && (out || out_hi), FGT_ERR_ARG, "fold: C=%d", C);
  FGT_REQUIRE(C / 4 <= 64, FGT_ERR_ARG, "fold: C=%d > 256", C);
  FGT_REQUIRE(out16_ok(out_hi, out_plane), FGT_ERR_ARG,
              "fold: 16-bit output misaligned or plane offset %lld not a non-negative multiple of 4", out_plane);
  const int gx = (C / 4 + 1) / 2 * 2;  // channel groups per row of the thread block
  const dim3 blk(gx, 256 / gx);
  launch_k(fold_kernel, dim3(bt * OH), dim3(blk), 0, reinterpret_cast<cudaStream_t>(stream), 
      hid, bt, th, tw, C, kh, kw, stride, pad, OH, OW, normalize, add, out, reinterpret_cast<__nv_bfloat16*>(out_hi),
      out_plane);
  FGT_CUDA(cudaGetLastError());
  return FGT_OK;
}

extern "C" int fgt_unfold(const float* img, int bt, int th, int tw, int C, int kh, int kw, int stride, int pad,
                          int OH, int OW, int relu, void* out_hi, long long out_plane, fgt_stream_t stream) {
  FGT_REQUIRE(img && out_hi && C % 4 == 0, FGT_ERR_ARG, "unfold: C=%d", C);
  FGT_REQUIRE(C / 4 <= 64, FGT_ERR_ARG, "unfold: C=%d > 256", C);
  const int gx = (C / 4 + 1) / 2 * 2;
  const dim3 blk(gx, 256 / gx);
  launch_k(unfold_kernel, dim3(bt * th * tw), dim3(blk), 0, reinterpret_cast<cudaStream_t>(stream), 
      img, bt, th, tw, C, kh, kw, stride, pad, OH, OW, relu, reinterpret_cast<__nv_bfloat16*>(out_hi), out_plane);
  FGT_CUDA(cudaGetLastError());
  return FGT_OK;
}

extern "C" int fgt_fold_unfold(const float* hid, int bt, int th, int tw, int C, int kh, int kw, int stride, int pad,
                               int OH, int OW, int relu, void* out_hi, long long out_plane, fgt_stream_t stream) {
  FGT_REQUIRE(hid && out_hi && C % 4 == 0 && C / 4 <= 64, FGT_ERR_ARG, "fold_unfold: C=%d", C);
  FGT_REQUIRE(kh >= stride && kw >= stride, FGT_ERR_ARG, "fold_unfold: kernel %dx%d must cover the stride %d", kh, kw, stride);
  FGT_REQUIRE(out16_ok(out_hi, out_plane), FGT_ERR_ARG,
              "fold_unfold: output misaligned or plane offset %lld not a non-negative multiple of 4", out_plane);
  // every pixel of the map must lie under at least one patch (last patch ends at (th-1)*stride + kh - 1 - pad)
  FGT_REQUIRE((th - 1) * stride + kh - pad >= OH && (tw - 1) * stride + kw - pad >= OW && pad < kh && pad < kw, FGT_ERR_ARG,
              "fold_unfold: patches do not cover the %dx%d map", OH, OW);
  const int gx = (C / 4 + 1) / 2 * 2;
  const dim3 blk(gx, 256 / gx);
  launch_k(fold_unfold_kernel, dim3(bt * (OH + 2 * pad), 4), dim3(blk), 0, reinterpret_cast<cudaStream_t>(stream), hid, bt, th, tw, C, kh,
           kw, stride, pad, OH, OW, relu, reinterpret_cast<__nv_bfloat16*>(out_hi), out_plane);
  FGT_CUDA(cudaGetLastError());
  return FGT_OK;
}

extern "C" int fgt_upsample2x(const void* in_hi, long long in_plane, int n, int H, int W, int C, void* out_hi,
                              long long out_plane, fgt_stream_t stream) {
  FGT_REQUIRE(in_hi && out_hi && C % 8 == 0, FGT_ERR_ARG, "upsample2x: C=%d", C);
  FGT_REQUIRE((in_plane == 0) == (out_plane == 0) && in_plane >= 0 && out_plane >= 0, FGT_ERR_ARG,
              "upsample2x: plane offsets %lld -> %lld (both 0: fp16, both > 0: split-bf16)", in_plane, out_plane);
  const long long total = (in_plane == 0 ? 1LL : 2LL) * n * (2 * H) * (2 * W) * (C / 8);
  launch_k(upsample2x_kernel, dim3(grid_for(total, 256)), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream), 
      reinterpret_cast<const __nv_bfloat16*>(in_hi), in_plane, n, H, W, C, reinterpret_cast<__nv_bfloat16*>(out_hi),
      out_plane);
  FGT_CUDA(cudaGetLastError());
  return FGT_OK;
}

extern "C" int fgt_tapsum(const float* y, int n, int H, int W, int cout, int kx, int ky, int pad_x, int pad_y,
                          long long ycol, const float* bias, int act, float* out, long long os_n, long long os_y,
                          long long os_x, long long os_c, fgt_stream_t stream) {
  FGT_REQUIRE(y && out && n >= 1 && H >= 1 && W >= 1, FGT_ERR_ARG, "tapsum: null / empty argument");
  FGT_REQUIRE(cout >= 1 && cout <= kTapsumMaxC && kx >= 1 && ky >= 1 && ycol >= static_cast<long long>(n) * H * W,
              FGT_ERR_ARG, "tapsum: cout=%d (max %d) taps %dx%d column stride %lld", cout, kTapsumMaxC, kx, ky, ycol);
  FGT_REQUIRE(act == FGT_ACT_NONE || act == FGT_ACT_TANH || act == FGT_ACT_RELU || act == FGT_ACT_SIGMOID ||
                  act == FGT_ACT_LEAKY02, FGT_ERR_ARG, "tapsum: act=%d", act);
  const dim3 grid((W + 31) / 32, (H + 7) / 8, n);
  launch_k(tapsum_kernel, grid, dim3(32, 8), 0, reinterpret_cast<cudaStream_t>(stream), y, H, W, cout, kx, ky, pad_x,
           pad_y, ycol, bias, act, out, os_n, os_y, os_x, os_c);
  FGT_CUDA(cudaGetLastError());
  return FGT_OK;
}
