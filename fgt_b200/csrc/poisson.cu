// Batched gradient-domain (Poisson) blending: tool/utils/Poisson_blend_img.py:19-270, called per frame by the
// driver (tool/video_inpainting.py:645-656). The reference assembles a sparse over-determined system per frame
// (one equation per hole pixel and 4-neighbour with a known gradient, :176-266) and runs scipy's LSQR with default
// tolerances per colour channel; its result is the LSQR iterate at which the stopping rule fires. Here all
// F frames x 3 channels are solved together, matrix-free, by the same LSQR recurrences and stopping tests in
// fp64 (the reference's float32 operands make scipy run its bidiagonalisation in float32; fp64 iterates stop at
// the same iteration and agree to ~1e-6, tests/golden/poisson_*.npz).
//
// Layout: thread = pixel, its 3 channels in registers; pixel-space vectors v, w, x are [F, H*W, 3] doubles,
// the equation-space vector u is [F, 4, H*W, 3] (n = 0 right, 1 down, 2 left, 3 up). `code` [F, H*W] holds per
// hole pixel bit n = "equation (p, n) exists" and bit 4+n = "its neighbour lies inside the hole"; because an
// in-hole edge yields the same equation from both of its ends, (A^T u)[p] only needs p's own bits.
// Vectors are kept UNNORMALISED (u^ = beta*u, v^ = alfa*v) with the scale applied on read, so one LSQR iteration
// is two kernels, each ending in a block reduction + one double atomic per (block, channel):
//   psn_v_kernel (k): v^ = A^T u^ / beta_k - beta_k * v,          aa[k]   += |v^|^2   (alfa_k^2)
//   psn_ux_kernel(k): scalar recurrences + stopping tests of iteration k (every block recomputes them from the
//                     previous state and the finished sums; block 0 stores the new state, ping-pong by parity),
//                     x += t1 w, w = v + t2 w,                      ww[k+1] += |w|^2
//                     u^ = A v - alfa_k * u,                        bb[k+1] += |u^|^2 (beta_{k+1}^2)
// Per-iteration sums live in zero-initialised slot arrays indexed by iteration, so nothing is ever reset, and a
// system that has stopped (its own istop) is frozen while the others continue. The iteration index is a device
// counter, so a chunk of iterations is captured once as a CUDA graph and replayed. HBM/L2-bound fp64 streaming.
#include "common.h"

#include <math.h>

namespace fgt {

constexpr int kPsnThreads = 256;
constexpr int kPsnC = 3;          // colour channels (the reference hard-codes 3 columns of b, :112)
constexpr int kPsnState = 16;     // doubles per system and parity
// state slots
enum { PS_ALFA = 0, PS_RHOBAR, PS_PHIBAR, PS_ANORM, PS_DDNORM, PS_XXNORM, PS_Z, PS_CS2, PS_SN2, PS_VSCALE, PS_USCALE,
       PS_BNORM, PS_DONE, PS_ISTOP, PS_ITN, PS_BETA };

struct PsnStep {   // what the vector part of psn_ux_kernel needs
  double t1, t2, vscale, au;   // au = alfa_k * uscale_k
  int skip_all, skip_u;
};

__host__ __device__ inline double psn_sign(double a) { return a > 0.0 ? 1.0 : (a < 0.0 ? -1.0 : 0.0); }

// scipy/sparse/linalg/_isolve/lsqr.py:_sym_ortho — stable Givens rotation.
__host__ __device__ inline void psn_sym_ortho(double a, double b, double* c, double* s, double* r) {
  if (b == 0.0) { *c = psn_sign(a); *s = 0.0; *r = fabs(a); return; }
  if (a == 0.0) { *c = 0.0; *s = psn_sign(b); *r = fabs(b); return; }
  if (fabs(b) > fabs(a)) {
    const double tau = a / b;
    *s = psn_sign(b) / sqrt(1.0 + tau * tau);
    *c = *s * tau;
    *r = b / *s;
  } else {
    const double tau = b / a;
    *c = psn_sign(a) / sqrt(1.0 + tau * tau);
    *s = *c * tau;
    *r = a / *c;
  }
}

// One LSQR iteration's scalar work (scipy lsqr.py main loop, damp = 0, default-style tolerances passed in).
// prev: state after iteration k-1 (ignored for k == 0); bbk/aak/wwk: |u^_k|^2, |v^_k|^2, |w|^2 at the start of
// iteration k. Writes the state after iteration k to cur and the coefficients of the vector updates to step.
__host__ __device__ inline void psn_advance(const double* prev, double* cur, PsnStep* step, int k, double bbk,
                                            double aak, double wwk, double atol, double btol, double ctol,
                                            int iter_lim) {
  const double eps = 2.220446049250313e-16;
  if (k == 0) {   // set-up: beta u = b, alfa v = A^T u, w = v, x = 0
    const double beta = sqrt(bbk), alfa = sqrt(aak);
    for (int i = 0; i < kPsnState; ++i) cur[i] = 0.0;
    cur[PS_ALFA] = alfa;
    cur[PS_RHOBAR] = alfa;
    cur[PS_PHIBAR] = beta;
    cur[PS_CS2] = -1.0;
    cur[PS_VSCALE] = alfa > 0.0 ? 1.0 / alfa : 1.0;
    cur[PS_USCALE] = beta > 0.0 ? 1.0 / beta : 1.0;
    cur[PS_BNORM] = beta;
    cur[PS_BETA] = beta;
    cur[PS_DONE] = (alfa * beta == 0.0) ? 1.0 : 0.0;   // "the exact solution is x = 0" (istop 0)
    step->t1 = 0.0;
    step->t2 = 0.0;
    step->vscale = cur[PS_VSCALE];
    step->au = alfa * cur[PS_USCALE];
    step->skip_all = cur[PS_DONE] != 0.0;
    step->skip_u = step->skip_all;
    return;
  }
  if (prev[PS_DONE] != 0.0) {   // frozen: carry the final state forward
    for (int i = 0; i < kPsnState; ++i) cur[i] = prev[i];
    step->t1 = step->t2 = step->au = 0.0;
    step->vscale = 1.0;
    step->skip_all = step->skip_u = 1;
    return;
  }
  const double alfa_prev = prev[PS_ALFA];
  const double beta = sqrt(bbk);
  double alfa = alfa_prev, anorm = prev[PS_ANORM], vscale = prev[PS_VSCALE], uscale = 1.0;
  if (beta > 0.0) {
    anorm = sqrt(anorm * anorm + alfa_prev * alfa_prev + beta * beta);
    alfa = sqrt(aak);
    vscale = alfa > 0.0 ? 1.0 / alfa : 1.0;
    uscale = 1.0 / beta;
  }
  double cs, sn, rho;
  psn_sym_ortho(prev[PS_RHOBAR], beta, &cs, &sn, &rho);
  const double theta = sn * alfa;
  const double rhobar = -cs * alfa;
  const double phi = cs * prev[PS_PHIBAR];
  const double phibar = sn * prev[PS_PHIBAR];
  const double tau = sn * phi;
  const double t1 = phi / rho, t2 = -theta / rho;
  const double ddnorm = prev[PS_DDNORM] + wwk / (rho * rho);
  // plane rotation on the right -> estimate of |x|
  const double delta = prev[PS_SN2] * rho;
  const double gambar = -prev[PS_CS2] * rho;
  const double rhs = phi - delta * prev[PS_Z];
  const double zbar = rhs / gambar;
  const double xnorm = sqrt(prev[PS_XXNORM] + zbar * zbar);
  const double gamma = sqrt(gambar * gambar + theta * theta);
  const double z = rhs / gamma;
  // stopping tests
  const double bnorm = prev[PS_BNORM];
  const double acond = anorm * sqrt(ddnorm);
  const double rnorm = fabs(phibar);
  const double arnorm = alfa * fabs(tau);
  const double test1 = rnorm / bnorm;
  const double test2 = arnorm / (anorm * rnorm + eps);
  const double test3 = 1.0 / (acond + eps);
  const double t1_ = test1 / (1.0 + anorm * xnorm / bnorm);
  const double rtol = btol + atol * anorm * xnorm / bnorm;
  int istop = 0;
  if (k >= iter_lim) istop = 7;
  if (1.0 + test3 <= 1.0) istop = 6;
  if (1.0 + test2 <= 1.0) istop = 5;
  if (1.0 + t1_ <= 1.0) istop = 4;
  if (test3 <= ctol) istop = 3;
  if (test2 <= atol) istop = 2;
  if (test1 <= rtol) istop = 1;
  cur[PS_ALFA] = alfa;
  cur[PS_RHOBAR] = rhobar;
  cur[PS_PHIBAR] = phibar;
  cur[PS_ANORM] = anorm;
  cur[PS_DDNORM] = ddnorm;
  cur[PS_XXNORM] = prev[PS_XXNORM] + z * z;
  cur[PS_Z] = z;
  cur[PS_CS2] = gambar / gamma;
  cur[PS_SN2] = theta / gamma;
  cur[PS_VSCALE] = vscale;
  cur[PS_USCALE] = uscale;
  cur[PS_BNORM] = bnorm;
  cur[PS_DONE] = istop != 0 ? 1.0 : 0.0;
  cur[PS_ISTOP] = static_cast<double>(istop);
  cur[PS_ITN] = static_cast<double>(k);
  cur[PS_BETA] = beta;
  step->t1 = t1;
  step->t2 = t2;
  step->vscale = vscale;
  step->au = alfa * uscale;
  step->skip_all = 0;
  step->skip_u = istop != 0;
}

#ifdef __CUDACC__

// Sums kPsnC per-thread values over the block; results valid in thread 0.
__device__ __forceinline__ void psn_block_sum(double (&v)[kPsnC], double (*red)[kPsnThreads / 32]) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int c = 0; c < kPsnC; ++c) {
    double t = v[c];
    for (int o = 16; o > 0; o >>= 1) t += __shfl_down_sync(0xffffffffu, t, o);
    if (lane == 0) red[c][warp] = t;
  }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int c = 0; c < kPsnC; ++c) {
      double t = lane < (kPsnThreads >> 5) ? red[c][lane] : 0.0;
      for (int o = 4; o > 0; o >>= 1) t += __shfl_down_sync(0xffffffffu, t, o);
      v[c] = t;
    }
  }
}

__device__ __forceinline__ int psn_nb(int n, int W) { return n == 0 ? 1 : (n == 1 ? W : (n == 2 ? -1 : -W)); }

// code, u^_0 = b, bb[0] += |b|^2 (constructEquation, Poisson_blend_img.py:176-266). trg [F,H,W,3], gx [F,H,W-1,3],
// gy [F,H-1,W,3] doubles; hole / gmask / edge uint8 [F,H,W] (gmask, edge may be null = all zero).
__global__ void psn_setup_kernel(const double* __restrict__ trg, const double* __restrict__ gx,
                                 const double* __restrict__ gy, const unsigned char* __restrict__ hole,
                                 const unsigned char* __restrict__ gmask, const unsigned char* __restrict__ edge, int H,
                                 int W, int S, unsigned char* __restrict__ code, double* __restrict__ u,
                                 double* __restrict__ bb, unsigned* __restrict__ list, int* __restrict__ cnt) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ double red[kPsnC][kPsnThreads / 32];
  __shared__ int s_woff[kPsnThreads / 32], s_base;
  const int f = blockIdx.y, HW = H * W;
  const long long fb = static_cast<long long>(f) * HW;
  const int i = blockIdx.x * kPsnThreads + threadIdx.x;
  double acc[kPsnC] = {0.0, 0.0, 0.0};
  bool owns = false;
  unsigned cd = 0;
  if (i < HW) {
    if (hole[fb + i]) {
      const int y = i / W, x = i - y * W;
      const bool e_p = edge && edge[fb + i];
#pragma unroll
      for (int n = 0; n < 4; ++n) {
        const int qy = y + (n == 1) - (n == 3), qx = x + (n == 0) - (n == 2);
        if (qy < 0 || qy >= H || qx < 0 || qx >= W) continue;
        const int q = qy * W + qx;
        if (e_p || (edge && edge[fb + q])) continue;
        const int owner = (n == 0 || n == 1) ? i : q;   // pixel owning the forward difference between p and q
        if (gmask && gmask[fb + owner]) continue;
        const bool inh = hole[fb + q] != 0;
        cd |= (1u << n) | (inh ? (16u << n) : 0u);
        const int oy = owner / W, ox = owner - oy * W;
        const double* g = (n == 0 || n == 2) ? gx + (static_cast<long long>(f) * H * (W - 1) + oy * (W - 1) + ox) * kPsnC
                                             : gy + (static_cast<long long>(f) * (H - 1) * W + oy * W + ox) * kPsnC;
        const double sgn = (n == 0 || n == 1) ? -1.0 : 1.0;
#pragma unroll
        for (int c = 0; c < kPsnC; ++c) {
          const double b = sgn * g[c] + (inh ? 0.0 : trg[(fb + q) * kPsnC + c]);
          u[((static_cast<long long>(f) * 4 + n) * HW + i) * kPsnC + c] = b;
          acc[c] += b * b;
        }
      }
    }
    code[fb + i] = static_cast<unsigned char>(cd);
    owns = (cd & 15u) != 0u;
  }
  // compaction: pixels owning equations are appended to list[f] (raster order inside a block, blocks in
  // arrival order), so the iteration kernels only launch threads that have work
  {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned bal = __ballot_sync(0xffffffffu, owns);
    if (lane == 0) s_woff[warp] = __popc(bal);
    __syncthreads();
    if (threadIdx.x == 0) {
      int tot = 0;
      for (int k = 0; k < kPsnThreads / 32; ++k) {
        const int c = s_woff[k];
        s_woff[k] = tot;
        tot += c;
      }
      s_base = tot ? atomicAdd(&cnt[f], tot) : 0;
    }
    __syncthreads();
    if (owns) list[fb + s_base + s_woff[warp] + __popc(bal & ((1u << lane) - 1u))] = static_cast<unsigned>(i) | (cd << 24);
    __syncthreads();
  }
  psn_block_sum(acc, red);
  if (threadIdx.x == 0)
    for (int c = 0; c < kPsnC; ++c)
      if (acc[c] != 0.0) atomicAdd(&bb[f * kPsnC + c], acc[c]);
}

// Iteration kernels. The iteration index lives on the device (kctr[0]: read by psn_v, written by psn_ux; kctr[1]:
// read by psn_ux, written by psn_v — no kernel reads a word it writes), so the launch sequence has no changing
// parameter and a chunk of iterations replays as ONE CUDA graph. A list entry packs the pixel index (low 24 bits)
// and its equation code (high 8 bits); entries past a frame's count are 0 = "no equation".
__global__ void psn_v_kernel(const unsigned* __restrict__ list, int H, int W, int S, const double* __restrict__ u,
                             double* __restrict__ v, const double* __restrict__ bb, double* __restrict__ aa,
                             const double* __restrict__ state, int* __restrict__ kctr) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ double red[kPsnC][kPsnThreads / 32];
  __shared__ double s_inv[kPsnC], s_coef[kPsnC];
  __shared__ int s_act[kPsnC];
  const int f = blockIdx.y, HW = H * W;
  const int k = kctr[0];
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) kctr[1] = k;
  const long long fb = static_cast<long long>(f) * HW;
  const int j = blockIdx.x * kPsnThreads + threadIdx.x;
  const unsigned entry = j < HW ? list[fb + j] : 0u;      // issued before the scalar prologue
  if (threadIdx.x < kPsnC) {
    const int s = f * kPsnC + threadIdx.x;
    const double* st = state + (static_cast<long long>((k + 1) & 1) * S + s) * kPsnState;   // parity of k-1
    const bool done = k >= 1 && st[PS_DONE] != 0.0;
    const double beta = sqrt(bb[static_cast<long long>(k) * S + s]);
    const bool act = !done && beta > 0.0;
    s_act[threadIdx.x] = act;
    s_inv[threadIdx.x] = act ? 1.0 / beta : 0.0;
    s_coef[threadIdx.x] = (act && k >= 1) ? beta * st[PS_VSCALE] : 0.0;
  }
  const unsigned cd = entry >> 24;
  const int i = static_cast<int>(entry & 0xffffffu);
  double acc[kPsnC] = {0.0, 0.0, 0.0};
  double s[kPsnC] = {0.0, 0.0, 0.0}, vo[kPsnC] = {0.0, 0.0, 0.0};
  if (cd & 15u) {
#pragma unroll
    for (int n = 0; n < 4; ++n) {
      if (!((cd >> n) & 1u)) continue;
      const double* up = u + ((static_cast<long long>(f) * 4 + n) * HW + i) * kPsnC;
#pragma unroll
      for (int c = 0; c < kPsnC; ++c) s[c] += up[c];
      if ((cd >> (4 + n)) & 1u) {   // the neighbour's equation towards p: coefficient -1 at p
        const double* uq = u + ((static_cast<long long>(f) * 4 + ((n + 2) & 3)) * HW + i + psn_nb(n, W)) * kPsnC;
#pragma unroll
        for (int c = 0; c < kPsnC; ++c) s[c] -= uq[c];
      }
    }
#pragma unroll
    for (int c = 0; c < kPsnC; ++c) vo[c] = v[(fb + i) * kPsnC + c];
  }
  __syncthreads();
  if (cd & 15u) {
    double* vp = v + (fb + i) * kPsnC;
#pragma unroll
    for (int c = 0; c < kPsnC; ++c) {
      if (!s_act[c]) continue;
      const double nv = s[c] * s_inv[c] - s_coef[c] * vo[c];
      vp[c] = nv;
      acc[c] = nv * nv;
    }
  }
  psn_block_sum(acc, red);
  if (threadIdx.x == 0)
    for (int c = 0; c < kPsnC; ++c)
      if (acc[c] != 0.0) atomicAdd(&aa[static_cast<long long>(k) * S + f * kPsnC + c], acc[c]);
}

__global__ void psn_ux_kernel(const unsigned* __restrict__ list, int H, int W, int S, double* __restrict__ u,
                              const double* __restrict__ v, double* __restrict__ w, double* __restrict__ x,
                              double* __restrict__ bb, const double* __restrict__ aa, double* __restrict__ ww,
                              double* __restrict__ state, int* __restrict__ kctr, double atol, double btol, double ctol,
                              int iter_lim) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ double red[kPsnC][kPsnThreads / 32];
  __shared__ PsnStep s_step[kPsnC];
  const int f = blockIdx.y, HW = H * W;
  const int k = kctr[1];
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) kctr[0] = k + 1;
  const long long fb = static_cast<long long>(f) * HW;
  const int j = blockIdx.x * kPsnThreads + threadIdx.x;
  const unsigned entry = j < HW ? list[fb + j] : 0u;
  const unsigned cd = entry >> 24;
  const int i = static_cast<int>(entry & 0xffffffu);
  // the u / v operands (27 of this thread's 33 loads) are issued before the barrier, i.e. while threads 0..2 run
  // the scalar recurrence; w and x are touched after it
  double vown[kPsnC] = {0.0, 0.0, 0.0};
  double uo[4][kPsnC], vq[4][kPsnC];
#pragma unroll
  for (int n = 0; n < 4; ++n)
#pragma unroll
    for (int c = 0; c < kPsnC; ++c) uo[n][c] = vq[n][c] = 0.0;
  if (cd & 15u) {
#pragma unroll
    for (int c = 0; c < kPsnC; ++c) vown[c] = v[(fb + i) * kPsnC + c];
#pragma unroll
    for (int n = 0; n < 4; ++n) {
      if (!((cd >> n) & 1u)) continue;
#pragma unroll
      for (int c = 0; c < kPsnC; ++c) uo[n][c] = u[((static_cast<long long>(f) * 4 + n) * HW + i) * kPsnC + c];
      if ((cd >> (4 + n)) & 1u) {
#pragma unroll
        for (int c = 0; c < kPsnC; ++c) vq[n][c] = v[(fb + i + psn_nb(n, W)) * kPsnC + c];
      }
    }
  }
  if (threadIdx.x < kPsnC) {
    const int s = f * kPsnC + threadIdx.x;
    const double* prev = state + (static_cast<long long>((k + 1) & 1) * S + s) * kPsnState;
    double cur[kPsnState];
    PsnStep st;
    const long long slot = static_cast<long long>(k) * S + s;
    psn_advance(prev, cur, &st, k, bb[slot], aa[slot], ww[slot], atol, btol, ctol, iter_lim);
    s_step[threadIdx.x] = st;
    if (blockIdx.x == 0) {
      double* dst = state + (static_cast<long long>(k & 1) * S + s) * kPsnState;
      for (int q = 0; q < kPsnState; ++q) dst[q] = cur[q];
    }
  }
  __syncthreads();
  double accw[kPsnC] = {0.0, 0.0, 0.0}, accu[kPsnC] = {0.0, 0.0, 0.0};
  if (cd & 15u) {
    double vn[kPsnC];
#pragma unroll
    for (int c = 0; c < kPsnC; ++c) {
      const PsnStep& st = s_step[c];
      vn[c] = vown[c] * st.vscale;
      if (st.skip_all) continue;
      const double wo = w[(fb + i) * kPsnC + c];
      x[(fb + i) * kPsnC + c] += st.t1 * wo;
      const double wn = vn[c] + st.t2 * wo;
      w[(fb + i) * kPsnC + c] = wn;
      accw[c] = wn * wn;
    }
#pragma unroll
    for (int n = 0; n < 4; ++n) {
      if (!((cd >> n) & 1u)) continue;
#pragma unroll
      for (int c = 0; c < kPsnC; ++c) {
        const PsnStep& st = s_step[c];
        if (st.skip_u) continue;
        const double av = vn[c] - vq[n][c] * st.vscale;   // vq is 0 when the neighbour lies outside the hole
        const double nu = av - st.au * uo[n][c];
        u[((static_cast<long long>(f) * 4 + n) * HW + i) * kPsnC + c] = nu;
        accu[c] += nu * nu;
      }
    }
  }
  psn_block_sum(accw, red);
  __syncthreads();
  if (threadIdx.x == 0)
    for (int c = 0; c < kPsnC; ++c)
      if (accw[c] != 0.0) atomicAdd(&ww[static_cast<long long>(k + 1) * S + f * kPsnC + c], accw[c]);
  psn_block_sum(accu, red);
  if (threadIdx.x == 0)
    for (int c = 0; c < kPsnC; ++c)
      if (accu[c] != 0.0) atomicAdd(&bb[static_cast<long long>(k + 1) * S + f * kPsnC + c], accu[c]);
}

// out = hole ? float64(float32(x)) : trg — the reference stores the reconstruction in a float32 image before
// blending in float64 (Poisson_blend_img.py:29,40-44). unf = hole & !clr_fwd & !clr_bwd (:172).
__global__ void psn_finish_kernel(const double* __restrict__ trg, const unsigned char* __restrict__ hole,
                                  const double* __restrict__ x, long long pixels, double* __restrict__ out,
                                  const unsigned char* __restrict__ clr, unsigned char* __restrict__ unf) {
  pdl_launch_dependents();
  pdl_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < pixels;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const bool h = hole[i] != 0;
#pragma unroll
    for (int c = 0; c < kPsnC; ++c)
      out[i * kPsnC + c] = h ? static_cast<double>(static_cast<float>(x[i * kPsnC + c])) : trg[i * kPsnC + c];
    if (unf) unf[i] = h && !clr[i] && !clr[pixels + i];
  }
}

// The two raster sweeps of solvePoisson's connectivity check (Poisson_blend_img.py:139-172): a hole pixel is
// cleared when a cleared 4-neighbour earlier in the sweep has a known gradient towards it. One warp per
// (frame, sweep): rows in sweep order, 32 columns per step as ballot words, the in-row dependency
//   cleared[j] = G[j] | (P[j] & cleared[j-1])   solved by a Kogge-Stone prefix on the words.
// Sweep 0 (forward): G = !hole | (cleared_above & ok_above), P = ok[i, j-1]; sweep 1 (backward, columns mirrored):
// G = !hole | (cleared_below & ok[i, j]), P = ok[i, j] (the reference tests the pixel's own gradientMask there).
__global__ void psn_sweep_kernel(const unsigned char* __restrict__ hole, const unsigned char* __restrict__ gmask, int F,
                                 int H, int W, unsigned char* __restrict__ clr) {
  pdl_launch_dependents();
  pdl_wait();
  const int f = blockIdx.x, back = blockIdx.y, lane = threadIdx.x;
  const long long fb = static_cast<long long>(f) * H * W;
  unsigned char* out = clr + (static_cast<long long>(back) * F + f) * H * W;
  for (int r = 0; r < H; ++r) {
    const int y = back ? H - 1 - r : r;
    const int yp = back ? y + 1 : y - 1;   // row already swept
    unsigned carry = 0;
    for (int g0 = 0; g0 < W; g0 += 32) {
      const int jj = g0 + lane;            // position along the sweep direction
      const int xcol = back ? W - 1 - jj : jj;
      bool G = false, P = false;
      if (jj < W) {
        const long long p = fb + static_cast<long long>(y) * W + xcol;
        G = !hole[p];
        if (!G && r > 0) {
          const long long pv = fb + static_cast<long long>(yp) * W + xcol;
          const bool okv = !(gmask && gmask[back ? p : pv]);
          G = out[static_cast<long long>(yp) * W + xcol] && okv;
        }
        if (jj > 0) P = !(gmask && gmask[back ? p : p - 1]);
      }
      unsigned g = __ballot_sync(0xffffffffu, G), pr = __ballot_sync(0xffffffffu, P);
      g |= pr & carry;                     // carry enters at bit 0
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        g |= pr & (g << d);
        pr &= pr << d;
      }
      if (jj < W) out[static_cast<long long>(y) * W + xcol] = (g >> lane) & 1u;
      carry = g >> 31;
    }
    __syncwarp();
  }
}

#endif  // __CUDACC__

}  // namespace fgt

using namespace fgt;

static dim3 psn_grid(int F, int H, int W) { return dim3((H * W + kPsnThreads - 1) / kPsnThreads, F); }

extern "C" int fgt_poisson_setup(const double* trg, const double* gx, const double* gy, const unsigned char* hole,
                                 const unsigned char* gmask, const unsigned char* edge, int F, int H, int W,
                                 unsigned char* code, double* u, double* bb, unsigned* list, int* cnt,
                                 fgt_stream_t stream) {
  FGT_REQUIRE(trg && gx && gy && hole && code && u && bb && list && cnt && F >= 1 && H >= 2 && W >= 2, FGT_ERR_ARG,
              "poisson_setup: bad argument");
  FGT_REQUIRE(static_cast<long long>(H) * W < (1LL << 24), FGT_ERR_ARG, "poisson_setup: H*W must be below 2^24");
  FGT_LAUNCH(psn_setup_kernel, psn_grid(F, H, W), dim3(kPsnThreads), 0, stream, trg, gx, gy, hole, gmask, edge, H, W,
             F * kPsnC, code, u, bb, list, cnt);
  return FGT_OK;
}

static int psn_enqueue(const unsigned* list, int max_cnt, int F, int H, int W, double* u, double* v, double* w, double* x,
                       double* bb, double* aa, double* ww, double* state, int* kctr, int iters, double atol, double btol,
                       double conlim, int iter_lim, fgt_stream_t st) {
  // one block column even when no pixel owns an equation: block 0 of every frame carries the scalar state
  const dim3 grid(max_cnt > 0 ? (max_cnt + kPsnThreads - 1) / kPsnThreads : 1, F);
  const int S = F * kPsnC;
  const double ctol = conlim > 0.0 ? 1.0 / conlim : 0.0;
  for (int it = 0; it < iters; ++it) {
    FGT_LAUNCH(psn_v_kernel, grid, dim3(kPsnThreads), 0, st, list, H, W, S, static_cast<const double*>(u), v,
               static_cast<const double*>(bb), aa, static_cast<const double*>(state), kctr);
    FGT_LAUNCH(psn_ux_kernel, grid, dim3(kPsnThreads), 0, st, list, H, W, S, u, static_cast<const double*>(v), w, x, bb,
               static_cast<const double*>(aa), ww, state, kctr, atol, btol, ctol, iter_lim);
  }
  return FGT_OK;
}

#define PSN_ITER_ARGS_OK                                                                                              \
  (list && u && v && w && x && bb && aa && ww && state && kctr && F >= 1 && iters >= 1 && max_cnt >= 0 && max_cnt <= H * W)

extern "C" int fgt_poisson_iters(const unsigned* list, int max_cnt, int F, int H, int W, double* u, double* v, double* w,
                                 double* x, double* bb, double* aa, double* ww, double* state, int* kctr, int iters,
                                 double atol, double btol, double conlim, int iter_lim, fgt_stream_t stream) {
  FGT_REQUIRE(PSN_ITER_ARGS_OK, FGT_ERR_ARG, "poisson_iters: bad argument");
  return psn_enqueue(list, max_cnt, F, H, W, u, v, w, x, bb, aa, ww, state, kctr, iters, atol, btol, conlim, iter_lim,
                     stream);
}

// The same `iters` iteration pairs captured once into an executable CUDA graph (the iteration index is on the
// device, so every replay continues where the previous one stopped).
extern "C" int fgt_poisson_graph_create(const unsigned* list, int max_cnt, int F, int H, int W, double* u, double* v,
                                        double* w, double* x, double* bb, double* aa, double* ww, double* state,
                                        int* kctr, int iters, double atol, double btol, double conlim, int iter_lim,
                                        void** exec_out) {
  FGT_REQUIRE(PSN_ITER_ARGS_OK && exec_out, FGT_ERR_ARG, "poisson_graph_create: bad argument");
  *exec_out = nullptr;
  cudaStream_t cs;
  FGT_CUDA(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t exec = nullptr;
  int rc = FGT_OK;
  cudaError_t e = cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal);
  if (e == cudaSuccess) {
    rc = psn_enqueue(list, max_cnt, F, H, W, u, v, w, x, bb, aa, ww, state, kctr, iters, atol, btol, conlim, iter_lim, cs);
    e = cudaStreamEndCapture(cs, &graph);   // always end the capture, also after a failed launch
    if (rc == FGT_OK && e == cudaSuccess) e = cudaGraphInstantiate(&exec, graph, 0);
  }
  if (graph) cudaGraphDestroy(graph);
  cudaStreamDestroy(cs);
  if (rc != FGT_OK) return rc;
  if (e != cudaSuccess) return set_err(FGT_ERR_CUDA, "poisson_graph_create: %s", cudaGetErrorString(e));
  *exec_out = exec;
  return FGT_OK;
}

extern "C" int fgt_poisson_graph_launch(void* exec, fgt_stream_t stream) {
  FGT_REQUIRE(exec, FGT_ERR_ARG, "poisson_graph_launch: null graph");
  FGT_CUDA(cudaGraphLaunch(reinterpret_cast<cudaGraphExec_t>(exec), stream));
  return FGT_OK;
}

extern "C" int fgt_poisson_graph_destroy(void* exec) {
  if (exec) FGT_CUDA(cudaGraphExecDestroy(reinterpret_cast<cudaGraphExec_t>(exec)));
  return FGT_OK;
}

extern "C" int fgt_poisson_unfilled(const unsigned char* hole, const unsigned char* gmask, int F, int H, int W,
                                    unsigned char* clr, fgt_stream_t stream) {
  FGT_REQUIRE(hole && clr && F >= 1 && H >= 1 && W >= 1, FGT_ERR_ARG, "poisson_unfilled: bad argument");
  FGT_LAUNCH(psn_sweep_kernel, dim3(F, 2), dim3(32), 0, stream, hole, gmask, F, H, W, clr);
  return FGT_OK;
}

extern "C" int fgt_poisson_finish(const double* trg, const unsigned char* hole, const double* x, int F, int H, int W,
                                  double* out, const unsigned char* clr, unsigned char* unf, fgt_stream_t stream) {
  FGT_REQUIRE(trg && hole && x && out && F >= 1 && H >= 1 && W >= 1 && (!unf || clr), FGT_ERR_ARG,
              "poisson_finish: bad argument");
  const long long pixels = static_cast<long long>(F) * H * W;
  FGT_LAUNCH(psn_finish_kernel, dim3(grid_stride(pixels, 256)), dim3(256), 0, stream, trg, hole, x, pixels, out, clr,
             unf);
  return FGT_OK;
}

// Host-side execution of the SAME scalar recurrence the kernels run (psn_advance is __host__ __device__), so the
// stopping logic can be tested without a GPU: prev / cur are 16 doubles, step_out = {t1, t2, vscale, au, skip_all,
// skip_u}. No device work.
extern "C" int fgt_poisson_advance_host(const double* prev_host, double* cur_host, double* step_out_host, int k,
                                        double bbk, double aak, double wwk, double atol, double btol, double conlim,
                                        int iter_lim) {
  FGT_REQUIRE(cur_host && step_out_host && (k == 0 || prev_host), FGT_ERR_ARG, "poisson_advance_host: bad argument");
  PsnStep st;
  double zero[kPsnState] = {0};
  psn_advance(prev_host ? prev_host : zero, cur_host, &st, k, bbk, aak, wwk, atol, btol,
              conlim > 0.0 ? 1.0 / conlim : 0.0, iter_lim);
  step_out_host[0] = st.t1;
  step_out_host[1] = st.t2;
  step_out_host[2] = st.vscale;
  step_out_host[3] = st.au;
  step_out_host[4] = st.skip_all;
  step_out_host[5] = st.skip_u;
  return FGT_OK;
}
