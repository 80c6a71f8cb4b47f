// cv2.inpaint(img, mask, radius, cv2.INPAINT_TELEA) on uint8 images, byte-identical to OpenCV's fast-marching
// implementation (tool/video_inpainting.py:316-320, 591-599, 663-671), plus the float32 glue around the call in the
// driver's gradient preparation (:583-614).
//
// Everything in TELEA except the pixel values depends on the mask alone: the order in which hole pixels are filled,
// their distances T, which neighbours count as known when a pixel is filled and every weight. So the work is split:
//   plan (one CTA per distinct mask): the two fast marches (outward over the ring -> negative T, inward over the hole
//       -> fill rank and T of every hole pixel) run serially on one thread with a binary heap ordered by
//       (T, insertion sequence), which reproduces OpenCV's sorted list with first-in-first-out ties. Then every hole
//       pixel gets a level: one more than the highest level among the earlier-filled pixels its stencil reads.
//   fill (one CTA per image): level by level, every pixel of a level is filled at once with exactly the serial
//       arithmetic (per channel, the stencil summed in OpenCV's raster order; no reductions, no FMA contraction).
// A pixel that the serial algorithm reads before it is filled is read from the input image, every other one from the
// output, so the result does not depend on the order inside a level.
//
// Coordinates follow OpenCV: a 1-pixel frame around the image (padded rows R = H+2, columns Cc = W+2).
// fgt_inpaint_telea_host runs plan + fill for one image on the CPU through the same __host__ __device__ routines.
#include <math.h>

#include <climits>
#include <vector>

#include "common.h"

namespace fgt {
namespace telea {

#define TL_HD __host__ __device__ __forceinline__

// IEEE arithmetic without contraction on the device (nvcc fuses a*b+c into FMA by default); plain operators on the
// host, where x86-64 code does not fuse.
#ifdef __CUDA_ARCH__
#define F_ADD(a, b) __fadd_rn((a), (b))
#define F_SUB(a, b) __fsub_rn((a), (b))
#define F_MUL(a, b) __fmul_rn((a), (b))
#define F_DIV(a, b) __fdiv_rn((a), (b))
#define F_SQRT(a) __fsqrt_rn(a)
#define D_ADD(a, b) __dadd_rn((a), (b))
#define D_MUL(a, b) __dmul_rn((a), (b))
#define D_DIV(a, b) __ddiv_rn((a), (b))
#define D_SQRT(a) __dsqrt_rn(a)
#else
#define F_ADD(a, b) ((a) + (b))
#define F_SUB(a, b) ((a) - (b))
#define F_MUL(a, b) ((a) * (b))
#define F_DIV(a, b) ((a) / (b))
#define F_SQRT(a) sqrtf(a)
#define D_ADD(a, b) ((a) + (b))
#define D_MUL(a, b) ((a) * (b))
#define D_DIV(a, b) ((a) / (b))
#define D_SQRT(a) sqrt(a)
#endif

enum : uint8_t { KNOWN = 0, BAND = 1, INSIDE = 2, CHANGE = 3 };
constexpr float kFar = 1.0e6f;
constexpr int kUnfilled = INT_MAX;  // rank of a hole pixel the march never reaches (a mask covering the whole image)

// Per-mask plan in the workspace. P = (H+2)*(W+2).
struct Plan {
  float* T;          // [P] distance (ring negative, band -0, hole >= 0)
  int* rank;         // [P] fill rank of a hole pixel, -1 outside the hole, kUnfilled if never filled
  int* level;        // [P] fill level of a hole pixel
  int* by_rank;      // [P] padded index of the pixel filled at each rank
  int* by_level;     // [P] the filled pixels grouped by level
  int* level_start;  // [P+2] offsets into by_level
  int* info;         // [4] filled pixels, levels
  uint8_t* flags;    // [P] inward-march flags
  uint8_t* ring;     // [P] outward-march flags
  uint8_t* rowdil;   // [P] row pass of the (2r+1)^2 dilation
  float* hkey;       // [P] heap: T
  int* hseq;         // [P] heap: insertion sequence
  int* hidx;         // [P] heap: padded index
};

TL_HD size_t align_up(size_t v) { return (v + 255) & ~static_cast<size_t>(255); }

TL_HD size_t plan_bytes(int H, int W) {
  const size_t P = static_cast<size_t>(H + 2) * (W + 2);
  return align_up(P * 4) * 8 + align_up((P + 2) * 4) + align_up(16) + align_up(P) * 3;
}

TL_HD Plan plan_at(void* base, int H, int W) {
  const size_t P = static_cast<size_t>(H + 2) * (W + 2);
  char* p = static_cast<char*>(base);
  Plan pl;
  auto take = [&](size_t n) { char* q = p; p += align_up(n); return q; };
  pl.T = reinterpret_cast<float*>(take(P * 4));
  pl.rank = reinterpret_cast<int*>(take(P * 4));
  pl.level = reinterpret_cast<int*>(take(P * 4));
  pl.by_rank = reinterpret_cast<int*>(take(P * 4));
  pl.by_level = reinterpret_cast<int*>(take(P * 4));
  pl.hkey = reinterpret_cast<float*>(take(P * 4));
  pl.hseq = reinterpret_cast<int*>(take(P * 4));
  pl.hidx = reinterpret_cast<int*>(take(P * 4));
  pl.level_start = reinterpret_cast<int*>(take((P + 2) * 4));
  pl.info = reinterpret_cast<int*>(take(16));
  pl.flags = reinterpret_cast<uint8_t*>(take(P));
  pl.ring = reinterpret_cast<uint8_t*>(take(P));
  pl.rowdil = reinterpret_cast<uint8_t*>(take(P));
  return pl;
}

// ---------------------------------------------------------------------------------------------- heap
// Min-heap on (T, seq): OpenCV's CvPriorityQueueFloat is a sorted list that inserts after every element with T <= t
// and pops the head, i.e. ascending T with first-in-first-out ties.
struct Heap {
  float* key;
  int* seq;
  int* idx;
  int n, next;
  TL_HD bool less(int a, int b) const { return key[a] < key[b] || (key[a] == key[b] && seq[a] < seq[b]); }
  TL_HD void swap(int a, int b) {
    float k = key[a]; key[a] = key[b]; key[b] = k;
    int s = seq[a]; seq[a] = seq[b]; seq[b] = s;
    int i = idx[a]; idx[a] = idx[b]; idx[b] = i;
  }
  TL_HD void push(int p, float t) {
    int c = n++;
    key[c] = t; seq[c] = next++; idx[c] = p;
    while (c > 0) {
      const int par = (c - 1) >> 1;
      if (!less(c, par)) break;
      swap(c, par);
      c = par;
    }
  }
  TL_HD int pop() {
    const int top = idx[0];
    --n;
    if (n > 0) {
      key[0] = key[n]; seq[0] = seq[n]; idx[0] = idx[n];
      int c = 0;
      for (;;) {
        const int l = 2 * c + 1, r = l + 1;
        int m = c;
        if (l < n && less(l, m)) m = l;
        if (r < n && less(r, m)) m = r;
        if (m == c) break;
        swap(c, m);
        c = m;
      }
    }
    return top;
  }
};

// FastMarching_solve: distance from two neighbours, in double.
TL_HD float solve(int p1, int p2, const uint8_t* f, const float* T) {
  const double a11 = T[p1], a22 = T[p2];
  const double m12 = a11 < a22 ? a11 : a22;
  double sol;
  if (f[p1] != INSIDE) {
    if (f[p2] != INSIDE) {
      const double d = a11 - a22;
      if (fabs(d) >= 1.0) sol = D_ADD(1.0, m12);
      else sol = D_MUL(D_ADD(D_ADD(a11, a22), D_SQRT(2.0 - D_MUL(d, d))), 0.5);
    } else {
      sol = D_ADD(1.0, a11);
    }
  } else if (f[p2] != INSIDE) {
    sol = D_ADD(1.0, a22);
  } else {
    sol = D_ADD(1.0, m12);
  }
  return static_cast<float>(sol);
}

TL_HD float min4(float a, float b, float c, float d) {
  const float ab = a < b ? a : b, cd = c < d ? c : d;
  return ab < cd ? ab : cd;
}

TL_HD float dist_at(int p, int Cc, const uint8_t* f, const float* T) {
  return min4(solve(p - Cc, p - 1, f, T), solve(p + Cc, p - 1, f, T), solve(p - Cc, p + 1, f, T),
              solve(p + Cc, p + 1, f, T));
}

// ---------------------------------------------------------------------------------------------- plan
// The three set-up passes are element-wise; `tid` / `nthr` stride them over a CTA (or run them on one host thread).
// hole(y,x) for padded coordinates (frame = not hole).
TL_HD bool hole_at(const uint8_t* mask, int H, int W, int y, int x) {
  return y >= 1 && x >= 1 && y <= H && x <= W && mask[static_cast<size_t>(y - 1) * W + (x - 1)] != 0;
}

// Pass 1: rowdil = hole dilated along rows by +-r; T, rank, level reset.
TL_HD void setup_rows(const uint8_t* mask, int H, int W, int r, const Plan& pl, int tid, int nthr) {
  const int R = H + 2, Cc = W + 2, P = R * Cc;
  for (int p = tid; p < P; p += nthr) {
    const int y = p / Cc, x = p - y * Cc;
    uint8_t v = 0;
    if (y >= 1 && y <= H)
      for (int xx = x - r; xx <= x + r && !v; ++xx) v = hole_at(mask, H, W, y, xx) ? 1 : 0;
    pl.rowdil[p] = v;
    pl.T[p] = kFar;
    pl.rank[p] = hole_at(mask, H, W, y, x) ? kUnfilled : -1;
    pl.level[p] = 0;
  }
}

// Pass 2: flags (hole INSIDE, band = cross dilation minus hole minus frame BAND, else KNOWN); ring flags (square
// dilation minus hole minus band minus frame INSIDE, else KNOWN); band T = 0.
TL_HD void setup_flags(const uint8_t* mask, int H, int W, int r, const Plan& pl, int tid, int nthr) {
  const int R = H + 2, Cc = W + 2, P = R * Cc;
  for (int p = tid; p < P; p += nthr) {
    const int y = p / Cc, x = p - y * Cc;
    const bool frame = y == 0 || x == 0 || y == R - 1 || x == Cc - 1;
    const bool h = hole_at(mask, H, W, y, x);
    const bool band = !frame && !h &&
                      (hole_at(mask, H, W, y - 1, x) || hole_at(mask, H, W, y + 1, x) ||
                       hole_at(mask, H, W, y, x - 1) || hole_at(mask, H, W, y, x + 1));
    bool sq = false;
    for (int yy = y - r; yy <= y + r && !sq; ++yy)
      if (yy >= 0 && yy < R) sq = pl.rowdil[yy * Cc + x] != 0;
    pl.flags[p] = h ? INSIDE : (band ? BAND : KNOWN);
    pl.ring[p] = (!frame && !h && !band && sq) ? INSIDE : KNOWN;
    if (band) pl.T[p] = 0.f;
  }
}

// Serial part: outward march over the ring, inward march over the hole (fill ranks and T). Returns the pixel count.
TL_HD int march(int H, int W, const Plan& pl) {
  const int R = H + 2, Cc = W + 2, P = R * Cc;
  Heap hp{pl.hkey, pl.hseq, pl.hidx, 0, 0};
  // icvCalcFMM(ring, t, Out, negate = true): the band pushed in raster order with T = 0
  for (int p = 0; p < P; ++p)
    if (pl.flags[p] == BAND) hp.push(p, 0.f);
  const int nb[4] = {-Cc, -1, Cc, 1};  // up, left, down, right
  while (hp.n > 0) {
    const int pp = hp.pop();
    pl.ring[pp] = CHANGE;
    const int ii = pp / Cc, jj = pp - ii * Cc;
    for (int q = 0; q < 4; ++q) {
      const int p = pp + nb[q];
      const int i = ii + (q == 0 ? -1 : q == 2 ? 1 : 0), j = jj + (q == 1 ? -1 : q == 3 ? 1 : 0);
      if (i <= 0 || j <= 0 || i > R - 1 || j > Cc - 1) continue;
      if (pl.ring[p] == INSIDE) {
        const float d = dist_at(p, Cc, pl.ring, pl.T);
        pl.T[p] = d;
        pl.ring[p] = BAND;
        hp.push(p, d);
      }
    }
  }
  for (int p = 0; p < P; ++p)
    if (pl.ring[p] == CHANGE) pl.T[p] = -pl.T[p];
  // icvTeleaInpaintFMM: the band again, a fresh heap; a pixel's rank is the order in which it is filled
  hp.n = 0;
  hp.next = 0;
  for (int p = 0; p < P; ++p)
    if (pl.flags[p] == BAND) hp.push(p, 0.f);
  int filled = 0;
  while (hp.n > 0) {
    const int pp = hp.pop();
    pl.flags[pp] = KNOWN;
    const int ii = pp / Cc, jj = pp - ii * Cc;
    for (int q = 0; q < 4; ++q) {
      const int p = pp + nb[q];
      const int i = ii + (q == 0 ? -1 : q == 2 ? 1 : 0), j = jj + (q == 1 ? -1 : q == 3 ? 1 : 0);
      if (i <= 0 || j <= 0 || i > R - 1 || j > Cc - 1) continue;
      if (pl.flags[p] == INSIDE) {
        const float d = dist_at(p, Cc, pl.flags, pl.T);
        pl.T[p] = d;
        pl.rank[p] = filled;
        pl.by_rank[filled++] = p;
        pl.flags[p] = BAND;
        hp.push(p, d);
      }
    }
  }
  return filled;
}

// ---------------------------------------------------------------------------------------------- one pixel
// Fills hole pixel p (padded index) the way icvTeleaInpaintFMM does when it reaches it. A neighbour is INSIDE at that
// moment iff it is a hole pixel of rank >= rank(p) (p itself included). `src` reads image values (image coordinates)
// and receives the results; the plan's level pass uses the same routine with a source that only records reads.
template <class Src>
TL_HD void fill_pixel(int p, int H, int W, int range, int nch, const float* T, const int* rank, Src& src) {
  const int R = H + 2, Cc = W + 2;
  const int i = p / Cc, j = p - i * Cc;
  const int rp = rank[p];
  auto inside = [&](int y, int x) { return rank[y * Cc + x] >= rp; };
  auto Tat = [&](int y, int x) { return T[y * Cc + x]; };
  const float Tij = T[p];
  float gTx, gTy;
  if (!inside(i, j + 1)) gTx = !inside(i, j - 1) ? F_MUL(F_SUB(Tat(i, j + 1), Tat(i, j - 1)), 0.5f) : F_SUB(Tat(i, j + 1), Tij);
  else gTx = !inside(i, j - 1) ? F_SUB(Tij, Tat(i, j - 1)) : 0.f;
  if (!inside(i + 1, j)) gTy = !inside(i - 1, j) ? F_MUL(F_SUB(Tat(i + 1, j), Tat(i - 1, j)), 0.5f) : F_SUB(Tat(i + 1, j), Tij);
  else gTy = !inside(i - 1, j) ? F_SUB(Tij, Tat(i - 1, j)) : 0.f;

  float Ia[3] = {0.f, 0.f, 0.f}, Jx[3] = {0.f, 0.f, 0.f}, Jy[3] = {0.f, 0.f, 0.f};
  float s = 1.0e-20f;
  for (int k = i - range; k <= i + range; ++k) {
    const int km = k - 1 + (k == 1), kp = k - 1 - (k == R - 2);
    for (int l = j - range; l <= j + range; ++l) {
      const int lm = l - 1 + (l == 1), lp = l - 1 - (l == Cc - 2);
      if (!(k > 0 && l > 0 && k < R - 1 && l < Cc - 1)) continue;
      if (inside(k, l) || (l - j) * (l - j) + (k - i) * (k - i) > range * range) continue;
      const float ry = static_cast<float>(i - k), rx = static_cast<float>(j - l);
      const float len2 = F_ADD(F_MUL(rx, rx), F_MUL(ry, ry));
      const float dst = static_cast<float>(D_DIV(1.0, D_MUL(static_cast<double>(len2), D_SQRT(static_cast<double>(len2)))));
      // 1 + |dT| in double (the difference itself in float): a float sum here is off by one level in ~6 % of images
      const float lev = static_cast<float>(D_DIV(1.0, D_ADD(1.0, fabs(static_cast<double>(F_SUB(Tat(k, l), Tij))))));
      float dir = F_ADD(F_MUL(rx, gTx), F_MUL(ry, gTy));
      if (fabs(static_cast<double>(dir)) <= 0.01) dir = 0.000001f;
      const float w = fabsf(F_MUL(F_MUL(dst, lev), dir));
      const bool rin = inside(k, l + 1), lin = inside(k, l - 1), din = inside(k + 1, l), uin = inside(k - 1, l);
      for (int c = 0; c < nch; ++c) {
        float gIx, gIy;
        if (!rin) gIx = !lin ? F_MUL(static_cast<float>(src.read(km, lp + 1, c) - src.read(km, lm - 1, c)), 2.0f)
                             : static_cast<float>(src.read(km, lp + 1, c) - src.read(km, lm, c));
        else gIx = !lin ? static_cast<float>(src.read(km, lp, c) - src.read(km, lm - 1, c)) : 0.f;
        if (!din) gIy = !uin ? F_MUL(static_cast<float>(src.read(kp + 1, lm, c) - src.read(km - 1, lm, c)), 2.0f)
                             : static_cast<float>(src.read(kp + 1, lm, c) - src.read(km, lm, c));
        else gIy = !uin ? static_cast<float>(src.read(kp, lm, c) - src.read(km - 1, lm, c)) : 0.f;
        Ia[c] = F_ADD(Ia[c], F_MUL(w, static_cast<float>(src.read(k - 1, l - 1, c))));
        Jx[c] = F_SUB(Jx[c], F_MUL(w, F_MUL(gIx, rx)));
        Jy[c] = F_SUB(Jy[c], F_MUL(w, F_MUL(gIy, ry)));
      }
      s = F_ADD(s, w);
    }
  }
  for (int c = 0; c < nch; ++c) {
    const float nrm = F_ADD(F_SQRT(F_ADD(F_MUL(Jx[c], Jx[c]), F_MUL(Jy[c], Jy[c]))), 1.0e-20f);
    const float sat = F_ADD(F_ADD(F_DIV(Ia[c], s), F_DIV(F_ADD(Jx[c], Jy[c]), nrm)), 0.5f);
#ifdef __CUDA_ARCH__
    const int iv = __float2int_rn(sat);
#else
    const int iv = static_cast<int>(lrintf(sat));
#endif
    src.write(i - 1, j - 1, c, static_cast<uint8_t>(iv < 0 ? 0 : iv > 255 ? 255 : iv));
  }
}

// Image source of the fill: hole pixels filled before p come from `out`, everything else from `in`.
struct ImageSrc {
  const uint8_t* in;
  uint8_t* out;
  const int* rank;
  int W, C, rp;
  TL_HD int read(int y, int x, int c) const {
    const int q = rank[(y + 1) * (W + 2) + x + 1];
    const size_t e = (static_cast<size_t>(y) * W + x) * C + c;
    return (q >= 0 && q < rp) ? out[e] : in[e];
  }
  TL_HD void write(int y, int x, int c, uint8_t v) { out[(static_cast<size_t>(y) * W + x) * C + c] = v; }
};

// Dependency source of the level pass: the highest level among the earlier-filled pixels read.
struct LevelSrc {
  const int* rank;
  const int* level;
  int W, rp, maxlev;
  TL_HD int read(int y, int x, int) {
    const int q = (y + 1) * (W + 2) + x + 1;
    const int rq = rank[q];
    if (rq >= 0 && rq < rp && level[q] > maxlev) maxlev = level[q];
    return 0;
  }
  TL_HD void write(int, int, int, uint8_t) {}
};

// Levels in rank order, then the pixels grouped by level (counting sort). Returns the number of levels.
TL_HD int levels(int H, int W, int range, int filled, const Plan& pl) {
  int nlev = 0;
  for (int k = 0; k < filled; ++k) {
    const int p = pl.by_rank[k];
    LevelSrc ls{pl.rank, pl.level, W, k, -1};
    fill_pixel(p, H, W, range, 1, pl.T, pl.rank, ls);
    pl.level[p] = ls.maxlev + 1;
    if (ls.maxlev + 2 > nlev) nlev = ls.maxlev + 2;
  }
  for (int L = 0; L <= nlev; ++L) pl.level_start[L] = 0;
  for (int k = 0; k < filled; ++k) pl.level_start[pl.level[pl.by_rank[k]] + 1]++;
  for (int L = 0; L < nlev; ++L) pl.level_start[L + 1] += pl.level_start[L];
  for (int k = 0; k < filled; ++k) {
    const int p = pl.by_rank[k];
    pl.by_level[pl.level_start[pl.level[p]]++] = p;
  }
  for (int L = nlev; L > 0; --L) pl.level_start[L] = pl.level_start[L - 1];
  pl.level_start[0] = 0;
  return nlev;
}

// ---------------------------------------------------------------------------------------------- kernels
__global__ void __launch_bounds__(256) march_kernel(const uint8_t* __restrict__ masks, long long mask_stride, int H,
                                                    int W, int range, char* ws, size_t stride) {
  const int b = blockIdx.x;
  const uint8_t* mask = masks + b * mask_stride;
  const Plan pl = plan_at(ws + b * stride, H, W);
  setup_rows(mask, H, W, range, pl, threadIdx.x, blockDim.x);
  __syncthreads();
  setup_flags(mask, H, W, range, pl, threadIdx.x, blockDim.x);
  __syncthreads();
  if (threadIdx.x == 0) pl.info[0] = march(H, W, pl);
}

// Serial as well: a pixel's level needs the levels of every earlier-filled pixel its stencil reads.
__global__ void levels_kernel(int H, int W, int range, char* ws, size_t stride) {
  const Plan pl = plan_at(ws + blockIdx.x * stride, H, W);
  if (threadIdx.x == 0) pl.info[1] = levels(H, W, range, pl.info[0], pl);
}

__global__ void __launch_bounds__(512) fill_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int H,
                                                   int W, int C, int range, const char* ws, size_t stride, int shared) {
  const int b = blockIdx.x;
  const size_t img = static_cast<size_t>(H) * W * C;
  const uint8_t* src = in + b * img;
  uint8_t* dst = out + b * img;
  for (size_t e = threadIdx.x; e < img; e += blockDim.x) dst[e] = src[e];
  const Plan pl = plan_at(const_cast<char*>(ws) + (shared ? 0 : b) * stride, H, W);
  const int nlev = pl.info[1];
  __syncthreads();
  for (int L = 0; L < nlev; ++L) {
    const int e = pl.level_start[L + 1];
    for (int t = pl.level_start[L] + threadIdx.x; t < e; t += blockDim.x) {
      const int p = pl.by_level[t];
      ImageSrc is{src, dst, pl.rank, W, C, pl.rank[p]};
      fill_pixel(p, H, W, range, C, pl.T, pl.rank, is);
    }
    __syncthreads();
  }
}

// Gradient preparation, before TELEA: zero the hole, then (img * 255).astype(uint8) (float32 multiply, truncation).
__global__ void grad_pre_kernel(const float* __restrict__ video, const uint8_t* __restrict__ mask, uint8_t* __restrict__ u8,
                                long long n_pix) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n_pix * 3;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float v = mask[i / 3] ? 0.f : video[i];
    u8[i] = static_cast<uint8_t>(static_cast<int>(__fmul_rn(v, 255.f)));
  }
}

// After TELEA: / 255 in float32, forward differences (last column / row zero), zero under mask_dilated.
__global__ void grad_post_kernel(const uint8_t* __restrict__ u8, const uint8_t* __restrict__ mask_dilated, int B, int H,
                                 int W, float* __restrict__ gx, float* __restrict__ gy) {
  const long long total = static_cast<long long>(B) * H * W * 3;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long pix = i / 3;
    const int x = static_cast<int>(pix % W), y = static_cast<int>((pix / W) % H);
    const float v = __fdiv_rn(static_cast<float>(u8[i]), 255.f);
    float dx = 0.f, dy = 0.f;
    if (!mask_dilated[pix]) {
      if (x + 1 < W) dx = __fsub_rn(__fdiv_rn(static_cast<float>(u8[i + 3]), 255.f), v);
      if (y + 1 < H) dy = __fsub_rn(__fdiv_rn(static_cast<float>(u8[i + 3LL * W]), 255.f), v);
    }
    gx[i] = dx;
    gy[i] = dy;
  }
}

// cv2.inpaint's radius: cvRound, then clamped to [1, 100] (only 3 is then accepted, see telea_check).
inline int radius_of(double radius) {
  int r = static_cast<int>(lrint(radius));
  return r < 1 ? 1 : r > 100 ? 100 : r;
}

}  // namespace telea
}  // namespace fgt

using namespace fgt::telea;

static int telea_check(int H, int W, int C, double radius, int* range) {
  FGT_REQUIRE(H >= 2 && W >= 2 && (C == 1 || C == 3), FGT_ERR_ARG,
              "inpaint_telea: images must be at least 2x2 with 1 or 3 channels (got %dx%dx%d)", H, W, C);
  FGT_REQUIRE(radius == radius, FGT_ERR_ARG, "inpaint_telea: radius is NaN");
  *range = radius_of(radius);
  // Only radius 3 (the driver's) has been found byte-identical on every case tried. Radii 1, 2, 4 and 6 each miss cv2
  // by one level on roughly 1 in 1000 to 1 in 20000 small speckled masks, where the final sum falls within a float ulp
  // of x.5 and some operation of OpenCV's rounds differently; they are refused rather than served approximately.
  FGT_REQUIRE(*range == 3, FGT_ERR_ARG,
              "inpaint_telea: radius %g rounds to %d; only radius 3 is supported (the only radius verified "
              "byte-identical to cv2.inpaint)", radius, *range);
  return FGT_OK;
}

extern "C" long long fgt_inpaint_telea_workspace(int n_masks, int H, int W) {
  if (n_masks < 1 || H < 1 || W < 1) return fgt::set_err(FGT_ERR_ARG, "inpaint_telea_workspace: bad argument");
  return static_cast<long long>(plan_bytes(H, W)) * n_masks;
}

static int ws_check(int n_masks, int H, int W, long long workspace_bytes) {
  const long long need = static_cast<long long>(plan_bytes(H, W)) * n_masks;
  FGT_REQUIRE(workspace_bytes >= need, FGT_ERR_ARG, "inpaint_telea: workspace of %lld bytes, %lld needed",
              workspace_bytes, need);
  return FGT_OK;
}

extern "C" int fgt_inpaint_telea_plan(const unsigned char* masks, int n_masks, int H, int W, double radius,
                                      void* workspace, long long workspace_bytes, fgt_stream_t stream) {
  FGT_REQUIRE(masks && workspace && n_masks >= 1, FGT_ERR_ARG, "inpaint_telea_plan: bad argument");
  int range = 0;
  int rc = telea_check(H, W, 1, radius, &range);
  if (rc == FGT_OK) rc = ws_check(n_masks, H, W, workspace_bytes);
  if (rc != FGT_OK) return rc;
  char* ws = static_cast<char*>(workspace);
  const size_t stride = plan_bytes(H, W);
  FGT_LAUNCH(march_kernel, dim3(n_masks), dim3(256), 0, stream, masks, static_cast<long long>(H) * W, H, W, range, ws,
             stride);
  FGT_LAUNCH(levels_kernel, dim3(n_masks), dim3(32), 0, stream, H, W, range, ws, stride);
  return FGT_OK;
}

extern "C" int fgt_inpaint_telea_fill(const unsigned char* images, int B, int H, int W, int C, int shared_plan,
                                      double radius, const void* workspace, long long workspace_bytes,
                                      unsigned char* out, fgt_stream_t stream) {
  FGT_REQUIRE(images && out && workspace && B >= 1, FGT_ERR_ARG, "inpaint_telea_fill: bad argument");
  FGT_REQUIRE(images != out, FGT_ERR_ARG, "inpaint_telea: out must not alias the images");
  int range = 0;
  int rc = telea_check(H, W, C, radius, &range);
  if (rc == FGT_OK) rc = ws_check(shared_plan ? 1 : B, H, W, workspace_bytes);
  if (rc != FGT_OK) return rc;
  FGT_LAUNCH(fill_kernel, dim3(B), dim3(512), 0, stream, images, out, H, W, C, range,
             static_cast<const char*>(workspace), plan_bytes(H, W), shared_plan ? 1 : 0);
  return FGT_OK;
}

extern "C" int fgt_inpaint_telea(const unsigned char* images, const unsigned char* masks, int B, int H, int W, int C,
                                 long long mask_stride, double radius, void* workspace, long long workspace_bytes,
                                 unsigned char* out, fgt_stream_t stream) {
  FGT_REQUIRE(images && masks && out && workspace && B >= 1, FGT_ERR_ARG, "inpaint_telea: bad argument");
  FGT_REQUIRE(mask_stride == 0 || mask_stride == static_cast<long long>(H) * W, FGT_ERR_ARG,
              "inpaint_telea: mask batch stride must be 0 (one mask for every image) or H*W");
  const int rc = fgt_inpaint_telea_plan(masks, mask_stride == 0 ? 1 : B, H, W, radius, workspace, workspace_bytes, stream);
  if (rc != FGT_OK) return rc;
  return fgt_inpaint_telea_fill(images, B, H, W, C, mask_stride == 0 ? 1 : 0, radius, workspace, workspace_bytes, out,
                                stream);
}

extern "C" int fgt_inpaint_telea_host(const unsigned char* image_host, const unsigned char* mask_host, int H, int W, int C,
                                      double radius, unsigned char* out_host) {
  FGT_REQUIRE(image_host && mask_host && out_host && image_host != out_host, FGT_ERR_ARG, "inpaint_telea_host: bad argument");
  int range = 0;
  const int rc = telea_check(H, W, C, radius, &range);
  if (rc != FGT_OK) return rc;
  std::vector<char> ws(plan_bytes(H, W) + 256);
  char* base = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(ws.data()) + 255) & ~static_cast<uintptr_t>(255));
  const Plan pl = plan_at(base, H, W);
  setup_rows(mask_host, H, W, range, pl, 0, 1);
  setup_flags(mask_host, H, W, range, pl, 0, 1);
  const int filled = march(H, W, pl);
  const int nlev = levels(H, W, range, filled, pl);
  memcpy(out_host, image_host, static_cast<size_t>(H) * W * C);
  for (int L = 0; L < nlev; ++L)  // the same order as the kernel (any order within a level gives the same bytes)
    for (int t = pl.level_start[L]; t < pl.level_start[L + 1]; ++t) {
      const int p = pl.by_level[t];
      ImageSrc is{image_host, out_host, pl.rank, W, C, pl.rank[p]};
      fill_pixel(p, H, W, range, C, pl.T, pl.rank, is);
    }
  return FGT_OK;
}

extern "C" int fgt_grad_prep_pre(const float* video, const unsigned char* mask, int B, int H, int W, unsigned char* u8,
                                 fgt_stream_t stream) {
  FGT_REQUIRE(video && mask && u8 && B >= 1 && H >= 1 && W >= 1, FGT_ERR_ARG, "grad_prep_pre: bad argument");
  const long long n = static_cast<long long>(B) * H * W;
  FGT_LAUNCH(grad_pre_kernel, dim3(fgt::grid_stride(n * 3, 256)), dim3(256), 0, stream, video, mask, u8, n);
  return FGT_OK;
}

extern "C" int fgt_grad_prep_post(const unsigned char* u8, const unsigned char* mask_dilated, int B, int H, int W, float* gx,
                                  float* gy, fgt_stream_t stream) {
  FGT_REQUIRE(u8 && mask_dilated && gx && gy && B >= 1 && H >= 1 && W >= 1, FGT_ERR_ARG, "grad_prep_post: bad argument");
  const long long n = static_cast<long long>(B) * H * W * 3;
  FGT_LAUNCH(grad_post_kernel, dim3(fgt::grid_stride(n, 256)), dim3(256), 0, stream, u8, mask_dilated, B, H, W, gx, gy);
  return FGT_OK;
}
