// 3x3 convolution with a handful of output channels (the decoder's final 64 -> 3 conv + tanh, model.py:185-193; RAFT's
// flow head 256 -> 2, update.py:13-14) as ONE kernel: tensor cores for the contraction, shared memory for the taps.
//
// A convolution with <= 3 output channels has no N extent for an implicit GEMM (N = 3 would waste most of every MMA
// and re-read the activation once per tap). Instead the taps become the N dimension: for every input position p the
// tensor core computes Y[p, tap*cout + c] = sum_ch x[p, ch] * W[c, ch, tap]  (N = 9*cout <= 32, K = Cin), reading the
// activation ONCE, and the output pixel is the sum of its 9 neighbours' matching columns:
//     out[c, y, x] = act(bias[c] + sum_{ty,tx} Y[(y+ty-1, x+tx-1), (ty*3+tx)*cout + c]).
// Y of a 16x8 output tile plus its 1-pixel halo (18x10 = 180 positions = three M=64 wgmma blocks) goes from registers
// to shared memory and never leaves the SM: HBM traffic = the activation once + the 3-channel image.
//
//   warp 4     : TMA producer (halo box (64 ch, 18, 10) per 64-channel chunk and plane; zero fill = the conv's padding)
//   warps 0..3 : one warpgroup: wgmma (3-term split-bf16, M=64 x N=32, three M blocks per chunk, fp32 accumulators in
//                registers) -> Y rows in smem (pitch 33 floats: conflict-free both ways) -> 9-tap sums -> bias,
//                activation, coalesced stores
// kF16 (mixed precision): activation and weights are single-plane fp16, one fp16 wgmma per K step.
#include "common.h"
#include "ptx.cuh"

namespace fgt {

constexpr int kTailTW = 16, kTailTH = 8;               // output tile
constexpr int kTailHW = kTailTW + 2, kTailHH = kTailTH + 2;
constexpr int kTailRows = kTailHW * kTailHH;           // 180 halo positions
constexpr int kTailMBlocks = 3;                        // M=64 blocks covering the 180 rows
constexpr int kTailAPlane = kTailMBlocks * 64 * 128;   // smem per plane and stage: 192 rows x 128 B
constexpr int kTailAStage = 2 * kTailAPlane;           // 48 KB
constexpr int kTailStages = 2;
constexpr int kTailMaxChunks = 4;                      // Cin <= 256
constexpr int kTailBBlk = 32 * 128;                    // one (chunk, plane) block of the weights: 32 rows x 128 B
constexpr int kTailYPitch = 33;
constexpr int kTailYBuf = ((kTailRows * kTailYPitch * 4 + 1023) / 1024) * 1024;
constexpr int kTailSmemA = 0;
constexpr int kTailSmemB = kTailSmemA + kTailStages * kTailAStage;
constexpr int kTailSmemY = kTailSmemB + kTailMaxChunks * 2 * kTailBBlk;
constexpr int kTailSmemBar = kTailSmemY + 2 * kTailYBuf;
constexpr int kTailSmem = kTailSmemBar + 256 + 1024;
constexpr int kTailThreads = 160;                      // one consumer warpgroup + one producer warp

struct TailParams {
  CUtensorMap a_map, b_map;
  int chunks, tiles_x, tiles_y, total_tiles;
  int H, W, cout, act;
  const float* bias;
  float* out;
  long long os_n, os_c, os_y, os_x;
};

template <bool kF16>
__global__ void __launch_bounds__(kTailThreads, 1) conv_tail_kernel(const __grid_constant__ TailParams p) {
  constexpr int kPlanes = kF16 ? 1 : 2;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* sgen = smem_raw + (sbase - smem_u32(smem_raw));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t bar = sbase + kTailSmemBar;
  auto full_bar = [&](int s) { return bar + 8u * s; };
  auto empty_bar = [&](int s) { return bar + 8u * (2 + s); };
  const uint32_t w_bar = bar + 8u * 4;

  if (warp == 4 && lane == 0) {
    for (int s = 0; s < kTailStages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 4);  // one arrival per consumer warp
    }
    mbar_init(w_bar, 1);
    fence_mbar_init();
    tma_prefetch_desc(&p.a_map);
    tma_prefetch_desc(&p.b_map);
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  const int tiles_per_z = p.tiles_x * p.tiles_y;

  if (warp == 4) {
    // ------------------------------------------------------------ TMA producer
    if (elect_one()) {
      // weights: every (chunk, plane) block once per CTA
      mbar_expect_tx(w_bar, static_cast<uint32_t>(p.chunks) * kPlanes * kTailBBlk);
      for (int c = 0; c < p.chunks; ++c)
        for (int pl = 0; pl < kPlanes; ++pl)
          tma_load_3d(sbase + kTailSmemB + (c * 2 + pl) * kTailBBlk, &p.b_map, w_bar, c * 64, 0, pl);
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        const int z = tile / tiles_per_z;
        const int rem = tile - z * tiles_per_z;
        const int ty = rem / p.tiles_x, tx = rem - ty * p.tiles_x;
        for (int c = 0; c < p.chunks; ++c) {
          mbar_wait_quiet(empty_bar(stage), phase ^ 1u);
          const uint32_t sa = sbase + kTailSmemA + stage * kTailAStage;
          mbar_expect_tx(full_bar(stage), kPlanes * kTailRows * 128u);
          tma_load_5d(sa, &p.a_map, full_bar(stage), c * 64, tx * kTailTW - 1, ty * kTailTH - 1, z, 0);
          if (!kF16) tma_load_5d(sa + kTailAPlane, &p.a_map, full_bar(stage), c * 64, tx * kTailTW - 1, ty * kTailTH - 1, z, 1);
          if (++stage == kTailStages) { stage = 0; phase ^= 1u; }
        }
      }
    }
    __syncwarp();
    return;
  }

  // -------------------------------------------------------------- warpgroup: MMA + tap sums (warps 0..3)
  const int r = threadIdx.x;  // output pixel of the tile for the tap sums
  const int py = r / kTailTW, px = r - py * kTailTW;
  const int g = lane >> 2, qc = lane & 3;
  const int cout = p.cout;
  float bias[4];
#pragma unroll
  for (int c = 0; c < 4; ++c) bias[c] = c < cout ? __ldg(p.bias + c) : 0.f;
  mbar_wait_quiet(w_bar, 0);
  int stage = 0, lt = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x, ++lt) {
    const int buf = lt & 1;
    const int z = tile / tiles_per_z;
    const int rem = tile - z * tiles_per_z;
    const int ty = rem / p.tiles_x, tx = rem - ty * p.tiles_x;
    float acc[kTailMBlocks][16];
    for (int c = 0; c < p.chunks; ++c) {
      mbar_wait_quiet(full_bar(stage), phase);
      const uint32_t sa = sbase + kTailSmemA + stage * kTailAStage;
      const uint64_t b_hi = gmma_desc_sw128(sbase + kTailSmemB + (c * 2 + 0) * kTailBBlk);
      const uint64_t b_lo = gmma_desc_sw128(sbase + kTailSmemB + (c * 2 + 1) * kTailBBlk);
#pragma unroll
      for (int mb = 0; mb < kTailMBlocks; ++mb) fence_regs(acc[mb]);
      wgmma_fence();
#pragma unroll
      for (int mb = 0; mb < kTailMBlocks; ++mb) {
        const uint64_t a_hi = gmma_desc_sw128(sa + mb * 64 * 128);
        const uint64_t a_lo = gmma_desc_sw128(sa + kTailAPlane + mb * 64 * 128);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint64_t ko = static_cast<uint64_t>(k * 2);
          if (kF16) {
            wgmma_ss<32, true>(acc[mb], a_hi + ko, b_hi + ko, (c | k) != 0);
            continue;
          }
          wgmma_ss<32, false>(acc[mb], a_lo + ko, b_hi + ko, (c | k) != 0);
          wgmma_ss<32, false>(acc[mb], a_hi + ko, b_lo + ko, 1u);
          wgmma_ss<32, false>(acc[mb], a_hi + ko, b_hi + ko, 1u);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int mb = 0; mb < kTailMBlocks; ++mb) fence_regs(acc[mb]);
      if (lane == 0) mbar_arrive(empty_bar(stage));
      if (++stage == kTailStages) { stage = 0; phase ^= 1u; }
    }
    // accumulator fragment -> Y rows (acc[mb][4 jj + 2 h + e] = Y[64 mb + 16 warp + g + 8 h][8 jj + 2 qc + e])
    float* Y = reinterpret_cast<float*>(sgen + kTailSmemY + buf * kTailYBuf);
#pragma unroll
    for (int mb = 0; mb < kTailMBlocks; ++mb)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = mb * 64 + warp * 16 + g + 8 * h;
        if (row < kTailRows) {
          float* yr = Y + row * kTailYPitch + 2 * qc;
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            yr[8 * jj] = acc[mb][4 * jj + 2 * h];
            yr[8 * jj + 1] = acc[mb][4 * jj + 2 * h + 1];
          }
        }
      }
    asm volatile("bar.sync 1, 128;\n" ::: "memory");  // all 180 rows of Y are in shared memory
    const int oy = ty * kTailTH + py, ox = tx * kTailTW + px;
    if (oy < p.H && ox < p.W) {
      float a[4] = {bias[0], bias[1], bias[2], bias[3]};
#pragma unroll
      for (int t = 0; t < 9; ++t) {
        const float* yr = Y + ((py + t / 3) * kTailHW + px + t % 3) * kTailYPitch + t * cout;
#pragma unroll
        for (int c = 0; c < 4; ++c)
          if (c < cout) a[c] += yr[c];
      }
      float* op = p.out + z * p.os_n + oy * p.os_y + ox * p.os_x;
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (c < cout) {
          float v = a[c];
          if (p.act == FGT_ACT_TANH) v = tanhf(v);
          else if (p.act == FGT_ACT_LEAKY02) v = v > 0.f ? v : 0.2f * v;
          else if (p.act == FGT_ACT_RELU) v = fmaxf(v, 0.f);
          else if (p.act == FGT_ACT_SIGMOID) v = 1.f / (1.f + expf(-v));
          op[c * p.os_c] = v;
        }
    }
    // Y is double-buffered: the barrier of the next tile orders these reads before tile lt+2 rewrites this buffer
  }
}

}  // namespace fgt

extern "C" int fgt_conv_tail(const void* x_hi, long long x_plane, int n, int H, int W, int cin, const void* w_hi,
                             long long w_plane, int k_pad, int cout, const float* bias, int act, float* out,
                             long long os_n, long long os_c, long long os_y, long long os_x, fgt_stream_t stream) {
  using namespace fgt;
  FGT_REQUIRE(x_hi && w_hi && bias && out, FGT_ERR_ARG, "conv_tail: null argument");
  FGT_REQUIRE(cin % 64 == 0 && cin >= 64 && cin <= 64 * kTailMaxChunks, FGT_ERR_ARG,
              "conv_tail: cin=%d must be a multiple of 64, <= %d", cin, 64 * kTailMaxChunks);
  FGT_REQUIRE(cout >= 1 && cout <= 3, FGT_ERR_ARG, "conv_tail: cout=%d (1..3: nine taps times cout must fit 32 columns)", cout);
  FGT_REQUIRE(k_pad == cin, FGT_ERR_ARG, "conv_tail: weights must be packed [32, cin] (k_pad=%d, cin=%d)", k_pad, cin);
  FGT_REQUIRE(n >= 1 && H >= 1 && W >= 1, FGT_ERR_ARG, "conv_tail: empty problem");
  FGT_REQUIRE(act == FGT_ACT_NONE || act == FGT_ACT_TANH || act == FGT_ACT_RELU || act == FGT_ACT_SIGMOID ||
                  act == FGT_ACT_LEAKY02, FGT_ERR_ARG, "conv_tail: act=%d", act);
  if (const int rc = fgt::check_act16("conv_tail: x", x_hi, x_plane, 8, true)) return rc;
  if (const int rc = fgt::check_act16("conv_tail: weights", w_hi, w_plane, 8, true)) return rc;
  FGT_REQUIRE((x_plane == 0) == (w_plane == 0), FGT_ERR_ARG,
              "conv_tail: activation and weights are both split-bf16 (plane > 0) or both single-plane fp16 (plane 0), "
              "got x_plane=%lld w_plane=%lld", x_plane, w_plane);
  const bool f16 = x_plane == 0;
  const uint64_t planes = f16 ? 1 : 2;
  TailParams p;
  memset(&p, 0, sizeof(p));
  {
    uint64_t dims[5] = {static_cast<uint64_t>(cin), static_cast<uint64_t>(W), static_cast<uint64_t>(H),
                        static_cast<uint64_t>(n), planes};
    uint64_t str[4] = {static_cast<uint64_t>(cin) * 2, static_cast<uint64_t>(W) * cin * 2,
                       static_cast<uint64_t>(H) * W * cin * 2, static_cast<uint64_t>(x_plane) * 2};
    if (f16) str[3] = str[2] * dims[3];  // single plane: the plane dimension has extent 1
    uint32_t box[5] = {64, kTailHW, kTailHH, 1, 1};
    int rc = encode_map_bf16(&p.a_map, x_hi, 5, dims, str, box);
    if (rc) return rc;
  }
  {
    uint64_t dims[3] = {static_cast<uint64_t>(k_pad), 32, planes};
    uint64_t str[2] = {static_cast<uint64_t>(k_pad) * 2, static_cast<uint64_t>(w_plane) * 2};
    if (f16) str[1] = str[0] * dims[1];
    uint32_t box[3] = {64, 32, 1};
    int rc = encode_map_bf16(&p.b_map, w_hi, 3, dims, str, box);
    if (rc) return rc;
  }
  p.chunks = cin / 64;
  p.tiles_x = (W + kTailTW - 1) / kTailTW;
  p.tiles_y = (H + kTailTH - 1) / kTailTH;
  p.total_tiles = p.tiles_x * p.tiles_y * n;
  p.H = H; p.W = W; p.cout = cout; p.act = act; p.bias = bias; p.out = out;
  p.os_n = os_n; p.os_c = os_c; p.os_y = os_y; p.os_x = os_x;
  auto kern = f16 ? conv_tail_kernel<true> : conv_tail_kernel<false>;
  if (const int rc = allow_dynamic_smem(kern, kTailSmem, "conv_tail_kernel")) return rc;
  int grid = num_sms();
  if (grid > p.total_tiles) grid = p.total_tiles;
  return launch("conv_tail_kernel", kern, dim3(grid), dim3(kTailThreads), kTailSmem, stream, p);
}
