// Persistent, warp-specialised implicit-GEMM engine for sm_90a.
//
//   warps 0..7 : two consumer warpgroups (wgmma.mma_async, 3-term split-bf16 or 1-term fp16, fp32 accumulators in
//                registers); warpgroup w owns rows [64 w, 64 w + 64) of the 128-row tile and runs the epilogue of
//                those rows straight from its registers (bias / activation / aux operand, rows scattered through a
//                rowmap, transposed / NCHW outputs, launches with two outputs)
//   warp 8     : TMA producer (cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier tx)
//
// One CTA per SM loops over output tiles (128 output positions x bn channels); the producer runs ahead through the
// stage ring while the consumers finish the previous tile's epilogue. The epilogue loads its bias / aux operands in
// batches before the accumulators are final, and up to bn = 64 the consumers issue the next tile's first K stage before
// it. Used for every Linear/Conv on the path (see include/fgt_b200.h).
#include "common.h"
#include "ptx.cuh"

#include <mutex>
#include <unordered_set>

namespace fgt {

constexpr int kMaxAMaps = 18;  // 2 segments x up to 9 stride phases
constexpr int kMaxTaps = 64;   // up to 7x7 (=49) taps
constexpr int kBK = 64;        // K elements per pipeline stage (128 bytes of bf16)
constexpr int kAPlaneBytes = 128 * 128;  // one A plane per stage: 128 rows x 128 B
constexpr int kGemmThreads = 288;        // 2 consumer warpgroups + 1 producer warp
constexpr int kProducerWarp = 8;

struct TapDesc {
  int8_t phase;  // which stride-phase view
  int8_t dx, dy, dz;
};
struct SegDesc {
  int map_base;     // first tensor map of this segment (+ phase)
  int c_base;       // channel coordinate for group 0
  int c_per_group;  // channel advance per group
  int chunks;       // 64-channel chunks per tap
};

struct GemmParams {
  CUtensorMap a_maps[kMaxAMaps];
  CUtensorMap b_map;
  TapDesc taps[kMaxTaps];
  SegDesc segs[2];
  int num_taps, num_segs, num_maps, k_iters;
  int tiles_x, tiles_y, tiles_z, n_tiles, total_tiles;
  int bn, stages;
  int box_w, box_h, a_rows;
  int N, cout_per_group;
  int out_w, out_h;
  int linear;  // 1: rows on x only (rowmap / lin_batch addressing)
  int lin_batch;
  int vec_ok;   // channel pairs stored (and aux pairs loaded) as one 8-byte / 4-byte access
  int aux_vec;  // aux pairs loaded as one access (debugging aid: 0 = per-element loads)
  int vec4_ok;  // 4-channel accesses (16-byte fp32 / 8-byte 16-bit) are aligned: the batched epilogue may run
  long long os_z, os_y, os_x, os_c;
  const int* rowmap;
  float* out_f32;
  __nv_bfloat16* out_hi;
  long long out_plane;
  const float* aux;
  const float* aux2;
  int aux_mode;
  const float* bias;
  int act;
  float alpha;
  int out_half;  // the 16-bit output is ONE plane of fp16 (input of a 1-term layer) instead of split-bf16
  int r16;       // FGT_OUT_HALF_AUTOCAST: every fp16 tensor of the layer under autocast is rounded (kExt = 1 or 2)
};

// Epilogue parameters hoisted into registers once per CTA.
struct EpiArgs {
  float* out_f32;
  __nv_bfloat16* out_hi;
  const float* aux;
  const float* aux2;
  long long out_plane, os_c;
  float alpha;
  int act, aux_mode, vec_ok, aux_vec, N, out_half, r16;
};

__device__ __forceinline__ float act_one(float v, int act) {
  switch (act) {
    case FGT_ACT_LEAKY02: return v > 0.f ? v : 0.2f * v;
    case FGT_ACT_LEAKY001: return v > 0.f ? v : 0.01f * v;
    case FGT_ACT_RELU: return fmaxf(v, 0.f);
    case FGT_ACT_SIGMOID: return 1.f / (1.f + expf(-v));
    case FGT_ACT_TANH: return tanhf(v);
    default: return v;
  }
}

// Nearest fp16 value, as fp32. Mixed-precision RAFT (out_half): the fp32 copy of an output equals its fp16 output, as
// autocast's fp16 tensors do.
__device__ __forceinline__ float round_f16(float v) { return __half2float(__float2half_rn(v)); }

__device__ __forceinline__ void load_pair(const float* src, long long o0, long long o1, bool two, bool vec, float& x0,
                                          float& x1) {
  if (vec) {
    const float2 a = __ldg(reinterpret_cast<const float2*>(src + o0));
    x0 = a.x;
    x1 = a.y;
  } else {
    x0 = __ldg(src + o0);
    x1 = two ? __ldg(src + o1) : 0.f;
  }
}

// Output channels (col, col + 1) of one output row at element offset `off`: bias + alpha * acc, activation, aux
// operand, stores. `two`: col + 1 < N. kExt = 1 adds the rarely used modes (pre-activation add, add+ReLU, GRU
// updates, slope-0.01 LeakyReLU); keeping them out of the common instantiation keeps its register count down. kExt = 2
// (FGT_OUT_HALF_AUTOCAST without those modes) has the activations and the r16 rounding only.
template <int kExt>
__device__ __forceinline__ void epi_pair(const EpiArgs& e, float v0, float v1, long long off, int col, bool two) {
  const bool vec = e.vec_ok && two;  // vec_ok implies a unit channel stride and even element offsets
  const long long o0 = off + static_cast<long long>(col) * e.os_c;
  const long long o1 = o0 + e.os_c;
  const bool avec = vec && e.aux_vec;
  float a0 = 0.f, a1 = 0.f;
  if (kExt && e.r16) {  // autocast (LAFC): the conv's output is an fp16 tensor, also before a pre-activation add
    v0 = round_f16(v0);
    v1 = round_f16(v1);
  }
  if (kExt == 1 && e.aux_mode == FGT_AUX_ADD_PRE) {  // residual added BEFORE the activation (LAFC edge head)
    load_pair(e.aux, o0, o1, two, avec, a0, a1);
    v0 += a0;
    v1 += a1;
  }
  if (kExt && (e.out_half || e.r16)) {  // mixed precision: the conv's output is an fp16 tensor before its activation (autocast)
    v0 = round_f16(v0);
    v1 = round_f16(v1);
  }
  if (kExt) {
    v0 = act_one(v0, e.act);
    v1 = act_one(v1, e.act);
    if (e.r16) {  // autocast (LAFC): the activation's output is an fp16 tensor before the residual add
      v0 = round_f16(v0);
      v1 = round_f16(v1);
    }
  } else if (e.act == FGT_ACT_LEAKY02) {
    v0 = v0 > 0.f ? v0 : 0.2f * v0;
    v1 = v1 > 0.f ? v1 : 0.2f * v1;
  } else if (e.act != FGT_ACT_NONE) {
    v0 = act_one(v0, e.act);
    v1 = act_one(v1, e.act);
  }
  if (kExt == 1 && e.out_half && (e.aux_mode == FGT_AUX_GRU_ZR || e.aux_mode == FGT_AUX_GRU)) {
    // mixed-precision GRU (update.py:45-60 under autocast): the gates z, r and the candidate q are fp16
    v0 = round_f16(v0);
    v1 = round_f16(v1);
  }
  if (kExt == 1 && e.aux_mode == FGT_AUX_GRU_ZR) {  // fused z | r gates: two C-channel outputs (host guarantees vec)
    const int half = e.N >> 1;
    if (col < half) {
      *reinterpret_cast<float2*>(e.out_f32 + o0) = make_float2(v0, v1);
    } else if (e.out_half) {  // r * h as the fp16 operand of the q conv
      const long long o = off + (col - half);
      load_pair(e.aux, o, o + 1, true, e.aux_vec != 0, a0, a1);
      *reinterpret_cast<uint32_t*>(e.out_hi + o) = pack_f16x2(v0 * a0, v1 * a1);
    } else {
      const long long o = off + (col - half);
      load_pair(e.aux, o, o + 1, true, e.aux_vec != 0, a0, a1);
      uint32_t hw, lw;
      split_bf16x2(v0 * a0, v1 * a1, hw, lw);
      *reinterpret_cast<uint32_t*>(e.out_hi + o) = hw;
      *reinterpret_cast<uint32_t*>(e.out_hi + e.out_plane + o) = lw;
    }
    return;
  }
  if (e.aux_mode == FGT_AUX_ADD) {
    load_pair(e.aux, o0, o1, two, avec, a0, a1);
    v0 += a0;
    v1 += a1;
  } else if (e.aux_mode == FGT_AUX_MUL) {
    load_pair(e.aux, o0, o1, two, avec, a0, a1);
    v0 *= a0;
    v1 *= a1;
  } else if (kExt == 1 && e.aux_mode == FGT_AUX_ADD_RELU) {
    load_pair(e.aux, o0, o1, two, avec, a0, a1);
    if (e.out_half) {  // mixed precision: act(v) is an fp16 tensor before the residual add (RAFT/extractor.py:55-56)
      v0 = round_f16(v0);
      v1 = round_f16(v1);
    }
    v0 = fmaxf(v0 + a0, 0.f);
    v1 = fmaxf(v1 + a1, 0.f);
  } else if (kExt == 1 && e.aux_mode == FGT_AUX_GRU) {  // h' = (1 - z) * h + z * q   (aux = h, aux2 = z, v = q)
    float z0, z1;
    load_pair(e.aux, o0, o1, two, avec, a0, a1);
    load_pair(e.aux2, o0, o1, two, avec, z0, z1);
    if (e.out_half) {  // mixed precision: each of the four fp16 tensor ops of update.py:52,58 rounds to fp16
      v0 = round_f16(round_f16(round_f16(1.f - z0) * a0) + round_f16(z0 * v0));
      v1 = round_f16(round_f16(round_f16(1.f - z1) * a1) + round_f16(z1 * v1));
    } else {
      v0 = (1.f - z0) * a0 + z0 * v0;
      v1 = (1.f - z1) * a1 + z1 * v1;
    }
  }
  if (kExt && (e.out_half || e.r16)) {  // the fp32 copy (a residual or GRU-state operand) holds the same fp16 value as the 16-bit output
    v0 = round_f16(v0);
    v1 = round_f16(v1);
  }
  if (vec) {
    if (e.out_f32) *reinterpret_cast<float2*>(e.out_f32 + o0) = make_float2(v0, v1);
    if (e.out_hi && e.out_half) {
      *reinterpret_cast<uint32_t*>(e.out_hi + o0) = pack_f16x2(v0, v1);
    } else if (e.out_hi) {
      uint32_t hw, lw;
      split_bf16x2(v0, v1, hw, lw);
      *reinterpret_cast<uint32_t*>(e.out_hi + o0) = hw;
      *reinterpret_cast<uint32_t*>(e.out_hi + e.out_plane + o0) = lw;
    }
  } else {
    // generic path: strided channel stores (transposed / NCHW outputs) and N tails
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      if (q == 1 && !two) break;
      const long long o = q ? o1 : o0;
      const float x = q ? v1 : v0;
      if (e.out_f32) e.out_f32[o] = x;
      if (e.out_hi && e.out_half) {
        reinterpret_cast<__half*>(e.out_hi)[o] = __float2half_rn(x);
      } else if (e.out_hi) {
        __nv_bfloat16 h, l;
        split_bf16(x, h, l);
        e.out_hi[o] = h;
        e.out_hi[e.out_plane + o] = l;
      }
    }
  }
}

// ---- Batched epilogue (kExt = 0 or 2, whole tile inside N, unit channel stride, 16-byte aligned rows: `vec4_ok`).
// The operands that do not depend on the accumulators (bias, aux) are loaded for a chunk of JC column groups j at once,
// before the accumulators are final, so the tile waits for global memory once per chunk instead of once per column
// pair. The quad of threads (qc = 0..3) that holds rows (r, r + 8) x channels [8 j, 8 j + 8) swaps pairs with
// `shfl_xor(1)` so that thread qc owns row r + 8 (qc & 1), channels [8 j + 4 (qc >> 1), + 4): one 16-byte fp32 store,
// 8 bytes per 16-bit plane. Each element gets exactly the arithmetic of epi_pair (bias fma, activation, aux), so the
// bits are the same. In-place residual (aux == out_f32): every element is read by the thread that writes it, before
// it writes it.
template <int JC>
struct EpiPre {
  float b[JC][2];  // bias of this thread's accumulator pair (channels 8 j + 2 qc, + 1)
  float4 a[JC];    // aux of the 4 channels this thread stores
};

__device__ __forceinline__ bool aux_loaded(int aux_mode) { return aux_mode == FGT_AUX_ADD || aux_mode == FGT_AUX_MUL; }

template <int JC>
__device__ __forceinline__ void epi_prefetch(EpiPre<JC>& pre, const EpiArgs& e, const float* bias, int j0, int n0,
                                             int qc, long long off, bool valid) {
#pragma unroll
  for (int jj = 0; jj < JC; ++jj) {
    const int col = n0 + (j0 + jj) * 8 + 2 * qc;
    pre.b[jj][0] = bias ? __ldg(bias + col) : 0.f;
    pre.b[jj][1] = bias ? __ldg(bias + col + 1) : 0.f;
  }
  if (aux_loaded(e.aux_mode)) {
    const float* src = e.aux + off + n0 + 4 * (qc >> 1);
#pragma unroll
    for (int jj = 0; jj < JC; ++jj)
      pre.a[jj] = valid ? __ldg(reinterpret_cast<const float4*>(src + (j0 + jj) * 8)) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// kAct: 0 = none, 1 = LeakyReLU(0.2), 2 = any other kExt = 0 activation (act_one).
template <int kAct>
__device__ __forceinline__ float epi_act(float v, int act) {
  if (kAct == 1) return v > 0.f ? v : 0.2f * v;
  if (kAct == 2) return act_one(v, act);
  return v;
}

// kR16: FGT_OUT_HALF_AUTOCAST (the kExt = 2 instantiation): the rounding points of epi_pair's r16 mode, for the modes
// the batched epilogue runs (activation, FGT_AUX_ADD / MUL).
template <int kAct, bool kR16, int JC, int R>
__device__ __forceinline__ void epi_chunk(const EpiArgs& e, const float (&acc)[R], const EpiPre<JC>& pre, int j0,
                                          int n0, int qc, long long off, bool valid) {
  const bool odd = qc & 1;
  const long long ob = off + n0 + 4 * (qc >> 1);
#pragma unroll
  for (int jj = 0; jj < JC; ++jj) {
    const int j = j0 + jj;
    const float b0 = pre.b[jj][0], b1 = pre.b[jj][1];
    const float v00 = fmaf(acc[4 * j], e.alpha, b0), v01 = fmaf(acc[4 * j + 1], e.alpha, b1);
    const float v10 = fmaf(acc[4 * j + 2], e.alpha, b0), v11 = fmaf(acc[4 * j + 3], e.alpha, b1);
    // keep the pair of row (qc & 1), trade the other row's pair with the neighbour qc ^ 1
    const float r0 = __shfl_xor_sync(0xffffffffu, odd ? v00 : v10, 1);
    const float r1 = __shfl_xor_sync(0xffffffffu, odd ? v01 : v11, 1);
    float x[4];
    x[0] = odd ? r0 : v00;
    x[1] = odd ? r1 : v01;
    x[2] = odd ? v10 : r0;
    x[3] = odd ? v11 : r1;
#pragma unroll
    for (int q = 0; q < 4; ++q) x[q] = kR16 ? round_f16(epi_act<kAct>(round_f16(x[q]), e.act)) : epi_act<kAct>(x[q], e.act);
    if (e.aux_mode == FGT_AUX_ADD) {
      x[0] += pre.a[jj].x; x[1] += pre.a[jj].y; x[2] += pre.a[jj].z; x[3] += pre.a[jj].w;
    } else if (e.aux_mode == FGT_AUX_MUL) {
      x[0] *= pre.a[jj].x; x[1] *= pre.a[jj].y; x[2] *= pre.a[jj].z; x[3] *= pre.a[jj].w;
    }
    if (kR16) {  // the fp32 copy holds the fp16 value of the 16-bit output
#pragma unroll
      for (int q = 0; q < 4; ++q) x[q] = round_f16(x[q]);
    }
    if (!valid) continue;
    const long long o = ob + j * 8;
    if (e.out_f32) *reinterpret_cast<float4*>(e.out_f32 + o) = make_float4(x[0], x[1], x[2], x[3]);
    if (e.out_hi && e.out_half) {
      *reinterpret_cast<uint2*>(e.out_hi + o) = make_uint2(pack_f16x2(x[0], x[1]), pack_f16x2(x[2], x[3]));
    } else if (e.out_hi) {
      uint32_t h0, l0, h1, l1;
      split_bf16x2(x[0], x[1], h0, l0);
      split_bf16x2(x[2], x[3], h1, l1);
      *reinterpret_cast<uint2*>(e.out_hi + o) = make_uint2(h0, h1);
      *reinterpret_cast<uint2*>(e.out_hi + e.out_plane + o) = make_uint2(l0, l1);
    }
  }
}

// BN: the wgmma N of the launch (== p.bn). kF16: single-plane fp16 operands (one MMA per K step) instead of
// split-bf16 (three). kSerial: the previous schedule (no early K stage, per-pair epilogue), kept for A/B comparisons.
template <int BN, bool kF16, int kExt, bool kSerial>
__global__ void __launch_bounds__(kGemmThreads, 1) gemm_tc_kernel(const __grid_constant__ GemmParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-byte alignment is required by the 128B swizzle atoms.
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  constexpr uint32_t nplanes = kF16 ? 1u : 2u;
  constexpr uint32_t b_plane_bytes = static_cast<uint32_t>(BN) * 128u;
  constexpr uint32_t stage_bytes = nplanes * (kAPlaneBytes + b_plane_bytes);
  const uint32_t bar_base = smem_base + static_cast<uint32_t>(p.stages) * stage_bytes;
  // barrier layout: full[stages], empty[stages]
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (p.stages + s); };

  if (warp == kProducerWarp && lane == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 8);  // one arrival per consumer warp
    }
    fence_mbar_init();
    for (int i = 0; i < p.num_maps; ++i) tma_prefetch_desc(&p.a_maps[i]);
    tma_prefetch_desc(&p.b_map);
  }
  __syncthreads();
  // PDL: the prologue above overlapped the previous kernel's tail; nothing before this line touches global data
  pdl_launch_dependents();
  pdl_wait();

  const int tiles_per_z = p.tiles_x * p.tiles_y;

  if (warp == kProducerWarp) {
    // ------------------------------------------------------------ TMA producer
    if (elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      const uint32_t tx_bytes = nplanes * (static_cast<uint32_t>(p.a_rows) + static_cast<uint32_t>(p.bn)) * 128u;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        const int nt = tile % p.n_tiles;
        const int mt = tile / p.n_tiles;
        const int z = mt / tiles_per_z;
        const int rem = mt - z * tiles_per_z;
        const int ty = rem / p.tiles_x;
        const int tx = rem - ty * p.tiles_x;
        const int x0 = tx * p.box_w, y0 = ty * p.box_h;
        const int n0 = nt * p.bn;
        const int group = n0 / p.cout_per_group;
        int kidx = 0;
        for (int t = 0; t < p.num_taps; ++t) {
          const TapDesc tap = p.taps[t];
          for (int sgi = 0; sgi < p.num_segs; ++sgi) {
            const SegDesc sg = p.segs[sgi];
            const CUtensorMap* amap = &p.a_maps[sg.map_base + tap.phase];
            const int c0 = sg.c_base + group * sg.c_per_group;
            for (int ch = 0; ch < sg.chunks; ++ch, ++kidx) {
              mbar_wait_quiet(empty_bar(stage), phase ^ 1u);
              const uint32_t sa = smem_base + stage * stage_bytes;
              const uint32_t sb = sa + nplanes * kAPlaneBytes;
              const uint32_t fb = full_bar(stage);
              mbar_expect_tx(fb, tx_bytes);
              const int cc = c0 + ch * kBK;
              tma_load_5d(sa, amap, fb, cc, x0 + tap.dx, y0 + tap.dy, z + tap.dz, 0);
              tma_load_3d(sb, &p.b_map, fb, kidx * kBK, n0, 0);
              if (nplanes == 2) {
                tma_load_5d(sa + kAPlaneBytes, amap, fb, cc, x0 + tap.dx, y0 + tap.dy, z + tap.dz, 1);
                tma_load_3d(sb + b_plane_bytes, &p.b_map, fb, kidx * kBK, n0, 1);
              }
              if (++stage == p.stages) { stage = 0; phase ^= 1u; }
            }
          }
        }
      }
    }
    __syncwarp();
  } else {
    // ------------------------------------------------------------ consumers: MMA + epilogue (warps 0..7)
    const int wg = warp >> 2;
    // Both warpgroups issue their MMAs unconditionally, also when all 64 rows of one lie beyond the tile's a_rows (boxes
    // of <= 64 positions): a branch around wgmma makes ptxas serialise every MMA of the kernel. Rows >= a_rows read
    // stale shared memory and are never stored.
    const uint32_t a_off = static_cast<uint32_t>(wg) * 64u * 128u;
    EpiArgs ep;
    ep.out_f32 = p.out_f32; ep.out_hi = p.out_hi; ep.aux = p.aux; ep.aux2 = p.aux2; ep.out_plane = p.out_plane; ep.os_c = p.os_c;
    ep.alpha = p.alpha; ep.act = p.act; ep.aux_mode = p.aux_mode; ep.vec_ok = p.vec_ok; ep.aux_vec = p.aux_vec; ep.N = p.N;
    ep.out_half = p.out_half;
    ep.r16 = p.r16;
    const int qc = lane & 3;
    int stage = 0;
    uint32_t phase = 0;
    int prev = -1;  // ring stage of the newest issued MMA group; released once a later group has been waited past
    // Schedule: after a tile's last K stage, each warpgroup issues the first K stage of its next tile into the other
    // accumulator array and runs the tile's epilogue while the tensor cores work on it. Stage release, the wgmma group
    // count and the MMA order are those of back-to-back tiles; only the issue point moves. The early stage is issued
    // unconditionally (a runtime trip count around a wgmma makes ptxas serialise all of them); without a next tile it
    // is a dummy stage that waits on no barrier and whose result is never read. Two accumulator arrays fit in the 168
    // registers a thread has at 288 threads (allocated as 12 warps) up to BN = 64.
    constexpr int early = (!kSerial && BN <= 64) ? 1 : 0;  // K stages of a tile issued before the previous epilogue
    // Registers cannot be indexed dynamically: the tile loop runs pairs of tiles with the two arrays in swapped roles.
    float acc0[BN / 2], acc1[BN / 2];

    // Issues the MMAs of K stage `it` of a tile into `acc` (the caller commits the group).
    auto mma_stage = [&](float (&acc)[BN / 2], int it, bool loaded) {
      if (loaded) mbar_wait_quiet(full_bar(stage), phase);
      const uint32_t sa = smem_base + stage * stage_bytes;
      const uint32_t sb = sa + nplanes * kAPlaneBytes;
      const uint64_t a_hi = gmma_desc_sw128(sa + a_off);
      const uint64_t b_hi = gmma_desc_sw128(sb);
      fence_regs(acc);
      wgmma_fence();
      if (nplanes == 2) {
        const uint64_t a_lo = gmma_desc_sw128(sa + kAPlaneBytes + a_off);
        const uint64_t b_lo = gmma_desc_sw128(sb + b_plane_bytes);
#pragma unroll
        for (int k = 0; k < kBK / 16; ++k) {
          const uint64_t ko = static_cast<uint64_t>(k * 2);  // 32 bytes >> 4
          wgmma_ss<BN, kF16>(acc, a_lo + ko, b_hi + ko, (it | k) != 0);
          wgmma_ss<BN, kF16>(acc, a_hi + ko, b_lo + ko, 1u);
          wgmma_ss<BN, kF16>(acc, a_hi + ko, b_hi + ko, 1u);
        }
      } else {
#pragma unroll
        for (int k = 0; k < kBK / 16; ++k) {
          const uint64_t ko = static_cast<uint64_t>(k * 2);
          wgmma_ss<BN, kF16>(acc, a_hi + ko, b_hi + ko, (it | k) != 0);
        }
      }
    };
    auto advance = [&]() {
      if (++stage == p.stages) { stage = 0; phase ^= 1u; }
    };

    // One tile: its remaining K stages into `cur`, the first stage of `next_tile` into `nxt`, the epilogue from `cur`.
    auto run_tile = [&](float (&cur)[BN / 2], float (&nxt)[BN / 2], int tile, int next_tile) {
      const int nt = tile % p.n_tiles;
      const int mt = tile / p.n_tiles;
      const int z = mt / tiles_per_z;
      const int rem = mt - z * tiles_per_z;
      const int ty = rem / p.tiles_x;
      const int tx = rem - ty * p.tiles_x;
      const int n0 = nt * p.bn;

      for (int it = early; it < p.k_iters; ++it) {
        mma_stage(cur, it, true);
        wgmma_commit();
        // the group of the previous stage has retired once at most this one is pending
        wgmma_wait<1>();
        fence_regs(cur);
        if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));
        prev = stage;
        advance();
      }

      // output positions of this thread's two accumulator rows
      long long off[2];
      bool valid[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
        bool v = r < p.a_rows;
        long long o = 0;
        if (p.linear) {
          int row = tx * p.box_w + r;
          v = v && row < p.out_w;
          if (v && p.rowmap) {
            row = p.rowmap[row];
            v = row >= 0;
          }
          if (v) {
            if (p.lin_batch > 0) {
              const int zb = row / p.lin_batch;
              o = zb * p.os_z + static_cast<long long>(row - zb * p.lin_batch) * p.os_x;
            } else {
              o = static_cast<long long>(row) * p.os_x;
            }
          }
        } else {
          const int ry = r / p.box_w;
          const int oy = ty * p.box_h + ry;
          const int ox = tx * p.box_w + (r - ry * p.box_w);
          v = v && oy < p.out_h && ox < p.out_w;
          o = z * p.os_z + static_cast<long long>(oy) * p.os_y + static_cast<long long>(ox) * p.os_x;
        }
        off[h] = o;
        valid[h] = v;
      }
      // The batched epilogue stores row (qc & 1) of the quad's two rows. Its first load batch goes out while the tile's
      // last MMA group runs.
      const bool batched = kExt != 1 && !kSerial && p.vec4_ok && n0 + BN <= p.N;
      const long long off_q = (qc & 1) ? off[1] : off[0];
      const bool valid_q = (qc & 1) ? valid[1] : valid[0];
      // column groups per load batch, as registers allow: 4 at BN = 64 next to two accumulator arrays, half the tile
      // above BN = 96
      constexpr int JC = (early && BN == 64) ? 4 : BN >= 112 ? BN / 16 : BN / 8;
      EpiPre<JC> pre;
      if (batched) epi_prefetch<JC>(pre, ep, p.bias, 0, n0, qc, off_q, valid_q);

      // The next tile's first stage goes to the tensor cores before this tile's epilogue.
      const int last = prev;
      const bool has_next = next_tile < p.total_tiles;
      prev = -1;
      for (int e = 0; e < early; ++e) {
        mma_stage(nxt, 0, has_next);
        if (has_next) {
          prev = stage;
          advance();
        }
      }
      // retire every group of `cur` with a count fixed at compile time (the commit is unconditional: a commit on a
      // divergent path, or a wait ptxas cannot prove covers `cur`, makes it serialise the MMAs)
      if constexpr (early) {
        wgmma_commit();
        wgmma_wait<1>();
      } else {
        wgmma_wait<0>();
      }
      fence_regs(cur);
      if (lane == 0) mbar_arrive(empty_bar(last));

      if (batched) {
        const int act_kind = ep.act == FGT_ACT_NONE ? 0 : ep.act == FGT_ACT_LEAKY02 ? 1 : 2;
#pragma unroll
        for (int j0 = 0; j0 < BN / 8; j0 += JC) {
          if (j0 > 0) epi_prefetch<JC>(pre, ep, p.bias, j0, n0, qc, off_q, valid_q);
          if (act_kind == 0) epi_chunk<0, kExt == 2>(ep, cur, pre, j0, n0, qc, off_q, valid_q);
          else if (act_kind == 1) epi_chunk<1, kExt == 2>(ep, cur, pre, j0, n0, qc, off_q, valid_q);
          else epi_chunk<2, kExt == 2>(ep, cur, pre, j0, n0, qc, off_q, valid_q);
        }
      } else {
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int cl = j * 8 + 2 * qc;
          const int col = n0 + cl;
          if (col < p.N) {
            const bool two = col + 1 < p.N;
            const float b0 = p.bias ? __ldg(p.bias + col) : 0.f;
            const float b1 = (p.bias && two) ? __ldg(p.bias + col + 1) : 0.f;
#pragma unroll
            for (int h = 0; h < 2; ++h)
              if (valid[h])
                epi_pair<kExt>(ep, fmaf(cur[4 * j + 2 * h], ep.alpha, b0), fmaf(cur[4 * j + 2 * h + 1], ep.alpha, b1),
                               off[h], col, two);
          }
        }
      }
    };

    const int step = gridDim.x;
    int tile = blockIdx.x;  // grid <= total_tiles: every CTA has a tile
    if constexpr (early) {
      mma_stage(acc0, 0, true);
      wgmma_commit();
      prev = stage;
      advance();
    }
    if constexpr (early) {
      for (; tile < p.total_tiles; tile += 2 * step) {
        run_tile(acc0, acc1, tile, tile + step);
        if (tile + step >= p.total_tiles) break;
        run_tile(acc1, acc0, tile + step, tile + 2 * step);
      }
    } else {
      // one array: a second one behind the pair loop's exit stays live (spills) and makes ptxas serialise the MMAs
      for (; tile < p.total_tiles; tile += step) run_tile(acc0, acc0, tile, tile + step);
    }
    wgmma_wait<0>();
  }
}

static int floordiv(int a, int b) { return (a >= 0) ? a / b : -((-a + b - 1) / b); }

static bool g_gemm_direct_epilogue = false;  // debugging aid: per-element stores only (A/B comparisons)
static bool g_gemm_direct_aux = false;       // debugging aid: aux operand by per-element loads on the paired path
static bool g_gemm_serial = false;           // debugging aid: the previous tile schedule (A/B timing)

// Widest channel tile. A 256-wide tile leaves room for only two 96 KB stages of the split-bf16 ring, too shallow to
// hide the TMA loads behind the MMAs on H100 (DESIGN.md 4.1).
constexpr int kMaxBN = 128;

// Channel tile of a launch: the requested bn, or, above kMaxBN, the widest multiple of 16 <= kMaxBN that divides it, so
// a requested tile runs as bn / tile equal tiles and never straddles a group boundary the request respects.
static int tile_bn(int bn) {
  int t = bn < kMaxBN ? bn : kMaxBN;
  while (bn % t) t -= 16;
  return t;
}

// wgmma N of a launch = its channel tile (every multiple of 16 up to kMaxBN has an instantiation).
template <bool kF16, int kExt, bool kSerial>
static void* gemm_kernel_for(int n) {
  switch (n) {
    case 16: return reinterpret_cast<void*>(gemm_tc_kernel<16, kF16, kExt, kSerial>);
    case 32: return reinterpret_cast<void*>(gemm_tc_kernel<32, kF16, kExt, kSerial>);
    case 48: return reinterpret_cast<void*>(gemm_tc_kernel<48, kF16, kExt, kSerial>);
    case 64: return reinterpret_cast<void*>(gemm_tc_kernel<64, kF16, kExt, kSerial>);
    case 80: return reinterpret_cast<void*>(gemm_tc_kernel<80, kF16, kExt, kSerial>);
    case 96: return reinterpret_cast<void*>(gemm_tc_kernel<96, kF16, kExt, kSerial>);
    case 112: return reinterpret_cast<void*>(gemm_tc_kernel<112, kF16, kExt, kSerial>);
    case 128: return reinterpret_cast<void*>(gemm_tc_kernel<128, kF16, kExt, kSerial>);
    default: return nullptr;
  }
}

int gemm_tc_launch(const FgtGemmDesc& d, cudaStream_t stream) {
  FGT_REQUIRE(d.num_segs >= 1 && d.num_segs <= 2, FGT_ERR_ARG, "gemm_tc: num_segs=%d", d.num_segs);
  FGT_REQUIRE(d.kx >= 1 && d.ky >= 1 && d.kz >= 1 && d.kx * d.ky * d.kz <= kMaxTaps, FGT_ERR_ARG,
              "gemm_tc: taps %dx%dx%d unsupported", d.kx, d.ky, d.kz);
  FGT_REQUIRE(d.stride >= 1 && d.stride <= 3 && d.dil >= 1, FGT_ERR_ARG, "gemm_tc: stride=%d dil=%d",
              d.stride, d.dil);
  FGT_REQUIRE(d.bn >= 16 && d.bn <= 256 && d.bn % 16 == 0, FGT_ERR_ARG, "gemm_tc: bn=%d", d.bn);
  FGT_REQUIRE(d.groups >= 1 && d.N % d.groups == 0, FGT_ERR_ARG, "gemm_tc: N=%d groups=%d", d.N, d.groups);
  const int cpg_out = d.N / d.groups;
  FGT_REQUIRE(d.groups == 1 || cpg_out % d.bn == 0, FGT_ERR_ARG,
              "gemm_tc: bn=%d must divide N/groups=%d", d.bn, cpg_out);
  const int a_rows = d.box_w * d.box_h;
  FGT_REQUIRE(d.box_w >= 1 && d.box_h >= 1 && a_rows <= 128 && a_rows % 8 == 0 && d.box_w <= 256,
              FGT_ERR_ARG, "gemm_tc: box %dx%d", d.box_w, d.box_h);
  FGT_REQUIRE(d.out_f32 || d.out_hi, FGT_ERR_ARG, "gemm_tc: no output");
  FGT_REQUIRE(d.aux_mode == FGT_AUX_NONE || d.aux, FGT_ERR_ARG, "gemm_tc: aux_mode without aux");
  FGT_REQUIRE(d.aux_mode != FGT_AUX_GRU || d.aux2, FGT_ERR_ARG, "gemm_tc: FGT_AUX_GRU needs aux2");
  FGT_REQUIRE((reinterpret_cast<uintptr_t>(d.w_hi) & 15) == 0 && d.k_pad % 64 == 0, FGT_ERR_ARG,
              "gemm_tc: weights misaligned / k_pad=%d", d.k_pad);
  const int bn = tile_bn(d.bn);

  GemmParams p;
  memset(&p, 0, sizeof(p));
  FGT_REQUIRE(d.terms == 0 || d.terms == 1 || d.terms == 3, FGT_ERR_ARG, "gemm_tc: terms=%d (1 or 3)", d.terms);
  const bool one_term = d.terms == 1;  // operands are single-plane fp16 tensors
  const int s = d.stride;
  const int phases = s * s;
  FGT_REQUIRE(d.num_segs * phases <= kMaxAMaps, FGT_ERR_ARG, "gemm_tc: too many A maps");

  // ---- A tensor maps: one per (segment, stride phase); dims (C, X', Y', Z, plane)
  int chunks_total = 0;
  for (int sgi = 0; sgi < d.num_segs; ++sgi) {
    const FgtASeg& sg = d.seg[sgi];
    FGT_REQUIRE((reinterpret_cast<uintptr_t>(sg.hi) & 15) == 0, FGT_ERR_ARG, "gemm_tc: A base misaligned");
    FGT_REQUIRE(sg.sx % 8 == 0 && (sg.DY == 1 || sg.sy % 8 == 0) && (sg.DZ == 1 || sg.sz % 8 == 0) &&
                    (one_term || sg.plane % 8 == 0),
                FGT_ERR_ARG, "gemm_tc: A strides must be multiples of 8 elements (sx=%lld sy=%lld sz=%lld)",
                sg.sx, sg.sy, sg.sz);
    FGT_REQUIRE(sg.c_count >= 1, FGT_ERR_ARG, "gemm_tc: c_count");
    for (int py = 0; py < s; ++py)
      for (int px = 0; px < s; ++px) {
        const uint64_t dx = static_cast<uint64_t>((sg.DX - px + s - 1) / s);
        const uint64_t dy = static_cast<uint64_t>((sg.DY - py + s - 1) / s);
        uint64_t dims[5] = {static_cast<uint64_t>(sg.C), dx > 0 ? dx : 1, dy > 0 ? dy : 1,
                            static_cast<uint64_t>(sg.DZ), one_term ? 1u : 2u};
        uint64_t strides[4] = {static_cast<uint64_t>(sg.sx) * s * 2, static_cast<uint64_t>(sg.sy) * s * 2,
                               static_cast<uint64_t>(sg.sz) * 2, static_cast<uint64_t>(sg.plane) * 2};
        if (sg.DY == 1) strides[1] = strides[0] * dims[1];
        if (sg.DZ == 1) strides[2] = strides[1] * dims[2];
        if (one_term) strides[3] = strides[2] * dims[3];  // single fp16 plane: the plane dimension has extent 1
        uint32_t box[5] = {kBK, static_cast<uint32_t>(d.box_w), static_cast<uint32_t>(d.box_h), 1, 1};
        const __nv_bfloat16* base =
            reinterpret_cast<const __nv_bfloat16*>(sg.hi) + py * sg.sy + px * sg.sx;
        int rc = encode_map_bf16(&p.a_maps[sgi * phases + py * s + px], base, 5, dims, strides, box);
        if (rc) return rc;
      }
    p.segs[sgi].map_base = sgi * phases;
    p.segs[sgi].c_base = sg.c_base;
    p.segs[sgi].c_per_group = sg.c_per_group;
    p.segs[sgi].chunks = (sg.c_count + kBK - 1) / kBK;
    chunks_total += p.segs[sgi].chunks;
  }
  // ---- taps (z-major, then y, then x: matches packing.py)
  int nt = 0;
  for (int kz = 0; kz < d.kz; ++kz)
    for (int ky = 0; ky < d.ky; ++ky)
      for (int kx = 0; kx < d.kx; ++kx) {
        const int ox = kx * d.dil - d.pad_x, oy = ky * d.dil - d.pad_y;
        const int qx = floordiv(ox, s), qy = floordiv(oy, s);
        TapDesc& t = p.taps[nt++];
        t.phase = static_cast<int8_t>((oy - qy * s) * s + (ox - qx * s));
        FGT_REQUIRE(qx >= -128 && qx <= 127 && qy >= -128 && qy <= 127, FGT_ERR_ARG, "gemm_tc: tap offset");
        t.dx = static_cast<int8_t>(qx);
        t.dy = static_cast<int8_t>(qy);
        t.dz = static_cast<int8_t>(kz - d.pad_z);
      }
  p.num_taps = nt;
  p.num_segs = d.num_segs;
  p.num_maps = d.num_segs * phases;
  p.k_iters = nt * chunks_total;
  FGT_REQUIRE(p.k_iters * kBK == d.k_pad, FGT_ERR_ARG, "gemm_tc: k_pad=%d but schedule needs %d", d.k_pad,
              p.k_iters * kBK);
  // ---- B map: (K, N, plane)
  {
    uint64_t dims[3] = {static_cast<uint64_t>(d.k_pad), static_cast<uint64_t>(d.N), one_term ? 1u : 2u};
    uint64_t strides[2] = {static_cast<uint64_t>(d.k_pad) * 2, static_cast<uint64_t>(d.w_plane) * 2};
    if (one_term) strides[1] = strides[0] * dims[1];
    uint32_t box[3] = {kBK, static_cast<uint32_t>(bn), 1};
    int rc = encode_map_bf16(&p.b_map, d.w_hi, 3, dims, strides, box);
    if (rc) return rc;
  }
  p.linear = (d.out_h == 1 && d.out_z == 1 && d.box_h == 1) ? 1 : 0;
  FGT_REQUIRE(p.linear || (!d.rowmap && d.lin_batch == 0), FGT_ERR_ARG, "gemm_tc: rowmap/lin_batch need linear mode");
  p.tiles_x = (d.out_w + d.box_w - 1) / d.box_w;
  p.tiles_y = (d.out_h + d.box_h - 1) / d.box_h;
  p.tiles_z = d.out_z;
  p.n_tiles = (d.N + bn - 1) / bn;
  p.total_tiles = p.tiles_x * p.tiles_y * p.tiles_z * p.n_tiles;
  p.bn = bn;
  p.box_w = d.box_w;
  p.box_h = d.box_h;
  p.a_rows = a_rows;
  p.N = d.N;
  p.cout_per_group = cpg_out;
  p.out_w = d.out_w;
  p.out_h = d.out_h;
  p.lin_batch = d.lin_batch;
  p.os_z = d.os_z; p.os_y = d.os_y; p.os_x = d.os_x; p.os_c = d.os_c;
  p.rowmap = d.rowmap;
  p.out_f32 = d.out_f32;
  p.out_hi = reinterpret_cast<__nv_bfloat16*>(d.out_hi);
  p.out_plane = d.out_plane;
  p.aux = d.aux;
  p.aux2 = d.aux2;
  p.aux_mode = d.aux_mode;
  p.bias = d.bias;
  p.act = d.act;
  p.alpha = d.alpha;
  // paired channel accesses (8-byte fp32 / 4-byte 16-bit): unit channel stride and every address component even
  auto al = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 7) == 0; };
  p.vec_ok = (d.os_c == 1 && d.os_x % 2 == 0 && d.os_y % 2 == 0 && d.os_z % 2 == 0 && (d.out_half || d.out_plane % 2 == 0) &&
              al(d.out_f32) && al(d.out_hi) && al(d.aux) && al(d.aux2) && !g_gemm_direct_epilogue)
                 ? 1
                 : 0;
  p.aux_vec = g_gemm_direct_aux ? 0 : 1;
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  p.vec4_ok = (p.vec_ok && p.aux_vec && d.os_x % 4 == 0 && d.os_y % 4 == 0 && d.os_z % 4 == 0 &&
               (d.out_half || d.out_plane % 4 == 0) && al16(d.out_f32) && al16(d.aux))
                  ? 1
                  : 0;

  // ---- numerics: 3-term split-bf16 (default) or single-plane fp16 operands (1 MMA per K step)
  const int planes = one_term ? 1 : 2;
  FGT_REQUIRE(d.out_half >= 0 && d.out_half <= FGT_OUT_HALF_AUTOCAST, FGT_ERR_ARG, "gemm_tc: out_half=%d", d.out_half);
  FGT_REQUIRE(d.out_half != 1 || d.out_hi, FGT_ERR_ARG, "gemm_tc: out_half without a 16-bit output");
  FGT_REQUIRE(d.out_half != FGT_OUT_HALF_AUTOCAST || one_term, FGT_ERR_ARG,
              "gemm_tc: FGT_OUT_HALF_AUTOCAST needs a 1-term (fp16) layer");
  p.out_half = (d.out_half && d.out_hi) ? 1 : 0;
  p.r16 = d.out_half == FGT_OUT_HALF_AUTOCAST ? 1 : 0;

  const uint32_t stage_bytes = static_cast<uint32_t>(planes) * (kAPlaneBytes + static_cast<uint32_t>(bn) * 128u);
  const uint32_t fixed = 1024u /*align*/ + 256u /*barriers*/;
  int stages = static_cast<int>((227u * 1024u - fixed) / stage_bytes);
  if (stages > 6) stages = 6;
  FGT_REQUIRE(stages >= 2, FGT_ERR_ARG, "gemm_tc: tile too large for shared memory");
  p.stages = stages;
  const size_t smem = static_cast<size_t>(stages) * stage_bytes + fixed;

  // out_half with an fp32 copy (mixed-precision RAFT): the fp16 rounding before the activation and of the fp32 copy lives
  // in the kExt = 1 epilogue, so the common instantiation keeps the previous code. FGT_OUT_HALF_AUTOCAST (mixed-precision
  // LAFC) has an instantiation of its own, kExt = 2: the batched epilogue with its rounding points, and epi_pair's r16
  // mode where the batched one does not apply; the modes only kExt = 1 has take kExt = 1.
  const bool ext_modes = d.aux_mode == FGT_AUX_ADD_PRE || d.aux_mode == FGT_AUX_ADD_RELU || d.aux_mode == FGT_AUX_GRU ||
                         d.aux_mode == FGT_AUX_GRU_ZR || d.act == FGT_ACT_LEAKY001;
  const bool ext = ext_modes || (d.out_half && d.out_f32 && !p.r16) || (p.r16 && g_gemm_serial);
  const bool r16_batched = p.r16 && !ext;
  if (d.aux_mode == FGT_AUX_GRU_ZR)
    FGT_REQUIRE(d.out_f32 && d.out_hi && p.vec_ok && d.N % 64 == 0 && (d.N / 2) % d.bn == 0 && d.groups == 1, FGT_ERR_ARG,
                "gemm_tc: FGT_AUX_GRU_ZR needs both outputs, aligned unit-stride channels, N=%d a multiple of 64 and "
                "bn=%d dividing N/2", d.N, d.bn);
  void* kern = g_gemm_serial
                   ? (one_term ? (ext ? gemm_kernel_for<true, 1, true>(bn) : gemm_kernel_for<true, 0, true>(bn))
                               : (ext ? gemm_kernel_for<false, 1, true>(bn) : gemm_kernel_for<false, 0, true>(bn)))
                   : (one_term ? (ext           ? gemm_kernel_for<true, 1, false>(bn)
                                  : r16_batched ? gemm_kernel_for<true, 2, false>(bn)
                                                : gemm_kernel_for<true, 0, false>(bn))
                               : (ext ? gemm_kernel_for<false, 1, false>(bn) : gemm_kernel_for<false, 0, false>(bn)));
  FGT_REQUIRE(kern, FGT_ERR_ARG, "gemm_tc: no instantiation for a %d-wide tile", bn);
  // raised once per instantiation: the attribute is per kernel
  static std::mutex attr_mu;
  static std::unordered_set<void*> attr_done;
  {
    std::lock_guard<std::mutex> lk(attr_mu);
    if (!attr_done.count(kern)) {
      FGT_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
      attr_done.insert(kern);
    }
  }
  int grid = num_sms();
  if (grid > p.total_tiles) grid = p.total_tiles;
  FGT_REQUIRE(grid >= 1, FGT_ERR_ARG, "gemm_tc: empty problem");
  launch_k(reinterpret_cast<void (*)(GemmParams)>(kern), dim3(grid), dim3(kGemmThreads), smem, stream, p);
  FGT_CUDA(cudaGetLastError());
  return FGT_OK;
}

}  // namespace fgt

extern "C" int fgt_gemm_tc(const FgtGemmDesc* desc, fgt_stream_t stream) {
  if (!desc) return fgt::set_err(FGT_ERR_ARG, "fgt_gemm_tc: null desc");
  return fgt::gemm_tc_launch(*desc, reinterpret_cast<cudaStream_t>(stream));
}

// Debugging aid (not part of the product interface): bit 0 forces per-element epilogue stores, bit 1 per-element aux
// loads on the paired path; both compute the same arithmetic as the default, so their outputs are bit-identical.
extern "C" int fgt_debug_gemm_direct_epilogue(int on) {
  fgt::g_gemm_direct_epilogue = (on & 1) != 0;
  fgt::g_gemm_direct_aux = (on & 2) != 0;
  return FGT_OK;
}

// Debugging aid (not part of the product interface): nonzero selects the previous tile schedule for launches that
// follow: no K stage of the next tile before a tile's epilogue, and the per-pair epilogue with its loads interleaved with
// the stores. Same MMAs in the same order, so the outputs are bit-identical; one build can time both schedules.
extern "C" int fgt_debug_gemm_serial_epilogue(int on) {
  fgt::g_gemm_serial = on != 0;
  return FGT_OK;
}
