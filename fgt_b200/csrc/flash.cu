// Fused softmax(QK^T * scale) V on wgmma for FGT's two attentions (never materialises scores).
//
// One CTA = 128 query rows x one head (head dim 128). Keys are consumed in tiles of 64:
//   warp 8     : TMA producer (K tiles and V tiles, two independent 2-deep rings; V stays row-major [keys, d] and is
//                consumed as an MN-major B operand, so the V projection GEMM stores through its paired path instead of
//                a transposed scatter)
//   warps 0..7 : two consumer warpgroups, warpgroup w owns query rows [64 w, 64 w + 64): S_j = Q K_j^T from shared
//                memory (Q staged there once, 128B-swizzled), online softmax on the accumulator registers, then
//                O += P_j V_j with P as the register A operand (the S accumulator layout is the A fragment layout),
//                all 3-term split-bf16 with fp32 accumulation; O stays in registers across key tiles
// The two warpgroups run independently, so one's softmax overlaps the other's MMAs. O is rescaled only when the
// running max outgrows the reference max by more than 2^8 (lazy rescaling; softmax is shift-invariant, so exact).
//
// kF16 (mixed precision): Q, K, V and the output are single-plane fp16; QK^T and P V take one fp16 wgmma per K step
// (P rounded to fp16 as the A operand). The scores, the online softmax and O stay fp32.
//
// mode DENSE    (TMHSA, attention_base.py:93-99): every key tile of the (batch=zone) sequence.
// mode WINDOWED (SWMHSA, attention_flow.py:130-164): a 128-row query tile is two 64-token windows;
//   its key list is [global tiles..., own window tile 2i, own window tile 2i+1] with a block-diagonal
//   mask on the two local tiles (warpgroup w attends to local tile w only). Global (pooled) tokens live after the
//   local rows of each frame.
#include "common.h"
#include "ptx.cuh"

namespace fgt {

constexpr int kKBlk = 64 * 128;       // one (plane, k-chunk) block of K: 64 keys x 128 B
constexpr int kVBlk = 128 * 128;      // one plane of a V tile: two [64 keys x 64 dims (128 B)] halves of 8 KB
constexpr int kVHalf = 64 * 128;
constexpr int kQBlk = 128 * 128;      // one (plane, k-chunk) block of Q: 128 rows x 128 B
constexpr int kKStage = 4 * kKBlk;    // 32 KB
constexpr int kVStage = 2 * kVBlk;    // 32 KB
constexpr int kStages = 2;            // K and V rings
constexpr int kSmemQ = 0;
constexpr int kSmemK = kSmemQ + 4 * kQBlk;            // +64 KB
constexpr int kSmemV = kSmemK + kStages * kKStage;    // +64 KB
constexpr int kSmemBar = kSmemV + kStages * kVStage;  // +64 KB = 192 KB
constexpr int kFlashSmem = kSmemBar + 256 + 1024;
constexpr int kFlashThreads = 288;    // 2 consumer warpgroups + 1 producer warp

struct FlashParams {
  CUtensorMap k_map, v_map;
  const __nv_bfloat16* q_hi;
  long long q_plane, q_batch_stride;
  int q_ld;
  int Lq, Lk, heads;
  int mode;  // 0 dense, 1 windowed
  int n_glob_tiles, glob_start, glob_count;
  float scale_log2;
  __nv_bfloat16* out_hi;
  long long out_plane, out_batch_stride;
  int out_ld;
  const int* out_rowmap;  // optional: query row (batch * Lq + row) -> output row of a [rows, out_ld] buffer, < 0 = dropped
};

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

template <bool kF16>
__global__ void __launch_bounds__(kFlashThreads, 1) flash_kernel(const __grid_constant__ FlashParams p) {
  constexpr int kPlanes = kF16 ? 1 : 2;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int qt = blockIdx.x, head = blockIdx.y, batch = blockIdx.z;

  const uint32_t bar = sbase + kSmemBar;
  auto k_full = [&](int s) { return bar + 8u * (0 + s); };
  auto k_empty = [&](int s) { return bar + 8u * (2 + s); };
  auto v_full = [&](int s) { return bar + 8u * (4 + s); };
  auto v_empty = [&](int s) { return bar + 8u * (6 + s); };

  const int n_tiles = (p.mode == 0) ? (p.Lk + 63) / 64 : p.n_glob_tiles + 2;

  if (warp == 8 && lane == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(k_full(s), 1);
      mbar_init(k_empty(s), 8);  // one arrival per consumer warp
      mbar_init(v_full(s), 1);
      mbar_init(v_empty(s), 8);
    }
    fence_mbar_init();
    tma_prefetch_desc(&p.k_map);
    tma_prefetch_desc(&p.v_map);
  }
  __syncthreads();
  // PDL: the prologue above overlapped the previous kernel's tail; nothing before this line touches global data
  pdl_launch_dependents();
  pdl_wait();

  auto key_row0 = [&](int j) -> int {
    if (p.mode == 0) return j * 64;
    if (j < p.n_glob_tiles) return p.glob_start + j * 64;
    return (2 * qt + (j - p.n_glob_tiles)) * 64;
  };

  if (warp == 8) {
    // ------------------------------------------------------------ K / V producer
    if (elect_one()) {
      int s = 0;
      uint32_t ph = 0;
      for (int j = 0; j < n_tiles; ++j) {
        const int r0 = key_row0(j);
        mbar_wait_quiet(k_empty(s), ph ^ 1u);
        mbar_expect_tx(k_full(s), kPlanes * 2 * kKBlk);
        for (int pl = 0; pl < kPlanes; ++pl)
          for (int kc = 0; kc < 2; ++kc)
            tma_load_4d(sbase + kSmemK + s * kKStage + (pl * 2 + kc) * kKBlk, &p.k_map, k_full(s),
                        head * 128 + kc * 64, r0, batch, pl);
        mbar_wait_quiet(v_empty(s), ph ^ 1u);
        mbar_expect_tx(v_full(s), kPlanes * kVBlk);
        for (int pl = 0; pl < kPlanes; ++pl)
          for (int hf = 0; hf < 2; ++hf)
            tma_load_4d(sbase + kSmemV + s * kVStage + pl * kVBlk + hf * kVHalf, &p.v_map, v_full(s),
                        head * 128 + hf * 64, r0, batch, pl);
        if (++s == kStages) { s = 0; ph ^= 1u; }
      }
    }
    __syncwarp();
    return;
  }

  // -------------------------------------------------------------- consumers (warps 0..7)
  const int wg = warp >> 2;
  {
    // Q tile -> shared memory as the K-major A operand: block (plane, 64-dim chunk) of 128 rows x 128 B, 16-byte chunk c
    // of row r at c ^ (r & 7) (the 128B swizzle). 256 threads x 16 chunks.
    uint8_t* sq = smem_raw + (sbase - smem_u32(smem_raw)) + kSmemQ;
    for (int i = threadIdx.x; i < kPlanes * 128 * 16; i += 256) {
      const int pl = i >> 11, r = (i >> 4) & 127, c = i & 15;
      const int qrow = qt * 128 + r;
      uint4 v = make_uint4(0u, 0u, 0u, 0u);
      if (qrow < p.Lq)
        v = __ldg(reinterpret_cast<const uint4*>(p.q_hi + pl * p.q_plane + batch * p.q_batch_stride +
                                                 static_cast<long long>(qrow) * p.q_ld + head * 128) + c);
      const int kc = c >> 3;
      *reinterpret_cast<uint4*>(sq + (pl * 2 + kc) * kQBlk + r * 128 + (((c & 7) ^ (r & 7)) << 4)) = v;
    }
    fence_proxy_async_smem();  // generic-proxy stores -> visible to the wgmma (async proxy) reads
    asm volatile("bar.sync 1, 256;\n" ::: "memory");
  }

  const int g = lane >> 2, qc = lane & 3;
  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  float m_ref[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const uint32_t q_off = static_cast<uint32_t>(wg) * 64u * 128u;
  int s = 0;
  uint32_t ph = 0;
  for (int j = 0; j < n_tiles; ++j) {
    int n_valid = 64;  // key columns [0, n_valid) of this tile are live for this warpgroup's rows
    if (p.mode == 0) {
      n_valid = min(64, p.Lk - j * 64);
    } else if (j < p.n_glob_tiles) {
      n_valid = min(64, p.glob_count - j * 64);
    } else {
      n_valid = (wg == j - p.n_glob_tiles) ? 64 : 0;
    }
    mbar_wait_quiet(k_full(s), ph);
    float sv[32];
    if (n_valid > 0) {
      fence_regs(sv);
      wgmma_fence();
#pragma unroll
      for (int kc = 0; kc < 2; ++kc) {
        const uint32_t kb = sbase + kSmemK + s * kKStage;
        const uint64_t b_hi = gmma_desc_sw128(kb + (0 * 2 + kc) * kKBlk);
        const uint64_t b_lo = gmma_desc_sw128(kb + (1 * 2 + kc) * kKBlk);
        const uint64_t a_hi = gmma_desc_sw128(sbase + kSmemQ + (0 * 2 + kc) * kQBlk + q_off);
        const uint64_t a_lo = gmma_desc_sw128(sbase + kSmemQ + (1 * 2 + kc) * kQBlk + q_off);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint64_t ko = static_cast<uint64_t>(k * 2);
          if (kF16) {
            wgmma_ss<64, true>(sv, a_hi + ko, b_hi + ko, (kc | k) != 0);
            continue;
          }
          wgmma_ss<64, false>(sv, a_lo + ko, b_hi + ko, (kc | k) != 0);  // Q_lo * K_hi
          wgmma_ss<64, false>(sv, a_hi + ko, b_lo + ko, 1u);             // Q_hi * K_lo
          wgmma_ss<64, false>(sv, a_hi + ko, b_hi + ko, 1u);             // Q_hi * K_hi
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(sv);
    }
    if (lane == 0) mbar_arrive(k_empty(s));

    uint32_t pa_hi[16], pa_lo[16];
    if (n_valid > 0) {
      // thread holds S[row g + 8 h][8 jj + 2 qc + e] in sv[4 jj + 2 h + e]; a row is spread over the 4 lanes of a quad
      if (n_valid != 64) {
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (8 * jj + 2 * qc + e >= n_valid) sv[4 * jj + e] = sv[4 * jj + 2 + e] = -INFINITY;
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float mx = -INFINITY;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) mx = fmaxf(mx, fmaxf(sv[4 * jj + 2 * h], sv[4 * jj + 2 * h + 1]));
        const float m_tile = quad_max(mx) * p.scale_log2;  // scale > 0
        const bool grow = m_tile > m_ref[h] + 8.f;          // also true for the first finite maximum
        const float alpha = grow ? ex2_approx(m_ref[h] - m_tile) : 1.f;  // m_ref = -inf -> 0
        if (grow) m_ref[h] = m_tile;
        const float neg_m = (m_ref[h] == -INFINITY) ? 0.f : -m_ref[h];
        float ps = 0.f;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          sv[4 * jj + 2 * h] = ex2_approx(fmaf(sv[4 * jj + 2 * h], p.scale_log2, neg_m));
          sv[4 * jj + 2 * h + 1] = ex2_approx(fmaf(sv[4 * jj + 2 * h + 1], p.scale_log2, neg_m));
          ps += sv[4 * jj + 2 * h] + sv[4 * jj + 2 * h + 1];
        }
        l_run[h] = l_run[h] * alpha + ps;
        if (grow) {
#pragma unroll
          for (int jj = 0; jj < 16; ++jj) {
            o[4 * jj + 2 * h] *= alpha;
            o[4 * jj + 2 * h + 1] *= alpha;
          }
        }
      }
      // P as the A operand: k16 chunk kk = sv[8 kk .. 8 kk + 7] -> {(g, 2qc), (g + 8, 2qc), (g, 2qc + 8), (g + 8, 2qc + 8)}
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        if (kF16) pa_hi[i] = pack_f16x2(sv[2 * i], sv[2 * i + 1]);
        else split_bf16x2(sv[2 * i], sv[2 * i + 1], pa_hi[i], pa_lo[i]);
      }
    }

    mbar_wait_quiet(v_full(s), ph);
    if (n_valid > 0) {
      const uint32_t vb = sbase + kSmemV + s * kVStage;
      const uint64_t b_hi = gmma_desc_sw128_mn(vb, kVHalf);
      const uint64_t b_lo = gmma_desc_sw128_mn(vb + kVBlk, kVHalf);
      fence_regs(o);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint64_t ko = static_cast<uint64_t>(k * 128);  // 16 keys = two 8-row swizzle atoms = 2048 B >> 4
        const uint32_t ah[4] = {pa_hi[4 * k], pa_hi[4 * k + 1], pa_hi[4 * k + 2], pa_hi[4 * k + 3]};
        if (kF16) {
          wgmma_rs_f16_mnb128(o, ah, b_hi + ko, 1u);
          continue;
        }
        const uint32_t al[4] = {pa_lo[4 * k], pa_lo[4 * k + 1], pa_lo[4 * k + 2], pa_lo[4 * k + 3]};
        wgmma_rs_bf16_mnb128(o, al, b_hi + ko, 1u);  // P_lo * V_hi
        wgmma_rs_bf16_mnb128(o, ah, b_lo + ko, 1u);  // P_hi * V_lo
        wgmma_rs_bf16_mnb128(o, ah, b_hi + ko, 1u);  // P_hi * V_hi
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(o);
    }
    if (lane == 0) mbar_arrive(v_empty(s));
    if (++s == kStages) { s = 0; ph ^= 1u; }
  }

  // normalise, store split-bf16. Output row: in place (batch-strided), or scattered through the row map — the
  // attention then undoes the zone / window regrouping itself (attention_base.py:100-103, attention_flow.py:165-168)
  // and the output projection is a plain row-major GEMM over the real tokens only.
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float inv = 1.f / quad_sum(l_run[h]);
    const int qrow = qt * 128 + wg * 64 + (warp & 3) * 16 + g + 8 * h;
    bool row_ok = qrow < p.Lq;
    long long orow = batch * p.out_batch_stride + static_cast<long long>(qrow) * p.out_ld;
    if (p.out_rowmap && row_ok) {
      const int m = __ldg(p.out_rowmap + static_cast<long long>(batch) * p.Lq + qrow);
      row_ok = m >= 0;
      orow = static_cast<long long>(m) * p.out_ld;
    }
    if (!row_ok) continue;
    __nv_bfloat16* oh = p.out_hi + orow + head * 128 + 2 * qc;
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
      if (kF16) {
        *reinterpret_cast<uint32_t*>(oh + 8 * jj) = pack_f16x2(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
        continue;
      }
      uint32_t hw, lw;
      split_bf16x2(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv, hw, lw);
      *reinterpret_cast<uint32_t*>(oh + 8 * jj) = hw;
      *reinterpret_cast<uint32_t*>(oh + p.out_plane + 8 * jj) = lw;
    }
  }
}

int attention_launch(const FgtAttnDesc& d, fgt_stream_t stream) {
  FGT_REQUIRE(d.head_dim == 128, FGT_ERR_ARG, "attention: head_dim=%d (only 128 supported)", d.head_dim);
  FGT_REQUIRE(d.batches >= 1 && d.heads >= 1 && d.Lq >= 1 && d.Lk >= 1, FGT_ERR_ARG, "attention: empty problem");
  FGT_REQUIRE(d.q_ld % 8 == 0 && d.k_ld % 8 == 0 && d.v_ld % 8 == 0 && d.out_ld % 8 == 0, FGT_ERR_ARG,
              "attention: leading dimensions must be multiples of 8 elements");
  FGT_REQUIRE(d.q_batch_stride % 8 == 0 && d.k_batch_stride % 8 == 0 && d.v_batch_stride % 8 == 0 &&
                  d.out_batch_stride % 8 == 0,
              FGT_ERR_ARG, "attention: batch strides must be multiples of 8 elements");
  FGT_REQUIRE(d.mode == 0 || d.mode == 1, FGT_ERR_ARG, "attention: mode=%d", d.mode);
  FGT_REQUIRE(d.f16 == 0 || d.f16 == 1, FGT_ERR_ARG, "attention: f16=%d (0 split-bf16, 1 single-plane fp16)", d.f16);
  const bool f16 = d.f16 != 0;
  FGT_REQUIRE(!f16 || (d.q_plane == 0 && d.k_plane == 0 && d.v_plane == 0 && d.out_plane == 0), FGT_ERR_ARG,
              "attention: f16 operands are single-plane (plane offsets must be 0)");
  FGT_REQUIRE(d.q_hi && d.k_hi && d.v_hi && d.out_hi, FGT_ERR_ARG, "attention: null operand");
  if (const int rc = check_act16("attention: Q", d.q_hi, d.q_plane, 8, f16)) return rc;
  if (const int rc = check_act16("attention: K", d.k_hi, d.k_plane, 8, f16)) return rc;
  if (const int rc = check_act16("attention: V", d.v_hi, d.v_plane, 8, f16)) return rc;
  if (const int rc = check_act16("attention: output", d.out_hi, d.out_plane, 8, f16)) return rc;
  FlashParams p;
  memset(&p, 0, sizeof(p));
  const uint64_t hd = static_cast<uint64_t>(d.heads) * 128;
  const uint64_t planes = f16 ? 1 : 2;
  p.q_hi = reinterpret_cast<const __nv_bfloat16*>(d.q_hi);
  p.q_plane = d.q_plane;
  p.q_batch_stride = d.q_batch_stride;
  p.q_ld = d.q_ld;
  {
    uint64_t dims[4] = {hd, static_cast<uint64_t>(d.Lk_rows), static_cast<uint64_t>(d.batches), planes};
    uint64_t str[3] = {static_cast<uint64_t>(d.k_ld) * 2, static_cast<uint64_t>(d.k_batch_stride) * 2,
                       static_cast<uint64_t>(d.k_plane) * 2};
    if (d.batches == 1) str[1] = str[0] * dims[1];
    if (f16) str[2] = str[1] * dims[2];  // single plane: the plane dimension has extent 1
    uint32_t box[4] = {64, 64, 1, 1};
    int rc = encode_map_bf16(&p.k_map, d.k_hi, 4, dims, str, box);
    if (rc) return rc;
  }
  {
    uint64_t dims[4] = {hd, static_cast<uint64_t>(d.Lk_rows), static_cast<uint64_t>(d.batches), planes};
    uint64_t str[3] = {static_cast<uint64_t>(d.v_ld) * 2, static_cast<uint64_t>(d.v_batch_stride) * 2,
                       static_cast<uint64_t>(d.v_plane) * 2};
    if (d.batches == 1) str[1] = str[0] * dims[1];
    if (f16) str[2] = str[1] * dims[2];
    uint32_t box[4] = {64, 64, 1, 1};
    int rc = encode_map_bf16(&p.v_map, d.v_hi, 4, dims, str, box);
    if (rc) return rc;
  }
  p.Lq = d.Lq;
  p.Lk = d.Lk;
  p.heads = d.heads;
  p.mode = d.mode;
  if (d.mode == 1) {
    FGT_REQUIRE(d.glob_count >= 1 && d.glob_start % 64 == 0 && d.Lq % 128 == 0, FGT_ERR_ARG,
                "attention: windowed mode needs glob_count>=1, glob_start%%64==0, Lq%%128==0");
    p.n_glob_tiles = (d.glob_count + 63) / 64;
    p.glob_start = d.glob_start;
    p.glob_count = d.glob_count;
  }
  p.scale_log2 = d.scale * 1.4426950408889634f;
  p.out_hi = reinterpret_cast<__nv_bfloat16*>(d.out_hi);
  p.out_plane = d.out_plane;
  p.out_batch_stride = d.out_batch_stride;
  p.out_ld = d.out_ld;
  p.out_rowmap = d.out_rowmap;

  auto kern = f16 ? flash_kernel<true> : flash_kernel<false>;
  if (const int rc = allow_dynamic_smem(kern, kFlashSmem, "flash_kernel")) return rc;
  const dim3 grid((d.Lq + 127) / 128, d.heads, d.batches);
  return launch("flash_kernel", kern, grid, dim3(kFlashThreads), kFlashSmem, stream, p);
}

}  // namespace fgt

extern "C" int fgt_attention(const FgtAttnDesc* desc, fgt_stream_t stream) {
  if (!desc) return fgt::set_err(FGT_ERR_ARG, "fgt_attention: null desc");
  return fgt::attention_launch(*desc, stream);
}
