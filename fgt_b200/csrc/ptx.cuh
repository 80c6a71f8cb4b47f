// Thin inline-PTX layer for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA).
// Everything here is device-side plumbing shared by gemm_tc.cu, flash.cu and conv_tail.cu.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace fgt {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait without a diagnostic print, for kernels that issue wgmma: any function call (printf) in such a kernel
// makes ptxas serialise its warpgroup MMAs. A broken pipeline traps (context error) instead of hanging.
__device__ __forceinline__ void mbar_wait_quiet(uint32_t bar, uint32_t parity) {
#pragma unroll 1
  for (int i = 0; i < 2048; ++i)
    if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) __trap();  // ~2 s at 2 GHz
  }
}
// Bounded wait: a broken pipeline prints which barrier stalled and traps (context error) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
#pragma unroll 1
  for (int i = 0; i < 2048; ++i)
    if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) {  // ~2 s at 2 GHz
      printf("fgt: mbarrier watchdog: block %d thread %d bar 0x%x parity %u\n", blockIdx.x, threadIdx.x, bar,
             parity);
      __trap();
    }
  }
}

// ---------------------------------------------------------------- fences
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];\n" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0,
                                            int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];\n" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0,
                                            int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];\n" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0,
                                            int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6, %7}], [%2];\n" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}

// ---------------------------------------------------------------- wgmma (bf16 / fp16 in, f32 accumulate in registers)
// Shared-memory matrix descriptor (sm_90 layout) for a K-major tile stored as rows of 128 bytes with the 128B swizzle
// (what TMA writes with CU_TENSOR_MAP_SWIZZLE_128B): 8-row atoms of 1024 B. Advance K by 16 elements with +2 (32 B >> 4).
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);         // start address  [0,14)
  d |= static_cast<uint64_t>(1) << 16;                         // LBO (unused for swizzled K-major)
  d |= static_cast<uint64_t>(1024 >> 4) << 32;                 // SBO = 8 rows * 128 B
  d |= static_cast<uint64_t>(1) << 62;                         // layout: SWIZZLE_128B
  return d;
}
// Same swizzle, MN-major operand (the N index is the contiguous one): a [K rows x 64 elements (128 B)] block per
// 64-wide slice of the N extent, 8-row atoms of 1024 B along K; `mn_block_bytes` = distance between the slices.
// Used for V [keys, d] as the B operand of P.V (K = keys, N = d). Advance K by 16 rows with +128 (2048 B >> 4).
__device__ __forceinline__ uint64_t gmma_desc_sw128_mn(uint32_t saddr, uint32_t mn_block_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);         // start address  [0,14)
  d |= static_cast<uint64_t>(mn_block_bytes >> 4) << 16;       // LBO: next 64-element slice along N
  d |= static_cast<uint64_t>(1024 >> 4) << 32;                 // SBO: next 8 rows along K
  d |= static_cast<uint64_t>(1) << 62;                         // layout: SWIZZLE_128B
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory");
}
// Keeps the compiler from moving reads / writes of accumulator registers across wgmma fences and waits.
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] * B[16 x N], A and B from shared memory (K-major descriptors). Accumulator fragment of
// thread t of the warpgroup: d[4 j + 2 h + e] = D[16 (t / 32) + (t % 32) / 4 + 8 h][8 j + 2 (t % 4) + e].
// kF16: fp16 operands instead of bf16. Specialisations for every N the engines use are in wgmma.cuh.
template <int N, bool kF16>
__device__ __forceinline__ void wgmma_ss(float (&d)[N / 2], uint64_t a, uint64_t b, uint32_t scale_d);

// ---------------------------------------------------------------- split-bf16 helpers
// A float v is carried as hi = bf16(v), lo = bf16(v - hi): hi + lo reproduces v to ~2^-17 relative.
__device__ __forceinline__ void split_bf16(float v, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(v);
  lo = __float2bfloat16_rn(v - __bfloat162float(hi));
}
// Two floats -> packed split-bf16 words: hi = {bf16(e0) | bf16(e1) << 16}, lo = residuals likewise.
// cvt.rn.bf16x2.f32 converts and packs two values in one instruction (first operand -> upper half).
__device__ __forceinline__ void split_bf16x2(float e0, float e1, uint32_t& hi, uint32_t& lo) {
  asm volatile("cvt.rn.bf16x2.f32 %0, %1, %2;\n" : "=r"(hi) : "f"(e1), "f"(e0));
  const float r0 = e0 - __uint_as_float(hi << 16);
  const float r1 = e1 - __uint_as_float(hi & 0xffff0000u);
  asm volatile("cvt.rn.bf16x2.f32 %0, %1, %2;\n" : "=r"(lo) : "f"(r1), "f"(r0));
}
// Two floats -> packed fp16 pair {f16(e0) | f16(e1) << 16}, round to nearest, saturating to the finite range.
__device__ __forceinline__ uint32_t pack_f16x2(float e0, float e1) {
  uint32_t r;
  asm volatile("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;\n" : "=r"(r) : "f"(e1), "f"(e0));
  return r;
}
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;\n" : "=f"(y) : "f"(x));
  return y;
}
// Nearest fp16 value, as fp32: where the reference under autocast makes an fp16 tensor.
__device__ __forceinline__ float round_f16(float v) { return __half2float(__float2half_rn(v)); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---------------------------------------------------------------- 16-bit activation stores
// A 16-bit activation is split-bf16 when plane > 0 (hi[i] = bf16(v), hi[plane + i] = bf16(v - hi)) and single-plane
// fp16 when plane == 0 (hi[i] = fp16(v)). store16* write 1, 2, 4 or 8 consecutive values at hi[0..]; a store of n
// values takes 2n-byte aligned addresses (the host's check_act16). Stores of two or more fp16 values saturate to the
// finite range (pack_f16x2), the single one rounds as __float2half_rn.
__device__ __forceinline__ void store16(__nv_bfloat16* hi, long long plane, float v) {
  if (plane == 0) {
    *reinterpret_cast<__half*>(hi) = __float2half_rn(v);
  } else {
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    hi[0] = h;
    hi[plane] = l;
  }
}

__device__ __forceinline__ void store16x2(__nv_bfloat16* hi, long long plane, float a, float b) {
  if (plane == 0) {
    *reinterpret_cast<uint32_t*>(hi) = pack_f16x2(a, b);
  } else {
    uint32_t h, l;
    split_bf16x2(a, b, h, l);
    *reinterpret_cast<uint32_t*>(hi) = h;
    *reinterpret_cast<uint32_t*>(hi + plane) = l;
  }
}

// Four values converted once, for a store to several places (lo is zero when plane == 0).
struct Packed16x4 {
  uint2 hi, lo;
};

__device__ __forceinline__ Packed16x4 pack16x4(long long plane, float a, float b, float c, float d) {
  Packed16x4 p = {};
  if (plane == 0) {
    p.hi = make_uint2(pack_f16x2(a, b), pack_f16x2(c, d));
  } else {
    split_bf16x2(a, b, p.hi.x, p.lo.x);
    split_bf16x2(c, d, p.hi.y, p.lo.y);
  }
  return p;
}

__device__ __forceinline__ void store16x4(__nv_bfloat16* hi, long long plane, const Packed16x4& p) {
  *reinterpret_cast<uint2*>(hi) = p.hi;
  if (plane) *reinterpret_cast<uint2*>(hi + plane) = p.lo;
}

__device__ __forceinline__ void store16x4(__nv_bfloat16* hi, long long plane, float a, float b, float c, float d) {
  store16x4(hi, plane, pack16x4(plane, a, b, c, d));
}

__device__ __forceinline__ void zero16x4(__nv_bfloat16* hi, long long plane) { store16x4(hi, plane, Packed16x4{}); }

__device__ __forceinline__ void store16x8(__nv_bfloat16* hi, long long plane, const float (&v)[8]) {
  if (plane == 0) {
    *reinterpret_cast<uint4*>(hi) =
        make_uint4(pack_f16x2(v[0], v[1]), pack_f16x2(v[2], v[3]), pack_f16x2(v[4], v[5]), pack_f16x2(v[6], v[7]));
  } else {
    uint32_t h[4], l[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) split_bf16x2(v[2 * t], v[2 * t + 1], h[t], l[t]);
    *reinterpret_cast<uint4*>(hi) = make_uint4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<uint4*>(hi + plane) = make_uint4(l[0], l[1], l[2], l[3]);
  }
}

}  // namespace fgt

#include "wgmma.cuh"
