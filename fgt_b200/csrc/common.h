// Host-side helpers shared by the C-ABI translation units: error reporting, TMA descriptor encode.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/fgt_b200.h"

namespace fgt {

// thread-local last-error text (returned by fgt_last_error()).
char* err_buf();
int set_err(int code, const char* fmt, ...);

#define FGT_REQUIRE(cond, code, ...)                   \
  do {                                                 \
    if (!(cond)) return fgt::set_err((code), __VA_ARGS__); \
  } while (0)

#define FGT_CUDA(call)                                                                  \
  do {                                                                                  \
    cudaError_t e__ = (call);                                                           \
    if (e__ != cudaSuccess)                                                             \
      return fgt::set_err(FGT_ERR_CUDA, "%s failed: %s (%s:%d)", #call,                 \
                          cudaGetErrorString(e__), __FILE__, __LINE__);                 \
  } while (0)

// A 16-bit activation argument: split-bf16 with the lo plane `plane` elements after `hi` (plane > 0) or, where
// `f16_ok`, single-plane fp16 (plane == 0). Its kernel accesses `vec` consecutive elements at a time, so hi must be
// 2*vec-byte aligned and plane a multiple of vec. A NULL hi (no such output) passes. FGT_OK, or FGT_ERR_ARG with the
// error text set.
int check_act16(const char* who, const void* hi, long long plane, int vec, bool f16_ok);

// Encode a bf16 tiled tensor map (rank <= 5) with the 128B swizzle and zero OOB fill.
// dims[0] is the contiguous dimension; strides_bytes has rank-1 entries (dims 1..rank-1).
int encode_map_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                    const uint64_t* strides_bytes, const uint32_t* box);

int num_sms();

// Programmatic dependent launch (PDL), opt-in with FGT_PDL=1: kernels are then launched with the
// programmatic-stream-serialization attribute; each calls pdl_launch_dependents() once its prologue is done
// (the next kernel may be scheduled onto SMs as they free up and run its own prologue: barrier init,
// descriptor prefetch) and pdl_wait() before its first global access (blocks until the preceding
// grid has completed and its memory is visible), so ordering is unchanged. Off by default (under CUDA-graph
// replay launch gaps are already small); without the attribute both instructions are no-ops.
bool pdl_enabled();

template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                            Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

#ifdef __CUDACC__
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
#endif

}  // namespace fgt
