// Host-side helpers shared by the C-ABI translation units: error reporting, TMA descriptor encode, kernel launch.
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

// Blocks of a grid-stride launch over `items` work items: ceil(items / block), capped at 16 per SM, at least 1.
int grid_stride(long long items, int block);

// Lets `kernel` use `bytes` of dynamic shared memory (needed above 48 KB). The limit belongs to the kernel as loaded on
// one device, so it is raised once per (kernel, current device); thread-safe. FGT_OK, or FGT_ERR_CUDA with an error
// naming the kernel.
int allow_dynamic_smem(const void* kernel, size_t bytes, const char* name);
template <typename... KArgs>
inline int allow_dynamic_smem(void (*kernel)(KArgs...), size_t bytes, const char* name) {
  return allow_dynamic_smem(reinterpret_cast<const void*>(kernel), bytes, name);
}

// Programmatic dependent launch (PDL), opt-in with FGT_PDL=1: kernels are then launched with the
// programmatic-stream-serialization attribute; each calls pdl_launch_dependents() once its prologue is done
// (the next kernel may be scheduled onto SMs as they free up and run its own prologue: barrier init,
// descriptor prefetch) and pdl_wait() before its first global access (blocks until the preceding
// grid has completed and its memory is visible), so ordering is unchanged. Off by default (under CUDA-graph
// replay launch gaps are already small); without the attribute both instructions are no-ops.
bool pdl_enabled();

// Sets an error naming the kernel, its configuration and `e`, and clears the runtime's last-error state, so the failure
// is reported once, by the entry that launched. Returns FGT_ERR_CUDA.
int launch_failed(const char* name, cudaError_t e, dim3 grid, dim3 block, size_t smem);

// Launches `kernel` on `stream`. FGT_OK, or FGT_ERR_CUDA with an error naming the kernel (`name`). Only the launch's
// own status is checked; a launch that succeeds leaves the runtime's last-error state as it was.
template <typename... KArgs, typename... Args>
inline int launch(const char* name, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, fgt_stream_t stream,
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
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
  return e == cudaSuccess ? FGT_OK : launch_failed(name, e, grid, block, smem);
}

// FGT_LAUNCH(kernel, grid, block, smem, stream, args...): fgt::launch named after `kernel`; a failure returns its code
// from the enclosing function.
#define FGT_LAUNCH(kernel, ...)                                                \
  do {                                                                         \
    if (const int rc__ = fgt::launch(#kernel, kernel, __VA_ARGS__)) return rc__; \
  } while (0)

#ifdef __CUDACC__
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
#endif

}  // namespace fgt
