// Peer memory and the device-side barrier of the multi-GPU exchange (include/fgt_b200.h, "Peer memory").
// One process per GPU; NVLink/NVSwitch P2P stores carry the data (fgt_rownorm_bcast), this file only
// provides the IPC plumbing and the release/acquire barrier that orders those stores against the peers'
// consumers. No reference counterpart (the reference's inference is single-device).
#include <cstring>

#include "common.h"

namespace fgt {

constexpr int kMaxPeers = 8;

struct PeerFlags {
  unsigned long long* flags[kMaxPeers];  // flags[q] = rank q's flag array (n entries), local or peer-mapped
  int n, rank;
};

__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// One warp. Lane q < n: publish "rank has reached epoch e" in peer q's flag array (slot = rank), then wait
// until peer q has published the same epoch in ours (slot = q). Epochs only grow, so `>=` is the test and
// no reset is ever needed. The epoch lives in device memory and is advanced here, which keeps the launch
// identical from call to call (CUDA-graph replay).
__global__ void peer_barrier_kernel(const PeerFlags pf, unsigned long long* __restrict__ epoch_ctr) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ unsigned long long epoch_s;
  if (threadIdx.x == 0) {
    epoch_s = *epoch_ctr + 1ull;
    *epoch_ctr = epoch_s;
  }
  __syncthreads();
  const unsigned long long epoch = epoch_s;
  const int q = threadIdx.x;
  if (q < pf.n) {
    __threadfence_system();  // peer stores of earlier kernels on this stream are performed before the flag
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(pf.flags[q] + pf.rank), "l"(epoch) : "memory");
    const unsigned long long* mine = pf.flags[pf.rank] + q;
    const unsigned long long t0 = global_ns();
    unsigned long long seen = 0;
    for (;;) {
      asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(seen) : "l"(mine) : "memory");
      if (seen >= epoch) break;
      if (global_ns() - t0 > 10000000000ull) {  // 10 s: a peer is gone — fail loudly instead of hanging the GPU
        printf("fgt_peer_barrier: rank %d timed out waiting for rank %d at epoch %llu (saw %llu)\n", pf.rank, q,
               epoch, seen);
        __trap();
      }
      __nanosleep(200);
    }
  }
  __syncthreads();
}

}  // namespace fgt

using namespace fgt;

extern "C" int fgt_peer_alloc(size_t bytes, void** ptr) {
  FGT_REQUIRE(ptr && bytes > 0, FGT_ERR_ARG, "peer_alloc: bad argument");
  FGT_CUDA(cudaMalloc(ptr, bytes));
  FGT_CUDA(cudaMemset(*ptr, 0, bytes));
  FGT_CUDA(cudaDeviceSynchronize());
  return FGT_OK;
}

extern "C" int fgt_peer_free(void* ptr) {
  if (ptr) FGT_CUDA(cudaFree(ptr));
  return FGT_OK;
}

extern "C" int fgt_peer_export(void* ptr, unsigned char handle[64]) {
  FGT_REQUIRE(ptr && handle, FGT_ERR_ARG, "peer_export: null argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handle size");
  cudaIpcMemHandle_t h;
  FGT_CUDA(cudaIpcGetMemHandle(&h, ptr));
  memcpy(handle, &h, 64);
  return FGT_OK;
}

extern "C" int fgt_peer_import(const unsigned char handle[64], void** ptr) {
  FGT_REQUIRE(ptr && handle, FGT_ERR_ARG, "peer_import: null argument");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, 64);
  FGT_CUDA(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return FGT_OK;
}

extern "C" int fgt_peer_unimport(void* ptr) {
  if (ptr) FGT_CUDA(cudaIpcCloseMemHandle(ptr));
  return FGT_OK;
}

extern "C" int fgt_peer_barrier(void* const* flags_host, int n, int rank, void* epoch_ctr, fgt_stream_t stream) {
  FGT_REQUIRE(flags_host && epoch_ctr && n >= 1 && n <= kMaxPeers && rank >= 0 && rank < n, FGT_ERR_ARG,
              "peer_barrier: n=%d rank=%d", n, rank);
  PeerFlags pf;
  for (int q = 0; q < kMaxPeers; ++q)
    pf.flags[q] = q < n ? reinterpret_cast<unsigned long long*>(flags_host[q]) : nullptr;
  pf.n = n;
  pf.rank = rank;
  for (int q = 0; q < n; ++q) FGT_REQUIRE(pf.flags[q], FGT_ERR_ARG, "peer_barrier: flags[%d] is NULL", q);
  FGT_LAUNCH(peer_barrier_kernel, dim3(1), dim3(32), 0, stream, pf, reinterpret_cast<unsigned long long*>(epoch_ctr));
  return FGT_OK;
}
