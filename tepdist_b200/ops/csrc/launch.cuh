// Kernel launch helper with programmatic dependent launch (PDL).
//
// A training step is ~600 short kernels in one stream (one CUDA graph); back-to-back dependent launches leave the GPU idle
// for the launch latency + the next kernel's prologue (barrier init, tensor-map prefetch) every time.
// Kernels launched through tepd::launch carry cudaLaunchAttributeProgrammaticStreamSerialization: they may be scheduled
// while their predecessor is still draining, run their prologue, and block in griddepcontrol.wait (sm90::pdl_wait) until
// the predecessor has completed and its writes are visible -- EVERY kernel launched this way calls pdl_wait() before its
// first global-memory access.  Persistent kernels (grid <= #SMs) call pdl_trigger() right after the wait so the successor
// can be scheduled as their CTAs retire; multi-wave kernels trigger at the end of each CTA.
// TEPDIST_PDL=0 turns the attribute off (plain stream order).
#pragma once
#include <cuda_runtime.h>
#include <stdlib.h>

namespace tepd {

// Streaming multiprocessors of the current device (grid sizes of persistent and grid-stride kernels).
inline int num_sms() {
  static int cached[16] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 16) dev = 0;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

inline bool pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("TEPDIST_PDL");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v == 1;
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

}  // namespace tepd
