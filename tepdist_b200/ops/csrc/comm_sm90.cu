// Peer-memory (NVLink / NVSwitch) collectives fused with compute, for one NVLink / NVSwitch node of H100s.
//
// The reference executes every collective as a separate in-stream NCCL call (DAPPLEAllReduceThunk etc., SURVEY
// §2.H K1-K3) and never emits reduce-scatter.  Here the hot collectives are kernels that read / write the peers'
// buffers directly (CUDA IPC mapped, P2P over NVLink 4):
//   * fused_rs_adamw_ag : gradient reduce-scatter (P2P loads of every peer's gradient chunk) + AdamW on the owned
//                         shard of the fp32 master weights / moments + bf16 cast + parameter all-gather (P2P stores
//                         of the updated bf16 shard into every peer's parameter buffer) in ONE pass over memory.
//   * symm_barrier      : flag barrier across ranks through peer memory (release/acquire at system scope).
// IPC plumbing (alloc / export / import) is exposed with a C ABI for the Python SymmetricMemory wrapper.
#include "launch.cuh"
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

namespace {

constexpr int MAX_PEERS = 8;
typedef __nv_bfloat16 bf16;

struct PeerPtrs {
  void* p[MAX_PEERS];
};

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ float4 ld_peer_f4(const float* p) {
  float4 v;
  asm volatile("ld.global.relaxed.sys.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}

// Every rank writes its epoch into slot [my_rank] of every peer's flag array, then waits until its own array shows
// that epoch from everybody.  One CTA, one thread per peer.  The epoch lives in device memory and is advanced by the
// kernel itself, so the launch is identical every time (CUDA-graph replay safe); all ranks advance in lock-step.
__global__ void symm_barrier_kernel(PeerPtrs flags, int n, int rank, uint32_t* local_epoch) {
  const int t = threadIdx.x;
  const uint32_t epoch = *local_epoch + 1;
  __syncthreads();
  if (t < n) {
    __threadfence_system();
    st_release_sys(reinterpret_cast<uint32_t*>(flags.p[t]) + rank, epoch);
    const uint32_t* mine = reinterpret_cast<const uint32_t*>(flags.p[rank]) + t;
    const long long t0 = clock64();
    while ((int32_t)(ld_acquire_sys(mine) - epoch) < 0) {
      if (clock64() - t0 > 20000000000LL) __trap();   // ~10 s of SM clocks: a peer that never arrives fails the launch loudly
    }
  }
  __syncthreads();
  if (t == 0) *local_epoch = epoch;
}

__device__ __forceinline__ void adamw_one(float& p, float g, float& m, float& v, float lr, float b1, float b2, float eps,
                                          float decay, float bc1, float bc2) {
  m = b1 * m + (1.f - b1) * g;
  v = b2 * v + (1.f - b2) * g * g;
  p -= lr * ((m / bc1) / (sqrtf(v / bc2) + eps) + decay * p);
}

// Flat element range [begin, end) is owned by this rank.  grads.p[r] / params.p[r] are rank r's full flat buffers.
// master / m / v are THIS rank's flat fp32 buffers (indexed with the same flat index).
__global__ void __launch_bounds__(256) fused_rs_adamw_ag_kernel(PeerPtrs grads, PeerPtrs params, float* __restrict__ master,
                                                                float* __restrict__ mom, float* __restrict__ var, int n,
                                                                long long begin, long long end, long long n_decay, float b1,
                                                                float b2, float eps, float wd, const float* __restrict__ hyper,
                                                                int n_grad) {
  const float lr = hyper[0], bc1 = hyper[1], bc2 = hyper[2], gscale = hyper[3];
  const long long nvec = (end - begin) >> 2;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    const long long e = begin + (i << 2);
    float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int r = 0; r < MAX_PEERS; ++r) {
      if (r < n_grad) {   // n_grad == n: reduce-scatter; n_grad == 1: the gradient is already complete on every rank
        float4 x = ld_peer_f4(reinterpret_cast<const float*>(grads.p[r]) + e);
        g.x += x.x; g.y += x.y; g.z += x.z; g.w += x.w;
      }
    }
    float4 pp = *reinterpret_cast<float4*>(master + e);
    float4 mm = *reinterpret_cast<float4*>(mom + e);
    float4 vv = *reinterpret_cast<float4*>(var + e);
    float pa[4] = {pp.x, pp.y, pp.z, pp.w}, ga[4] = {g.x, g.y, g.z, g.w};
    float ma[4] = {mm.x, mm.y, mm.z, mm.w}, va[4] = {vv.x, vv.y, vv.z, vv.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) adamw_one(pa[j], ga[j] * gscale, ma[j], va[j], lr, b1, b2, eps, (e + j < n_decay) ? wd : 0.f, bc1, bc2);
    *reinterpret_cast<float4*>(master + e) = make_float4(pa[0], pa[1], pa[2], pa[3]);
    *reinterpret_cast<float4*>(mom + e) = make_float4(ma[0], ma[1], ma[2], ma[3]);
    *reinterpret_cast<float4*>(var + e) = make_float4(va[0], va[1], va[2], va[3]);
    __nv_bfloat162 lo = __floats2bfloat162_rn(pa[0], pa[1]), hi = __floats2bfloat162_rn(pa[2], pa[3]);
    uint2 u;
    u.x = *reinterpret_cast<uint32_t*>(&lo);
    u.y = *reinterpret_cast<uint32_t*>(&hi);
#pragma unroll
    for (int r = 0; r < MAX_PEERS; ++r)
      if (r < n) *reinterpret_cast<uint2*>(reinterpret_cast<bf16*>(params.p[r]) + e) = u;  // all-gather by P2P store
  }
}

PeerPtrs MakePtrs(void* const* ptrs, int n) {
  PeerPtrs p;
  for (int i = 0; i < MAX_PEERS; ++i) p.p[i] = i < n ? ptrs[i] : nullptr;
  return p;
}

}  // namespace

#define CS(s) reinterpret_cast<cudaStream_t>(s)

// ---------------------------------------------------------------------------------------- IPC plumbing
extern "C" int tepd_symm_alloc(long long bytes, void** out) {
  cudaError_t e = cudaMalloc(out, (size_t)bytes);
  if (e != cudaSuccess) return (int)e;
  return (int)cudaMemset(*out, 0, (size_t)bytes);
}
extern "C" int tepd_symm_free(void* p) { return (int)cudaFree(p); }
extern "C" int tepd_ipc_get_handle(void* p, void* handle64) {
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) return (int)e;
  memcpy(handle64, &h, sizeof(h));
  return 0;
}
extern "C" int tepd_ipc_open(const void* handle64, void** out) {
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, sizeof(h));
  return (int)cudaIpcOpenMemHandle(out, h, cudaIpcMemLazyEnablePeerAccess);
}
extern "C" int tepd_ipc_close(void* p) { return (int)cudaIpcCloseMemHandle(p); }
extern "C" int tepd_ipc_handle_size() { return (int)sizeof(cudaIpcMemHandle_t); }

// ---------------------------------------------------------------------------------------- kernels
extern "C" int tepd_symm_barrier(void* const* flag_ptrs, int n, int rank, void* local_epoch, void* stream) {
  if (n > MAX_PEERS) return -2;
  symm_barrier_kernel<<<1, 32, 0, CS(stream)>>>(MakePtrs(flag_ptrs, n), n, rank, (uint32_t*)local_epoch);
  return (int)cudaGetLastError();
}
extern "C" int tepd_fused_rs_adamw_ag(void* const* grad_ptrs, void* const* param_ptrs, void* master, void* m, void* v, int n,
                                      long long begin, long long end, long long n_decay, float b1, float b2, float eps, float wd,
                                      const void* hyper, int ctas, void* stream, int n_grad) {
  if (n > MAX_PEERS || (begin & 3) || (end & 3)) return -2;
  if (ctas <= 0) ctas = tepd::num_sms() * 2;
  if (n_grad <= 0 || n_grad > n) n_grad = n;   // grad_ptrs[0 .. n_grad) are read (n_grad == 1: grad_ptrs[0] must be local)
  fused_rs_adamw_ag_kernel<<<ctas, 256, 0, CS(stream)>>>(MakePtrs(grad_ptrs, n_grad), MakePtrs(param_ptrs, n), (float*)master,
                                                        (float*)m, (float*)v, n, begin, end, n_decay, b1, b2, eps, wd,
                                                        (const float*)hyper, n_grad);
  return (int)cudaGetLastError();
}
