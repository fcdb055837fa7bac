// Peer-memory (NVLink / NVSwitch) collectives fused with compute, for one NVLink / NVSwitch node of H100s.
//
// The reference executes every collective as a separate in-stream NCCL call (DAPPLEAllReduceThunk etc., SURVEY
// §2.H K1-K3) and never emits reduce-scatter.  Here the hot collectives are kernels that read / write the peers'
// buffers directly (CUDA IPC mapped, P2P over NVLink 4):
//   * fused_rs_adamw_ag : gradient reduce-scatter (P2P loads of every peer's gradient chunk) + AdamW on the owned
//                         shard of the fp32 master weights / moments + bf16 cast + parameter all-gather (P2P stores
//                         of the updated bf16 shard into every peer's parameter buffer) in ONE pass over memory.
//   * symm_barrier      : flag barrier across ranks through peer memory (release/acquire at system scope).
//   * p2p_reduce_scatter / p2p_all_gather : standalone bucket collectives (used for non-optimizer tensors).
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

// out[begin:end) (local fp32) = sum_r in_r[begin:end)
__global__ void __launch_bounds__(256) p2p_reduce_scatter_kernel(PeerPtrs in, float* __restrict__ out, int n, long long begin,
                                                                 long long end) {
  const long long nvec = (end - begin) >> 2;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    const long long e = begin + (i << 2);
    float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int r = 0; r < MAX_PEERS; ++r)
      if (r < n) {
        float4 x = ld_peer_f4(reinterpret_cast<const float*>(in.p[r]) + e);
        g.x += x.x; g.y += x.y; g.z += x.z; g.w += x.w;
      }
    *reinterpret_cast<float4*>(out + e) = g;
  }
}

// every peer's buffer[begin:end) (16-byte units) = local buffer[begin:end)
__global__ void __launch_bounds__(256) p2p_all_gather_kernel(PeerPtrs bufs, int n, int rank, long long begin16, long long end16) {
  const uint4* src = reinterpret_cast<const uint4*>(bufs.p[rank]);
  for (long long i = begin16 + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < end16; i += (long long)gridDim.x * blockDim.x) {
    const uint4 v = src[i];
#pragma unroll
    for (int r = 0; r < MAX_PEERS; ++r)
      if (r < n && r != rank) reinterpret_cast<uint4*>(bufs.p[r])[i] = v;
  }
}

// out[i] = sum_s slots[s][i] (+ bias[col] + residual[i]); slots is THIS rank's staging buffer [n, rows, N] bf16 that the
// peers' GEMM epilogues (gemm_sm90.cu peer mode 3) filled with plain stores.  8 elements (16 B) per thread per step.
// `bcast`: when n_bcast > 0 the bf16 result is ALSO stored into every peer's buffer bcast.p[r] at element offset
// bcast_off (GEMM -> ALL-reduce: each rank reduces the row block it owns and publishes it to everybody).
__global__ void __launch_bounds__(256) slot_reduce_kernel(const bf16* __restrict__ slots, int n, long long per_slot, int N,
                                                          const float* __restrict__ bias, const bf16* __restrict__ residual,
                                                          bf16* __restrict__ out_bf16, float* __restrict__ out_f32,
                                                          PeerPtrs bcast, int n_bcast, long long bcast_off) {
  const long long nvec = per_slot >> 3;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
    for (int s = 0; s < MAX_PEERS; ++s) {
      if (s < n) {
        const uint4 u = *reinterpret_cast<const uint4*>(slots + s * per_slot + (i << 3));
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 f = __bfloat1622float2(h[e]);
          acc[2 * e] += f.x;
          acc[2 * e + 1] += f.y;
        }
      }
    }
    if (bias != nullptr) {
      const int col = (int)((i << 3) % N);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += __ldg(bias + col + j);
    }
    if (residual != nullptr) {
      const uint4 u = *reinterpret_cast<const uint4*>(residual + (i << 3));
      const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __bfloat1622float2(h[e]);
        acc[2 * e] += f.x;
        acc[2 * e + 1] += f.y;
      }
    }
    if (out_bf16 != nullptr) {
      uint4 u;
      __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
      for (int e = 0; e < 4; ++e) h[e] = __floats2bfloat162_rn(acc[2 * e], acc[2 * e + 1]);
      *reinterpret_cast<uint4*>(out_bf16 + (i << 3)) = u;
    }
    if (n_bcast > 0) {
      uint4 u;
      __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
      for (int e = 0; e < 4; ++e) h[e] = __floats2bfloat162_rn(acc[2 * e], acc[2 * e + 1]);
#pragma unroll
      for (int r = 0; r < MAX_PEERS; ++r)
        if (r < n_bcast) *reinterpret_cast<uint4*>(reinterpret_cast<bf16*>(bcast.p[r]) + bcast_off + (i << 3)) = u;
    }
    if (out_f32 != nullptr) {
      *reinterpret_cast<float4*>(out_f32 + (i << 3)) = make_float4(acc[0], acc[1], acc[2], acc[3]);
      *reinterpret_cast<float4*>(out_f32 + (i << 3) + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
    }
  }
}

// Pull every peer's shard (chunk_bytes each) into the local staging buffer `full` (chunk r at byte offset r*chunk_bytes),
// walking owners in the order rank+1, rank+2, ... -- the same order the chunk-major GEMM (peer mode 4) consumes them.
// All CTAs work on one chunk at a time; the last CTA to finish a chunk publishes flags[owner] = epoch (release, gpu scope).
// `epoch` is the device-resident counter of the SymmBarrier that ran just before (unique per launch, graph-replay safe).
__global__ void __launch_bounds__(512) p2p_gather_chunks_kernel(PeerPtrs shards, uint8_t* __restrict__ full, int n, int rank,
                                                                long long chunk_bytes, uint32_t* flags, uint32_t* cnt,
                                                                const uint32_t* epoch_ptr) {
  const uint32_t epoch = *epoch_ptr;
  const long long nvec = chunk_bytes >> 4;
  for (int c = 1; c < n; ++c) {
    int owner = rank + c;
    if (owner >= n) owner -= n;
    const uint4* src = reinterpret_cast<const uint4*>(shards.p[owner]);
    uint4* dst = reinterpret_cast<uint4*>(full + owner * chunk_bytes);
    long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    const long long step = (long long)gridDim.x * blockDim.x;
    for (; i + 3 * step < nvec; i += 4 * step) {  // 4 independent 16-byte NVLink loads in flight per thread
      uint4 v0, v1, v2, v3;
      asm volatile("ld.global.relaxed.sys.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v0.x), "=r"(v0.y), "=r"(v0.z), "=r"(v0.w) : "l"(src + i));
      asm volatile("ld.global.relaxed.sys.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v1.x), "=r"(v1.y), "=r"(v1.z), "=r"(v1.w) : "l"(src + i + step));
      asm volatile("ld.global.relaxed.sys.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v2.x), "=r"(v2.y), "=r"(v2.z), "=r"(v2.w) : "l"(src + i + 2 * step));
      asm volatile("ld.global.relaxed.sys.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v3.x), "=r"(v3.y), "=r"(v3.z), "=r"(v3.w) : "l"(src + i + 3 * step));
      dst[i] = v0; dst[i + step] = v1; dst[i + 2 * step] = v2; dst[i + 3 * step] = v3;
    }
    for (; i < nvec; i += step) {
      uint4 v;
      asm volatile("ld.global.relaxed.sys.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(src + i));
      dst[i] = v;
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
      const uint32_t prev = atomicAdd(cnt + owner, 1u);
      if (prev == gridDim.x - 1) {
        cnt[owner] = 0;
        __threadfence();
        asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(flags + owner), "r"(epoch) : "memory");
      }
    }
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
extern "C" int tepd_p2p_reduce_scatter(void* const* in_ptrs, void* out, int n, long long begin, long long end, int ctas, void* stream) {
  if (n > MAX_PEERS || (begin & 3) || (end & 3)) return -2;
  if (ctas <= 0) ctas = tepd::num_sms();
  p2p_reduce_scatter_kernel<<<ctas, 256, 0, CS(stream)>>>(MakePtrs(in_ptrs, n), (float*)out, n, begin, end);
  return (int)cudaGetLastError();
}
extern "C" int tepd_p2p_all_gather(void* const* buf_ptrs, int n, int rank, long long begin_bytes, long long end_bytes, int ctas,
                                   void* stream) {
  if (n > MAX_PEERS || (begin_bytes & 15) || (end_bytes & 15)) return -2;
  if (ctas <= 0) ctas = tepd::num_sms();
  p2p_all_gather_kernel<<<ctas, 256, 0, CS(stream)>>>(MakePtrs(buf_ptrs, n), n, rank, begin_bytes >> 4, end_bytes >> 4);
  return (int)cudaGetLastError();
}

// out (bf16 and/or fp32, either may be NULL) = sum over the n slots of `slots` [n, rows, N] (+ bias + residual)
extern "C" int tepd_slot_reduce(const void* slots, int n, long long rows, int N, const void* bias, const void* residual,
                                void* out_bf16, void* out_f32, int ctas, void* stream) {
  if (n > MAX_PEERS || (N & 7)) return -2;
  if (ctas <= 0) ctas = tepd::num_sms() * 4;
  PeerPtrs none;
  for (int i = 0; i < MAX_PEERS; ++i) none.p[i] = nullptr;
  slot_reduce_kernel<<<ctas, 256, 0, CS(stream)>>>((const bf16*)slots, n, rows * N, N, (const float*)bias, (const bf16*)residual,
                                                  (bf16*)out_bf16, (float*)out_f32, none, 0, 0);
  return (int)cudaGetLastError();
}
// GEMM -> all-reduce tail: sum this rank's n slots (+ bias + residual rows) and store the bf16 rows into EVERY peer's
// [M, N] buffer at row block `rank` (out_ptrs[r] + rank * rows * N).
extern "C" int tepd_slot_reduce_bcast(const void* slots, int n, long long rows, int N, const void* bias, const void* residual,
                                      void* const* out_ptrs, int rank, int ctas, void* stream) {
  if (n > MAX_PEERS || (N & 7)) return -2;
  if (ctas <= 0) ctas = tepd::num_sms() * 4;
  slot_reduce_kernel<<<ctas, 256, 0, CS(stream)>>>((const bf16*)slots, n, rows * N, N, (const float*)bias, (const bf16*)residual,
                                                  nullptr, nullptr, MakePtrs(out_ptrs, n), n, (long long)rank * rows * N);
  return (int)cudaGetLastError();
}
extern "C" int tepd_p2p_gather_chunks(void* const* shard_ptrs, void* full, int n, int rank, long long chunk_bytes, void* flags,
                                      void* cnt, const void* epoch, int ctas, void* stream) {
  if (n > MAX_PEERS || (chunk_bytes & 15)) return -2;
  if (ctas <= 0) ctas = 32;
  p2p_gather_chunks_kernel<<<ctas, 512, 0, CS(stream)>>>(MakePtrs(shard_ptrs, n), (uint8_t*)full, n, rank, chunk_bytes,
                                                        (uint32_t*)flags, (uint32_t*)cnt, (const uint32_t*)epoch);
  return (int)cudaGetLastError();
}
