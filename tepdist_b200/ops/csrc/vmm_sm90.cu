// NVLS substrate: symmetric memory out of the CUDA virtual-memory-management API, bound to an NVSwitch multicast object,
// plus the kernels that use it (`multimem.ld_reduce` / `multimem.st` / `multimem.red`: the reduction happens INSIDE the
// switch, a broadcast store leaves the GPU once).
//
//   host plumbing (C ABI, driver API resolved through cudaGetDriverEntryPoint -- no link-time libcuda dependency):
//     tepd_vmm_query / create / import_fd / map / unmap_release      physical allocation <-> POSIX fd <-> mapping
//     tepd_mc_create / add_device / bind                              multicast object over the same physical pages
//   kernels:
//     mc_barrier            cross-rank barrier: ONE multimem.red per rank signals every peer, bounded spin
//     mc_all_reduce_bf16    one-shot NVLS all-reduce of a symmetric bf16 buffer, fused with + bias + residual:
//                           each rank pulls its 1/n slice already reduced by the switch and broadcasts the result
//     mc_rs_adamw_ag        data-parallel optimizer step over NVLS: gradient reduce-scatter = multimem.ld_reduce (fp32 or
//                           bf16 wire), AdamW on the owned shard, bf16 parameter all-gather = multimem.st
//
// The reference reaches the same hardware only through NCCL (SURVEY 2.H K1-K3; dapple_all_reduce_thunk.cc:136-159); it has
// no reduce-scatter and never fuses a collective with the math around it.
#include <cuda.h>
#include "launch.cuh"
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

namespace {

// ------------------------------------------------------------------------------------------------ driver entry points
struct Drv {
  CUresult (*MemCreate)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long);
  CUresult (*MemRelease)(CUmemGenericAllocationHandle);
  CUresult (*MemExport)(void*, CUmemGenericAllocationHandle, CUmemAllocationHandleType, unsigned long long);
  CUresult (*MemImport)(CUmemGenericAllocationHandle*, void*, CUmemAllocationHandleType);
  CUresult (*MemAddressReserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long);
  CUresult (*MemAddressFree)(CUdeviceptr, size_t);
  CUresult (*MemMap)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long);
  CUresult (*MemUnmap)(CUdeviceptr, size_t);
  CUresult (*MemSetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t);
  CUresult (*MemGetGranularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags);
  CUresult (*McCreate)(CUmemGenericAllocationHandle*, const CUmulticastObjectProp*);
  CUresult (*McAddDevice)(CUmemGenericAllocationHandle, CUdevice);
  CUresult (*McBindMem)(CUmemGenericAllocationHandle, size_t, CUmemGenericAllocationHandle, size_t, size_t, unsigned long long);
  CUresult (*McGetGranularity)(size_t*, const CUmulticastObjectProp*, CUmulticastGranularity_flags);
  CUresult (*DeviceGet)(CUdevice*, int);
  CUresult (*DeviceGetAttribute)(int*, CUdevice_attribute, CUdevice);
  bool ok = false;
};

template <typename F>
bool resolve(const char* name, F& fn) {
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || p == nullptr) {
    fprintf(stderr, "[tepdist_b200] driver entry point %s unavailable\n", name);
    return false;
  }
  fn = reinterpret_cast<F>(p);
  return true;
}

Drv& drv() {
  static Drv d;
  static bool tried = false;
  if (!tried) {
    tried = true;
    cudaFree(nullptr);   // make sure the primary context exists and is current
    bool ok = resolve("cuMemCreate", d.MemCreate) && resolve("cuMemRelease", d.MemRelease) &&
              resolve("cuMemExportToShareableHandle", d.MemExport) && resolve("cuMemImportFromShareableHandle", d.MemImport) &&
              resolve("cuMemAddressReserve", d.MemAddressReserve) && resolve("cuMemAddressFree", d.MemAddressFree) &&
              resolve("cuMemMap", d.MemMap) && resolve("cuMemUnmap", d.MemUnmap) && resolve("cuMemSetAccess", d.MemSetAccess) &&
              resolve("cuMemGetAllocationGranularity", d.MemGetGranularity) && resolve("cuMulticastCreate", d.McCreate) &&
              resolve("cuMulticastAddDevice", d.McAddDevice) && resolve("cuMulticastBindMem", d.McBindMem) &&
              resolve("cuMulticastGetGranularity", d.McGetGranularity) && resolve("cuDeviceGet", d.DeviceGet) &&
              resolve("cuDeviceGetAttribute", d.DeviceGetAttribute);
    d.ok = ok;
  }
  return d;
}

CUmemAllocationProp mem_prop(int dev) {
  CUmemAllocationProp prop;
  memset(&prop, 0, sizeof(prop));
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = dev;
  prop.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  return prop;
}

#define DRV_CHECK(call)                                                                                  \
  do {                                                                                                   \
    CUresult r_ = (call);                                                                                \
    if (r_ != CUDA_SUCCESS) {                                                                            \
      fprintf(stderr, "[tepdist_b200] %s failed: CUresult %d (%s:%d)\n", #call, (int)r_, __FILE__, __LINE__); \
      return 1000 + (int)r_;                                                                             \
    }                                                                                                    \
  } while (0)

}  // namespace

// Is multicast available on `dev`, and what size granularity do symmetric allocations need?  (granularity = max of the
// physical-allocation and the multicast minimum granularities; 0 when the VMM API itself is unavailable.)
extern "C" int tepd_vmm_query(int dev, int n_devices, int* mc_supported, long long* granularity) {
  *mc_supported = 0;
  *granularity = 0;
  Drv& d = drv();
  if (!d.ok) return -1;
  CUdevice cd;
  DRV_CHECK(d.DeviceGet(&cd, dev));
  int sup = 0;
  DRV_CHECK(d.DeviceGetAttribute(&sup, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, cd));
  CUmemAllocationProp prop = mem_prop(dev);
  size_t g = 0;
  DRV_CHECK(d.MemGetGranularity(&g, &prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM));
  if (sup) {
    CUmulticastObjectProp mp;
    memset(&mp, 0, sizeof(mp));
    mp.numDevices = n_devices;
    mp.size = g;
    mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    size_t mg = 0;
    CUresult r = d.McGetGranularity(&mg, &mp, CU_MULTICAST_GRANULARITY_MINIMUM);
    if (r != CUDA_SUCCESS) sup = 0;
    else if (mg > g) g = mg;
  }
  *mc_supported = sup;
  *granularity = (long long)g;
  return 0;
}

extern "C" int tepd_vmm_create(int dev, long long bytes, unsigned long long* handle, int* fd) {
  Drv& d = drv();
  if (!d.ok) return -1;
  CUmemAllocationProp prop = mem_prop(dev);
  CUmemGenericAllocationHandle h;
  DRV_CHECK(d.MemCreate(&h, (size_t)bytes, &prop, 0));
  int f = -1;
  DRV_CHECK(d.MemExport(&f, h, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
  *handle = (unsigned long long)h;
  *fd = f;
  return 0;
}

extern "C" int tepd_vmm_import_fd(int fd, unsigned long long* handle) {
  Drv& d = drv();
  if (!d.ok) return -1;
  CUmemGenericAllocationHandle h;
  DRV_CHECK(d.MemImport(&h, (void*)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR));
  *handle = (unsigned long long)h;
  return 0;
}

// Map `handle` (a physical allocation of a peer / of this device, or a multicast object) read-write for `dev`.
extern "C" int tepd_vmm_map(unsigned long long handle, int dev, long long bytes, long long align, void** out) {
  Drv& d = drv();
  if (!d.ok) return -1;
  CUdeviceptr va = 0;
  DRV_CHECK(d.MemAddressReserve(&va, (size_t)bytes, (size_t)align, 0, 0));
  DRV_CHECK(d.MemMap(va, (size_t)bytes, 0, (CUmemGenericAllocationHandle)handle, 0));
  CUmemAccessDesc acc;
  memset(&acc, 0, sizeof(acc));
  acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  acc.location.id = dev;
  acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  DRV_CHECK(d.MemSetAccess(va, (size_t)bytes, &acc, 1));
  *out = (void*)va;
  return 0;
}

extern "C" int tepd_vmm_unmap(void* ptr, long long bytes) {
  Drv& d = drv();
  if (!d.ok) return -1;
  DRV_CHECK(d.MemUnmap((CUdeviceptr)ptr, (size_t)bytes));
  DRV_CHECK(d.MemAddressFree((CUdeviceptr)ptr, (size_t)bytes));
  return 0;
}

extern "C" int tepd_vmm_release(unsigned long long handle) {
  Drv& d = drv();
  if (!d.ok) return -1;
  DRV_CHECK(d.MemRelease((CUmemGenericAllocationHandle)handle));
  return 0;
}

extern "C" int tepd_mc_create(int n_devices, long long bytes, unsigned long long* handle, int* fd) {
  Drv& d = drv();
  if (!d.ok) return -1;
  CUmulticastObjectProp mp;
  memset(&mp, 0, sizeof(mp));
  mp.numDevices = n_devices;
  mp.size = (size_t)bytes;
  mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  CUmemGenericAllocationHandle h;
  DRV_CHECK(d.McCreate(&h, &mp));
  int f = -1;
  DRV_CHECK(d.MemExport(&f, h, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
  *handle = (unsigned long long)h;
  *fd = f;
  return 0;
}

extern "C" int tepd_mc_add_device(unsigned long long mc, int dev) {
  Drv& d = drv();
  if (!d.ok) return -1;
  CUdevice cd;
  DRV_CHECK(d.DeviceGet(&cd, dev));
  DRV_CHECK(d.McAddDevice((CUmemGenericAllocationHandle)mc, cd));
  return 0;
}

extern "C" int tepd_mc_bind(unsigned long long mc, unsigned long long mem, long long bytes) {
  Drv& d = drv();
  if (!d.ok) return -1;
  DRV_CHECK(d.McBindMem((CUmemGenericAllocationHandle)mc, 0, (CUmemGenericAllocationHandle)mem, 0, (size_t)bytes, 0));
  return 0;
}

// ================================================================================================ kernels
namespace {

typedef __nv_bfloat16 bf16;
constexpr long long SPIN_LIMIT = 20000000000LL;   // ~10 s of SM clocks: a peer that never arrives becomes an error flag, not a hang

__device__ __forceinline__ uint32_t ld_acquire_sys_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void mm_red_add_release(uint32_t* mc, uint32_t v) {
  asm volatile("multimem.red.release.sys.global.add.u32 [%0], %1;" ::"l"(mc), "r"(v) : "memory");
}
__device__ __forceinline__ float4 mm_ld_reduce_f32x4(const void* mc) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(mc) : "memory");
  return v;
}
// 8 bf16 summed across the ranks with an fp32 accumulator inside the switch
__device__ __forceinline__ uint4 mm_ld_reduce_bf16x8(const void* mc) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc) : "memory");
  return v;
}
__device__ __forceinline__ void mm_st_b128(void* mc, uint4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "f"(__uint_as_float(v.x)),
               "f"(__uint_as_float(v.y)), "f"(__uint_as_float(v.z)), "f"(__uint_as_float(v.w)) : "memory");
}

// Barrier between the CTAs with the same blockIdx on every rank.  flags_mc / flags_uc: multicast and local views of one
// symmetric u32 per CTA; `count` counts arrivals for ever (rank-count * barriers so far), so nothing is ever reset.
// Returns false after SPIN_LIMIT clocks (and raises *err).
__device__ __forceinline__ bool block_barrier(uint32_t* flags_mc, const uint32_t* flags_uc, uint32_t target, int* err) {
  __syncthreads();
  __shared__ int ok_s;
  if (threadIdx.x == 0) {
    __threadfence_system();
    mm_red_add_release(flags_mc + blockIdx.x, 1u);
    const long long t0 = clock64();
    int ok = 1;
    while ((int32_t)(ld_acquire_sys_u32(flags_uc + blockIdx.x) - target) < 0) {
      if (clock64() - t0 > SPIN_LIMIT) { ok = 0; atomicExch(err, 1); break; }
    }
    ok_s = ok;
  }
  __syncthreads();
  return ok_s != 0;
}

constexpr int MAX_CTAS = 512;   // flag slots per barrier array

// Every launch of a kernel below consumes `uses` barriers per CTA; the running count lives in device memory (epochs[blockIdx])
// so a captured launch is identical at every replay and all ranks advance in lock-step.
__global__ void mc_barrier_kernel(uint32_t* flags_mc, const uint32_t* flags_uc, uint32_t* epochs, int n, int* err) {
  const uint32_t e = epochs[blockIdx.x] + 1;
  block_barrier(flags_mc, flags_uc, e * n, err);
  if (threadIdx.x == 0) epochs[blockIdx.x] = e;
}

// buf: symmetric [total] bf16 holding this rank's partial values.  After the kernel every rank's buf holds
// sum over ranks (+ bias[col] + residual), rounded once to bf16.  total % (8 * n) == 0.
__global__ void __launch_bounds__(512) mc_all_reduce_bf16_kernel(bf16* __restrict__ buf_mc, uint32_t* flags_mc,
                                                                 const uint32_t* flags_uc, uint32_t* epochs, int n, int rank,
                                                                 long long total, int N, const float* __restrict__ bias,
                                                                 const bf16* __restrict__ residual, int* err) {
  const uint32_t e0 = epochs[blockIdx.x];
  if (!block_barrier(flags_mc, flags_uc, (e0 + 1) * n, err)) return;      // every rank's partials are written
  const long long per = total / n;                  // elements this rank reduces
  const long long base = (long long)rank * per;
  const long long nvec = per >> 3;
  const long long step = (long long)gridDim.x * blockDim.x;
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  for (; i + 3 * step < nvec; i += 4 * step) {      // 4 independent 16-byte switch reductions in flight per thread
    uint4 u[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) u[j] = mm_ld_reduce_bf16x8(buf_mc + base + ((i + j * step) << 3));
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long e = base + ((i + j * step) << 3);
      if (bias != nullptr || residual != nullptr) {
        __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u[j]);
        float f[8];
#pragma unroll
        for (int q = 0; q < 4; ++q) { const float2 t = __bfloat1622float2(h[q]); f[2 * q] = t.x; f[2 * q + 1] = t.y; }
        if (bias != nullptr) {
          const int col = (int)(e % N);
#pragma unroll
          for (int q = 0; q < 8; ++q) f[q] += __ldg(bias + col + q);
        }
        if (residual != nullptr) {
          const uint4 r = *reinterpret_cast<const uint4*>(residual + e);
          const __nv_bfloat162* rh = reinterpret_cast<const __nv_bfloat162*>(&r);
#pragma unroll
          for (int q = 0; q < 4; ++q) { const float2 t = __bfloat1622float2(rh[q]); f[2 * q] += t.x; f[2 * q + 1] += t.y; }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) h[q] = __floats2bfloat162_rn(f[2 * q], f[2 * q + 1]);
      }
      mm_st_b128(buf_mc + e, u[j]);
    }
  }
  for (; i < nvec; i += step) {
    const long long e = base + (i << 3);
    uint4 u = mm_ld_reduce_bf16x8(buf_mc + e);
    if (bias != nullptr || residual != nullptr) {
      __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
      float f[8];
#pragma unroll
      for (int q = 0; q < 4; ++q) { const float2 t = __bfloat1622float2(h[q]); f[2 * q] = t.x; f[2 * q + 1] = t.y; }
      if (bias != nullptr) {
        const int col = (int)(e % N);
#pragma unroll
        for (int q = 0; q < 8; ++q) f[q] += __ldg(bias + col + q);
      }
      if (residual != nullptr) {
        const uint4 r = *reinterpret_cast<const uint4*>(residual + e);
        const __nv_bfloat162* rh = reinterpret_cast<const __nv_bfloat162*>(&r);
#pragma unroll
        for (int q = 0; q < 4; ++q) { const float2 t = __bfloat1622float2(rh[q]); f[2 * q] += t.x; f[2 * q + 1] += t.y; }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) h[q] = __floats2bfloat162_rn(f[2 * q], f[2 * q + 1]);
    }
    mm_st_b128(buf_mc + e, u);
  }
  block_barrier(flags_mc, flags_uc, (e0 + 2) * n, err);                   // every rank's slice has landed everywhere
  if (threadIdx.x == 0) epochs[blockIdx.x] = e0 + 2;
}

__device__ __forceinline__ void adamw_one(float& p, float g, float& m, float& v, float lr, float b1, float b2, float eps,
                                          float decay, float bc1, float bc2) {
  m = b1 * m + (1.f - b1) * g;
  v = b2 * v + (1.f - b2) * g * g;
  p -= lr * ((m / bc1) / (sqrtf(v / bc2) + eps) + decay * p);
}

// Flat element range [begin, end) is owned by this rank (8-aligned).  grad_mc: multicast view of the symmetric gradient
// buffer (fp32, or bf16 when GRAD_BF16); param_mc: multicast view of the symmetric bf16 parameter buffer.  No barrier
// inside: the caller brackets a group of bucket launches with mc_barrier (gradients complete / parameters delivered).
template <bool GRAD_BF16>
__device__ __forceinline__ void mc_load_grad8(const void* grad_mc, long long e, float (&g)[8]) {
  if constexpr (GRAD_BF16) {
    const uint4 u = mm_ld_reduce_bf16x8(reinterpret_cast<const bf16*>(grad_mc) + e);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
    for (int q = 0; q < 4; ++q) { const float2 t = __bfloat1622float2(h[q]); g[2 * q] = t.x; g[2 * q + 1] = t.y; }
  } else {
    const float4 a = mm_ld_reduce_f32x4(reinterpret_cast<const float*>(grad_mc) + e);
    const float4 b = mm_ld_reduce_f32x4(reinterpret_cast<const float*>(grad_mc) + e + 4);
    g[0] = a.x; g[1] = a.y; g[2] = a.z; g[3] = a.w; g[4] = b.x; g[5] = b.y; g[6] = b.z; g[7] = b.w;
  }
}

__device__ __forceinline__ void adamw_update8(float (&g)[8], bf16* __restrict__ param_mc, float* __restrict__ master,
                                              float* __restrict__ mom, float* __restrict__ var, long long e, long long n_decay,
                                              float lr, float b1, float b2, float eps, float wd, float bc1, float bc2, float gscale) {
  float p[8], m[8], v[8];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float4 pp = *reinterpret_cast<const float4*>(master + e + 4 * h);
    const float4 mm = *reinterpret_cast<const float4*>(mom + e + 4 * h);
    const float4 vv = *reinterpret_cast<const float4*>(var + e + 4 * h);
    p[4 * h] = pp.x; p[4 * h + 1] = pp.y; p[4 * h + 2] = pp.z; p[4 * h + 3] = pp.w;
    m[4 * h] = mm.x; m[4 * h + 1] = mm.y; m[4 * h + 2] = mm.z; m[4 * h + 3] = mm.w;
    v[4 * h] = vv.x; v[4 * h + 1] = vv.y; v[4 * h + 2] = vv.z; v[4 * h + 3] = vv.w;
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) adamw_one(p[j], g[j] * gscale, m[j], v[j], lr, b1, b2, eps, (e + j < n_decay) ? wd : 0.f, bc1, bc2);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    *reinterpret_cast<float4*>(master + e + 4 * h) = make_float4(p[4 * h], p[4 * h + 1], p[4 * h + 2], p[4 * h + 3]);
    *reinterpret_cast<float4*>(mom + e + 4 * h) = make_float4(m[4 * h], m[4 * h + 1], m[4 * h + 2], m[4 * h + 3]);
    *reinterpret_cast<float4*>(var + e + 4 * h) = make_float4(v[4 * h], v[4 * h + 1], v[4 * h + 2], v[4 * h + 3]);
  }
  uint4 u;
  __nv_bfloat162* h2 = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
  for (int q = 0; q < 4; ++q) h2[q] = __floats2bfloat162_rn(p[2 * q], p[2 * q + 1]);
  mm_st_b128(param_mc + e, u);     // all-gather: one store, the switch replicates it to every rank
}

// Flat element range [begin, end) is owned by this rank (8-aligned).  grad_mc: multicast view of the symmetric gradient
// buffer (fp32, or bf16 when GRAD_BF16); param_mc: multicast view of the symmetric bf16 parameter buffer.  No barrier
// inside: the caller brackets a group of bucket launches with mc_barrier (gradients complete / parameters delivered).
// A switch reduction has several microseconds of latency: every thread keeps UNROLL independent ones in flight.
template <bool GRAD_BF16>
__global__ void __launch_bounds__(256, 2) mc_rs_adamw_ag_kernel(const void* __restrict__ grad_mc, bf16* __restrict__ param_mc,
                                                             float* __restrict__ master, float* __restrict__ mom,
                                                             float* __restrict__ var, long long begin, long long end,
                                                             long long n_decay, float b1, float b2, float eps, float wd,
                                                             const float* __restrict__ hyper) {
  constexpr int UNROLL = 4;
  const float lr = hyper[0], bc1 = hyper[1], bc2 = hyper[2], gscale = hyper[3];
  const long long nvec = (end - begin) >> 3;
  const long long step = (long long)gridDim.x * blockDim.x;
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  for (; i + (UNROLL - 1) * step < nvec; i += UNROLL * step) {
    float g[UNROLL][8];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) mc_load_grad8<GRAD_BF16>(grad_mc, begin + ((i + u * step) << 3), g[u]);
#pragma unroll
    for (int u = 0; u < UNROLL; ++u)
      adamw_update8(g[u], param_mc, master, mom, var, begin + ((i + u * step) << 3), n_decay, lr, b1, b2, eps, wd, bc1, bc2, gscale);
  }
  for (; i < nvec; i += step) {
    float g[8];
    mc_load_grad8<GRAD_BF16>(grad_mc, begin + (i << 3), g);
    adamw_update8(g, param_mc, master, mom, var, begin + (i << 3), n_decay, lr, b1, b2, eps, wd, bc1, bc2, gscale);
  }
}

}  // namespace

#define CS(s) reinterpret_cast<cudaStream_t>(s)

// flags_*: symmetric u32[MAX_CTAS] (multicast / local view); epochs: LOCAL u32[MAX_CTAS]; err: local int.
extern "C" int tepd_mc_barrier(void* flags_mc, const void* flags_uc, void* epochs, int n, void* err, void* stream) {
  mc_barrier_kernel<<<1, 32, 0, CS(stream)>>>((uint32_t*)flags_mc, (const uint32_t*)flags_uc, (uint32_t*)epochs, n, (int*)err);
  return (int)cudaGetLastError();
}

extern "C" int tepd_mc_all_reduce_bf16(void* buf_mc, void* flags_mc, const void* flags_uc, void* epochs, int n, int rank,
                                       long long total, int N, const void* bias, const void* residual, void* err, int ctas,
                                       void* stream) {
  if (total % (8LL * n) || (N & 7)) return -2;
  // 16 CTAs x 512 threads at n >= 4, 32 at n = 2: the switch is the bottleneck and more CTAs only add barrier traffic
  // (not re-measured on H100; tests/mc_worker.py times the choices)
  if (ctas <= 0) ctas = n >= 4 ? 16 : 32;
  if (ctas > MAX_CTAS) ctas = MAX_CTAS;
  mc_all_reduce_bf16_kernel<<<ctas, 512, 0, CS(stream)>>>((bf16*)buf_mc, (uint32_t*)flags_mc, (const uint32_t*)flags_uc,
                                                          (uint32_t*)epochs, n, rank, total, N, (const float*)bias,
                                                          (const bf16*)residual, (int*)err);
  return (int)cudaGetLastError();
}

extern "C" int tepd_mc_rs_adamw_ag(const void* grad_mc, void* param_mc, void* master, void* m, void* v, long long begin,
                                   long long end, long long n_decay, float b1, float b2, float eps, float wd, const void* hyper,
                                   int grad_bf16, int ctas, void* stream) {
  if ((begin & 7) || (end & 7)) return -2;
  if (ctas <= 0) ctas = tepd::num_sms();
  if (grad_bf16)
    mc_rs_adamw_ag_kernel<true><<<ctas, 256, 0, CS(stream)>>>(grad_mc, (bf16*)param_mc, (float*)master, (float*)m, (float*)v, begin,
                                                              end, n_decay, b1, b2, eps, wd, (const float*)hyper);
  else
    mc_rs_adamw_ag_kernel<false><<<ctas, 256, 0, CS(stream)>>>(grad_mc, (bf16*)param_mc, (float*)master, (float*)m, (float*)v, begin,
                                                               end, n_decay, b1, b2, eps, wd, (const float*)hyper);
  return (int)cudaGetLastError();
}
