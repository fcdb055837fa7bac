// Mixture-of-experts hot path for sm_90a: peer-memory all-to-all dispatch fused with fp8 quantisation, fp8 (e4m3)
// grouped expert GEMM (wgmma e4m3, tepd_gemm_fp8 in gemm_sm90.cu) with per-token / per-expert scales applied in the
// epilogue, and a
// peer-memory combine that pulls expert outputs back and applies the gate weights.
//
// The reference implements expert parallelism as einsum dispatch/combine + a hand-rolled ncclSend/ncclRecv all-to-all
// (DAPPLEAllToAllThunk, SURVEY K3; examples/gpt_moe/layers/moe_layers.py:425-446).  Here a token row travels exactly
// once over NVLink, already quantised, straight into the owning expert's input buffer:
//   dispatch : x[t, :] (bf16) --row amax--> e4m3 + fp32 scale --P2P st--> rank(e).xin[e_local, src*C + slot, :]
//   expert FC: h = gelu((xin . w1^T) * row_scale * w_scale + b1)      wgmma fp8, register accumulators, bf16 out
//   combine  : out[t, :] = sum_k gate[t,k] * rank(e_k).y[e_local, src*C + slot, :]        P2P loads
// Slots are assigned per (expert, source rank) region, so ranks never contend for a slot (GShard local groups).
#include "sm90_ptx.cuh"
#include "launch.cuh"
#include <cuda_fp8.h>
#include <stdio.h>

using namespace sm90;

namespace {

constexpr int MAXP = 8;
struct Peers {
  void* p[MAXP];
};

// ------------------------------------------------------------------ dispatch (quantise + all-to-all push)
// route[t*K + k] = e * 65536 + slot, or -1 when the token was dropped for that choice.
__global__ void __launch_bounds__(256) moe_dispatch_kernel(const __nv_bfloat16* __restrict__ x, const int* __restrict__ route, Peers xin,
                                                          Peers xscale, int T, int M, int top_k, int experts_per_rank, int cap_per_src,
                                                          int n_ranks, int src_rank) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= T * top_k) return;
  const int r = route[warp];
  if (r < 0) return;
  const int t = warp / top_k, e = r >> 16, slot = r & 0xFFFF;
  const int owner = e / experts_per_rank, el = e % experts_per_rank;
  const __nv_bfloat16* row = x + (size_t)t * M;
  // pass 1: row amax (M <= 8192: each lane keeps its values in registers, 8 per 16-byte vector)
  float amax = 0.f;
  for (int v = lane; v < (M >> 3); v += 32) {
    uint4 u = __ldg(reinterpret_cast<const uint4*>(row) + v);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float2 f = __bfloat1622float2(h[i]);
      amax = fmaxf(amax, fmaxf(fabsf(f.x), fabsf(f.y)));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  const float scale = amax > 0.f ? amax / 448.f : 1.f, inv = 1.f / scale;
  const size_t drow = ((size_t)el * n_ranks + src_rank) * cap_per_src + slot;
  uint8_t* dst = reinterpret_cast<uint8_t*>(xin.p[owner]) + drow * M;
  for (int v = lane; v < (M >> 3); v += 32) {
    uint4 u = __ldg(reinterpret_cast<const uint4*>(row) + v);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
    uint2 q;
    uint8_t* qb = reinterpret_cast<uint8_t*>(&q);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float2 f = __bfloat1622float2(h[i]);
      qb[2 * i] = (uint8_t)__nv_cvt_float_to_fp8(f.x * inv, __NV_SATFINITE, __NV_E4M3);
      qb[2 * i + 1] = (uint8_t)__nv_cvt_float_to_fp8(f.y * inv, __NV_SATFINITE, __NV_E4M3);
    }
    reinterpret_cast<uint2*>(dst)[v] = q;  // 8 fp8 values per store, straight into the expert owner's memory
  }
  if (lane == 0) reinterpret_cast<float*>(xscale.p[owner])[drow] = scale;
}

// ------------------------------------------------------------------ combine (pull + gate)
__global__ void __launch_bounds__(256) moe_combine_kernel(Peers y, const int* __restrict__ route, const float* __restrict__ gate,
                                                         __nv_bfloat16* __restrict__ out, int T, int M, int top_k, int experts_per_rank,
                                                         int cap_per_src, int n_ranks, int src_rank) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= T) return;
  for (int v = lane; v < (M >> 3); v += 32) {
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int k = 0; k < top_k; ++k) {
      const int r = route[warp * top_k + k];
      if (r < 0) continue;
      const int e = r >> 16, slot = r & 0xFFFF;
      const int owner = e / experts_per_rank, el = e % experts_per_rank;
      const size_t srow = ((size_t)el * n_ranks + src_rank) * cap_per_src + slot;
      const uint4 u = *(reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(y.p[owner]) + srow * M) + v);
      const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
      const float g = gate[warp * top_k + k];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float2 f = __bfloat1622float2(h[i]);
        acc[2 * i] += g * f.x;
        acc[2 * i + 1] += g * f.y;
      }
    }
    uint4 o;
    o.x = pack_bf16x2(acc[0], acc[1]); o.y = pack_bf16x2(acc[2], acc[3]);
    o.z = pack_bf16x2(acc[4], acc[5]); o.w = pack_bf16x2(acc[6], acc[7]);
    reinterpret_cast<uint4*>(out + (size_t)warp * M)[v] = o;
  }
}

// per-tensor (per-expert) weight quantisation: w[b] (bf16 [rows, K]) -> e4m3 + scale[b]
__global__ void quant_weight_kernel(const __nv_bfloat16* __restrict__ w, uint8_t* __restrict__ q, const float* __restrict__ scale_inv,
                                    long long per_batch, long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
    q[i] = (uint8_t)__nv_cvt_float_to_fp8(__bfloat162float(w[i]) * scale_inv[i / per_batch], __NV_SATFINITE, __NV_E4M3);
}

Peers mk(void* const* ptrs, int n) {
  Peers p;
  for (int i = 0; i < MAXP; ++i) p.p[i] = i < n ? ptrs[i] : nullptr;
  return p;
}

}  // namespace

#define CS(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int tepd_moe_dispatch(const void* x, const void* route, void* const* xin_ptrs, void* const* xscale_ptrs, int T, int M,
                                 int top_k, int experts_per_rank, int cap_per_src, int n_ranks, int src_rank, void* stream) {
  if (M % 8 || n_ranks > MAXP) return -2;
  const int warps = T * top_k;
  moe_dispatch_kernel<<<(warps * 32 + 255) / 256, 256, 0, CS(stream)>>>((const __nv_bfloat16*)x, (const int*)route, mk(xin_ptrs, n_ranks),
                                                                      mk(xscale_ptrs, n_ranks), T, M, top_k, experts_per_rank, cap_per_src,
                                                                      n_ranks, src_rank);
  return (int)cudaGetLastError();
}
extern "C" int tepd_moe_combine(void* const* y_ptrs, const void* route, const void* gate, void* out, int T, int M, int top_k,
                                int experts_per_rank, int cap_per_src, int n_ranks, int src_rank, void* stream) {
  if (M % 8 || n_ranks > MAXP) return -2;
  moe_combine_kernel<<<(T * 32 + 255) / 256, 256, 0, CS(stream)>>>(mk(y_ptrs, n_ranks), (const int*)route, (const float*)gate,
                                                                  (__nv_bfloat16*)out, T, M, top_k, experts_per_rank, cap_per_src, n_ranks,
                                                                  src_rank);
  return (int)cudaGetLastError();
}
extern "C" int tepd_quant_weight_fp8(const void* w, void* q, const void* scale_inv, long long per_batch, long long total, void* stream) {
  quant_weight_kernel<<<tepd::num_sms() * 4, 256, 0, CS(stream)>>>((const __nv_bfloat16*)w, (uint8_t*)q, (const float*)scale_inv, per_batch, total);
  return (int)cudaGetLastError();
}
// ================================================================================================ route-table dispatch / combine
// GShard writes dispatch and combine as dense einsums with a [G, S, E, C] one-hot mask (and so does the planner graph, which is
// what lets the planner see the G <-> E re-distribution).  Every slot (e, c) of a group holds at most ONE token and every token
// occupies at most top_k slots, so at run time the four dense einsums (and the four their gradients need) are row gathers:
//   gather_scale : out[e, g, c, :] = w[g, e, c] * src[g, slot_src[g, e, c], :]                 (dispatch; d combine / d y)
//   combine_sum  : out[g, s, :]    = sum_k gw[g, s, k] * y[e_k, g, c_k, :]                      (combine; d dispatch / d x)
//   route_dots   : dots[g, s, k]   = < a[g, s, :], b[e_k, g, c_k, :] >                          (d / d mask weights)
// 2 * G*S*E*C*M FLOPs per einsum (25.8 GFLOP per group at the reference shape) become G*E*C*M bytes of row traffic.
namespace {

__global__ void __launch_bounds__(256) moe_gather_scale_kernel(const __nv_bfloat16* __restrict__ src, const int* __restrict__ slot_src,
                                                              const float* __restrict__ w, __nv_bfloat16* __restrict__ out, int G, int S,
                                                              int E, int C, int M) {
  const long long row = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= (long long)E * G * C) return;
  const int c = (int)(row % C), g = (int)((row / C) % G), e = (int)(row / ((long long)G * C));
  const long long si = ((long long)g * E + e) * C + c;
  const int s = slot_src[si];
  const float ws = s >= 0 ? w[si] : 0.f;
  uint4* dst = reinterpret_cast<uint4*>(out + row * M);
  const uint4* sp = reinterpret_cast<const uint4*>(src + ((long long)g * S + (s >= 0 ? s : 0)) * M);
  for (int v = lane; v < (M >> 3); v += 32) {
    uint4 o = make_uint4(0u, 0u, 0u, 0u);
    if (s >= 0) {
      const uint4 u = __ldg(sp + v);
      const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
      float2 f0 = __bfloat1622float2(h[0]), f1 = __bfloat1622float2(h[1]), f2 = __bfloat1622float2(h[2]), f3 = __bfloat1622float2(h[3]);
      o.x = pack_bf16x2(ws * f0.x, ws * f0.y); o.y = pack_bf16x2(ws * f1.x, ws * f1.y);
      o.z = pack_bf16x2(ws * f2.x, ws * f2.y); o.w = pack_bf16x2(ws * f3.x, ws * f3.y);
    }
    dst[v] = o;
  }
}

__global__ void __launch_bounds__(256) moe_combine_sum_kernel(const __nv_bfloat16* __restrict__ y, const int* __restrict__ re,
                                                             const int* __restrict__ rc, const float* __restrict__ gw,
                                                             __nv_bfloat16* __restrict__ out, int G, int S, int E, int C, int M, int K) {
  const long long row = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;   // (g, s)
  const int lane = threadIdx.x & 31;
  if (row >= (long long)G * S) return;
  const int g = (int)(row / S);
  for (int v = lane; v < (M >> 3); v += 32) {
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int k = 0; k < K; ++k) {
      const int e = re[row * K + k];
      if (e < 0) continue;
      const int c = rc[row * K + k];
      const float wk = gw[row * K + k];
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(y + (((long long)e * G + g) * C + c) * M) + v);
      const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = __bfloat1622float2(h[i]);
        acc[2 * i] += wk * f.x;
        acc[2 * i + 1] += wk * f.y;
      }
    }
    uint4 o;
    o.x = pack_bf16x2(acc[0], acc[1]); o.y = pack_bf16x2(acc[2], acc[3]);
    o.z = pack_bf16x2(acc[4], acc[5]); o.w = pack_bf16x2(acc[6], acc[7]);
    reinterpret_cast<uint4*>(out + row * M)[v] = o;
  }
}

__global__ void __launch_bounds__(256) moe_route_dots_kernel(const __nv_bfloat16* __restrict__ a, const __nv_bfloat16* __restrict__ b,
                                                            const int* __restrict__ re, const int* __restrict__ rc,
                                                            float* __restrict__ dots, int G, int S, int E, int C, int M, int K) {
  const long long wid = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;   // (g, s, k)
  const int lane = threadIdx.x & 31;
  if (wid >= (long long)G * S * K) return;
  const long long row = wid / K;
  const int g = (int)(row / S);
  const int e = re[wid];
  float acc = 0.f;
  if (e >= 0) {
    const int c = rc[wid];
    const uint4* ap = reinterpret_cast<const uint4*>(a + row * M);
    const uint4* bp = reinterpret_cast<const uint4*>(b + (((long long)e * G + g) * C + c) * M);
    for (int v = lane; v < (M >> 3); v += 32) {
      const uint4 ua = __ldg(ap + v), ub = __ldg(bp + v);
      const __nv_bfloat162* ha = reinterpret_cast<const __nv_bfloat162*>(&ua);
      const __nv_bfloat162* hb = reinterpret_cast<const __nv_bfloat162*>(&ub);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 fa = __bfloat1622float2(ha[i]), fb = __bfloat1622float2(hb[i]);
        acc += fa.x * fb.x + fa.y * fb.y;
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) dots[wid] = acc;
}

}  // namespace

extern "C" int tepd_moe_gather_scale(const void* src, const void* slot_src, const void* w, void* out, int G, int S, int E, int C, int M,
                                     void* stream) {
  if (M % 8) return -2;
  const long long rows = (long long)E * G * C;
  moe_gather_scale_kernel<<<(unsigned)((rows * 32 + 255) / 256), 256, 0, CS(stream)>>>((const __nv_bfloat16*)src, (const int*)slot_src,
                                                                                        (const float*)w, (__nv_bfloat16*)out, G, S, E, C, M);
  return (int)cudaGetLastError();
}
extern "C" int tepd_moe_combine_sum(const void* y, const void* re, const void* rc, const void* gw, void* out, int G, int S, int E, int C,
                                    int M, int K, void* stream) {
  if (M % 8) return -2;
  const long long rows = (long long)G * S;
  moe_combine_sum_kernel<<<(unsigned)((rows * 32 + 255) / 256), 256, 0, CS(stream)>>>((const __nv_bfloat16*)y, (const int*)re, (const int*)rc,
                                                                                       (const float*)gw, (__nv_bfloat16*)out, G, S, E, C, M, K);
  return (int)cudaGetLastError();
}
extern "C" int tepd_moe_route_dots(const void* a, const void* b, const void* re, const void* rc, void* dots, int G, int S, int E, int C,
                                   int M, int K, void* stream) {
  if (M % 8) return -2;
  const long long warps = (long long)G * S * K;
  moe_route_dots_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, CS(stream)>>>((const __nv_bfloat16*)a, (const __nv_bfloat16*)b,
                                                                                       (const int*)re, (const int*)rc, (float*)dots, G, S, E, C, M, K);
  return (int)cudaGetLastError();
}
