// Mixture-of-experts dispatch and combine for sm_90a, as route-table row gathers.
//
// The reference implements expert parallelism as einsum dispatch/combine + a hand-rolled ncclSend/ncclRecv all-to-all
// (DAPPLEAllToAllThunk, SURVEY K3; examples/gpt_moe/layers/moe_layers.py:425-446).  GShard writes dispatch and combine as
// dense einsums with a [G, S, E, C] one-hot mask (and so does the planner graph, which is what lets the planner see the
// G <-> E re-distribution).  Every slot (e, c) of a group holds at most ONE token and every token occupies at most top_k
// slots, so at run time the four dense einsums (and the four their gradients need) are row gathers:
//   gather_scale : out[e, g, c, :] = w[g, e, c] * src[g, slot_src[g, e, c], :]                 (dispatch; d combine / d y)
//   combine_sum  : out[g, s, :]    = sum_k gw[g, s, k] * y[e_k, g, c_k, :]                      (combine; d dispatch / d x)
//   route_dots   : dots[g, s, k]   = < a[g, s, :], b[e_k, g, c_k, :] >                          (d / d mask weights)
// 2 * G*S*E*C*M FLOPs per einsum (25.8 GFLOP per group at the reference shape) become G*E*C*M bytes of row traffic.  The
// expert FCs run on the batched wgmma GEMM (gemm_sm90.cu) and the all-to-all between ranks on NCCL.
#include "sm90_ptx.cuh"
#include <stdio.h>

using namespace sm90;

#define CS(s) reinterpret_cast<cudaStream_t>(s)

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
