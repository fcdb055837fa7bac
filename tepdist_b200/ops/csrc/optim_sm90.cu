// Multi-tensor optimizer updates for sm_90a: momentum, LAMB, Adafactor and SM3 over the flat variable buffers
// (runtime/optimizers.py is the specification; the executor's whole-variable path drives these).
//
// One launch sequence per step covers every variable of the graph: a device-resident work table (built once when the
// executor plans, ops.OptimPlan) lists the variables (OptVar: offset, [B, R, C] view, slot pointers) and their chunks
// (OptChunk), and every kernel runs one CTA per chunk.  Elementwise kinds cut a variable into flat chunks of
// kFlatChunk elements; Adafactor's factored variables and SM3's rank >= 2 variables into chunks of 32 whole rows of the
// [B * R, C] view, so a row's reduction completes inside one CTA.
//
// Determinism: every per-variable sum is written as a per-chunk partial to a fixed slot of the work space, and every CTA
// that needs the total adds the partials of that variable in the same fixed order -- no float atomics.  SM3's maxima of
// non-negative values use integer atomicMax on the float bits, which is exact.  So replicas stay bit-identical and a
// captured CUDA graph replays the eager bits.
//
// Step-dependent scalars (learning rate, bias corrections, Adafactor's decay and relative step) are read from the device
// tensor `hyper`, per-graph constants (betas, eps, weight decay, ...) are launch arguments.
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <string.h>
#include <type_traits>
#include "launch.cuh"

namespace {

typedef __nv_bfloat16 bf16;

constexpr int kThreads = 256, kWarps = 8, kRowsPerWarp = 4;     // row chunks: kWarps * kRowsPerWarp = 32 rows
enum { H_LR = 0, H_BC1 = 1, H_BC2 = 2, H_AF_DECAY = 4, H_AF_REL_LR = 5 };   // slots of `hyper` (runtime/optimizers.py)
enum { F_DECAY = 1, F_ROWS = 2, F_MOM = 4 };
enum { P_PSQ = 0, P_USQ = 1, P_VR = 2 };                          // per-chunk partials: 4 floats per chunk at ws[4 * chunk]

// Layouts shared with ops/__init__.py (OptimPlan): all fields 64-bit.
struct OptVar {
  long long off;        // element offset of the variable in the flat master / grad / bf16 buffers
  long long n;          // elements
  long long B, R, C;    // [B, R, C] view: rank 1 -> [1, 1, n]; rank 2 -> [1, R, C]; rank r > 2 -> [prod(leading), R, C]
  long long flags;      // F_DECAY: weight decay applies; F_ROWS: row-chunked; F_MOM: SM3 momentum slot in s[3]
  long long c0, nc;     // first chunk, number of chunks
  long long sc;         // work-space offset (floats): Adafactor column partials [nc, C]; SM3 new accumulators [B + R + C]
  long long rank;
  float* s[4];          // slots: momentum {mom}; LAMB {m, v}; Adafactor {vr, vc} | {vf}; SM3 {acc0.., , , mom}
  long long cpb;        // chunks per batch entry (row-chunked)
  long long pad;
};
struct OptChunk {
  long long var, b, r0, nr;   // row chunks: batch entry b, rows [r0, r0 + nr)
  long long e0, ne;           // elements [e0, e0 + ne) of the variable
};
struct OptHP {          // per-graph constants, in the order ops.OptimPlan packs them
  float b1;             // LAMB beta1; momentum / SM3: momentum
  float b2, eps, wd, eps1, eps2;
  float clip;           // Adafactor clipping threshold; <= 0: no clipping
  float decay_rate;     // Adafactor; < 0: hyper[H_AF_DECAY]
  float rel_lr, param_scale, adapt_all, nesterov;   // flags (0 / 1)
};
struct Bufs {
  float* p;
  const float* g;
  bf16* pb;             // bf16 compute copy (may be null)
  float* ws;            // work space: partials, column partials, new SM3 accumulators
  const float* hyper;
  const OptVar* vars;
  const OptChunk* chunks;
};

__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// fixed-order block reduction: lane 0 of every warp, then the 8 warp results in warp order; every thread gets the total
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) t += red[w];
  __syncthreads();
  return t;
}
// sum of partial `which` over chunks [c0, c0 + nc) in a fixed order (identical bits in every CTA that asks)
__device__ __forceinline__ float chunk_total(const float* ws, long long c0, long long nc, int which, float* red) {
  float s = 0.f;
  for (long long k = threadIdx.x; k < nc; k += kThreads) s += ws[4 * (c0 + k) + which];
  return block_sum(s, red);
}
__device__ __forceinline__ void atomic_max_nonneg(float* a, float x) {   // exact for x >= 0
  atomicMax(reinterpret_cast<int*>(a), __float_as_int(x));
}

template <int VEC> __device__ __forceinline__ void ldv(const float* p, float (&x)[VEC]) {
  if constexpr (VEC == 4) {
    const float4 t = *reinterpret_cast<const float4*>(p);
    x[0] = t.x; x[1] = t.y; x[2] = t.z; x[3] = t.w;
  } else {
    x[0] = *p;
  }
}
template <int VEC> __device__ __forceinline__ void stv(float* p, const float (&x)[VEC]) {
  if constexpr (VEC == 4) *reinterpret_cast<float4*>(p) = make_float4(x[0], x[1], x[2], x[3]);
  else *p = x[0];
}
template <int VEC> __device__ __forceinline__ void stb(bf16* p, const float (&x)[VEC]) {
  if (!p) return;
  if constexpr (VEC == 4) {
    __nv_bfloat162 lo = __floats2bfloat162_rn(x[0], x[1]), hi = __floats2bfloat162_rn(x[2], x[3]);
    uint2 u;
    u.x = *reinterpret_cast<uint32_t*>(&lo);
    u.y = *reinterpret_cast<uint32_t*>(&hi);
    *reinterpret_cast<uint2*>(p) = u;
  } else {
    *p = __float2bfloat16(x[0]);
  }
}

using V4 = std::integral_constant<int, 4>;
using V1 = std::integral_constant<int, 1>;

// elements [0, ne) of a flat chunk whose first element is 16-byte aligned: f(VEC, i) for 4-vectors, then a scalar tail
template <class F> __device__ __forceinline__ void flat_loop(long long ne, F&& f) {
  const long long nv = ne >> 2;
  for (long long i = threadIdx.x; i < nv; i += kThreads) f(V4(), i << 2);
  for (long long i = (nv << 2) + threadIdx.x; i < ne; i += kThreads) f(V1(), i);
}
// a row chunk: warp w owns local rows w + 8k (k < kRowsPerWarp, a compile-time index after unrolling); lanes cover 32 * VEC
// columns at a time.  f(VEC, k, rl, c) handles columns [c, c + VEC) of local row rl; colend(cb) runs in every thread after
// each column block (column reductions).  VEC = 4 needs C % 4 == 0.
template <int VEC, class F, class G> __device__ __forceinline__ void rows_loop(long long nr, long long C, F&& f, G&& colend) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (long long cb = 0; cb < C; cb += 32 * VEC) {
    const long long c = cb + lane * VEC;
#pragma unroll
    for (int k = 0; k < kRowsPerWarp; ++k) {
      const int rl = warp + kWarps * k;
      if (rl < nr && c < C) f(std::integral_constant<int, VEC>(), k, rl, c);
    }
    colend(cb);
  }
}

// ------------------------------------------------------------------ momentum (one pass)
__global__ void __launch_bounds__(kThreads) optim_momentum_kernel(Bufs bu, OptHP hp) {
  pdl_wait();
  const OptChunk ch = bu.chunks[blockIdx.x];
  const OptVar& v = bu.vars[ch.var];
  const long long base = v.off + ch.e0;
  float* p = bu.p + base;
  const float* g = bu.g + base;
  bf16* pb = bu.pb ? bu.pb + base : nullptr;
  float* mo = v.s[0] + ch.e0;
  const float lr = bu.hyper[H_LR], mu = hp.b1;
  const bool nesterov = hp.nesterov != 0.f;
  flat_loop(ch.ne, [&](auto vt, long long i) {
    constexpr int VEC = decltype(vt)::value;
    float pv[VEC], gv[VEC], mv[VEC];
    ldv(p + i, pv); ldv(g + i, gv); ldv(mo + i, mv);
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      mv[j] = mv[j] * mu + gv[j];
      const float u = nesterov ? gv[j] + mu * mv[j] : mv[j];
      pv[j] = pv[j] - lr * u;
    }
    stv(mo + i, mv); stv(p + i, pv); stb(pb ? pb + i : nullptr, pv);
  });
}

// ------------------------------------------------------------------ LAMB (two passes: moments + norms, then the scaled step)
__device__ __forceinline__ float lamb_dir(float m, float v, float p, float bc1, float bc2, float eps, float wd) {
  float u = (m / bc1) / (sqrtf(v / bc2) + eps);
  if (wd != 0.f) u = u + wd * p;
  return u;
}
__global__ void __launch_bounds__(kThreads) optim_lamb_moments_kernel(Bufs bu, OptHP hp) {
  __shared__ float red[kWarps];
  pdl_wait();
  const long long chunk = blockIdx.x;
  const OptChunk ch = bu.chunks[chunk];
  const OptVar& v = bu.vars[ch.var];
  const long long base = v.off + ch.e0;
  const float* p = bu.p + base;
  const float* g = bu.g + base;
  float* m = v.s[0] + ch.e0;
  float* vv = v.s[1] + ch.e0;
  const float bc1 = bu.hyper[H_BC1], bc2 = bu.hyper[H_BC2];
  const float wd = (v.flags & F_DECAY) ? hp.wd : 0.f;
  float psq = 0.f, usq = 0.f;
  flat_loop(ch.ne, [&](auto vt, long long i) {
    constexpr int VEC = decltype(vt)::value;
    float pv[VEC], gv[VEC], mv[VEC], vw[VEC];
    ldv(p + i, pv); ldv(g + i, gv); ldv(m + i, mv); ldv(vv + i, vw);
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      mv[j] = mv[j] * hp.b1 + (1.f - hp.b1) * gv[j];
      vw[j] = vw[j] * hp.b2 + (1.f - hp.b2) * gv[j] * gv[j];
      const float u = lamb_dir(mv[j], vw[j], pv[j], bc1, bc2, hp.eps, wd);
      psq += pv[j] * pv[j];
      usq += u * u;
    }
    stv(m + i, mv); stv(vv + i, vw);
  });
  psq = block_sum(psq, red);
  usq = block_sum(usq, red);
  if (threadIdx.x == 0) { bu.ws[4 * chunk + P_PSQ] = psq; bu.ws[4 * chunk + P_USQ] = usq; }
}
__global__ void __launch_bounds__(kThreads) optim_lamb_apply_kernel(Bufs bu, OptHP hp) {
  __shared__ float red[kWarps];
  pdl_wait();
  const OptChunk ch = bu.chunks[blockIdx.x];
  const OptVar& v = bu.vars[ch.var];
  const long long base = v.off + ch.e0;
  float* p = bu.p + base;
  bf16* pb = bu.pb ? bu.pb + base : nullptr;
  const float* m = v.s[0] + ch.e0;
  const float* vv = v.s[1] + ch.e0;
  const float bc1 = bu.hyper[H_BC1], bc2 = bu.hyper[H_BC2];
  const float wd = (v.flags & F_DECAY) ? hp.wd : 0.f;
  float ratio = 1.f;
  if ((v.flags & F_DECAY) || hp.adapt_all != 0.f) {      // layer adaptation (skipped for no-decay variables unless adapt_all)
    const float wn = sqrtf(chunk_total(bu.ws, v.c0, v.nc, P_PSQ, red));
    const float un = sqrtf(chunk_total(bu.ws, v.c0, v.nc, P_USQ, red));
    ratio = wn > 0.f ? (un > 0.f ? wn / un : 1.f) : 1.f;
  }
  const float lr = bu.hyper[H_LR] * ratio;
  flat_loop(ch.ne, [&](auto vt, long long i) {
    constexpr int VEC = decltype(vt)::value;
    float pv[VEC], mv[VEC], vw[VEC];
    ldv(p + i, pv); ldv(m + i, mv); ldv(vv + i, vw);
#pragma unroll
    for (int j = 0; j < VEC; ++j) pv[j] = pv[j] - lr * lamb_dir(mv[j], vw[j], pv[j], bc1, bc2, hp.eps, wd);
    stv(p + i, pv); stb(pb ? pb + i : nullptr, pv);
  });
}

// ------------------------------------------------------------------ Adafactor (four launches)
__device__ __forceinline__ float af_beta2(const Bufs& bu, const OptHP& hp) {
  return hp.decay_rate < 0.f ? bu.hyper[H_AF_DECAY] : hp.decay_rate;
}
// mean over rows of the (new) vr of batch entry b: the fixed-order total of the chunks' P_VR partials
__device__ __forceinline__ float af_row_mean(const Bufs& bu, const OptVar& v, long long b, float* red) {
  return chunk_total(bu.ws, v.c0 + b * v.cpb, v.cpb, P_VR, red) / (float)v.R;
}

// pass 1: factored: row sums (-> new vr), per-chunk column partials, sum of the new vr, sum of p^2;
//         unfactored: vf update, sums of u^2 and p^2
template <int VEC>
__device__ __forceinline__ void af_stats_rows(const Bufs& bu, const OptHP& hp, const OptVar& v, const OptChunk& ch, long long chunk,
                                              float beta2, float* sm, float* red) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long C = v.C;
  const long long row0 = ch.b * v.R + ch.r0;
  const float* g = bu.g + v.off;
  const float* p = bu.p + v.off;
  float* colpart = bu.ws + v.sc + (chunk - v.c0) * C;
  const bool want_p = hp.param_scale != 0.f;
  float racc[kRowsPerWarp] = {};
  float cacc[VEC] = {};
  float psq = 0.f;
  rows_loop<VEC>(ch.nr, C, [&](auto, int k, int rl, long long c) {
    const long long e = (row0 + rl) * C + c;
    float gv[VEC];
    ldv(g + e, gv);
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const float x = gv[j] * gv[j] + hp.eps1;
      racc[k] += x;
      cacc[j] += x;
    }
    if (want_p) {
      float pv[VEC];
      ldv(p + e, pv);
#pragma unroll
      for (int j = 0; j < VEC; ++j) psq += pv[j] * pv[j];
    }
  }, [&](long long cb) {
#pragma unroll
    for (int j = 0; j < VEC; ++j) { sm[warp * 32 * VEC + lane * VEC + j] = cacc[j]; cacc[j] = 0.f; }
    __syncthreads();
    for (int t = threadIdx.x; t < 32 * VEC; t += kThreads) {
      if (cb + t < C) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < kWarps; ++w) s += sm[w * 32 * VEC + t];
        colpart[cb + t] = s;
      }
    }
    __syncthreads();
  });
  float vrs = 0.f;
#pragma unroll
  for (int k = 0; k < kRowsPerWarp; ++k) {
    const float s = warp_sum(racc[k]);
    const int rl = warp + kWarps * k;
    if (lane == 0 && rl < ch.nr) {
      float* vr = v.s[0] + row0 + rl;
      const float nv = *vr * beta2 + (s / (float)C) * (1.f - beta2);
      *vr = nv;
      vrs += nv;
    }
  }
  psq = block_sum(psq, red);
  vrs = block_sum(vrs, red);
  if (threadIdx.x == 0) { bu.ws[4 * chunk + P_PSQ] = psq; bu.ws[4 * chunk + P_VR] = vrs; }
}
__global__ void __launch_bounds__(kThreads) optim_af_stats_kernel(Bufs bu, OptHP hp) {
  __shared__ float sm[kWarps * 128];
  __shared__ float red[kWarps];
  pdl_wait();
  const long long chunk = blockIdx.x;
  const OptChunk ch = bu.chunks[chunk];
  const OptVar& v = bu.vars[ch.var];
  const float beta2 = af_beta2(bu, hp);
  if (v.flags & F_ROWS) {
    if (v.C % 4 == 0) af_stats_rows<4>(bu, hp, v, ch, chunk, beta2, sm, red);
    else af_stats_rows<1>(bu, hp, v, ch, chunk, beta2, sm, red);
    return;
  }
  const long long base = v.off + ch.e0;
  const float* p = bu.p + base;
  const float* g = bu.g + base;
  float* vf = v.s[0] + ch.e0;
  const bool want_p = hp.param_scale != 0.f;
  float psq = 0.f, usq = 0.f;
  flat_loop(ch.ne, [&](auto vt, long long i) {
    constexpr int VEC = decltype(vt)::value;
    float gv[VEC], fv[VEC];
    ldv(g + i, gv); ldv(vf + i, fv);
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      fv[j] = fv[j] * beta2 + (gv[j] * gv[j] + hp.eps1) * (1.f - beta2);
      const float u = gv[j] * rsqrtf(fv[j]);
      usq += u * u;
    }
    stv(vf + i, fv);
    if (want_p) {
      float pv[VEC];
      ldv(p + i, pv);
#pragma unroll
      for (int j = 0; j < VEC; ++j) psq += pv[j] * pv[j];
    }
  });
  psq = block_sum(psq, red);
  usq = block_sum(usq, red);
  if (threadIdx.x == 0) { bu.ws[4 * chunk + P_PSQ] = psq; bu.ws[4 * chunk + P_USQ] = usq; }
}

// pass 2 (factored variables): vc from the column partials of the chunks of each batch entry, in chunk order
__global__ void __launch_bounds__(kThreads) optim_af_cols_kernel(Bufs bu, OptHP hp) {
  pdl_wait();
  const OptVar& v = bu.vars[blockIdx.x];
  if (!(v.flags & F_ROWS)) return;
  const float beta2 = af_beta2(bu, hp);
  const long long C = v.C, BC = v.B * v.C, cpb = v.cpb;
  for (long long i = (long long)blockIdx.y * kThreads + threadIdx.x; i < BC; i += (long long)gridDim.y * kThreads) {
    const long long b = i / C, c = i - b * C;
    const float* cp = bu.ws + v.sc + b * cpb * C + c;
    float s = 0.f;
    for (long long k = 0; k < cpb; ++k) s += cp[k * C];
    float* vc = v.s[1] + i;
    *vc = *vc * beta2 + (s / (float)v.R) * (1.f - beta2);
  }
}

// the factored update before clipping: g * rsqrt(vr / row_mean) * rsqrt(vc)
template <int VEC> __device__ __forceinline__ void af_factored_u(const float (&gv)[VEC], float rfac, const float* vc, float (&u)[VEC]) {
  float cv[VEC];
  ldv(vc, cv);
#pragma unroll
  for (int j = 0; j < VEC; ++j) u[j] = gv[j] * rfac * rsqrtf(cv[j]);
}

// pass 3 (factored variables): per-chunk sums of u^2
template <int VEC>
__device__ __forceinline__ void af_usq_rows(const Bufs& bu, const OptVar& v, const OptChunk& ch, long long chunk, float* red) {
  const long long C = v.C;
  const long long row0 = ch.b * v.R + ch.r0;
  const float rm = af_row_mean(bu, v, ch.b, red);
  const float* g = bu.g + v.off;
  const float* vc = v.s[1] + ch.b * C;
  float usq = 0.f;
  rows_loop<VEC>(ch.nr, C, [&](auto, int, int rl, long long c) {
    float gv[VEC], u[VEC];
    ldv(g + (row0 + rl) * C + c, gv);
    af_factored_u(gv, rsqrtf(v.s[0][row0 + rl] / rm), vc + c, u);
#pragma unroll
    for (int j = 0; j < VEC; ++j) usq += u[j] * u[j];
  }, [](long long) {});
  usq = block_sum(usq, red);
  if (threadIdx.x == 0) bu.ws[4 * chunk + P_USQ] = usq;
}
__global__ void __launch_bounds__(kThreads) optim_af_usq_kernel(Bufs bu, OptHP hp) {
  __shared__ float red[kWarps];
  pdl_wait();
  const long long chunk = blockIdx.x;
  const OptChunk ch = bu.chunks[chunk];
  const OptVar& v = bu.vars[ch.var];
  if (!(v.flags & F_ROWS)) return;
  if (v.C % 4 == 0) af_usq_rows<4>(bu, v, ch, chunk, red);
  else af_usq_rows<1>(bu, v, ch, chunk, red);
}

// pass 4: clip by RMS(u), step size (relative or hyper[H_LR], times max(RMS(p), eps2)), weight decay, write p and bf16
template <int VEC> __device__ __forceinline__ void af_write(float* p, bf16* pb, const float (&u)[VEC], float den, float wd, float lr) {
  float pv[VEC];
  ldv(p, pv);
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    float x = u[j] / den;
    if (wd != 0.f) x = x + wd * pv[j];
    pv[j] = pv[j] - lr * x;
  }
  stv(p, pv);
  stb(pb, pv);
}
template <int VEC>
__device__ __forceinline__ void af_apply_rows(const Bufs& bu, const OptVar& v, const OptChunk& ch, float den, float wd, float lr, float* red) {
  const long long C = v.C;
  const long long row0 = ch.b * v.R + ch.r0;
  const float rm = af_row_mean(bu, v, ch.b, red);
  const float* g = bu.g + v.off;
  float* p = bu.p + v.off;
  bf16* pb = bu.pb ? bu.pb + v.off : nullptr;
  const float* vc = v.s[1] + ch.b * C;
  rows_loop<VEC>(ch.nr, C, [&](auto, int, int rl, long long c) {
    const long long e = (row0 + rl) * C + c;
    float gv[VEC], u[VEC];
    ldv(g + e, gv);
    af_factored_u(gv, rsqrtf(v.s[0][row0 + rl] / rm), vc + c, u);
    af_write(p + e, pb ? pb + e : nullptr, u, den, wd, lr);
  }, [](long long) {});
}
__global__ void __launch_bounds__(kThreads) optim_af_apply_kernel(Bufs bu, OptHP hp) {
  __shared__ float red[kWarps];
  pdl_wait();
  const OptChunk ch = bu.chunks[blockIdx.x];
  const OptVar& v = bu.vars[ch.var];
  const float nf = (float)v.n;
  float den = 1.f;
  if (hp.clip > 0.f) den = fmaxf(sqrtf(chunk_total(bu.ws, v.c0, v.nc, P_USQ, red) / nf) / hp.clip, 1.f);
  float lr = bu.hyper[hp.rel_lr != 0.f ? H_AF_REL_LR : H_LR];
  if (hp.param_scale != 0.f) lr = lr * fmaxf(sqrtf(chunk_total(bu.ws, v.c0, v.nc, P_PSQ, red) / nf), hp.eps2);
  const float wd = (v.flags & F_DECAY) ? hp.wd : 0.f;
  if (v.flags & F_ROWS) {
    if (v.C % 4 == 0) af_apply_rows<4>(bu, v, ch, den, wd, lr, red);
    else af_apply_rows<1>(bu, v, ch, den, wd, lr, red);
    return;
  }
  const long long base = v.off + ch.e0;
  float* p = bu.p + base;
  const float* g = bu.g + base;
  bf16* pb = bu.pb ? bu.pb + base : nullptr;
  const float* vf = v.s[0] + ch.e0;
  flat_loop(ch.ne, [&](auto vt, long long i) {
    constexpr int VEC = decltype(vt)::value;
    float gv[VEC], fv[VEC], u[VEC];
    ldv(g + i, gv); ldv(vf + i, fv);
#pragma unroll
    for (int j = 0; j < VEC; ++j) u[j] = gv[j] * rsqrtf(fv[j]);
    af_write(p + i, pb ? pb + i : nullptr, u, den, wd, lr);
  });
}

// ------------------------------------------------------------------ SM3 (update + maxima, then the accumulator copy)
// rank >= 2: nu = min_i acc_i + g^2 from the OLD accumulators; the new ones (max of nu over the other dims) collect in the
// work space (ws[sc ..]: [B] batch, [R] rows, [C] columns) and replace the old ones in the second launch
template <int VEC>
__device__ __forceinline__ void sm3_rows(const Bufs& bu, const OptHP& hp, const OptVar& v, const OptChunk& ch, float lr, float* sm) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long C = v.C;
  const long long row0 = ch.b * v.R + ch.r0;
  const bool r3 = v.rank == 3;
  const float accb = r3 ? v.s[0][ch.b] : __int_as_float(0x7f800000);
  const float* accr = v.s[r3 ? 1 : 0];
  const float* accc = v.s[r3 ? 2 : 1];
  float* nb = bu.ws + v.sc;
  float* nr_ = nb + v.B;
  float* nc_ = nr_ + v.R;
  float* p = bu.p + v.off;
  const float* g = bu.g + v.off;
  bf16* pb = bu.pb ? bu.pb + v.off : nullptr;
  float* mo = (v.flags & F_MOM) ? v.s[3] : nullptr;
  const float mu = hp.b1;
  float rmax[kRowsPerWarp] = {};
  float cmax[VEC] = {};
  rows_loop<VEC>(ch.nr, C, [&](auto, int k, int rl, long long c) {
    const long long e = (row0 + rl) * C + c;
    const float ar = fminf(accb, accr[ch.r0 + rl]);
    float gv[VEC], pv[VEC], cv[VEC];
    ldv(g + e, gv); ldv(p + e, pv); ldv(accc + c, cv);
    float u[VEC];
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const float nu = fminf(ar, cv[j]) + gv[j] * gv[j];
      rmax[k] = fmaxf(rmax[k], nu);
      cmax[j] = fmaxf(cmax[j], nu);
      u[j] = (1.f - mu) * gv[j] * rsqrtf(nu + 1e-30f);
    }
    if (mo) {
      float mv[VEC];
      ldv(mo + e, mv);
#pragma unroll
      for (int j = 0; j < VEC; ++j) { mv[j] = mv[j] * mu + u[j]; u[j] = mv[j]; }
      stv(mo + e, mv);
    }
#pragma unroll
    for (int j = 0; j < VEC; ++j) pv[j] = pv[j] - lr * u[j];
    stv(p + e, pv);
    stb(pb ? pb + e : nullptr, pv);
  }, [&](long long cb) {
#pragma unroll
    for (int j = 0; j < VEC; ++j) { sm[warp * 32 * VEC + lane * VEC + j] = cmax[j]; cmax[j] = 0.f; }
    __syncthreads();
    for (int t = threadIdx.x; t < 32 * VEC; t += kThreads) {
      if (cb + t < C) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < kWarps; ++w) s = fmaxf(s, sm[w * 32 * VEC + t]);
        atomic_max_nonneg(nc_ + cb + t, s);
      }
    }
    __syncthreads();
  });
  float bm = 0.f;
#pragma unroll
  for (int k = 0; k < kRowsPerWarp; ++k) {
    const float s = warp_max(rmax[k]);
    const int rl = warp + kWarps * k;
    if (lane == 0 && rl < ch.nr) atomic_max_nonneg(nr_ + ch.r0 + rl, s);
    bm = fmaxf(bm, s);
  }
  if (r3 && lane == 0) atomic_max_nonneg(nb + ch.b, bm);
}
__global__ void __launch_bounds__(kThreads) optim_sm3_kernel(Bufs bu, OptHP hp) {
  __shared__ float sm[kWarps * 128];
  pdl_wait();
  const OptChunk ch = bu.chunks[blockIdx.x];
  const OptVar& v = bu.vars[ch.var];
  const float lr = bu.hyper[H_LR];
  if (v.flags & F_ROWS) {
    if (v.C % 4 == 0) sm3_rows<4>(bu, hp, v, ch, lr, sm);
    else sm3_rows<1>(bu, hp, v, ch, lr, sm);
    return;
  }
  const long long base = v.off + ch.e0;
  float* p = bu.p + base;
  const float* g = bu.g + base;
  bf16* pb = bu.pb ? bu.pb + base : nullptr;
  float* acc = v.s[0] + ch.e0;
  float* mo = (v.flags & F_MOM) ? v.s[3] + ch.e0 : nullptr;
  const float mu = hp.b1;
  flat_loop(ch.ne, [&](auto vt, long long i) {
    constexpr int VEC = decltype(vt)::value;
    float gv[VEC], pv[VEC], av[VEC], u[VEC];
    ldv(g + i, gv); ldv(p + i, pv); ldv(acc + i, av);
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      av[j] = av[j] + gv[j] * gv[j];
      u[j] = (1.f - mu) * gv[j] * rsqrtf(av[j] + 1e-30f);
    }
    stv(acc + i, av);
    if (mo) {
      float mv[VEC];
      ldv(mo + i, mv);
#pragma unroll
      for (int j = 0; j < VEC; ++j) { mv[j] = mv[j] * mu + u[j]; u[j] = mv[j]; }
      stv(mo + i, mv);
    }
#pragma unroll
    for (int j = 0; j < VEC; ++j) pv[j] = pv[j] - lr * u[j];
    stv(p + i, pv);
    stb(pb ? pb + i : nullptr, pv);
  });
}
// the new accumulators replace the old ones; the work space is cleared for the next step
__global__ void __launch_bounds__(kThreads) optim_sm3_finish_kernel(Bufs bu) {
  pdl_wait();
  const OptVar& v = bu.vars[blockIdx.x];
  if (!(v.flags & F_ROWS)) return;
  const bool r3 = v.rank == 3;
  const long long B = v.B, R = v.R, tot = v.B + v.R + v.C;
  float* w = bu.ws + v.sc;
  for (long long i = (long long)blockIdx.y * kThreads + threadIdx.x; i < tot; i += (long long)gridDim.y * kThreads) {
    const float x = w[i];
    w[i] = 0.f;
    if (i < B) {
      if (r3) v.s[0][i] = x;
    } else if (i < B + R) {
      v.s[r3 ? 1 : 0][i - B] = x;
    } else {
      v.s[r3 ? 2 : 1][i - B - R] = x;
    }
  }
}

}  // namespace

#define CS(s) reinterpret_cast<cudaStream_t>(s)

// kind: 0 momentum (1 launch), 1 LAMB (2), 2 Adafactor (4), 3 SM3 (2).  vars / chunks: device tables (OptVar / OptChunk);
// p, g: flat fp32 master / gradient buffers, p_bf16: flat bf16 compute copy (or null); ws: work space (zero-initialised
// once; SM3 keeps it zero between steps); hyper: device fp32 [8]; hp: host fp32 [12] (OptHP).  col_blocks: grid.y of the
// per-variable launches (Adafactor's column pass, SM3's accumulator copy).
extern "C" int tepd_optim_step(int kind, const void* vars, const void* chunks, int nvars, int nchunks, int col_blocks,
                               void* p, const void* g, void* p_bf16, void* ws, const void* hyper, const float* hp, void* stream) {
  if (((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g)) & 15) || (reinterpret_cast<uintptr_t>(p_bf16) & 7)) return -2;
  if (nvars <= 0 || nchunks <= 0 || col_blocks <= 0 || !hp || !hyper || !ws) return -3;
  OptHP h;
  memcpy(&h, hp, sizeof(h));
  Bufs bu{(float*)p, (const float*)g, (bf16*)p_bf16, (float*)ws, (const float*)hyper, (const OptVar*)vars, (const OptChunk*)chunks};
  const dim3 grid(nchunks), per_var(nvars, col_blocks), blk(kThreads);
  cudaStream_t s = CS(stream);
  cudaError_t e = cudaSuccess;
  switch (kind) {
    case 0:
      e = tepd::launch(optim_momentum_kernel, grid, blk, 0, s, bu, h);
      break;
    case 1:
      if ((e = tepd::launch(optim_lamb_moments_kernel, grid, blk, 0, s, bu, h)) != cudaSuccess) break;
      e = tepd::launch(optim_lamb_apply_kernel, grid, blk, 0, s, bu, h);
      break;
    case 2:
      if ((e = tepd::launch(optim_af_stats_kernel, grid, blk, 0, s, bu, h)) != cudaSuccess) break;
      if ((e = tepd::launch(optim_af_cols_kernel, per_var, blk, 0, s, bu, h)) != cudaSuccess) break;
      if ((e = tepd::launch(optim_af_usq_kernel, grid, blk, 0, s, bu, h)) != cudaSuccess) break;
      e = tepd::launch(optim_af_apply_kernel, grid, blk, 0, s, bu, h);
      break;
    case 3:
      if ((e = tepd::launch(optim_sm3_kernel, grid, blk, 0, s, bu, h)) != cudaSuccess) break;
      e = tepd::launch(optim_sm3_finish_kernel, per_var, blk, 0, s, bu);
      break;
    default:
      return -4;
  }
  return (int)e;
}
