// Convolution as implicit-GEMM pieces for the wgmma GEMM kernels (Wide-ResNet; reference K9 runs cuDNN custom-calls,
// SURVEY 2.H).  Activations live in NHWC memory (torch channels_last), so
//   * a 1x1 / stride-1 convolution IS a GEMM  Y[N*H*W, Cout] = X[N*H*W, Cin] . W[Cout, Cin]^T  -- no data movement at all;
//   * every other shape goes through `im2col` (rows = output pixels, columns = (tap, cin) with cin fastest: each tap is one
//     contiguous Cin-vector of the source, copied with 16-byte accesses) followed by the same GEMM;
//   * the input gradient is  dcol = dY . W  (GEMM) followed by `col2im`, written as a GATHER over the taps that touch an
//     input pixel (no atomics, every dX element written exactly once);
//   * the weight gradient is  dW[Cout, taps*Cin] = dY^T . col  (the MN-major x MN-major GEMM used for linear layers).
// The GEMMs run in gemm_sm90.cu; this file holds the data-movement kernels.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "launch.cuh"

namespace {

typedef __nv_bfloat16 bf16;

__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

struct ConvGeom {
  int N, H, W, C;       // input  [N, H, W, C]
  int Ho, Wo;           // output spatial size
  int kh, kw, stride, pad;
  int Kpad;             // row length of the column matrix (>= kh*kw*C, multiple of 8)
};

// col[(n, ho, wo), (tap, c)] = x[n, ho*stride - pad + ky, wo*stride - pad + kx, c]   (0 outside the image / in the K padding)
// One thread per 8 channels of one (row, tap); VEC = 8 needs C % 8 == 0, VEC = 1 is the generic path (stem conv, C = 3).
template <int VEC>
__global__ void __launch_bounds__(256) im2col_nhwc_kernel(const bf16* __restrict__ x, bf16* __restrict__ col, ConvGeom g) {
  pdl_wait();
  const int taps = g.kh * g.kw;
  const int cv = (g.C + VEC - 1) / VEC;                       // channel vectors per tap
  const long long per_row = (long long)taps * cv;
  const long long rows = (long long)g.N * g.Ho * g.Wo;
  const long long total = rows * per_row;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / per_row;
    const int r = (int)(i - row * per_row);
    const int tap = r / cv, c0 = (r - tap * cv) * VEC;
    const int ky = tap / g.kw, kx = tap - ky * g.kw;
    const int wo = (int)(row % g.Wo);
    const int ho = (int)((row / g.Wo) % g.Ho);
    const int n = (int)(row / ((long long)g.Wo * g.Ho));
    const int hi = ho * g.stride - g.pad + ky, wi = wo * g.stride - g.pad + kx;
    const bool in = hi >= 0 && hi < g.H && wi >= 0 && wi < g.W;
    bf16* dst = col + row * g.Kpad + (long long)tap * g.C + c0;
    if (VEC == 8) {
      uint4 v = make_uint4(0u, 0u, 0u, 0u);
      if (in) v = __ldg(reinterpret_cast<const uint4*>(x + (((long long)n * g.H + hi) * g.W + wi) * g.C + c0));
      *reinterpret_cast<uint4*>(dst) = v;
    } else {
      *dst = in ? x[(((long long)n * g.H + hi) * g.W + wi) * g.C + c0] : __float2bfloat16(0.f);
    }
  }
  // zero the K padding (generic path only: taps*C is not a multiple of 8)
  if (VEC == 1 && g.Kpad > taps * g.C) {
    const int padk = g.Kpad - taps * g.C;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < rows * padk; i += (long long)gridDim.x * blockDim.x) {
      const long long row = i / padk;
      col[row * g.Kpad + taps * g.C + (int)(i - row * padk)] = __float2bfloat16(0.f);
    }
  }
}

// dx[n, hi, wi, c] = sum over taps (ky, kx) with (hi + pad - ky) % stride == 0 etc. of dcol[(n, ho, wo), (tap, c)]
template <int VEC>
__global__ void __launch_bounds__(256) col2im_nhwc_kernel(const bf16* __restrict__ dcol, bf16* __restrict__ dx, ConvGeom g) {
  pdl_wait();
  const int cv = (g.C + VEC - 1) / VEC;
  const long long total = (long long)g.N * g.H * g.W * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c0 = (int)(i % cv) * VEC;
    long long p = i / cv;
    const int wi = (int)(p % g.W); p /= g.W;
    const int hi = (int)(p % g.H);
    const int n = (int)(p / g.H);
    float acc[VEC];
#pragma unroll
    for (int j = 0; j < VEC; ++j) acc[j] = 0.f;
    for (int ky = 0; ky < g.kh; ++ky) {
      const int hn = hi + g.pad - ky;
      if (hn < 0 || hn % g.stride) continue;
      const int ho = hn / g.stride;
      if (ho >= g.Ho) continue;
      for (int kx = 0; kx < g.kw; ++kx) {
        const int wn = wi + g.pad - kx;
        if (wn < 0 || wn % g.stride) continue;
        const int wo = wn / g.stride;
        if (wo >= g.Wo) continue;
        const bf16* src = dcol + (((long long)n * g.Ho + ho) * g.Wo + wo) * g.Kpad + (long long)(ky * g.kw + kx) * g.C + c0;
        if (VEC == 8) {
          const uint4 u = __ldg(reinterpret_cast<const uint4*>(src));
          const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float2 f = __bfloat1622float2(h[e]);
            acc[2 * e] += f.x;
            acc[2 * e + 1] += f.y;
          }
        } else {
          acc[0] += __bfloat162float(*src);
        }
      }
    }
    bf16* dst = dx + (((long long)n * g.H + hi) * g.W + wi) * g.C + c0;
    if (VEC == 8) {
      uint4 u;
      __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
      for (int e = 0; e < 4; ++e) h[e] = __floats2bfloat162_rn(acc[2 * e], acc[2 * e + 1]);
      *reinterpret_cast<uint4*>(dst) = u;
    } else {
      *dst = __float2bfloat16(acc[0]);
    }
  }
}

inline int grid_for(long long work) {
  long long b = (work + 255) / 256;
  const long long cap = (long long)tepd::num_sms() * 16;
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

// ---- pooling, NHWC bf16, C % 8 == 0, one thread per 8 channels (reference K9: XLA reduce-window / select-and-scatter on cuDNN-era
// codegen).  Max pool backward is a GATHER (no atomics): an input pixel looks at the <= ceil(k/stride)^2 windows that cover it,
// re-scans each window and takes dy when it is that window's FIRST maximum in row-major scan order (torch's tie rule).
__device__ __forceinline__ void ld8(const bf16* p, float (&f)[8]) {
  const uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) { const float2 t = __bfloat1622float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
}
__device__ __forceinline__ void st8(bf16* p, const float (&f)[8]) {
  uint4 u;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  *reinterpret_cast<uint4*>(p) = u;
}
__global__ void __launch_bounds__(256) maxpool_fwd_nhwc_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, ConvGeom g) {
  const int cv = g.C / 8;
  const long long total = (long long)g.N * g.Ho * g.Wo * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cv) * 8;
    long long r = i / cv;
    const int wo = (int)(r % g.Wo); r /= g.Wo;
    const int ho = (int)(r % g.Ho);
    const int n = (int)(r / g.Ho);
    float m[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) m[j] = -INFINITY;
    for (int ky = 0; ky < g.kh; ++ky) {
      const int ih = ho * g.stride - g.pad + ky;
      if (ih < 0 || ih >= g.H) continue;
      for (int kx = 0; kx < g.kw; ++kx) {
        const int iw = wo * g.stride - g.pad + kx;
        if (iw < 0 || iw >= g.W) continue;
        float v[8];
        ld8(x + (((long long)n * g.H + ih) * g.W + iw) * g.C + c, v);
#pragma unroll
        for (int j = 0; j < 8; ++j) m[j] = fmaxf(m[j], v[j]);
      }
    }
    st8(y + i * 8, m);
  }
}
__global__ void __launch_bounds__(256) maxpool_bwd_nhwc_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x,
                                                               const bf16* __restrict__ y, bf16* __restrict__ dx, ConvGeom g) {
  const int cv = g.C / 8;
  const long long total = (long long)g.N * g.H * g.W * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cv) * 8;
    long long r = i / cv;
    const int iw = (int)(r % g.W); r /= g.W;
    const int ih = (int)(r % g.H);
    const int n = (int)(r / g.H);
    float xv[8], acc[8];
    ld8(x + i * 8, xv);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    // output rows / columns whose window contains (ih, iw):  ho*stride - pad <= ih <= ho*stride - pad + k - 1
    const int ho_lo = max(0, (ih + g.pad - g.kh + g.stride) / g.stride), ho_hi = min(g.Ho - 1, (ih + g.pad) / g.stride);
    const int wo_lo = max(0, (iw + g.pad - g.kw + g.stride) / g.stride), wo_hi = min(g.Wo - 1, (iw + g.pad) / g.stride);
    for (int ho = ho_lo; ho <= ho_hi; ++ho)
      for (int wo = wo_lo; wo <= wo_hi; ++wo) {
        const long long oidx = (((long long)n * g.Ho + ho) * g.Wo + wo) * g.C + c;
        float yv[8], gv[8];
        ld8(y + oidx, yv);
        ld8(dy + oidx, gv);
        unsigned cand = 0;                       // channels where this pixel holds the window maximum
#pragma unroll
        for (int j = 0; j < 8; ++j) cand |= (xv[j] == yv[j]) ? (1u << j) : 0u;
        if (!cand) continue;
        // an EARLIER pixel of the window (row-major) with the same value wins the tie
        const int my = (ih - (ho * g.stride - g.pad)) * g.kw + (iw - (wo * g.stride - g.pad));
        for (int t = 0; t < my && cand; ++t) {
          const int ph = ho * g.stride - g.pad + t / g.kw, pw = wo * g.stride - g.pad + t % g.kw;
          if (ph < 0 || ph >= g.H || pw < 0 || pw >= g.W) continue;
          float pv[8];
          ld8(x + (((long long)n * g.H + ph) * g.W + pw) * g.C + c, pv);
#pragma unroll
          for (int j = 0; j < 8; ++j) if (pv[j] == yv[j]) cand &= ~(1u << j);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) if (cand & (1u << j)) acc[j] += gv[j];
      }
    st8(dx + i * 8, acc);
  }
}
// global average pool: y[n, c] = mean over H*W (fp32 accumulation); backward: dx[n, h, w, c] = dy[n, c] / (H*W)
__global__ void __launch_bounds__(256) gap_fwd_nhwc_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, int N, int HW, int C) {
  const int cv = C / 8;
  const long long total = (long long)N * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cv) * 8, n = (int)(i / cv);
    float s[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j] = 0.f;
    for (int p = 0; p < HW; ++p) {
      float v[8];
      ld8(x + ((long long)n * HW + p) * C + c, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) s[j] += v[j];
    }
    const float inv = 1.f / (float)HW;
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j] *= inv;
    st8(y + (long long)n * C + c, s);
  }
}
__global__ void __launch_bounds__(256) gap_bwd_nhwc_kernel(const bf16* __restrict__ dy, bf16* __restrict__ dx, int N, int HW, int C) {
  const int cv = C / 8;
  const long long total = (long long)N * HW * cv;
  const float inv = 1.f / (float)HW;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cv) * 8, n = (int)(i / ((long long)cv * HW));
    float v[8];
    ld8(dy + (long long)n * C + c, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] *= inv;
    st8(dx + i * 8, v);
  }
}

ConvGeom MakeGeom(int N, int H, int W, int C, int Ho, int Wo, int kh, int kw, int stride, int pad, int Kpad) {
  ConvGeom g;
  g.N = N; g.H = H; g.W = W; g.C = C; g.Ho = Ho; g.Wo = Wo; g.kh = kh; g.kw = kw; g.stride = stride; g.pad = pad; g.Kpad = Kpad;
  return g;
}

}  // namespace

#define CS(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int tepd_im2col_nhwc(const void* x, void* col, int N, int H, int W, int C, int Ho, int Wo, int kh, int kw, int stride,
                                int pad, int Kpad, void* stream) {
  if (Kpad % 8 || Kpad < kh * kw * C) return -2;
  const ConvGeom g = MakeGeom(N, H, W, C, Ho, Wo, kh, kw, stride, pad, Kpad);
  const long long rows = (long long)N * Ho * Wo;
  if (C % 8 == 0) {
    if (Kpad != kh * kw * C) return -3;
    return (int)tepd::launch(im2col_nhwc_kernel<8>, dim3(grid_for(rows * kh * kw * (C / 8))), dim3(256), 0, CS(stream),
                             (const bf16*)x, (bf16*)col, g);
  }
  return (int)tepd::launch(im2col_nhwc_kernel<1>, dim3(grid_for(rows * kh * kw * C)), dim3(256), 0, CS(stream), (const bf16*)x,
                           (bf16*)col, g);
}

extern "C" int tepd_col2im_nhwc(const void* dcol, void* dx, int N, int H, int W, int C, int Ho, int Wo, int kh, int kw, int stride,
                                int pad, int Kpad, void* stream) {
  if (Kpad % 8 || Kpad < kh * kw * C) return -2;
  const ConvGeom g = MakeGeom(N, H, W, C, Ho, Wo, kh, kw, stride, pad, Kpad);
  const long long px = (long long)N * H * W;
  if (C % 8 == 0)
    return (int)tepd::launch(col2im_nhwc_kernel<8>, dim3(grid_for(px * (C / 8))), dim3(256), 0, CS(stream), (const bf16*)dcol,
                             (bf16*)dx, g);
  return (int)tepd::launch(col2im_nhwc_kernel<1>, dim3(grid_for(px * C)), dim3(256), 0, CS(stream), (const bf16*)dcol, (bf16*)dx, g);
}

extern "C" int tepd_maxpool_nhwc(const void* x, void* y, int N, int H, int W, int C, int Ho, int Wo, int k, int stride, int pad, void* stream) {
  if (C % 8) return -2;
  const ConvGeom g = MakeGeom(N, H, W, C, Ho, Wo, k, k, stride, pad, 0);
  maxpool_fwd_nhwc_kernel<<<grid_for((long long)N * Ho * Wo * (C / 8)), 256, 0, CS(stream)>>>((const bf16*)x, (bf16*)y, g);
  return (int)cudaGetLastError();
}
extern "C" int tepd_maxpool_bwd_nhwc(const void* dy, const void* x, const void* y, void* dx, int N, int H, int W, int C, int Ho, int Wo,
                                     int k, int stride, int pad, void* stream) {
  if (C % 8) return -2;
  const ConvGeom g = MakeGeom(N, H, W, C, Ho, Wo, k, k, stride, pad, 0);
  maxpool_bwd_nhwc_kernel<<<grid_for((long long)N * H * W * (C / 8)), 256, 0, CS(stream)>>>((const bf16*)dy, (const bf16*)x, (const bf16*)y,
                                                                                          (bf16*)dx, g);
  return (int)cudaGetLastError();
}
extern "C" int tepd_gap_nhwc(const void* x, void* y, int N, int HW, int C, void* stream) {
  if (C % 8) return -2;
  gap_fwd_nhwc_kernel<<<grid_for((long long)N * (C / 8)), 256, 0, CS(stream)>>>((const bf16*)x, (bf16*)y, N, HW, C);
  return (int)cudaGetLastError();
}
extern "C" int tepd_gap_bwd_nhwc(const void* dy, void* dx, int N, int HW, int C, void* stream) {
  if (C % 8) return -2;
  gap_bwd_nhwc_kernel<<<grid_for((long long)N * HW * (C / 8)), 256, 0, CS(stream)>>>((const bf16*)dy, (bf16*)dx, N, HW, C);
  return (int)cudaGetLastError();
}
