// Fused (flash) attention for sm_90a, head_dim 64 or 128, bf16, with wgmma.mma_async on register accumulators.
// Forward, one CTA per (128-query block, batch, head): two warpgroups own 64 query rows each, a producer warpgroup streams
// K / V tiles through a TMA + mbarrier ring.
//   S = Q K^T            wgmma m64n128k16 (A = Q, B = K, both K-major in smem)        -> registers
//   P = online softmax   in registers (quad shuffles for the row max / sum)
//   O += P V             wgmma m64nDk16 with A = P from registers (the S fragment repacked to bf16), B = V MN-major
// Q/K/V are read straight out of the fused qkv projection buffer [B, S, H, 3, D] (heads-major) with 4-D TMA maps
// (no head-split transposes), O is written as [B, S, H, D] so it feeds the output projection GEMM.
// A D-wide row tile is D / 64 SW128 column chunks of [rows x 64] (128 B per row), each loaded by one TMA box.
// The producer warpgroup drops to 24 registers with setmaxnreg and the two consumer warpgroups take 240 each, so no kernel
// spills even where the O (fwd) and dK + dV (bwd) accumulators double at D = 128.
// The reference gets attention from XLA-fused batched dots + softmax fusions (SURVEY Appendix C);
// this kernel is the H100-native replacement.
#include "sm90_ptx.cuh"
#include "launch.cuh"
#include <math.h>
#include <stdio.h>

using namespace sm90;

namespace {

constexpr int BQ = 128;       // query rows per forward CTA
constexpr int BKV = 128;      // kv rows per forward iteration / per backward CTA
constexpr int CHUNK = 128 * 128;  // 16 KB: one [128 x 64] bf16 SW128 column chunk of a 128-row tile

template <int HD>
struct AttnCfg;
template <>
struct AttnCfg<64> {
  static constexpr int THREADS = 384;  // warpgroups 0, 1: compute (240 registers), warpgroup 2: TMA producer (24)
  static constexpr int KV_STAGES = 3;
  static constexpr int Q_STAGES = 3;
};
template <>
struct AttnCfg<128> {
  static constexpr int THREADS = 384;  // warpgroups 0, 1: compute (240 registers), warpgroup 2: TMA producer (24)
  static constexpr int KV_STAGES = 2;  // 32 KB Q + 2 x 64 KB K / V
  static constexpr int Q_STAGES = 3;   // 64 KB K / V + 16 KB dS^T + 3 x 32 KB Q / dO
};

template <int HD>
struct FwdSmem {
  static constexpr int TILE_BYTES = 128 * HD * 2;  // a [128 x HD] bf16 tile (HD / 64 chunks)
  static constexpr int SM_Q = 0;
  static constexpr int SM_K = SM_Q + TILE_BYTES;
  static constexpr int SM_V = SM_K + AttnCfg<HD>::KV_STAGES * TILE_BYTES;
  static constexpr int SM_BAR = SM_V + AttnCfg<HD>::KV_STAGES * TILE_BYTES;
  static constexpr int BYTES = SM_BAR + 256 + 1024;
};

struct AttnFwdParams {
  void* O;      // bf16 [B, S, H, D]
  float* lse;   // fp32 [B, H, S]   (natural-log domain, scaled scores)
  int B, H, S, causal;
  float scale_log2;  // softmax scale * log2(e)
  float scale;
  const int* doc_start;   // int32 [B, S], DOC kernels only: query s sees keys [doc_start[b, s], s]
};

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// DOC (document-masked causal attention): a query tile starts its KV loop at the tile holding the document start of its
// first row (doc_start is non-decreasing along the sequence), and tiles below the document start of its last row get an
// element mask.  A row can then see a fully masked tile, so the softmax subtracts 0 instead of a -inf running max.
template <int HD, bool DOC>
__global__ void __launch_bounds__(AttnCfg<HD>::THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                const __grid_constant__ CUtensorMap tmap_v, const AttnFwdParams p) {
  using L = FwdSmem<HD>;
  constexpr int KV_STAGES = AttnCfg<HD>::KV_STAGES;
  constexpr int NC = HD / 64;   // column chunks per row tile
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::SM_BAR);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;               // [KV_STAGES]
  uint64_t* kv_empty = bars + 1 + KV_STAGES;  // [KV_STAGES]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nq = p.S / BQ;
  const int BH = p.B * p.H;
  const int qi = p.causal ? nq - 1 - (int)(blockIdx.x / BH) : (int)(blockIdx.x / BH);  // longest causal rows first
  const int bh = blockIdx.x % BH;
  const int b = bh / p.H, h = bh % p.H;
  const int nkv = p.causal ? qi + 1 : p.S / BKV;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_k);
    tma_prefetch_desc(&tmap_v);
    mbar_init(q_full, 1);
    for (int s = 0; s < KV_STAGES; ++s) {
      mbar_init(&kv_full[s], 1);
      mbar_init(&kv_empty[s], 2);   // one arrival per compute warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  int j0 = 0;   // first KV tile (stage and phase indices count from it)
  if constexpr (DOC) j0 = __ldg(p.doc_start + (size_t)b * p.S + qi * BQ) / BKV;

  if (warp >= 8) {   // producer warpgroup
    setmaxnreg_dec<24>();
    if (lane == 0 && warp == 8) {
      mbar_expect_tx(q_full, L::TILE_BYTES);
#pragma unroll
      for (int c = 0; c < NC; ++c) tma_load_4d(smem + L::SM_Q + c * CHUNK, &tmap_q, q_full, c * 64, qi * BQ, h, b);
      for (int j = j0; j < nkv; ++j) {
        const int st = (j - j0) % KV_STAGES;
        mbar_wait(&kv_empty[st], (((j - j0) / KV_STAGES) & 1) ^ 1);
        mbar_expect_tx(&kv_full[st], 2 * L::TILE_BYTES);
#pragma unroll
        for (int c = 0; c < NC; ++c)
          tma_load_4d(smem + L::SM_K + st * L::TILE_BYTES + c * CHUNK, &tmap_k, &kv_full[st], c * 64, j * BKV, h, b);
#pragma unroll
        for (int c = 0; c < NC; ++c)
          tma_load_4d(smem + L::SM_V + st * L::TILE_BYTES + c * CHUNK, &tmap_v, &kv_full[st], c * 64, j * BKV, h, b);
      }
    }
    pdl_trigger();
    return;
  }
  setmaxnreg_inc<240>();

  const int wg = warp >> 2;
  const int g = lane >> 2, q = lane & 3;
  const int row0 = wg * 64 + (warp & 3) * 16 + g;   // query row (in the tile) of fragment rows e < 2; +8 for e >= 2
  const uint32_t sq = smem_u32(smem + L::SM_Q) + wg * 64 * 128;
  float o[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  int ds[2] = {0, 0}, ds_last = 0;   // DOC: document starts of this thread's two rows and of the tile's last row
  if constexpr (DOC) {
    const int* dsb = p.doc_start + (size_t)b * p.S + qi * BQ;
    ds[0] = __ldg(dsb + row0);
    ds[1] = __ldg(dsb + row0 + 8);
    ds_last = __ldg(dsb + BQ - 1);
  }
  // online softmax of the score tile of KV tile j: s -> P (fp32), running max / sum updated, alpha = the factor O is rescaled by
  auto softmax = [&](float (&s)[64], int j, float (&alpha)[2]) {
    const bool diag = p.causal && j == qi;
    if (DOC && j * BKV < ds_last) {   // some key of this tile lies before the document start of some row (a separate pass:
                                      // the tiles without one run the plain softmax)
#pragma unroll
      for (int jj = 0; jj < 16; ++jj)
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (j * BKV + 8 * jj + 2 * q + (e & 1) < ds[e >> 1]) s[4 * jj + e] = -INFINITY;
    }
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int r = row0 + hr * 8;
      float mx = m[hr];
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int idx = 4 * jj + 2 * hr + e;
          float x = s[idx] * p.scale_log2;
          if (diag && 8 * jj + 2 * q + e > r) x = -INFINITY;
          s[idx] = x;
          mx = fmaxf(mx, x);
        }
      }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      // safe max: a row that has seen only masked keys keeps m = -inf, and subtracting 0 instead gives p = 0, alpha = 0
      const float mxs = DOC && mx == -INFINITY ? 0.f : mx;
      alpha[hr] = exp2f(m[hr] - mxs);
      m[hr] = mx;
      float sum = 0.f;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int idx = 4 * jj + 2 * hr + e;
          const float pv = exp2f(s[idx] - mxs);
          s[idx] = pv;
          sum += pv;
        }
      }
      l[hr] = l[hr] * alpha[hr] + sum;
    }
  };
  auto rescale_o = [&](const float (&alpha)[2]) {
#pragma unroll
    for (int hr = 0; hr < 2; ++hr)
#pragma unroll
      for (int jj = 0; jj < HD / 8; ++jj) {
        o[4 * jj + 2 * hr] *= alpha[hr];
        o[4 * jj + 2 * hr + 1] *= alpha[hr];
      }
  };
  auto issue_s = [&](float (&s)[64], int j) {   // S = Q K_j^T (one commit group)
    const int st = (j - j0) % KV_STAGES;
    mbar_wait(&kv_full[st], ((j - j0) / KV_STAGES) & 1);
    const uint32_t sk = smem_u32(smem + L::SM_K + st * L::TILE_BYTES);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < HD / 16; ++k)
      wgmma_m64n128k16_bf16_ss<0, 0>(s, make_smem_desc_sw128(sq + (k / 4) * CHUNK + (k % 4) * 32, 0, 1024),
                                     make_smem_desc_sw128(sk + (k / 4) * CHUNK + (k % 4) * 32, 0, 1024), k > 0 ? 1u : 0u);
    wgmma_commit();
  };
  auto issue_pv = [&](const uint32_t (&pa)[32], int j) {   // O += P V_j (one commit group); P packed to bf16 A fragments
    const uint32_t sv = smem_u32(smem + L::SM_V + ((j - j0) % KV_STAGES) * L::TILE_BYTES);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      const uint32_t a[4] = {pa[4 * kk], pa[4 * kk + 1], pa[4 * kk + 2], pa[4 * kk + 3]};
      // V MN-major: LBO = the next 64-column chunk (the field is unused at N = 64)
      wgmma_m64nXk16_bf16_rs<1>(o, a, make_smem_desc_sw128(sv + kk * 16 * 128, HD == 64 ? 8192 : CHUNK, 1024), 1u);
    }
    wgmma_commit();
  };
  auto pack_p = [&](const float (&s)[64], uint32_t (&pa)[32]) {
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      uint32_t a[4];
      frag_a_from_acc(s, kk, a);
#pragma unroll
      for (int t = 0; t < 4; ++t) pa[4 * kk + t] = a[t];
    }
  };
  auto release = [&](int j) {
    if ((threadIdx.x & 127) == 0) mbar_arrive(&kv_empty[(j - j0) % KV_STAGES]);
  };
  mbar_wait(q_full, 0);
  if constexpr (HD == 64) {
    // Software-pipelined: S_{j+1} = Q K_{j+1}^T and O += P_j V_j are in flight while the softmax of S_{j+1} runs; O is
    // rescaled once P_j V_j has landed, so every tile sees the same arithmetic in the same order as the unpipelined loop.
    float s[64], alpha[2];
    uint32_t pa[32];
    issue_s(s, j0);
    wgmma_wait<0>();
    fence_regs(s);
    softmax(s, j0, alpha);
    rescale_o(alpha);
    pack_p(s, pa);
    for (int j = j0 + 1; j < nkv; ++j) {
      issue_s(s, j);
      issue_pv(pa, j - 1);
      wgmma_wait<1>();
      fence_regs(s);
      softmax(s, j, alpha);
      wgmma_wait<0>();
      fence_regs(o);
      release(j - 1);
      rescale_o(alpha);
      pack_p(s, pa);
    }
    issue_pv(pa, nkv - 1);
    wgmma_wait<0>();
    fence_regs(o);
    release(nkv - 1);
  } else {
    for (int j = j0; j < nkv; ++j) {
      const int st = (j - j0) % KV_STAGES;
      mbar_wait(&kv_full[st], ((j - j0) / KV_STAGES) & 1);
      const uint32_t sk = smem_u32(smem + L::SM_K + st * L::TILE_BYTES), sv = smem_u32(smem + L::SM_V + st * L::TILE_BYTES);
      float s[64];
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < HD / 16; ++k)
        wgmma_m64n128k16_bf16_ss<0, 0>(s, make_smem_desc_sw128(sq + (k / 4) * CHUNK + (k % 4) * 32, 0, 1024),
                                       make_smem_desc_sw128(sk + (k / 4) * CHUNK + (k % 4) * 32, 0, 1024), k > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(s);
      const bool diag = p.causal && j == qi;
      if (DOC && j * BKV < ds_last) {   // some key of this tile lies before the document start of some row (a separate pass:
                                        // the tiles without one run the plain softmax)
#pragma unroll
        for (int jj = 0; jj < 16; ++jj)
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (j * BKV + 8 * jj + 2 * q + (e & 1) < ds[e >> 1]) s[4 * jj + e] = -INFINITY;
      }
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int r = row0 + hr * 8;
        float mx = m[hr];
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int idx = 4 * jj + 2 * hr + e;
            float x = s[idx] * p.scale_log2;
            if (diag && 8 * jj + 2 * q + e > r) x = -INFINITY;
            s[idx] = x;
            mx = fmaxf(mx, x);
          }
        }
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        // safe max: a row that has seen only masked keys keeps m = -inf, and subtracting 0 instead gives p = 0, alpha = 0
        const float mxs = DOC && mx == -INFINITY ? 0.f : mx;
        const float alpha = exp2f(m[hr] - mxs);
        m[hr] = mx;
        float sum = 0.f;
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int idx = 4 * jj + 2 * hr + e;
            const float pv = exp2f(s[idx] - mxs);
            s[idx] = pv;
            sum += pv;
          }
        }
        l[hr] = l[hr] * alpha + sum;
#pragma unroll
        for (int jj = 0; jj < HD / 8; ++jj) {
          o[4 * jj + 2 * hr] *= alpha;
          o[4 * jj + 2 * hr + 1] *= alpha;
        }
      }
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        uint32_t a[4];
        frag_a_from_acc(s, kk, a);
        // V MN-major: LBO = the next 64-column chunk (the field is unused at N = 64)
        wgmma_m64nXk16_bf16_rs<1>(o, a, make_smem_desc_sw128(sv + kk * 16 * 128, HD == 64 ? 8192 : CHUNK, 1024), 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(o);
      if ((threadIdx.x & 127) == 0) mbar_arrive(&kv_empty[st]);
    }
  }
  pdl_trigger();
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    float lsum = l[hr];
    lsum += __shfl_xor_sync(0xffffffffu, lsum, 1);
    lsum += __shfl_xor_sync(0xffffffffu, lsum, 2);
    const float inv = 1.f / lsum;
    const int row = qi * BQ + row0 + hr * 8;
    __nv_bfloat16* op = reinterpret_cast<__nv_bfloat16*>(p.O) + (((size_t)b * p.S + row) * p.H + h) * HD;
#pragma unroll
    for (int jj = 0; jj < HD / 8; ++jj)
      *reinterpret_cast<uint32_t*>(op + 8 * jj + 2 * q) = pack_bf16x2(o[4 * jj + 2 * hr] * inv, o[4 * jj + 2 * hr + 1] * inv);
    if (q == 0) p.lse[((size_t)b * p.H + h) * p.S + row] = (m[hr] + log2f(lsum)) * 0.6931471805599453f;
  }
}

// =====================================================================================================
// Backward.  One CTA per (128-row kv block j, batch, head); two warpgroups own 64 kv rows each and loop over 64-row query
// blocks i (those that see block j when causal), streamed by the producer.  Per warpgroup and block:
//   S^T = K Q^T, dP^T = V dO^T                      wgmma m64n64k16, both operands K-major in smem
//   P^T = exp2(S^T c - lse), dS^T = P^T (dP^T - delta)          in registers
//   dV += P^T dO, dK += dS^T Q                      wgmma m64nDk16 with A from registers, B (dO / Q) MN-major in smem
//   dQ  = dS K over this warpgroup's 64 kv rows      dS^T goes through smem (read as an MN-major A operand) ->
//                                                   summed into dq_acc over kv blocks / warpgroups: at D = 128 by fp32
//                                                   red.add from the fragments, one 64-column half of D at a time (keeps
//                                                   it within 240 registers); at D = 64 staged in smem and added by one
//                                                   bulk reduce-add per warpgroup and block
// At D = 64 lse / delta come from smem (bulk-copied by the producer with each Q / dO stage), S^T and dP^T are separate
// commit groups, and dV += P^T dO runs while dS^T is formed.
// =====================================================================================================
constexpr int BQB = 64;                          // query rows per backward iteration

template <int HD>
struct BwdSmem {
  static constexpr int KV_BYTES = 128 * HD * 2;   // K or V: [128 kv x HD]
  static constexpr int DS_BYTES = 128 * 64 * 2;   // dS^T [128 kv][64 q] bf16, SW128
  static constexpr int QB_BYTES = BQB * HD * 2;   // Q or dO: [64 q x HD]
  static constexpr int QB_CHUNK = BQB * 128;      // 8 KB: one [64 x 64] column chunk
  static constexpr int SB_K = 0;
  static constexpr int SB_V = SB_K + KV_BYTES;
  static constexpr int SB_DS = SB_V + KV_BYTES;
  static constexpr int SB_Q = SB_DS + DS_BYTES;   // [Q_STAGES]
  static constexpr int SB_DO = SB_Q + AttnCfg<HD>::Q_STAGES * QB_BYTES;
  // D = 64 only: each warpgroup's fp32 [64 q x 64] dQ partial, and per Q / dO stage the block's 64 lse + 64 delta values
  static constexpr int DQ_BYTES = HD == 64 ? BQB * 64 * 4 : 0;
  static constexpr int STAT_BYTES = HD == 64 ? 2 * BQB * 4 : 0;
  static constexpr int SB_DQ = SB_DO + AttnCfg<HD>::Q_STAGES * QB_BYTES;   // [2 warpgroups]
  static constexpr int SB_STAT = SB_DQ + 2 * DQ_BYTES;                     // [Q_STAGES]
  static constexpr int SB_BAR = SB_STAT + AttnCfg<HD>::Q_STAGES * STAT_BYTES;
  static constexpr int BYTES = SB_BAR + 256 + 1024;
};

struct AttnBwdParams {
  const float* lse;    // [B,H,S]
  const float* delta;  // [B,H,S]
  float* dq_acc;       // fp32, zero-initialised: [B, S, H, 128] at D = 128, [B, H, S, 64] (see attn_dq_cast_kernel) at D = 64
  void* dk;            // bf16, strided [B,S,H,D] view
  void* dv;
  long long dstride_b, dstride_s, dstride_h;
  int B, H, S, causal;
  float scale_log2, scale;
  const int* doc_start;   // int32 [B, S], DOC kernels only
};

// DOC: the query blocks of KV block j end at the first block whose first row starts its document after the block's last
// key (binary search, doc_start is non-decreasing).  Inside the range P = 0 where key < doc_start[query]; since doc_start is
// monotone, those queries are a suffix for each key row, so a thread keeps one bound per kv row instead of loading
// doc_start per query column.
template <int HD, bool DOC>
__global__ void __launch_bounds__(AttnCfg<HD>::THREADS, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ CUtensorMap tmap_do,
                const AttnBwdParams p) {
  using L = BwdSmem<HD>;
  constexpr int Q_STAGES = AttnCfg<HD>::Q_STAGES;
  constexpr int NC = HD / 64;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::SB_BAR);
  uint64_t* kv_full = bars;
  uint64_t* q_full = bars + 1;              // [Q_STAGES]
  uint64_t* q_empty = bars + 1 + Q_STAGES;  // [Q_STAGES]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int BH = p.B * p.H;
  const int j = (int)(blockIdx.x / BH);  // kv block; small j = most work, scheduled first
  const int bh = blockIdx.x % BH;
  const int b = bh / p.H, h = bh % p.H;
  const int nqb = p.S / BQB;
  const int i0 = p.causal ? j * (BKV / BQB) : 0;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_k);
    tma_prefetch_desc(&tmap_v);
    tma_prefetch_desc(&tmap_do);
    mbar_init(kv_full, 1);
    for (int s = 0; s < Q_STAGES; ++s) {
      mbar_init(&q_full[s], 1);
      mbar_init(&q_empty[s], 2);
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  int i_end = nqb;   // producer and consumers walk the same query blocks [i0, i_end)
  const int* ds_b = DOC ? p.doc_start + (size_t)b * p.S : nullptr;
  if constexpr (DOC) {
    const int last_key = j * BKV + BKV - 1;
    int lo = i0;   // block i0 starts at key j * BKV and sees itself: the range is never empty
    while (lo < i_end) {
      const int mid = (lo + i_end) >> 1;
      if (__ldg(ds_b + mid * BQB) > last_key) i_end = mid;
      else lo = mid + 1;
    }
  }

  if (warp >= 8) {   // producer warpgroup
    setmaxnreg_dec<24>();
    if (lane == 0 && warp == 8) {
      mbar_expect_tx(kv_full, 2 * L::KV_BYTES);
#pragma unroll
      for (int c = 0; c < NC; ++c) tma_load_4d(smem + L::SB_K + c * CHUNK, &tmap_k, kv_full, c * 64, j * BKV, h, b);
#pragma unroll
      for (int c = 0; c < NC; ++c) tma_load_4d(smem + L::SB_V + c * CHUNK, &tmap_v, kv_full, c * 64, j * BKV, h, b);
      for (int i = i0, it = 0; i < i_end; ++i, ++it) {
        const int st = it % Q_STAGES;
        mbar_wait(&q_empty[st], ((it / Q_STAGES) & 1) ^ 1);
        mbar_expect_tx(&q_full[st], 2 * L::QB_BYTES + L::STAT_BYTES);
        if constexpr (HD == 64) {
          float* stat = reinterpret_cast<float*>(smem + L::SB_STAT + st * L::STAT_BYTES);
          const size_t row = ((size_t)b * p.H + h) * p.S + i * BQB;
          bulk_load(stat, p.lse + row, BQB * 4, &q_full[st]);
          bulk_load(stat + BQB, p.delta + row, BQB * 4, &q_full[st]);
        }
#pragma unroll
        for (int c = 0; c < NC; ++c)
          tma_load_4d(smem + L::SB_Q + st * L::QB_BYTES + c * L::QB_CHUNK, &tmap_q, &q_full[st], c * 64, i * BQB, h, b);
#pragma unroll
        for (int c = 0; c < NC; ++c)
          tma_load_4d(smem + L::SB_DO + st * L::QB_BYTES + c * L::QB_CHUNK, &tmap_do, &q_full[st], c * 64, i * BQB, h, b);
      }
    }
    pdl_trigger();
    return;
  }
  setmaxnreg_inc<240>();

  const int wg = warp >> 2;
  const int g = lane >> 2, q = lane & 3;
  const int r0 = (warp & 3) * 16 + g;      // fragment row inside the warpgroup's 64 rows (+8 for e >= 2)
  const uint32_t sk = smem_u32(smem + L::SB_K) + wg * 64 * 128, sv = smem_u32(smem + L::SB_V) + wg * 64 * 128;
  uint8_t* ds_tile = smem + L::SB_DS + wg * 64 * 128;   // this warpgroup's 64 kv rows of dS^T
  const uint32_t sds = smem_u32(ds_tile);
  const float* lse_bh = p.lse + ((size_t)b * p.H + h) * p.S;
  const float* delta_bh = p.delta + ((size_t)b * p.H + h) * p.S;
  float dv[HD / 2], dk[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) { dv[i] = 0.f; dk[i] = 0.f; }
  int qend[2] = {0, 0};   // DOC: first query whose document starts after kv row r0 + 8 hr (from there on P = 0)
  if constexpr (DOC) {
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int key = j * BKV + wg * 64 + r0 + 8 * hr;
      int lo = key + 1, hi = i_end * BQB;   // doc_start[key] <= key; no query at or past i_end * BQB sees this block
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(ds_b + mid) > key) hi = mid;
        else lo = mid + 1;
      }
      qend[hr] = lo;
    }
  }
  mbar_wait(kv_full, 0);
  for (int i = i0, it = 0; i < i_end; ++i, ++it) {
    const int st = it % Q_STAGES;
    mbar_wait(&q_full[st], (it / Q_STAGES) & 1);
    const uint32_t sq = smem_u32(smem + L::SB_Q + st * L::QB_BYTES), sdo = smem_u32(smem + L::SB_DO + st * L::QB_BYTES);
    float s[32], dp[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < HD / 16; ++k)
      wgmma_m64n64k16_bf16_ss<0, 0>(s, make_smem_desc_sw128(sk + (k / 4) * CHUNK + (k % 4) * 32, 0, 1024),
                                    make_smem_desc_sw128(sq + (k / 4) * L::QB_CHUNK + (k % 4) * 32, 0, 1024), k > 0 ? 1u : 0u);
    if constexpr (HD == 64) wgmma_commit();   // S^T and dP^T in separate groups: P^T is computed while dP^T runs
#pragma unroll
    for (int k = 0; k < HD / 16; ++k)
      wgmma_m64n64k16_bf16_ss<0, 0>(dp, make_smem_desc_sw128(sv + (k / 4) * CHUNK + (k % 4) * 32, 0, 1024),
                                    make_smem_desc_sw128(sdo + (k / 4) * L::QB_CHUNK + (k % 4) * 32, 0, 1024), k > 0 ? 1u : 0u);
    wgmma_commit();
    const bool masked = p.causal && i * BQB < j * BKV + BKV;   // query block overlaps the kv block
    const bool dmask = DOC && i * BQB + BQB > min(qend[0], qend[1]);   // some query of the block is past a kv row's document
    if constexpr (HD == 64) {
      const float* stat = reinterpret_cast<const float*>(smem + L::SB_STAT + st * L::STAT_BYTES);
      wgmma_wait<1>();
      fence_regs(s);
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
        for (int e1 = 0; e1 < 2; ++e1) {
          const int qt = 8 * jj + 2 * q + e1;
          const float L2 = stat[qt] * 1.4426950408889634f;
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            const int idx = 4 * jj + 2 * hr + e1;
            float pv = exp2f(s[idx] * p.scale_log2 - L2);
            if (masked && i * BQB + qt < j * BKV + wg * 64 + r0 + 8 * hr) pv = 0.f;
            if (dmask && i * BQB + qt >= qend[hr]) pv = 0.f;
            s[idx] = pv;
          }
        }
      }
      // dV += P^T dO runs while dS^T is formed
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        uint32_t a[4];
        frag_a_from_acc(s, kk, a);
        wgmma_m64nXk16_bf16_rs<1>(dv, a, make_smem_desc_sw128(sdo + kk * 16 * 128, L::QB_CHUNK, 1024), 1u);
      }
      wgmma_commit();
      wgmma_wait<1>();
      fence_regs(dp);
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
        for (int e1 = 0; e1 < 2; ++e1) {
          const float dl = stat[BQB + 8 * jj + 2 * q + e1];
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            const int idx = 4 * jj + 2 * hr + e1;
            dp[idx] = s[idx] * (dp[idx] - dl);
          }
        }
      }
    } else {
    wgmma_wait<0>();
    fence_regs(s);
    fence_regs(dp);
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
      for (int e1 = 0; e1 < 2; ++e1) {
        const int qt = 8 * jj + 2 * q + e1;
        const float L2 = __ldg(lse_bh + i * BQB + qt) * 1.4426950408889634f;
        const float dl = __ldg(delta_bh + i * BQB + qt);
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int idx = 4 * jj + 2 * hr + e1;
          float pv = exp2f(s[idx] * p.scale_log2 - L2);
          if (masked && i * BQB + qt < j * BKV + wg * 64 + r0 + 8 * hr) pv = 0.f;
          if (dmask && i * BQB + qt >= qend[hr]) pv = 0.f;
          s[idx] = pv;
          dp[idx] = pv * (dp[idx] - dl);
        }
      }
    }
    }
    // dS^T -> smem: element (kv row r, query column c) at byte r * 128 + 2c of the SW128 tile (16-byte chunk index XOR r % 8)
    if (HD == 64 && (threadIdx.x & 127) == 0) bulk_wait_group_read<0>();   // the last dQ reduce has read its partial
    named_bar_sync(1 + wg, 128);   // this warpgroup's previous dQ MMA has finished reading the tile
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int r = r0 + 8 * hr;
        const uint32_t byte = r * 128 + (8 * jj + 2 * q) * 2;
        *reinterpret_cast<uint32_t*>(ds_tile + (byte ^ ((r & 7) << 4))) = pack_bf16x2(dp[4 * jj + 2 * hr], dp[4 * jj + 2 * hr + 1]);
      }
    }
    fence_proxy_async();
    named_bar_sync(1 + wg, 128);
    wgmma_fence();
    // dO / Q MN-major: LBO = the next 64-column chunk (the field is unused at N = 64)
    if constexpr (HD == 128) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t a[4];
      frag_a_from_acc(s, kk, a);
      wgmma_m64nXk16_bf16_rs<1>(dv, a, make_smem_desc_sw128(sdo + kk * 16 * 128, L::QB_CHUNK, 1024), 1u);
    }
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t a[4];
      frag_a_from_acc(dp, kk, a);
      wgmma_m64nXk16_bf16_rs<1>(dk, a, make_smem_desc_sw128(sq + kk * 16 * 128, L::QB_CHUNK, 1024), 1u);
    }
#pragma unroll
    for (int n = 0; n < NC; ++n) {   // dQ columns [64 n, 64 n + 64); the first half shares the dV / dK commit group
      float dq[32];
      if (n > 0) wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
        wgmma_m64n64k16_bf16_ss<1, 1>(dq, make_smem_desc_sw128(sds + kk * 16 * 128, 8192, 1024),
                                      make_smem_desc_sw128(sk + n * CHUNK + kk * 16 * 128, 8192, 1024), kk > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      if (n == 0) {
        fence_regs(dv);
        fence_regs(dk);
      }
      fence_regs(dq);
      if (n == 0 && (threadIdx.x & 127) == 0) mbar_arrive(&q_empty[st]);
      if constexpr (HD == 64) {
        // the warpgroup's [64 q x 64] partial -> smem (8-column groups XOR row % 4: conflict-free float2 stores), one bulk
        // reduce-add of the contiguous 16 KB block into dq_acc [B, H, S, 64]
        float* dq_tile = reinterpret_cast<float*>(smem + L::SB_DQ + wg * L::DQ_BYTES);
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int r = r0 + 8 * hr;
#pragma unroll
          for (int jj = 0; jj < 8; ++jj)
            *reinterpret_cast<float2*>(dq_tile + r * 64 + 8 * (jj ^ (r & 3)) + 2 * q) =
                make_float2(dq[4 * jj + 2 * hr] * p.scale, dq[4 * jj + 2 * hr + 1] * p.scale);
        }
        fence_proxy_async();
        named_bar_sync(1 + wg, 128);
        if ((threadIdx.x & 127) == 0) {
          bulk_reduce_add_f32(p.dq_acc + (((size_t)b * p.H + h) * p.S + i * BQB) * 64, dq_tile, L::DQ_BYTES);
          bulk_commit_group();
        }
      } else {
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int row = i * BQB + r0 + 8 * hr;
        float* dqp = p.dq_acc + (((size_t)b * p.S + row) * p.H + h) * HD + n * 64;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
          asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dqp + 8 * jj + 2 * q), "f"(dq[4 * jj + 2 * hr] * p.scale),
                       "f"(dq[4 * jj + 2 * hr + 1] * p.scale)
                       : "memory");
      }
      }
    }
  }
  pdl_trigger();
  if (HD == 64 && (threadIdx.x & 127) == 0) bulk_wait_group<0>();   // the dQ partials live until the last reduce is done
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int row = j * BKV + wg * 64 + r0 + 8 * hr;
    const size_t off = (size_t)b * p.dstride_b + (size_t)row * p.dstride_s + (size_t)h * p.dstride_h;
    __nv_bfloat16* dkp = reinterpret_cast<__nv_bfloat16*>(p.dk) + off;
    __nv_bfloat16* dvp = reinterpret_cast<__nv_bfloat16*>(p.dv) + off;
#pragma unroll
    for (int jj = 0; jj < HD / 8; ++jj) {
      *reinterpret_cast<uint32_t*>(dkp + 8 * jj + 2 * q) = pack_bf16x2(dk[4 * jj + 2 * hr] * p.scale, dk[4 * jj + 2 * hr + 1] * p.scale);
      *reinterpret_cast<uint32_t*>(dvp + 8 * jj + 2 * q) = pack_bf16x2(dv[4 * jj + 2 * hr], dv[4 * jj + 2 * hr + 1]);
    }
  }
}

// delta[b,h,s] = sum_d dO * O ; HD / 8 lanes per (b, s, h) row (one 16-byte load per lane and tensor).
template <int HD>
__global__ void attn_delta_kernel(const __nv_bfloat16* __restrict__ dO, const __nv_bfloat16* __restrict__ O,
                                  float* __restrict__ delta, int B, int S, int H) {
  constexpr int LANES = HD / 8, LANES_LOG2 = HD == 64 ? 3 : 4;
  static_assert(LANES == 1 << LANES_LOG2, "HD = 64 or 128");
  const long long gid = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long row = gid >> LANES_LOG2;
  const int sub = (int)(gid & (LANES - 1));
  pdl_wait();
  if (row >= (long long)B * S * H) return;
  const int hh = row % H, s = (row / H) % S, bb = row / ((long long)H * S);
  const uint4 a = __ldg(reinterpret_cast<const uint4*>(dO + row * HD) + sub);
  const uint4 c = __ldg(reinterpret_cast<const uint4*>(O + row * HD) + sub);
  const __nv_bfloat162* ha = reinterpret_cast<const __nv_bfloat162*>(&a);
  const __nv_bfloat162* hc = reinterpret_cast<const __nv_bfloat162*>(&c);
  float v = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 fa = __bfloat1622float2(ha[i]), fc = __bfloat1622float2(hc[i]);
    v += fa.x * fc.x + fa.y * fc.y;
  }
#pragma unroll
  for (int off = LANES / 2; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  if (sub == 0) delta[((size_t)bb * H + hh) * S + s] = v;
}

// dq (bf16, strided) = dq_acc, fp32 contiguous: [B, S, H, 128] at D = 128; [B, H, S, 64] at D = 64, with the 8-column
// groups of row s stored at group index (v ^ s % 4) (the layout the backward's bulk reduce-adds write).
// (the accumulator is zeroed again on the way out, so the persistent workspace never needs a separate memset)
template <int HD>
__global__ void attn_dq_cast_kernel(float* __restrict__ acc, __nv_bfloat16* __restrict__ dq, int B, int S, int H,
                                    long long sb, long long ss, long long sh) {
  const size_t n8 = (size_t)B * S * H * (HD / 8);
  pdl_wait();
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n8; i += (size_t)gridDim.x * blockDim.x) {
    const int v = i % (HD / 8);
    size_t r = i / (HD / 8);
    const int hh = r % H; r /= H;
    const int s = r % S;
    const int bb = r / S;
    const size_t a = HD == 64 ? (((size_t)bb * H + hh) * S + s) * 8 + (v ^ (s & 3)) : i;   // 8-float group in acc
    const float4 x = reinterpret_cast<const float4*>(acc)[a * 2], y = reinterpret_cast<const float4*>(acc)[a * 2 + 1];
    uint4 u;
    u.x = pack_bf16x2(x.x, x.y); u.y = pack_bf16x2(x.z, x.w); u.z = pack_bf16x2(y.x, y.y); u.w = pack_bf16x2(y.z, y.w);
    *reinterpret_cast<uint4*>(dq + (size_t)bb * sb + (size_t)s * ss + (size_t)hh * sh + v * 8) = u;
    reinterpret_cast<float4*>(acc)[a * 2] = make_float4(0.f, 0.f, 0.f, 0.f);
    reinterpret_cast<float4*>(acc)[a * 2 + 1] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);
EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) != cudaSuccess) return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

}  // namespace

// 4-D map over a [B, S, H, D]-addressable bf16 tensor given element strides; box = {64, box_rows, 1, 1}.
extern "C" int tepd_make_tmap_bshd(CUtensorMap* out, const void* ptr, int B, int S, int H, int D, long long stride_b,
                                   long long stride_s, long long stride_h, int box_rows) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return -1;
  cuuint64_t dims[4] = {(cuuint64_t)D, (cuuint64_t)S, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)stride_s * 2, (cuuint64_t)stride_h * 2, (cuuint64_t)stride_b * 2};
  cuuint32_t box[4] = {64, (cuuint32_t)box_rows, 1, 1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)r;
}

namespace {

template <auto Kern>
cudaError_t set_smem(int bytes) {   // once per kernel instantiation
  static bool cfg = false;
  if (!cfg) {
    cudaError_t e = cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) return e;
    cfg = true;
  }
  return cudaSuccess;
}

template <int HD>
int attn_fwd(const void* q, const void* k, const void* v, void* o, void* lse, int B, int H, int S, float scale, int causal,
             long long stride_b, long long stride_s, long long stride_h, const int* doc_start, cudaStream_t stream) {
  CUtensorMap tq, tk, tv;
  int rc = tepd_make_tmap_bshd(&tq, q, B, S, H, HD, stride_b, stride_s, stride_h, BQ);
  if (rc) return 100 + rc;
  rc = tepd_make_tmap_bshd(&tk, k, B, S, H, HD, stride_b, stride_s, stride_h, BKV);
  if (rc) return 200 + rc;
  rc = tepd_make_tmap_bshd(&tv, v, B, S, H, HD, stride_b, stride_s, stride_h, BKV);
  if (rc) return 300 + rc;
  auto kern = doc_start ? attn_fwd_kernel<HD, true> : attn_fwd_kernel<HD, false>;
  cudaError_t e = doc_start ? set_smem<attn_fwd_kernel<HD, true>>(FwdSmem<HD>::BYTES)
                            : set_smem<attn_fwd_kernel<HD, false>>(FwdSmem<HD>::BYTES);
  if (e != cudaSuccess) return (int)e;
  AttnFwdParams p;
  p.O = o; p.lse = (float*)lse; p.B = B; p.H = H; p.S = S; p.causal = causal;
  p.scale = scale; p.scale_log2 = scale * 1.4426950408889634f;
  p.doc_start = doc_start;
  return (int)tepd::launch(kern, dim3((S / BQ) * B * H), dim3(AttnCfg<HD>::THREADS), FwdSmem<HD>::BYTES, stream,
                           tq, tk, tv, p);
}

template <int HD>
int attn_bwd(const void* dO, const void* q, const void* k, const void* v, const void* o, const void* lse, float* delta,
             float* dq_acc, void* dq, void* dk, void* dv, int B, int H, int S, float scale, int causal, long long stride_b,
             long long stride_s, long long stride_h, long long dstride_b, long long dstride_s, long long dstride_h,
             const int* doc_start, cudaStream_t st) {
  CUtensorMap tq, tk, tv, tdo;
  int rc = tepd_make_tmap_bshd(&tq, q, B, S, H, HD, stride_b, stride_s, stride_h, BQB);
  if (rc) return 100 + rc;
  rc = tepd_make_tmap_bshd(&tk, k, B, S, H, HD, stride_b, stride_s, stride_h, BKV);
  if (rc) return 200 + rc;
  rc = tepd_make_tmap_bshd(&tv, v, B, S, H, HD, stride_b, stride_s, stride_h, BKV);
  if (rc) return 300 + rc;
  rc = tepd_make_tmap_bshd(&tdo, dO, B, S, H, HD, (long long)S * H * HD, (long long)H * HD, HD, BQB);
  if (rc) return 400 + rc;
  {
    const long long rows = (long long)B * S * H;
    cudaError_t le = tepd::launch(attn_delta_kernel<HD>, dim3((unsigned)((rows * (HD / 8) + 255) / 256)), dim3(256), 0, st,
                                  (const __nv_bfloat16*)dO, (const __nv_bfloat16*)o, delta, B, S, H);
    if (le != cudaSuccess) return (int)le;
  }
  auto kern = doc_start ? attn_bwd_kernel<HD, true> : attn_bwd_kernel<HD, false>;
  cudaError_t e = doc_start ? set_smem<attn_bwd_kernel<HD, true>>(BwdSmem<HD>::BYTES)
                            : set_smem<attn_bwd_kernel<HD, false>>(BwdSmem<HD>::BYTES);
  if (e != cudaSuccess) return (int)e;
  AttnBwdParams p;
  p.lse = (const float*)lse; p.delta = delta; p.dq_acc = dq_acc; p.dk = dk; p.dv = dv;
  p.dstride_b = dstride_b; p.dstride_s = dstride_s; p.dstride_h = dstride_h;
  p.B = B; p.H = H; p.S = S; p.causal = causal; p.scale = scale; p.scale_log2 = scale * 1.4426950408889634f;
  p.doc_start = doc_start;
  cudaError_t le = tepd::launch(kern, dim3((S / BKV) * B * H), dim3(AttnCfg<HD>::THREADS), BwdSmem<HD>::BYTES, st,
                                tq, tk, tv, tdo, p);
  if (le != cudaSuccess) return (int)le;
  return (int)tepd::launch(attn_dq_cast_kernel<HD>, dim3(tepd::num_sms() * 4), dim3(256), 0, st, dq_acc, (__nv_bfloat16*)dq, B, S,
                           H, dstride_b, dstride_s, dstride_h);
}

}  // namespace

// q, k, v: bf16 pointers addressed as [B, S, H, D] with the given element strides (shared by q/k/v).  D = 64 or 128.
// doc_start: nullptr, or int32 [B, S] non-decreasing document starts (causal only): query s sees keys [doc_start[b, s], s].
extern "C" int tepd_attn_fwd(const void* q, const void* k, const void* v, void* o, void* lse, int B, int H, int S, int D,
                             float scale, int causal, long long stride_b, long long stride_s, long long stride_h,
                             void* stream, const int* doc_start) {
  if (S % 128 != 0 || (doc_start && !causal)) return -2;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (D == 64) return attn_fwd<64>(q, k, v, o, lse, B, H, S, scale, causal, stride_b, stride_s, stride_h, doc_start, st);
  if (D == 128) return attn_fwd<128>(q, k, v, o, lse, B, H, S, scale, causal, stride_b, stride_s, stride_h, doc_start, st);
  return -2;
}

// do, o: contiguous [B,S,H,D]; q/k/v strided views; dq/dk/dv strided views (shared strides).  D = 64 or 128.
// lse: contiguous fp32 [B, H, S] (16-byte aligned at D = 64).  dq_acc: nullptr (a persistent, self-clearing workspace of the
// library's) or a zeroed fp32 buffer of B * S * H * D elements in the layout attn_dq_cast_kernel reads; left zeroed.
extern "C" int tepd_attn_bwd(const void* dO, const void* q, const void* k, const void* v, const void* o, const void* lse,
                             void* dq_acc, void* dq, void* dk, void* dv, int B, int H, int S, int D, float scale,
                             int causal, long long stride_b, long long stride_s, long long stride_h, long long dstride_b,
                             long long dstride_s, long long dstride_h, void* stream, const int* doc_start) {
  if ((D != 64 && D != 128) || S % 128 != 0 || (doc_start && !causal)) return -2;
  if (D == 64 && (reinterpret_cast<uintptr_t>(lse) & 15)) return -2;   // lse rows are bulk-copied (16-byte alignment)
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  static float* delta_buf = nullptr;
  static size_t delta_cap = 0;
  const size_t need = (size_t)B * H * S;
  if (need > delta_cap) {
    if (delta_buf) cudaFree(delta_buf);
    if (cudaMalloc(&delta_buf, need * sizeof(float)) != cudaSuccess) return -5;
    delta_cap = need;
  }
  // persistent, self-clearing fp32 dQ accumulator (used when the caller passes no buffer)
  static float* dq_ws = nullptr;
  static size_t dq_cap = 0;
  if (dq_acc == nullptr) {
    const size_t needq = (size_t)B * S * H * D;
    if (needq > dq_cap) {
      if (dq_ws) cudaFree(dq_ws);
      if (cudaMalloc(&dq_ws, needq * sizeof(float)) != cudaSuccess) return -6;
      cudaMemsetAsync(dq_ws, 0, needq * sizeof(float), st);
      dq_cap = needq;
    }
    dq_acc = dq_ws;
  }
  if (D == 64)
    return attn_bwd<64>(dO, q, k, v, o, lse, delta_buf, (float*)dq_acc, dq, dk, dv, B, H, S, scale, causal, stride_b, stride_s,
                        stride_h, dstride_b, dstride_s, dstride_h, doc_start, st);
  return attn_bwd<128>(dO, q, k, v, o, lse, delta_buf, (float*)dq_acc, dq, dk, dv, B, H, S, scale, causal, stride_b, stride_s,
                       stride_h, dstride_b, dstride_s, dstride_h, doc_start, st);
}
