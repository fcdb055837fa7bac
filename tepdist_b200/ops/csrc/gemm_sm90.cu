// Persistent warp-specialised GEMM for sm_90a: TMA -> smem (SWIZZLE_128B, multi-stage mbarrier ring) -> wgmma.mma_async
// into register accumulators of two consumer warpgroups -> epilogue from the accumulator fragments (bias / GELU /
// residual / fp32 split-K or stream-K reduction fused).  bf16 outputs, and the fp32 weight-gradient outputs, whose layout
// TMA can address go through a swizzled shared-memory staging buffer and TMA stores (or TMA reduce-adds) that overlap the
// next tile's MMAs; the other outputs are stored straight from the fragments.  Operands are bf16.  This is the
// device-op layer that replaces the reference's cuBLAS GemmThunk
// (reference: tensorflow/compiler/xla/service/gpu/gemm_thunk.cc, SURVEY §2.H K8).
//
//   D[b, M, N] = epilogue( alpha * A[b] (M x K)  *  B[b] (K x N) )
//
// Operand storage is described per operand by a "major" flag:
//   A K-major : memory [b, M, K] (K contiguous)       A MN-major: memory [b, K, M] (M contiguous)
//   B K-major : memory [b, N, K] (K contiguous)       B MN-major: memory [b, K, N] (N contiguous)
// which covers forward (x @ W^T), dgrad (dy @ W) and wgrad (dy^T @ x) without any transposes.
#include "sm90_ptx.cuh"
#include "launch.cuh"
#include <stdio.h>

using namespace sm90;

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;   // 64 bf16 = 128 B = one swizzle row
constexpr int NUM_THREADS = 384;  // warpgroups 0, 1: consumers (232 registers), warpgroup 2: TMA producer (40)
constexpr int CONSUMER_REGS = 232, PRODUCER_REGS = 40;   // 2 x 128 x 232 + 128 x 40 = 384 x 168, the launch allocation
constexpr int STORE_BOX = 64;     // TMA store box: 64 columns (128 B, one swizzle row) x 64 rows = 8 KB
constexpr int STORE_BOX_F32 = 32; // the same 8 KB box for fp32 outputs: 32 columns (128 B) x 64 rows

struct GemmParams {
  int M, N, K, batch;
  int m_blocks, n_blocks, k_blocks, split_k;
  long long ldd, stride_d;       // output leading dim / batch stride (elements)
  long long ld_res, stride_res;  // residual
  void* D;
  const void* bias;      // fp32 [N] or nullptr
  const void* residual;  // bf16 [b, M, N] or nullptr
  float alpha;
  int out_fp32;    // 0: bf16 output, 1: fp32 output
  int accumulate;  // 1: red.add into fp32 output (split-K / gradient accumulation)
  int act;         // 0 none, 1 tanh-GELU, 2 multiply by GELU'(aux)  (fused gelu backward on a dgrad GEMM)
  int bias_bf16;
  void* D2;        // act 1: when set, D receives the pre-activation and D2 the activated value (saved for backward)
  const void* aux; // act 2: bf16 [b, M, N] pre-activation
  int stream_k;    // > 0: stream-K -- CTA c owns the contiguous range [c, c+1) * stream_k of the (tile, k-block) iteration
                   // space and flushes its accumulator with red.add at every tile boundary (fp32 accumulate outputs only):
                   // every SM gets the same number of k-blocks whatever the tile count (no wave quantisation)
};

// One unit of work for a CTA: k-blocks [kb0, kb1) of output tile (m_blk, n_blk, b).  `lead` = this unit holds k-block 0
// (it adds bias / residual).  Data-parallel + split-K: cursor walks tile indices blockIdx.x, +gridDim.x, ...;
// stream-K: cursor walks this CTA's iteration range and a unit ends at the tile boundary or at the end of the range.
struct Work {
  int m_blk, n_blk, b, kb0, kb1;
  bool lead;
};
__device__ __forceinline__ void work_range(const GemmParams& p, int& cursor, int& end) {
  if (p.stream_k > 0) {
    const long long total = (long long)p.m_blocks * p.n_blocks * p.batch * p.k_blocks;
    const long long c0 = (long long)blockIdx.x * p.stream_k;
    cursor = (int)(c0 < total ? c0 : total);
    end = (int)(c0 + p.stream_k < total ? c0 + p.stream_k : total);
  } else {
    cursor = blockIdx.x;
    end = p.m_blocks * p.n_blocks * p.batch * p.split_k;
  }
}
__device__ __forceinline__ void next_work(const GemmParams& p, int& cursor, int end, Work& w) {
  int t;
  if (p.stream_k > 0) {
    t = cursor / p.k_blocks;
    w.kb0 = cursor - t * p.k_blocks;
    w.kb1 = min(p.k_blocks, w.kb0 + (end - cursor));
    w.lead = w.kb0 == 0;
    cursor += w.kb1 - w.kb0;
  } else {
    t = cursor;
    cursor += gridDim.x;
  }
  w.m_blk = t % p.m_blocks; t /= p.m_blocks;
  w.n_blk = t % p.n_blocks; t /= p.n_blocks;
  w.b = t % p.batch;
  if (p.stream_k <= 0) {
    const int split = t / p.batch;
    const int per = (p.k_blocks + p.split_k - 1) / p.split_k;
    w.kb0 = split * per;
    w.kb1 = min(p.k_blocks, w.kb0 + per);
    w.lead = split == 0;
  }
}

__device__ __forceinline__ float gelu_tanh_grad(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(k0 * (x + k1 * x * x * x)));
  return 0.5f * (1.0f + t) + 0.5f * x * (1.0f - t * t) * k0 * (1.0f + 3.0f * k1 * x * x);
}
__device__ __forceinline__ float gelu_tanh(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  float u = k0 * (x + k1 * x * x * x);
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(u));
  return 0.5f * x * (1.0f + t);
}

// Epilogue kinds, fixed at compile time.  EPI_DIRECT stores straight from the accumulator fragments and reads its options
// (bias, GELU, GELU', residual, fp32 store, red.add) at run time.  The other kinds write their output through a
// shared-memory staging buffer (one 64 x BLOCK_N bf16 buffer per consumer warpgroup, in the TMA store box layout) and TMA
// stores; their inputs are in shared memory before the epilogue starts: the bias (zeros when there is none) is
// copied there at the start of the tile, the residual / GELU' aux tile is TMA-loaded into the staging buffer itself.  The
// fp32 kinds fill the same buffer with half the tile's columns at a time (64 x BLOCK_N / 2 fp32) and store it in two rounds.
enum Epi : int {
  EPI_DIRECT = 0,
  EPI_PLAIN,       // alpha * acc
  EPI_BIAS,        // + bias
  EPI_BIAS_RES,    // + bias + residual
  EPI_GELU_DUAL,   // D = alpha * acc + bias, D2 = GELU(D)
  EPI_GELU_BWD,    // alpha * acc * GELU'(aux)
  EPI_F32,         // fp32 D = alpha * acc
  EPI_F32_ADD,     // fp32 D += alpha * acc (TMA reduce-add: split-K, stream-K and gradient accumulation)
};
template <int EPI> __host__ __device__ constexpr bool epi_bias() { return EPI == EPI_BIAS || EPI == EPI_BIAS_RES || EPI == EPI_GELU_DUAL; }
template <int EPI> __host__ __device__ constexpr bool epi_tile_in() { return EPI == EPI_BIAS_RES || EPI == EPI_GELU_BWD; }
template <int EPI> __host__ __device__ constexpr bool epi_f32() { return EPI == EPI_F32 || EPI == EPI_F32_ADD; }

// At BLOCK_N = 256 the 64 KB of staging cost one pipeline stage (3 x 48 KB + 64 KB + 2 KB of bias of the 227 KB).
template <int BLOCK_N, bool STAGED>
struct Cfg {
  static constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;
  static constexpr int B_BYTES = BLOCK_N * BLOCK_K * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = (BLOCK_N == 256) ? (STAGED ? 3 : 4) : 6;
  static constexpr int STAGING_WG_BYTES = STAGED ? 64 * BLOCK_N * 2 : 0;
  static constexpr int STAGING_OFF = STAGES * STAGE_BYTES;
  static constexpr int BIAS_OFF = STAGING_OFF + 2 * STAGING_WG_BYTES;   // fp32 [2][BLOCK_N]
  static constexpr int BAR_OFF = BIAS_OFF + (STAGED ? 2 * BLOCK_N * 4 : 0);
  static constexpr int SMEM_BYTES = BAR_OFF + 1024 /*align*/ + 256 /*barriers*/;
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory");
};

__device__ __forceinline__ void st_bf16x2(void* p, float a, float b) { *reinterpret_cast<uint32_t*>(p) = pack_bf16x2(a, b); }
__device__ __forceinline__ float2 ldg_bf16x2(const void* p) {
  return __bfloat1622float2(__ldg(reinterpret_cast<const __nv_bfloat162*>(p)));
}

// named barrier of one consumer warpgroup (ids 2, 3)
__device__ __forceinline__ void wg_bar_sync(int wg) {
  if (wg == 0) asm volatile("bar.sync 2, 128;" ::: "memory");
  else         asm volatile("bar.sync 3, 128;" ::: "memory");
}

// Epilogue math + store for two adjacent columns (col, col + 1) of one output row.  v0 / v1 already hold the scaled
// accumulator.  N % 8 == 0 and col is even, so col < N covers both columns.
__device__ __forceinline__ void epilogue_pair(float v0, float v1, const GemmParams& p, int row, int col, int b, bool add_bias,
                                              bool add_res) {
  if (add_bias) {
    if (p.bias_bf16) {
      const float2 f = ldg_bf16x2(reinterpret_cast<const __nv_bfloat16*>(p.bias) + col);
      v0 += f.x; v1 += f.y;
    } else {
      const float2 f = __ldg(reinterpret_cast<const float2*>(reinterpret_cast<const float*>(p.bias) + col));
      v0 += f.x; v1 += f.y;
    }
  }
  const long long off = (long long)b * p.stride_d + (long long)row * p.ldd + col;
  if (p.act == 1) {
    if (p.D2 != nullptr) st_bf16x2(reinterpret_cast<__nv_bfloat16*>(p.D) + off, v0, v1);  // pre-activation for backward
    v0 = gelu_tanh(v0); v1 = gelu_tanh(v1);
  } else if (p.act == 2) {
    const float2 f = ldg_bf16x2(reinterpret_cast<const __nv_bfloat16*>(p.aux) + off);
    v0 *= gelu_tanh_grad(f.x); v1 *= gelu_tanh_grad(f.y);
  }
  if (add_res) {
    const float2 f = ldg_bf16x2(reinterpret_cast<const __nv_bfloat16*>(p.residual) + (long long)b * p.stride_res +
                                (long long)row * p.ld_res + col);
    v0 += f.x; v1 += f.y;
  }
  if (!p.out_fp32) {
    __nv_bfloat16* dp = reinterpret_cast<__nv_bfloat16*>(p.D2 != nullptr && p.act == 1 ? p.D2 : p.D) + off;
    st_bf16x2(dp, v0, v1);
  } else if (!p.accumulate) {
    *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.D) + off) = make_float2(v0, v1);
  } else {
    float* dp = reinterpret_cast<float*>(p.D) + off;
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dp), "f"(v0), "f"(v1) : "memory");
  }
}

// One k-block (BLOCK_K = 128 bytes of K) of this warpgroup's 64 x BLOCK_N accumulator: four wgmma k-steps of 16 bf16
// (32 bytes of K), each one m64n256k16 (BLOCK_N = 256) or m64n128k16 (BLOCK_N = 128).  The B descriptor covers all
// BLOCK_N rows: K-major B rows follow each other in the swizzled tile (SBO), MN-major B is BLOCK_N / 64 chunks of 64
// columns LBO apart.
template <int BLOCK_N, bool A_MN, bool B_MN>
__device__ __forceinline__ void mma_kblock(float (&acc)[BLOCK_N / 2], uint32_t sa, uint32_t sb, int wg, bool first) {
  static_assert(BLOCK_N == 128 || BLOCK_N == 256, "tile width");
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    uint64_t da, db;
    if constexpr (!A_MN) da = make_smem_desc_sw128(sa + wg * 64 * 128 + k * 32, 0, 1024);
    else                 da = make_smem_desc_sw128(sa + wg * 64 * BLOCK_K * 2 + k * 16 * 128, 64 * BLOCK_K * 2, 1024);
    if constexpr (!B_MN) db = make_smem_desc_sw128(sb + k * 32, 0, 1024);
    else                 db = make_smem_desc_sw128(sb + k * 16 * 128, 64 * BLOCK_K * 2, 1024);
    const uint32_t scale_d = (first && k == 0) ? 0u : 1u;
    if constexpr (BLOCK_N == 256) wgmma_m64n256k16_bf16_ss<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, scale_d);
    else                          wgmma_m64n128k16_bf16_ss<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, scale_d);
  }
}

// Warp roles: warpgroups 0, 1 = consumers (wgmma into registers, rows [64 wg, +64) of the 128-row tile, then the
// epilogue); warpgroup 2 = TMA producer (one elected thread), which hands most of its registers to the consumers.
template <int BLOCK_N, bool A_MN, bool B_MN, int EPI>
__device__ __forceinline__ void gemm_body(const CUtensorMap& tmap_a, const CUtensorMap& tmap_b, const CUtensorMap& tmap_d,
                                          const CUtensorMap& tmap_d2, const CUtensorMap& tmap_in, const GemmParams& p) {
  constexpr bool STAGED = EPI != EPI_DIRECT;
  using C = Cfg<BLOCK_N, STAGED>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + C::BAR_OFF);
  uint64_t* empty_bar = full_bar + C::STAGES;
  uint64_t* in_bar = empty_bar + C::STAGES;   // [2]: residual / aux tile of consumer warpgroup 0 / 1 has landed

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if constexpr (STAGED) {
      tma_prefetch_desc(&tmap_d);
      if constexpr (EPI == EPI_GELU_DUAL) tma_prefetch_desc(&tmap_d2);
      if constexpr (epi_tile_in<EPI>()) tma_prefetch_desc(&tmap_in);
    }
    mbar_init(&in_bar[0], 1);
    mbar_init(&in_bar[1], 1);
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);   // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();      // everything above overlapped the previous kernel's tail; its outputs are visible from here on
  pdl_trigger();   // persistent grid: the next kernel may be scheduled as these CTAs retire

  if (warp >= 8) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == 8 && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      int cursor, cend;
      work_range(p, cursor, cend);
      while (cursor < cend) {
        Work w;
        next_work(p, cursor, cend, w);
        const int m_blk = w.m_blk, n_blk = w.n_blk;
        const int b = w.b, kb0 = w.kb0, kb1 = w.kb1;
        const int a_row = m_blk * BLOCK_M;
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * C::STAGE_BYTES;
          uint8_t* sb = sa + C::A_BYTES;
          mbar_expect_tx(&full_bar[stage], C::STAGE_BYTES);
          if constexpr (!A_MN) {
            tma_load_3d(sa, &tmap_a, &full_bar[stage], kb * BLOCK_K, a_row, b);
          } else {
#pragma unroll
            for (int j = 0; j < BLOCK_M / 64; ++j)
              tma_load_3d(sa + j * (64 * BLOCK_K * 2), &tmap_a, &full_bar[stage],
                          m_blk * BLOCK_M + j * 64, kb * BLOCK_K, b);
          }
          if constexpr (!B_MN) {
            tma_load_3d(sb, &tmap_b, &full_bar[stage], kb * BLOCK_K, n_blk * BLOCK_N, b);
          } else {
#pragma unroll
            for (int j = 0; j < BLOCK_N / 64; ++j)
              tma_load_3d(sb + j * (64 * BLOCK_K * 2), &tmap_b, &full_bar[stage],
                          n_blk * BLOCK_N + j * 64, kb * BLOCK_K, b);
          }
          if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }
  {
    // ===================== consumers: MMA + epilogue =====================
    setmaxnreg_inc<CONSUMER_REGS>();
    const int wg = warp >> 2;                 // rows [64 wg, 64 wg + 64) of the tile
    const int t128 = threadIdx.x & 127;
    const int g = lane >> 2, q = lane & 3;
    const int row_base = wg * 64 + (warp & 3) * 16 + g;   // + 8 for the second half of each fragment
    uint8_t* staging = smem + C::STAGING_OFF + wg * C::STAGING_WG_BYTES;
    float* sbias = reinterpret_cast<float*>(smem + C::BIAS_OFF) + wg * BLOCK_N;
    uint32_t in_phase = 0;
    int stage = 0;
    uint32_t phase = 0;
    int cursor, cend;
    work_range(p, cursor, cend);
    while (cursor < cend) {
      Work w;
      next_work(p, cursor, cend, w);
      const int m_blk = w.m_blk, n_blk = w.n_blk;
      const int b = w.b;
      const bool has_k = w.kb0 < w.kb1;
      if constexpr (STAGED) {
        // the previous tile's epilogue is done with the bias copy and the staging buffer (every thread of the warpgroup
        // passed its last barrier); once its TMA stores have read the buffer, the next input tile may land in it
        if constexpr (epi_bias<EPI>()) {
          for (int c = t128; c < BLOCK_N; c += 128) {
            const int col = n_blk * BLOCK_N + c;
            float v = 0.f;
            if (p.bias != nullptr && col < p.N)
              v = p.bias_bf16 ? __bfloat162float(__ldg(reinterpret_cast<const __nv_bfloat16*>(p.bias) + col))
                              : __ldg(reinterpret_cast<const float*>(p.bias) + col);
            sbias[c] = v;
          }
        }
        if (t128 == 0) {
          bulk_wait_group_read<0>();
          if constexpr (epi_tile_in<EPI>()) {
            mbar_expect_tx(&in_bar[wg], C::STAGING_WG_BYTES);
#pragma unroll
            for (int c = 0; c < BLOCK_N / STORE_BOX; ++c)
              tma_load_3d(staging + c * (64 * 128), &tmap_in, &in_bar[wg], n_blk * BLOCK_N + c * STORE_BOX,
                          m_blk * BLOCK_M + wg * 64, b);
          }
        }
      }
      float acc[BLOCK_N / 2];
      int prev = -1;
      for (int kb = w.kb0; kb < w.kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * C::STAGE_BYTES);
        wgmma_fence();
        mma_kblock<BLOCK_N, A_MN, B_MN>(acc, sa, sa + C::A_BYTES, wg, kb == w.kb0);
        wgmma_commit();
        wgmma_wait<1>();   // the previous k-block's MMAs have retired: its slot may be refilled
        if (prev >= 0 && t128 == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      fence_regs(acc);
      if (prev >= 0 && t128 == 0) mbar_arrive(&empty_bar[prev]);

      const bool add_bias = p.bias != nullptr && w.lead;
      const bool add_res = p.residual != nullptr && w.lead;
      if constexpr (STAGED) {
        // bf16 tile -> swizzled staging buffer (the TMA store box layout: 64-column boxes of 64 rows x 128 B, 16-byte
        // chunk c of row r at chunk c ^ (r & 7)) -> TMA stores.  A thread reads its residual / aux pair from the address it
        // then overwrites.  The stores drain while this warpgroup runs the next tile's MMAs.  Rows / columns outside the
        // output are not written here and clipped by the store.  The dual-output GELU epilogue stores D, then D2.  The
        // fp32 kinds store columns [0, BLOCK_N / 2) of the tile, then [BLOCK_N / 2, BLOCK_N), in 32-column boxes; the
        // accumulate kind adds each box into the output with a TMA reduce-add (a stream-K or split-K unit adds its partial).
        if constexpr (epi_tile_in<EPI>()) {
          mbar_wait(&in_bar[wg], in_phase);
          in_phase ^= 1;
        }
        wg_bar_sync(wg);   // the bias copy is visible
        if (has_k) {
#pragma unroll
          for (int r = 0; r < (EPI == EPI_GELU_DUAL || epi_f32<EPI>() ? 2 : 1); ++r) {
            if (r == 1) {
              if (t128 == 0) bulk_wait_group_read<0>();
              wg_bar_sync(wg);
            }
#pragma unroll
            for (int hr = 0; hr < 2; ++hr) {
              const int row_in_tile = row_base + hr * 8;
              if (m_blk * BLOCK_M + row_in_tile >= p.M) continue;
              const uint32_t srow = smem_u32(staging) + (row_in_tile - wg * 64) * 128;
              if constexpr (epi_f32<EPI>()) {
                // fragment column pair jj of this round: box jj / 4, 16-byte chunk 2 (jj & 3) + q / 2, 8 bytes in
#pragma unroll
                for (int jj = 0; jj < BLOCK_N / 16; ++jj) {
                  const int j = r * (BLOCK_N / 16) + jj;
                  if (n_blk * BLOCK_N + j * 8 + 2 * q >= p.N) continue;
                  const uint32_t addr = srow + (jj / 4) * (64 * 128) + ((((jj & 3) * 2 + (q >> 1)) ^ g) << 4) + 8 * (q & 1);
                  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(acc[4 * j + 2 * hr] * p.alpha),
                               "f"(acc[4 * j + 2 * hr + 1] * p.alpha));
                }
              } else {
#pragma unroll
                for (int j = 0; j < BLOCK_N / 8; ++j) {
                  const int cit = j * 8 + 2 * q;
                  if (n_blk * BLOCK_N + cit >= p.N) continue;
                  const uint32_t addr = srow + (j / 8) * (64 * 128) + (((j & 7) ^ g) << 4) + 4 * q;
                  float v0 = acc[4 * j + 2 * hr] * p.alpha, v1 = acc[4 * j + 2 * hr + 1] * p.alpha;
                  if constexpr (epi_bias<EPI>()) {
                    const float2 bb = *reinterpret_cast<const float2*>(sbias + cit);
                    v0 += bb.x; v1 += bb.y;
                  }
                  if constexpr (EPI == EPI_GELU_DUAL) {
                    if (r == 1) { v0 = gelu_tanh(v0); v1 = gelu_tanh(v1); }
                  }
                  if constexpr (epi_tile_in<EPI>()) {
                    uint32_t in;
                    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(in) : "r"(addr));
                    const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&in));
                    if constexpr (EPI == EPI_GELU_BWD) { v0 *= gelu_tanh_grad(f.x); v1 *= gelu_tanh_grad(f.y); }
                    else                               { v0 += f.x; v1 += f.y; }
                  }
                  asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(pack_bf16x2(v0, v1)));
                }
              }
            }
            fence_proxy_async();   // the generic-proxy writes above are read by the TMA unit
            wg_bar_sync(wg);
            if (t128 == 0) {
#pragma unroll
              for (int c = 0; c < BLOCK_N / STORE_BOX; ++c) {
                if constexpr (EPI == EPI_F32)
                  tma_store_3d(&tmap_d, staging + c * (64 * 128), n_blk * BLOCK_N + r * (BLOCK_N / 2) + c * STORE_BOX_F32,
                               m_blk * BLOCK_M + wg * 64, b);
                else if constexpr (EPI == EPI_F32_ADD)
                  tma_reduce_add_3d(&tmap_d, staging + c * (64 * 128), n_blk * BLOCK_N + r * (BLOCK_N / 2) + c * STORE_BOX_F32,
                                    m_blk * BLOCK_M + wg * 64, b);
                else
                  tma_store_3d(r == 1 ? &tmap_d2 : &tmap_d, staging + c * (64 * 128), n_blk * BLOCK_N + c * STORE_BOX,
                               m_blk * BLOCK_M + wg * 64, b);
              }
              bulk_commit_group();
            }
          }
        }
        continue;
      }
      if (has_k) {
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int row = m_blk * BLOCK_M + row_base + hr * 8;
          if (row >= p.M) continue;
#pragma unroll
          for (int j = 0; j < BLOCK_N / 8; ++j) {
            const int col = n_blk * BLOCK_N + j * 8 + 2 * q;
            if (col >= p.N) continue;
            epilogue_pair(acc[4 * j + 2 * hr] * p.alpha, acc[4 * j + 2 * hr + 1] * p.alpha, p, row, col, b, add_bias, add_res);
          }
        }
      }
    }
    if constexpr (STAGED) {
      if (t128 == 0) bulk_wait_group<0>();   // the staging buffers live until the last stores have read them
    }
  }
}

template <int BLOCK_N, bool A_MN, bool B_MN, int EPI>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                 const __grid_constant__ CUtensorMap tmap_d, const __grid_constant__ CUtensorMap tmap_d2,
                 const __grid_constant__ CUtensorMap tmap_in, const GemmParams p) {
  gemm_body<BLOCK_N, A_MN, B_MN, EPI>(tmap_a, tmap_b, tmap_d, tmap_d2, tmap_in, p);
}

// ------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p) {
      fprintf(stderr, "[tepdist] cuTensorMapEncodeTiled unavailable\n");
      return nullptr;
    }
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

}  // namespace

// 3-D tensor map of 2-byte (bf16) or 4-byte (fp32) elements: dims (inner, rows, batch); box (box_inner, box_rows, 1);
// SWIZZLE_128B.
static int make_tmap_3d(CUtensorMap* out, CUtensorMapDataType dtype, int elem_bytes, const void* ptr, long long inner,
                        long long rows, long long batch, long long ld_elems, long long batch_stride_elems, int box_inner,
                        int box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return -1;
  cuuint64_t dims[3] = {(cuuint64_t)inner, (cuuint64_t)rows, (cuuint64_t)batch};
  cuuint64_t strides[2] = {(cuuint64_t)ld_elems * elem_bytes,
                           (cuuint64_t)(batch > 1 ? batch_stride_elems : rows * ld_elems) * elem_bytes};
  cuuint32_t box[3] = {(cuuint32_t)box_inner, (cuuint32_t)box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(out, dtype, 3, const_cast<void*>(ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)r;
}

extern "C" int tepd_make_tmap_bf16_3d(CUtensorMap* out, const void* ptr, long long inner, long long rows,
                                      long long batch, long long ld_elems, long long batch_stride_elems,
                                      int box_inner, int box_rows) {
  return make_tmap_3d(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, ptr, inner, rows, batch, ld_elems, batch_stride_elems,
                      box_inner, box_rows);
}

struct Maps { CUtensorMap a, b, d, d2, in; };

template <int BLOCK_N, bool A_MN, bool B_MN, int EPI>
static int launch_gemm(const Maps& m, const GemmParams& p, int num_sms, cudaStream_t stream) {
  using C = Cfg<BLOCK_N, EPI != EPI_DIRECT>;
  auto kern = gemm_bf16_kernel<BLOCK_N, A_MN, B_MN, EPI>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    if (e != cudaSuccess) return (int)e;
    configured = true;
  }
  int total = p.m_blocks * p.n_blocks * p.batch * p.split_k;
  int grid = total < num_sms ? total : num_sms;
  if (p.stream_k > 0) {
    const long long iters = (long long)p.m_blocks * p.n_blocks * p.batch * p.k_blocks;
    grid = (int)((iters + p.stream_k - 1) / p.stream_k);
  }
  return (int)tepd::launch(kern, dim3(grid), dim3(NUM_THREADS), C::SMEM_BYTES, stream, m.a, m.b, m.d, m.d2, m.in, p);
}

// C ABI entry (called from Python via ctypes).  All leading dims / strides are in elements.
extern "C" int tepd_gemm_bf16(const void* A, const void* B, void* D, const void* bias, const void* residual,
                              int M, int N, int K, int batch, long long lda, long long ldb, long long ldd,
                              long long stride_a, long long stride_b, long long stride_d, long long ld_res,
                              long long stride_res, int a_mn, int b_mn, int out_fp32, int accumulate, int act,
                              int bias_bf16, float alpha, int split_k, int block_n, int num_sms, void* stream, void* D2,
                              const void* aux) {
  // K % 8 is a TMA row-pitch requirement of K-major operands only (MN-major operands have K as the outer dimension)
  if (N % 8 != 0 || M <= 0 || (K % 8 != 0 && !(a_mn && b_mn))) return -2;
  if ((D2 || aux) && out_fp32) return -5;
  if ((a_mn && (M % 8)) || (accumulate && !out_fp32)) return -3;
  GemmParams p;
  p.M = M; p.N = N; p.K = K; p.batch = batch;
  if (block_n != 128 && block_n != 256) block_n = (N % 256 == 0 || N > 1024) ? 256 : 128;
  p.m_blocks = (M + BLOCK_M - 1) / BLOCK_M;
  p.n_blocks = (N + block_n - 1) / block_n;
  p.k_blocks = (K + BLOCK_K - 1) / BLOCK_K;
  p.stream_k = 0;
  if (num_sms <= 0) num_sms = tepd::num_sms();
  if (split_k < 0) {  // stream-K requested: equal k-block ranges per SM
    // a unit that ends mid-tile adds its partial into the output, so only an accumulating fp32 output can take it
    if (!(out_fp32 && accumulate)) return -4;
    const long long iters = (long long)p.m_blocks * p.n_blocks * batch * p.k_blocks;
    long long per = (iters + num_sms - 1) / num_sms;
    if (per < 4) per = 4;   // do not shred tiny problems into sub-4-k-block units
    p.stream_k = (int)per;
    split_k = 1;
  }
  if (split_k < 1) split_k = 1;
  if (split_k > p.k_blocks) split_k = p.k_blocks;
  if (split_k > 1) {
    // make every split non-empty
    int per = (p.k_blocks + split_k - 1) / split_k;
    split_k = (p.k_blocks + per - 1) / per;
    if (!(out_fp32 && accumulate)) return -4;
  }
  p.split_k = split_k;
  p.ldd = ldd; p.stride_d = stride_d; p.ld_res = ld_res; p.stride_res = stride_res;
  p.D = D; p.bias = bias; p.residual = residual; p.alpha = alpha;
  p.out_fp32 = out_fp32; p.accumulate = accumulate; p.act = act; p.bias_bf16 = bias_bf16;
  p.D2 = D2; p.aux = aux;

  CUtensorMap ta, tb;
  int rc;
  if (!a_mn) rc = tepd_make_tmap_bf16_3d(&ta, A, K, M, batch, lda, stride_a, BLOCK_K, BLOCK_M);
  else       rc = tepd_make_tmap_bf16_3d(&ta, A, M, K, batch, lda, stride_a, 64, BLOCK_K);
  if (rc) return 100 + rc;
  if (!b_mn) rc = tepd_make_tmap_bf16_3d(&tb, B, K, N, batch, ldb, stride_b, BLOCK_K, block_n);
  else       rc = tepd_make_tmap_bf16_3d(&tb, B, N, K, batch, ldb, stride_b, 64, BLOCK_K);
  if (rc) return 200 + rc;
  // Epilogue kind.  bf16 outputs go through shared memory and TMA when TMA can address the output and the residual / aux
  // (16-byte aligned base, row pitch and batch stride; aux and D2 share D's layout) and a staged kind exists for the
  // flags and the operand layout: plain for every layout, bias / bias + residual / dual GELU for the forward layout
  // (A and B K-major), GELU' for the data-gradient layout (B MN-major).  fp32 outputs of the weight-gradient layout (A and B
  // MN-major) without bias, residual or activation go through shared memory too: plain stores, or TMA reduce-adds for
  // accumulating outputs (split-K, stream-K, gradient accumulation).  Everything else stores from the fragments.
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  const bool fwd = !a_mn && !b_mn, dgrad = !a_mn && b_mn, wgrad = a_mn && b_mn;
  int epi = EPI_DIRECT;
  if (!out_fp32 && ldd % 8 == 0 && (batch == 1 || stride_d % 8 == 0) && al16(D)) {
    const bool res_ok = residual != nullptr && al16(residual) && ld_res % 8 == 0 && (batch == 1 || stride_res % 8 == 0);
    if (act == 0 && !bias && !residual) epi = EPI_PLAIN;
    else if (act == 0 && !residual && fwd) epi = EPI_BIAS;
    else if (act == 0 && res_ok && fwd) epi = EPI_BIAS_RES;
    else if (act == 1 && D2 && al16(D2) && !residual && fwd) epi = EPI_GELU_DUAL;
    else if (act == 2 && al16(aux) && !bias && !residual && dgrad) epi = EPI_GELU_BWD;
  }
  if (out_fp32 && wgrad && act == 0 && !bias && !residual && ldd % 4 == 0 && (batch == 1 || stride_d % 4 == 0) && al16(D))
    epi = accumulate ? EPI_F32_ADD : EPI_F32;
  Maps m;
  m.a = ta; m.b = tb;
  m.d = m.d2 = m.in = CUtensorMap{};
  if (epi == EPI_F32 || epi == EPI_F32_ADD) {
    rc = make_tmap_3d(&m.d, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, D, N, M, batch, ldd, stride_d, STORE_BOX_F32, 64);
    if (rc) return 300 + rc;
  } else if (epi != EPI_DIRECT) {
    rc = tepd_make_tmap_bf16_3d(&m.d, D, N, M, batch, ldd, stride_d, STORE_BOX, 64);
    if (!rc && epi == EPI_GELU_DUAL) rc = tepd_make_tmap_bf16_3d(&m.d2, D2, N, M, batch, ldd, stride_d, STORE_BOX, 64);
    if (!rc && epi == EPI_BIAS_RES) rc = tepd_make_tmap_bf16_3d(&m.in, residual, N, M, batch, ld_res, stride_res, STORE_BOX, 64);
    if (!rc && epi == EPI_GELU_BWD) rc = tepd_make_tmap_bf16_3d(&m.in, aux, N, M, batch, ldd, stride_d, STORE_BOX, 64);
    if (rc) return 300 + rc;
  }
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
#define LAYOUTS(BN, E)                                                         \
  if (!a_mn && !b_mn) return launch_gemm<BN, false, false, E>(m, p, num_sms, s); \
  if (!a_mn && b_mn) return launch_gemm<BN, false, true, E>(m, p, num_sms, s);   \
  if (a_mn && !b_mn) return launch_gemm<BN, true, false, E>(m, p, num_sms, s);   \
  return launch_gemm<BN, true, true, E>(m, p, num_sms, s);
#define KINDS(BN)                                                                                  \
  switch (epi) {                                                                                   \
    case EPI_PLAIN: { LAYOUTS(BN, EPI_PLAIN) }                                                     \
    case EPI_BIAS: return launch_gemm<BN, false, false, EPI_BIAS>(m, p, num_sms, s);               \
    case EPI_BIAS_RES: return launch_gemm<BN, false, false, EPI_BIAS_RES>(m, p, num_sms, s);       \
    case EPI_GELU_DUAL: return launch_gemm<BN, false, false, EPI_GELU_DUAL>(m, p, num_sms, s);     \
    case EPI_GELU_BWD: return launch_gemm<BN, false, true, EPI_GELU_BWD>(m, p, num_sms, s);        \
    case EPI_F32: return launch_gemm<BN, true, true, EPI_F32>(m, p, num_sms, s);                   \
    case EPI_F32_ADD: return launch_gemm<BN, true, true, EPI_F32_ADD>(m, p, num_sms, s);           \
    default: { LAYOUTS(BN, EPI_DIRECT) }                                                           \
  }
  if (block_n == 256) { KINDS(256) } else { KINDS(128) }
#undef KINDS
#undef LAYOUTS
}
