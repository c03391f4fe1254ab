// Persistent warp-specialised bf16 GEMM for sm_90a: TMA -> smem ring -> wgmma (register accumulators) -> fused epilogue
// -> shared-memory staging -> TMA store.
//
// One kernel covers every dense contraction on the dual-encoder path:
//   forward linears   y = x W^T      A K-major [M,K],  B K-major [N,K]      (torch/nn/functional.py:6478,6690;
//                                                                            torch/nn/modules/transformer.py:980-982)
//   dgrad             dx = dy W      A K-major [M,N'], B MN-major [N',K']
//   wgrad             dW = dy^T x    A MN-major [tokens,N'], B MN-major [tokens,K']   (split-K, fp32 partials)
//   logits            a b^T * T      (modules/losses/contrastive_loss_with_temperature.py:90-95)
//
// Tile: BLOCK_M=128 x BLOCK_N=256 x BLOCK_K=64 per CTA, 4-stage smem ring (16 KB A + 32 KB B = 48 KB per stage).  Warp
// roles: warpgroup 0 = TMA producer (one elected thread; setmaxnreg drops it to 40 registers), warpgroups 1 and 2 =
// consumers (raised to 232 registers), each owning 64 rows of the tile (wgmma m64n256k16, 128 fp32 accumulator
// registers per thread) and running the epilogue of its rows.  While the consumers run an epilogue the producer is
// already filling the ring with the next tile's k-blocks.
// Epilogue: each consumer warpgroup converts its 64 x 256 accumulator chunk by chunk (64 bf16 or 32 fp32 columns =
// 128-byte rows) into one of its two 8 KB 128B-swizzled staging buffers, and one thread issues a TMA store (or, for an
// fp32 D += result, a TMA reduce-add) of the chunk.  A buffer is reused as soon as the store has READ it; the global
// writes drain while the warpgroup goes on.  EPI_BF16_DACT brings its pre-activation chunks into the same buffers by
// TMA (the first two are issued before the tile's main loop).  An fp32 output that TMA cannot address (base not
// 16-byte aligned) is written with direct stores instead.
// Shared memory: 4 x 48 KB ring + 32 KB staging + barriers = 225.3 KB of the 227 KB a block may use.  Four stages keep
// about 4 us of operands in flight per CTA at the measured rate (DESIGN.md §9); a 3-stage ring would free room for
// more staging but has not been measured.  ptxas: no spills except a few epilogue words in the DACT and CE_STATS
// instantiations (tests/test_gemm_sass_cpu.py).
// Cluster mode (CLU): two CTAs of a cluster compute a 256 x 256 tile; each loads its own 128 rows of A and HALF of
// the B tile, multicast into both CTAs' shared memory, which halves the L2 -> SM traffic for B.
#include "common.cuh"
#include "mmb200_internal.h"
#include <stdlib.h>
#include <mutex>

namespace mmb {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_N = 256;
constexpr int BLOCK_K = 64;
constexpr int WG_K = 16;
constexpr int STAGES = 4;
constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;   // 16 KB
constexpr int B_BYTES = BLOCK_N * BLOCK_K * 2;   // 32 KB
constexpr int GEMM_THREADS = 384;
constexpr int STG_BYTES = 64 * 128;             // one staging chunk: 64 rows x 128 B (64 bf16 / 32 fp32 columns)
constexpr int EPI_SMEM = 4 * STG_BYTES;         // two chunks per consumer warpgroup
constexpr int GEMM_SMEM_BYTES = 1024 /*align slack*/ + STAGES * (A_BYTES + B_BYTES) + EPI_SMEM + 256 /*barriers*/;
static_assert(GEMM_SMEM_BYTES <= 227 * 1024, "H100: at most 227 KB of shared memory per block");

struct GemmArgs {
  int M, N, K;
  int m_tiles, n_tiles, splits, kb_total, kb_per_split;
  float alpha;
  const float* bias;          // [N] fp32 or nullptr
  const __nv_bfloat16* aux;   // EPI_DACT: pre-activation [M, ld_aux]
  long long ld_aux;
  void* d0; void* d1;
  long long ldd0, ldd1;
  float* colsum_part;         // bf16 epilogues (not ACT), or nullptr: [ceil(M/128)][N] column sums of bf16(D0) per
                              // 128-row block; the host adds them into colsum[n] in block order (bias gradient)
  float* splitk_ws;           // fp32 epilogue with split-K: [splits][ws_rows][N] partial products, reduced in split order
  int ws_rows;                // rows per split in splitk_ws (M rounded up to whole tiles)
  int accumulate;             // fp32 epilogue without split-K: D0 += result (one writer per element)
  int f32_direct;             // fp32 epilogue without split-K whose D0 cannot take TMA stores: direct stores
  // ---- temperature-scaled cross-entropy epilogues (EPI_CE_STATS / EPI_CE_GRAD): logits = exp(*ce_log_scale) * acc
  // are consumed in registers and never written to HBM (contrastive_loss_with_temperature.py:90-107)
  const float* ce_log_scale;  // device scalar (logit_scale parameter)
  int ce_label0;              // the label column of output row r is ce_label0 + r in THIS launch's column space
  const int* ce_labels;       // CE_STATS, optional: explicit label column per row (any out-of-range value = none here)
  int ce_n_total;             // columns of the whole logits row (all launches), for the smoothing term eps / N
  float ce_smoothing;
  float ce_gs;                // CE_GRAD: loss_weight / rows (row scale when there are no row weights)
  float ce_loss_weight;
  const float* ce_lse_row;    // CE_GRAD: [M] row log-sum-exp (natural log)
  const float* ce_row_w;      // CE_GRAD: [M] masked-mean row weights or nullptr
  const float* ce_lse_col;    // CE_GRAD: [N] row-LSE of the other direction's global row j (transposed term) or nullptr
  const float* ce_col_w;      // CE_GRAD: [N] weights of those rows or nullptr
  int ce_col_lo, ce_col_hi;   // CE_GRAD: columns that receive the transposed term
  float4* ce_part;            // CE_STATS: [M][ce_part_ld] partial (max, sum e^(x-max), sum e^(x-max) x, sum x) per 128
  int ce_part_ld, ce_part0;   // CE_STATS: row pitch (in float4) and first part index of this launch     columns
  float* ce_xlabel;           // CE_STATS: [M] logit at the label column
};

// named barrier of one consumer warpgroup (ids 2, 3; id 1 spans both consumer warpgroups)
__device__ __forceinline__ void wg_bar_sync(int cw) { asm volatile("bar.sync %0, 128;" ::"r"(2 + cw) : "memory"); }

// tmC0: the output D0 (bf16 epilogues), the split-K workspace or D0 (fp32); tmC1: D1 (EPI_BF16_ACT) or the
// pre-activation aux (EPI_BF16_DACT).  Both are 128B-swizzled with a 64-row x 128-byte box.
template <bool A_MN, bool B_MN, int EPI, int ACT, bool CLU>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
            const __grid_constant__ CUtensorMap tmC0, const __grid_constant__ CUtensorMap tmC1, const GemmArgs p) {
  extern __shared__ uint8_t smem_raw[];
  // 1024 B alignment for the 128B-swizzle atoms (identical offset in both CTAs of a cluster: the multicast target)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * A_BYTES;
  uint8_t* sStg = smem + STAGES * (A_BYTES + B_BYTES);                                      // [2 wg][2][STG_BYTES]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sStg + EPI_SMEM);                        // [STAGES]
  uint64_t* empty_bar = full_bar + STAGES;                                                  // [STAGES]
  uint64_t* aux_bar = empty_bar + STAGES;                                                   // [2 wg][2]
  constexpr int TILE_M = CLU ? 2 * BLOCK_M : BLOCK_M;
  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], CLU ? 4 : 2);   // one arrive per consumer warpgroup (of both CTAs of a cluster)
    }
    for (int i = 0; i < 4; ++i) mbar_init(&aux_bar[i], 1);
    fence_mbar_init();
  }
  if (CLU) cluster_sync_all(); else __syncthreads();

  // tile schedule, computed in each role after setmaxnreg (a value live across the reallocation gets spilled)
#define MMB_TILE_SCHEDULE                                                      \
  const uint32_t rank = CLU ? cluster_ctarank() : 0u;                          \
  const int tiles_mn = p.m_tiles * p.n_tiles;                                  \
  const int total_tiles = tiles_mn * p.splits;                                 \
  const int tile_first = CLU ? (int)(blockIdx.x >> 1) : (int)blockIdx.x;       \
  const int tile_step = CLU ? (int)(gridDim.x >> 1) : (int)gridDim.x;

  if (wg == 0) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    MMB_TILE_SCHEDULE
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = tile_first; t < total_tiles; t += tile_step) {
        const int split = t / tiles_mn;
        const int rem = t - split * tiles_mn;
        const int m_blk = rem / p.n_tiles, n_blk = rem - m_blk * p.n_tiles;
        const int kb0 = split * p.kb_per_split;
        const int kb1 = min(kb0 + p.kb_per_split, p.kb_total);
        const int m_row = m_blk * TILE_M + (int)rank * BLOCK_M;
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait_quiet(&empty_bar[stage], phase ^ 1);
          // the B bytes of both CTAs' multicast halves land here too
          mbar_arrive_expect_tx(&full_bar[stage], A_BYTES + B_BYTES);
          uint8_t* a_dst = sA + stage * A_BYTES;
          uint8_t* b_dst = sB + stage * B_BYTES;
          if (!A_MN) {
            tma_load_2d(&tmA, &full_bar[stage], a_dst, kb * BLOCK_K, m_row);
          } else {
#pragma unroll
            for (int j = 0; j < BLOCK_M / 64; ++j)
              tma_load_2d(&tmA, &full_bar[stage], a_dst + j * (64 * BLOCK_K * 2), m_row + j * 64, kb * BLOCK_K);
          }
          // B: K-major -> rows [n0, n0 + 256) of [N][K]; MN-major -> four 64-column boxes of [K][N], 8 KB apart.
          // Either way 64 columns of the tile are 8 KB; a cluster CTA loads (and multicasts) the 16 KB half `rank`.
          const int n0 = n_blk * BLOCK_N;
          if (CLU) {
            const int h = (int)rank;
            if (!B_MN) {
              tma_load_2d_multicast(&tmB, &full_bar[stage], b_dst + h * 16384, kb * BLOCK_K, n0 + h * 128, 3);
            } else {
#pragma unroll
              for (int c = 2 * h; c < 2 * h + 2; ++c)
                tma_load_2d_multicast(&tmB, &full_bar[stage], b_dst + c * 8192, n0 + c * 64, kb * BLOCK_K, 3);
            }
          } else {
            if (!B_MN) {
              tma_load_2d(&tmB, &full_bar[stage], b_dst, kb * BLOCK_K, n0);
            } else {
#pragma unroll
              for (int c = 0; c < 4; ++c) tma_load_2d(&tmB, &full_bar[stage], b_dst + c * 8192, n0 + c * 64, kb * BLOCK_K);
            }
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== Consumers: wgmma main loop + epilogue =====================
    setmaxnreg_inc<232>();
    MMB_TILE_SCHEDULE
    const int cw = wg - 1;                       // 64-row half of the CTA's tile
    const int wq = (threadIdx.x >> 5) & 3;       // warp within the warpgroup: 16-row slice
    const int lane = threadIdx.x & 31;
    const int tq = lane & 3;
    const int rl = wq * 16 + (lane >> 2);        // this thread's first row within the warpgroup's 64 (second: +8)
    const bool elected = (threadIdx.x & 127) == 0;
    uint8_t* stg = sStg + cw * 2 * STG_BYTES;    // this warpgroup's two staging buffers
    // K-major SW128: 8-row groups 1024 B apart (SBO), LBO unused.  MN-major SW128: 64-element MN blocks (one TMA box,
    // BLOCK_K rows x 128 B) 8192 B apart (LBO); 8-row k groups 1024 B apart (SBO).
    constexpr uint32_t A_KSTEP = A_MN ? (WG_K / 8) * 1024 : WG_K * 2;   // bytes per k16 step
    constexpr uint32_t B_KSTEP = B_MN ? (WG_K / 8) * 1024 : WG_K * 2;
    constexpr uint32_t B_LBO = B_MN ? 64 * BLOCK_K * 2 : 16;
    int stage = 0;
    uint32_t phase = 0;
    uint32_t stg_next = 0;                       // staging buffer of the next stored chunk (alternates per store)
    uint32_t aux_phase = 0;                      // EPI_BF16_DACT: parity bit per staging buffer's load barrier
    float acc[128];
    for (int t = tile_first; t < total_tiles; t += tile_step) {
      const int split = t / tiles_mn;
      const int rem = t - split * tiles_mn;
      const int m_blk = rem / p.n_tiles, n_blk = rem - m_blk * p.n_tiles;
      const int kb0 = split * p.kb_per_split;
      const int kb1 = min(kb0 + p.kb_per_split, p.kb_total);
      const int row0 = m_blk * TILE_M + (int)rank * BLOCK_M + cw * 64;   // first row of this warpgroup
      const int col0 = n_blk * BLOCK_N;
      if (EPI == EPI_BF16_DACT && elected) {
        // the first two pre-activation chunks load during the main loop (the previous tile's stores have read both)
        tma_store_wait_read<0>();
#pragma unroll
        for (int b = 0; b < 2; ++b)
          if (col0 + 64 * b < p.N) {
            mbar_arrive_expect_tx(&aux_bar[2 * cw + b], STG_BYTES);
            tma_load_2d(&tmC1, &aux_bar[2 * cw + b], stg + b * STG_BYTES, col0 + 64 * b, row0);
          }
      }
      int prev_stage = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait_quiet(&full_bar[stage], phase);
        // this warpgroup's 64 rows of A: 64 K-major rows or one 64-wide MN box -- 8192 B in from the stage base either way
        const uint64_t adesc = make_smem_desc_sw128(smem_u32(sA + stage * A_BYTES + cw * 8192), 16, 1024);
        const uint64_t bdesc = make_smem_desc_sw128(smem_u32(sB + stage * B_BYTES), B_LBO, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / WG_K; ++k)
          wgmma_m64n256k16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, adesc + (uint64_t)((k * A_KSTEP) >> 4),
                                                      bdesc + (uint64_t)((k * B_KSTEP) >> 4), (kb > kb0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        // keep one k-block of MMAs in flight; the one before it has read its stage -> release that stage
        wgmma_wait<1>();
        if (prev_stage >= 0 && threadIdx.x % 128 == 0) {
          mbar_arrive(&empty_bar[prev_stage]);
          if (CLU) mbar_arrive_cluster(&empty_bar[prev_stage], rank ^ 1u);
        }
        prev_stage = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if (prev_stage >= 0 && threadIdx.x % 128 == 0) {
        mbar_arrive(&empty_bar[prev_stage]);
        if (CLU) mbar_arrive_cluster(&empty_bar[prev_stage], rank ^ 1u);
      }

      // ---------------- epilogue: rows r[0], r[1] of this thread, columns nq + 8j (+1) ----------------
      const int r[2] = {row0 + rl, row0 + rl + 8};
      const int nq = col0 + 2 * tq;
      const int n_left = p.N - nq;               // columns nq + c with c < n_left exist
      const bool add_bias = (p.bias != nullptr) && (split == 0);
      if (EPI == EPI_CE_STATS) {
        const float T = __expf(__ldg(p.ce_log_scale));
        const float T2 = T * 1.4426950408889634f;
        // one statistics part per 128 columns: the tile's columns j = 16h .. 16h + 15 form part h
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (col0 + 128 * h >= p.N) continue;
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const int lab = p.ce_labels ? __ldg(p.ce_labels + min(r[i], p.M - 1)) : p.ce_label0 + r[i];
            const int lab_off = r[i] < p.M ? lab - nq : -1;   // the label column's offset from nq (-1: none)
            float gm = -INFINITY;
#pragma unroll
            for (int j = 16 * h; j < 16 * h + 16; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e)
                if (8 * j + e < n_left) gm = fmaxf(gm, acc[4 * j + 2 * i + e]);
            float m2 = gm * T2, se = 0.f, sex = 0.f, sx = 0.f;
            if (gm > -INFINITY) {
#pragma unroll
              for (int j = 16 * h; j < 16 * h + 16; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  if (8 * j + e < n_left) {
                    const float a = acc[4 * j + 2 * i + e];
                    const float x = a * T;
                    const float pe = ex2_approx(fmaf(a, T2, -m2));
                    se += pe; sex = fmaf(pe, x, sex); sx += x;
                    if (8 * j + e == lab_off) p.ce_xlabel[r[i]] = x;
                  }
                }
            }
            // merge the four lanes of the quad (the row's 128 columns)
#pragma unroll
            for (int o = 1; o <= 2; o <<= 1) {
              const float mo = __shfl_xor_sync(0xffffffffu, m2, o);
              const float seo = __shfl_xor_sync(0xffffffffu, se, o);
              const float sexo = __shfl_xor_sync(0xffffffffu, sex, o);
              const float sxo = __shfl_xor_sync(0xffffffffu, sx, o);
              const float mn = fmaxf(m2, mo);
              const float f = (m2 == -INFINITY) ? 0.f : ex2_approx(m2 - mn);
              const float fo = (mo == -INFINITY) ? 0.f : ex2_approx(mo - mn);
              se = se * f + seo * fo; sex = sex * f + sexo * fo; sx += sxo; m2 = mn;
            }
            if (tq == 0 && r[i] < p.M)
              p.ce_part[(long long)r[i] * p.ce_part_ld + p.ce_part0 + 2 * n_blk + h] =
                  make_float4(m2 * 0.6931471805599453f, se, sex, sx);
          }
        }
      } else if (EPI == EPI_F32) {
        if (p.f32_direct) {
          float* D = reinterpret_cast<float*>(p.d0);
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const int n = nq + 8 * j;
            if (n >= p.N) continue;
            float b0 = 0.f, b1 = 0.f;
            if (add_bias) { b0 = __ldg(p.bias + n); b1 = __ldg(p.bias + n + 1); }
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              if (r[i] >= p.M) continue;
              const float v0 = fmaf(acc[4 * j + 2 * i], p.alpha, b0), v1 = fmaf(acc[4 * j + 2 * i + 1], p.alpha, b1);
              float* dst = D + (long long)r[i] * p.ldd0 + n;
              if (p.accumulate) { dst[0] += v0; dst[1] += v1; }
              else              { dst[0] = v0; dst[1] = v1; }
            }
          }
        } else {
          // eight chunks of 32 fp32 columns; 16-byte unit u of a 128-byte row sits at u ^ (row % 8) (SWIZZLE_128B)
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            if (col0 + 32 * q >= p.N) continue;
            uint8_t* buf = stg + (stg_next & 1u) * STG_BYTES;
            if (elected) tma_store_wait_read<1>();
            wg_bar_sync(cw);
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const int j = 4 * q + jj;
              const int n = nq + 8 * j;
              float b0 = 0.f, b1 = 0.f;
              if (add_bias && n < p.N) { b0 = __ldg(p.bias + n); b1 = __ldg(p.bias + n + 1); }
#pragma unroll
              for (int i = 0; i < 2; ++i) {
                const int rr = rl + 8 * i;
                float2* sp = reinterpret_cast<float2*>(buf + rr * 128 + (((2 * jj + (tq >> 1)) ^ (rr & 7)) << 4) + 8 * (tq & 1));
                *sp = make_float2(fmaf(acc[4 * j + 2 * i], p.alpha, b0), fmaf(acc[4 * j + 2 * i + 1], p.alpha, b1));
              }
            }
            fence_proxy_async_smem();
            wg_bar_sync(cw);
            if (elected) {
              if (p.splitk_ws)       tma_store_2d(&tmC0, buf, col0 + 32 * q, split * p.ws_rows + row0);
              else if (p.accumulate) tma_reduce_add_2d(&tmC0, buf, col0 + 32 * q, row0);
              else                   tma_store_2d(&tmC0, buf, col0 + 32 * q, row0);
              tma_store_commit();
            }
            ++stg_next;
          }
        }
      } else {
        // bf16 outputs.  EPI_CE_GRAD: per-row constants of this thread's two rows.
        float ce_T = 0.f, ce_T2 = 0.f, ce_eps_n = 0.f, ce_gcT = 0.f;
        float ce_lse2[2] = {0.f, 0.f}, ce_gsT[2] = {0.f, 0.f};
        if (EPI == EPI_CE_GRAD) {
          ce_T = __expf(__ldg(p.ce_log_scale));
          ce_T2 = ce_T * 1.4426950408889634f;
          ce_gcT = ce_T * p.ce_gs;
          ce_eps_n = p.ce_smoothing / (float)p.ce_n_total;
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const int gr = min(r[i], p.M - 1);
            ce_lse2[i] = __ldg(p.ce_lse_row + gr) * 1.4426950408889634f;
            ce_gsT[i] = ce_T * (p.ce_row_w ? p.ce_loss_weight * __ldg(p.ce_row_w + gr) : p.ce_gs);
          }
        }
        const bool do_colsum = (EPI == EPI_BF16 || EPI == EPI_BF16_DACT) && p.colsum_part != nullptr;
        // this warp's column sums over its 16 rows, column pair 8j + 2tq of j = 8q + lane / 4 kept by this lane
        float cs_keep[4][2];
        // EPI_BF16_ACT stores PRE in the first pass and act(PRE) (recomputed from the accumulators) in the second
        constexpr int PASSES = EPI == EPI_BF16_ACT ? 2 : 1;
#pragma unroll
        for (int ps = 0; ps < PASSES; ++ps) {
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            cs_keep[q][0] = cs_keep[q][1] = 0.f;
            if (col0 + 64 * q >= p.N) continue;
            // 64-column chunk q; 16-byte unit jj of a 128-byte row sits at jj ^ (row % 8) (SWIZZLE_128B)
            const uint32_t b = EPI == EPI_BF16_DACT ? (uint32_t)(q & 1) : (stg_next & 1u);
            uint8_t* buf = stg + b * STG_BYTES;
            if (EPI == EPI_BF16_DACT) {
              mbar_wait_quiet(&aux_bar[2 * cw + b], (aux_phase >> b) & 1u);
              aux_phase ^= 1u << b;
            } else {
              if (elected) tma_store_wait_read<1>();
              wg_bar_sync(cw);
            }
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const int j = 8 * q + jj;
              const int n = nq + 8 * j;
              const bool col_ok = n < p.N;
              float b0 = 0.f, b1 = 0.f;
              if (add_bias && col_ok) { b0 = __ldg(p.bias + n); b1 = __ldg(p.bias + n + 1); }
              float cs0 = 0.f, cs1 = 0.f;
#pragma unroll
              for (int i = 0; i < 2; ++i) {
                const int rr = rl + 8 * i;
                uint32_t* sp = reinterpret_cast<uint32_t*>(buf + rr * 128 + ((jj ^ (rr & 7)) << 4) + 4 * tq);
                float f0, f1;
                if (EPI == EPI_CE_GRAD) {
                  // d(loss_weight * mean CE) / d sims of this row block, plus (columns [col_lo, col_hi)) the transposed
                  // other-direction term rebuilt from the column LSEs -- see contrastive_ce_grad_kernel (loss.cu)
                  float f[2];
#pragma unroll
                  for (int e = 0; e < 2; ++e) {
                    const int c = n + e;
                    const float a = acc[4 * j + 2 * i + e];
                    const float tt = ((c == p.ce_label0 + r[i]) ? (1.f - p.ce_smoothing) : 0.f) + ce_eps_n;
                    float gsum = ce_gsT[i] * (ex2_approx(fmaf(a, ce_T2, -ce_lse2[i])) - tt);
                    if (p.ce_lse_col != nullptr && c >= p.ce_col_lo && c < p.ce_col_hi && c < p.N) {
                      const float wc = p.ce_col_w ? p.ce_loss_weight * ce_T * __ldg(p.ce_col_w + c) : ce_gcT;
                      if (wc != 0.f) gsum += wc * (ex2_approx(fmaf(a, ce_T2, -__ldg(p.ce_lse_col + c) * 1.4426950408889634f)) - tt);
                    }
                    f[e] = gsum;
                  }
                  f0 = f[0]; f1 = f[1];
                } else {
                  f0 = fmaf(acc[4 * j + 2 * i], p.alpha, b0);
                  f1 = fmaf(acc[4 * j + 2 * i + 1], p.alpha, b1);
                }
                if (EPI == EPI_BF16_DACT) {
                  const uint32_t av = *sp;   // pre-activation, loaded into this very slot by TMA
                  f0 = act_dgrad<ACT>(f0, bf16_lo(av));
                  f1 = act_dgrad<ACT>(f1, bf16_hi(av));
                }
                uint32_t o = pack_bf16x2(f0, f1);
                // the activation is applied to the bf16-ROUNDED pre-activation: exactly what the backward (which only
                // sees the stored bf16 pre-activation) differentiates
                if (EPI == EPI_BF16_ACT && ps == 1) o = pack_bf16x2(act_fn<ACT>(bf16_lo(o)), act_fn<ACT>(bf16_hi(o)));
                *sp = o;
                if (do_colsum && col_ok && r[i] < p.M) { cs0 += bf16_lo(o); cs1 += bf16_hi(o); }
              }
              if (do_colsum) {
                // column sums of the rounded output over the warp's 16 rows (lanes sharing tq)
#pragma unroll
                for (int o = 4; o <= 16; o <<= 1) {
                  cs0 += __shfl_xor_sync(0xffffffffu, cs0, o);
                  cs1 += __shfl_xor_sync(0xffffffffu, cs1, o);
                }
                if ((lane >> 2) == jj) { cs_keep[q][0] = cs0; cs_keep[q][1] = cs1; }
              }
            }
            fence_proxy_async_smem();
            wg_bar_sync(cw);
            if (elected) {
              tma_store_2d(EPI == EPI_BF16_ACT && ps == 1 ? &tmC1 : &tmC0, buf, col0 + 64 * q, row0);
              tma_store_commit();
              if (EPI == EPI_BF16_DACT && q + 2 < 4 && col0 + 64 * (q + 2) < p.N) {
                // this buffer's next pre-activation chunk, once the store has read it
                tma_store_wait_read<0>();
                mbar_arrive_expect_tx(&aux_bar[2 * cw + b], STG_BYTES);
                tma_load_2d(&tmC1, &aux_bar[2 * cw + b], buf, col0 + 64 * (q + 2), row0);
              }
            }
            if (EPI != EPI_BF16_DACT) ++stg_next;
          }
        }
        if (do_colsum) {
          // the 8 consumer warps' sums in warp order -> one partial row per 128-row block (no atomics: the host reduces
          // the blocks in order, so the result does not depend on which CTA finishes first).  The per-warp rows live
          // in the warpgroup's staging buffers, once their last store has read them.
          if (elected) tma_store_wait_read<0>();
          wg_bar_sync(cw);
          float* sCol = reinterpret_cast<float*>(stg) + wq * BLOCK_N;
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int c = 8 * (8 * q + (lane >> 2)) + 2 * tq;
            sCol[c] = cs_keep[q][0];
            sCol[c + 1] = cs_keep[q][1];
          }
          asm volatile("bar.sync 1, 256;" ::: "memory");
          const int ct = threadIdx.x - 128, blk_row = m_blk * TILE_M + (int)rank * BLOCK_M;
          if (blk_row < p.M && col0 + ct < p.N) {
            const float* all = reinterpret_cast<const float*>(sStg);
            float s = 0.f;
#pragma unroll
            for (int w = 0; w < 8; ++w) s += all[(w >> 2) * (2 * STG_BYTES / 4) + (w & 3) * BLOCK_N + ct];
            p.colsum_part[(long long)(blk_row / BLOCK_M) * p.N + col0 + ct] = s;
          }
          fence_proxy_async_smem();   // these generic reads come before the next TMA writes into the staging buffers
          asm volatile("bar.sync 1, 256;" ::: "memory");
        }
      }
    }
    // the global writes of the last stores complete before the CTA retires
    if (elected) tma_store_wait_all<0>();
  }
  // cluster: nobody exits while the peer may still multicast into it or arrive on its barriers
  if (CLU) cluster_sync_all();
}
#undef MMB_TILE_SCHEDULE

// ----------------------------------------------------------------------------------------------
// Host side
// ----------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess || !p)
      return nullptr;
    fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

// A tensor map is a pure function of (pointer, dims, pitch, box, dtype): the training step re-issues the same ~300
// GEMMs / attention launches on persistent workspaces every step, so the encoded descriptors are memoised (the
// driver call costs ~1-2 us each, 3-4 per launch).  Small direct-mapped cache; a miss simply re-encodes.
struct TmapKey {
  const void* ptr; uint64_t inner, outer, pitch; uint32_t box_inner, box_outer, kind;
  bool operator==(const TmapKey& o) const {
    return ptr == o.ptr && inner == o.inner && outer == o.outer && pitch == o.pitch && box_inner == o.box_inner &&
           box_outer == o.box_outer && kind == o.kind;
  }
};
struct TmapSlot { TmapKey key; CUtensorMap map; bool valid; };
constexpr int TMAP_CACHE_SLOTS = 4096;
static TmapSlot* g_tmap_cache = nullptr;
static std::mutex g_tmap_mu;

// 2-D row-major tensor [outer, inner] with row pitch `pitch_bytes`; box = [box_outer, box_inner]; 128B swizzle.
int make_tmap_2d(CUtensorMap* out, const void* ptr, int elem_bytes, bool is_f32, uint64_t inner, uint64_t outer,
                 uint64_t pitch_bytes, uint32_t box_inner, uint32_t box_outer) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return MMB_ERR_DRIVER;
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || (pitch_bytes & 15) || box_inner * elem_bytes != 128) return MMB_ERR_ARG;
  const TmapKey key{ptr, inner, outer, pitch_bytes, box_inner, box_outer, (uint32_t)(is_f32 ? 1 : 0)};
  uint64_t hsh = reinterpret_cast<uintptr_t>(ptr) * 0x9E3779B97F4A7C15ull;
  hsh ^= (inner * 0xC2B2AE3D27D4EB4Full) ^ (outer * 0x165667B19E3779F9ull) ^ (pitch_bytes << 17) ^
         ((uint64_t)box_outer << 40) ^ ((uint64_t)box_inner << 52) ^ key.kind;
  const int slot = (int)((hsh >> 20) % TMAP_CACHE_SLOTS);
  {
    std::lock_guard<std::mutex> lk(g_tmap_mu);
    if (!g_tmap_cache) g_tmap_cache = new TmapSlot[TMAP_CACHE_SLOTS]();
    if (g_tmap_cache[slot].valid && g_tmap_cache[slot].key == key) {
      *out = g_tmap_cache[slot].map;
      return MMB_OK;
    }
  }
  cuuint64_t gdim[2] = {inner, outer};
  cuuint64_t gstr[1] = {pitch_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, is_f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
                   const_cast<void*>(ptr), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return MMB_ERR_DRIVER;
  {
    std::lock_guard<std::mutex> lk(g_tmap_mu);
    g_tmap_cache[slot].key = key;
    g_tmap_cache[slot].map = *out;
    g_tmap_cache[slot].valid = true;
  }
  return MMB_OK;
}

// 3-D bf16 tensor [dim2, dim1, inner] (pitch1 / pitch2 in bytes), box = [1, box1, box_inner], 128B swizzle: a box never
// crosses a dim1 boundary, so per-batch row tiles are clipped at the sequence length (attention forward epilogue).
int make_tmap_3d_bf16(CUtensorMap* out, const void* ptr, uint64_t inner, uint64_t dim1, uint64_t dim2, uint64_t pitch1,
                      uint64_t pitch2, uint32_t box_inner, uint32_t box1) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return MMB_ERR_DRIVER;
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || (pitch1 & 15) || (pitch2 & 15) || box_inner * 2 != 128) return MMB_ERR_ARG;
  cuuint64_t gdim[3] = {inner, dim1, dim2};
  cuuint64_t gstr[2] = {pitch1, pitch2};
  cuuint32_t box[3] = {box_inner, box1, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(ptr), gdim, gstr, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? MMB_OK : MMB_ERR_DRIVER;
}

static int g_num_sms = 0;
int num_sms() {
  if (!g_num_sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
  }
  return g_num_sms;
}

template <bool A_MN, bool B_MN, int EPI, int ACT, bool CLU>
static int launch_impl(const CUtensorMap& tA, const CUtensorMap& tB, const CUtensorMap& tC0, const CUtensorMap& tC1,
                       const GemmArgs& args, cudaStream_t stream) {
  auto kfn = gemm_kernel<A_MN, B_MN, EPI, ACT, CLU>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM_BYTES);
    if (e != cudaSuccess) return (int)e;
    attr_set = true;
  }
  const int total = args.m_tiles * args.n_tiles * args.splits;
  cudaLaunchConfig_t cfg{};
  cudaLaunchAttribute attr[1];
  if (CLU) {
    const int clusters = total < num_sms() / 2 ? total : num_sms() / 2;
    cfg.gridDim = dim3(2 * clusters);
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
  } else {
    cfg.gridDim = dim3(total < num_sms() ? total : num_sms());
  }
  cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = GEMM_SMEM_BYTES;
  cfg.stream = stream;
  return (int)cudaLaunchKernelEx(&cfg, kfn, tA, tB, tC0, tC1, args);
}

}  // namespace mmb

using namespace mmb;

// Test / A-B hook: force the kernel variant mmb_gemm_bf16 dispatches to (process-wide).
//   cta2: -1 = automatic (size heuristic), 0 = one CTA per 128x256 tile, 1 = 2-CTA clusters (256x256 tiles, B multicast)
//   epilogue_warps: 0 or 8 (the two consumer warpgroups run the epilogue; kept for ABI compatibility)
static int g_force_cta2 = -1;
extern "C" int mmb_gemm_set_mode(int cta2, int epilogue_warps) {
  if (cta2 < -1 || cta2 > 1 || (epilogue_warps != 0 && epilogue_warps != 8)) return MMB_ERR_ARG;
  g_force_cta2 = cta2;
  return MMB_OK;
}

// D[m, n] = (accumulate ? D[m, n] : 0) + sum_{s = 0..S-1} ws[s][m][n], splits added in order (N % 4 == 0); a split
// holds ws_rows >= M rows
__global__ void splitk_reduce_kernel(const float* __restrict__ ws, int S, int M, int ws_rows, int N, float* __restrict__ D,
                                     long long ldd, int accumulate) {
  const int n = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (n >= N) return;
  for (int m = blockIdx.y; m < M; m += gridDim.y) {
    float* dst = D + (long long)m * ldd + n;
    float4 acc = accumulate ? make_float4(dst[0], dst[1], dst[2], dst[3]) : make_float4(0.f, 0.f, 0.f, 0.f);
    for (int s = 0; s < S; ++s) {
      const float4 v = *reinterpret_cast<const float4*>(ws + ((long long)s * ws_rows + m) * N + n);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    dst[0] = acc.x; dst[1] = acc.y; dst[2] = acc.z; dst[3] = acc.w;
  }
}

static int gemm_launch(int a_mn_major, int b_mn_major, int epilogue, int act, bool cta2, const CUtensorMap& tA,
                       const CUtensorMap& tB, const CUtensorMap& tC0, const CUtensorMap& tC1, const GemmArgs& g,
                       cudaStream_t stream);

static int gemm_dispatch(const void* A, long long lda, int a_mn_major, const void* B, long long ldb, int b_mn_major,
                         void* D0, long long ldd0, void* D1, long long ldd1, int M, int N, int K, int epilogue, int act,
                         float alpha, const float* bias, const void* aux, long long ld_aux, int splits, int accumulate,
                         float* colsum, const GemmArgs* ce, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0 || N <= 0 || K <= 0) return MMB_ERR_ARG;
  if ((epilogue == EPI_CE_STATS || epilogue == EPI_CE_GRAD) && (!ce || a_mn_major || b_mn_major)) return MMB_ERR_ARG;
  if ((lda & 7) || (ldb & 7)) return MMB_ERR_ARG;
  if (epilogue != EPI_CE_STATS && (epilogue == EPI_F32 ? (N & 3) : (N & 7))) return MMB_ERR_ARG;   // CE_STATS writes no tensor
  // only the fp32 epilogue adds into D0, and EPI_BF16_DACT takes no bias: refuse what the kernel would ignore
  if (accumulate && epilogue != EPI_F32) return MMB_ERR_ARG;
  if (bias && epilogue == EPI_BF16_DACT) return MMB_ERR_ARG;
  // 2-CTA clusters (256x256 tiles, B multicast) for everything large enough to fill the SM pairs at least once
  const long long big_tiles = (long long)((M + 2 * BLOCK_M - 1) / (2 * BLOCK_M)) * ((N + BLOCK_N - 1) / BLOCK_N);
  const bool cta2 = g_force_cta2 == 1 ||
                    (g_force_cta2 == -1 && M >= 512 && big_tiles * (splits < 1 ? 1 : splits) >= num_sms() / 2);
  GemmArgs g{};
  if (ce) g = *ce;   // cross-entropy epilogue parameters (the geometry fields below are overwritten)
  g.M = M; g.N = N; g.K = K;
  g.m_tiles = cta2 ? (M + 2 * BLOCK_M - 1) / (2 * BLOCK_M) : (M + BLOCK_M - 1) / BLOCK_M;
  g.n_tiles = (N + BLOCK_N - 1) / BLOCK_N;
  g.kb_total = (K + BLOCK_K - 1) / BLOCK_K;
  if (splits < 1) splits = 1;
  if (splits > g.kb_total) splits = g.kb_total;
  if (epilogue != EPI_F32) splits = 1;
  g.kb_per_split = (g.kb_total + splits - 1) / splits;
  g.splits = (g.kb_total + g.kb_per_split - 1) / g.kb_per_split;
  g.alpha = alpha;
  g.bias = bias;
  g.aux = reinterpret_cast<const __nv_bfloat16*>(aux);
  g.ld_aux = ld_aux;
  g.d0 = D0; g.d1 = D1; g.ldd0 = ldd0; g.ldd1 = ldd1;
  g.accumulate = accumulate ? 1 : 0;
  if (colsum && (epilogue == EPI_F32 || epilogue == EPI_BF16_ACT)) return MMB_ERR_ARG;
  const int col_blocks = (M + BLOCK_M - 1) / BLOCK_M;
  if (colsum) {
    g.colsum_part = static_cast<float*>(scratch(SCR_GEMM_COLSUM, (size_t)col_blocks * N * sizeof(float), stream));
    if (!g.colsum_part) return (int)cudaErrorMemoryAllocation;
  }
  if (epilogue == EPI_F32 && g.splits > 1) {
    g.ws_rows = g.m_tiles * (cta2 ? 2 * BLOCK_M : BLOCK_M);   // whole tiles: TMA stores need not clip inside a split
    g.splitk_ws = static_cast<float*>(scratch(SCR_GEMM_SPLITK, (size_t)g.splits * g.ws_rows * N * sizeof(float), stream));
    if (!g.splitk_ws) return (int)cudaErrorMemoryAllocation;
  }

  CUtensorMap tA, tB;
  int rc;
  // A: K-major -> global [M rows][K inner]; MN-major -> global [K rows][M inner]
  if (!a_mn_major) rc = make_tmap_2d(&tA, A, 2, false, K, M, lda * 2, 64, BLOCK_M);
  else             rc = make_tmap_2d(&tA, A, 2, false, M, K, lda * 2, 64, BLOCK_K);
  if (rc) return rc;
  // B: a cluster CTA loads (and multicasts) half of the 256-row tile
  if (!b_mn_major) rc = make_tmap_2d(&tB, B, 2, false, K, N, ldb * 2, 64, cta2 ? BLOCK_N / 2 : BLOCK_N);
  else             rc = make_tmap_2d(&tB, B, 2, false, N, K, ldb * 2, 64, BLOCK_K);
  if (rc) return rc;
  // epilogue tensor maps: 64-row x 128-byte boxes, clipped by TMA at M and N
  CUtensorMap tC0 = tA, tC1 = tA;   // unused ones stay a copy of tA and are never read
  if (epilogue == EPI_F32) {
    if (ldd0 & 3) return MMB_ERR_ARG;
    if (g.splitk_ws) {
      rc = make_tmap_2d(&tC0, g.splitk_ws, 4, true, N, (uint64_t)g.splits * g.ws_rows, (uint64_t)N * 4, 32, 64);
    } else if ((reinterpret_cast<uintptr_t>(D0) & 15) == 0 && (ldd0 & 3) == 0) {
      rc = make_tmap_2d(&tC0, D0, 4, true, N, M, ldd0 * 4, 32, 64);
    } else {
      g.f32_direct = 1;   // e.g. a column slice of an fp32 tensor: TMA needs a 16-byte aligned base
    }
    if (rc) return rc;
  } else if (epilogue != EPI_CE_STATS) {
    if ((ldd0 & 7) || (reinterpret_cast<uintptr_t>(D0) & 15)) return MMB_ERR_ARG;
    if (epilogue == EPI_BF16_ACT && (!D1 || (ldd1 & 7) || (reinterpret_cast<uintptr_t>(D1) & 15))) return MMB_ERR_ARG;
    if (epilogue == EPI_BF16_DACT && (!aux || (ld_aux & 7) || (reinterpret_cast<uintptr_t>(aux) & 15))) return MMB_ERR_ARG;
    rc = make_tmap_2d(&tC0, D0, 2, false, N, M, ldd0 * 2, 64, 64);
    if (!rc && epilogue == EPI_BF16_ACT) rc = make_tmap_2d(&tC1, D1, 2, false, N, M, ldd1 * 2, 64, 64);
    if (!rc && epilogue == EPI_BF16_DACT) rc = make_tmap_2d(&tC1, aux, 2, false, N, M, ld_aux * 2, 64, 64);
    if (rc) return rc;
  }

  int rc_launch = gemm_launch(a_mn_major, b_mn_major, epilogue, act, cta2, tA, tB, tC0, tC1, g, stream);
  if (rc_launch) return rc_launch;
  if (g.splitk_ws) {
    splitk_reduce_kernel<<<dim3((N / 4 + 127) / 128, M < 65535 ? M : 65535), 128, 0, stream>>>(
        g.splitk_ws, g.splits, M, g.ws_rows, N, reinterpret_cast<float*>(D0), ldd0, g.accumulate);
    rc_launch = (int)cudaGetLastError();
    if (rc_launch) return rc_launch;
  }
  if (colsum) return reduce_partials(g.colsum_part, col_blocks, N, N, colsum, 1, stream);
  return MMB_OK;
}

static int gemm_launch(int a_mn_major, int b_mn_major, int epilogue, int act, bool cta2, const CUtensorMap& tA,
                       const CUtensorMap& tB, const CUtensorMap& tC0, const CUtensorMap& tC1, const GemmArgs& g,
                       cudaStream_t stream) {
  const int am = a_mn_major ? 1 : 0, bm = b_mn_major ? 1 : 0;
  if (epilogue == EPI_CE_STATS)
    return cta2 ? launch_impl<false, false, EPI_CE_STATS, 0, true>(tA, tB, tC0, tC1, g, stream)
                : launch_impl<false, false, EPI_CE_STATS, 0, false>(tA, tB, tC0, tC1, g, stream);
  if (epilogue == EPI_CE_GRAD)
    return cta2 ? launch_impl<false, false, EPI_CE_GRAD, 0, true>(tA, tB, tC0, tC1, g, stream)
                : launch_impl<false, false, EPI_CE_GRAD, 0, false>(tA, tB, tC0, tC1, g, stream);
#define MMB_CASE(AM, BM, E, AC)                                                                                   \
  if (am == AM && bm == BM && epilogue == E && (AC < 0 || act == AC))                                             \
    return cta2 ? launch_impl<(AM != 0), (BM != 0), E, (AC < 0 ? 0 : AC), true>(tA, tB, tC0, tC1, g, stream)                \
                : launch_impl<(AM != 0), (BM != 0), E, (AC < 0 ? 0 : AC), false>(tA, tB, tC0, tC1, g, stream);
  MMB_CASE(0, 0, EPI_BF16, -1)
  MMB_CASE(0, 0, EPI_BF16_ACT, ACT_QUICK_GELU)
  MMB_CASE(0, 0, EPI_BF16_ACT, ACT_GELU_ERF)
  MMB_CASE(0, 0, EPI_BF16_ACT, ACT_RELU)
  MMB_CASE(0, 0, EPI_F32, -1)
  MMB_CASE(0, 1, EPI_BF16, -1)
  MMB_CASE(0, 1, EPI_BF16_DACT, ACT_QUICK_GELU)
  MMB_CASE(0, 1, EPI_BF16_DACT, ACT_GELU_ERF)
  MMB_CASE(0, 1, EPI_BF16_DACT, ACT_RELU)
  MMB_CASE(0, 1, EPI_F32, -1)
  MMB_CASE(1, 1, EPI_F32, -1)
  MMB_CASE(1, 0, EPI_F32, -1)
#undef MMB_CASE
  return MMB_ERR_UNSUPPORTED;
}
extern "C" int mmb_gemm_bf16(const void* A, long long lda, int a_mn_major, const void* B, long long ldb,
                             int b_mn_major, void* D0, long long ldd0, void* D1, long long ldd1, int M, int N, int K,
                             int epilogue, int act, float alpha, const float* bias, const void* aux,
                             long long ld_aux, int splits, int accumulate, float* colsum, void* stream_) {
  if (epilogue < EPI_BF16 || epilogue > EPI_F32) return MMB_ERR_ARG;
  return gemm_dispatch(A, lda, a_mn_major, B, ldb, b_mn_major, D0, ldd0, D1, ldd1, M, N, K, epilogue, act, alpha, bias,
                       aux, ld_aux, splits, accumulate, colsum, nullptr, stream_);
}

// ---- fused similarity GEMM + temperature-scaled cross-entropy (no logits in HBM) ------------------------------------
// Number of float4 partials per row one mmb_gemm_ce_stats launch over N columns writes (one per 128 columns: a
// 256-column tile writes two).
extern "C" int mmb_gemm_ce_num_parts(int N) { return N <= 0 ? 0 : (N + 127) / 128; }

static int gemm_ce_stats_impl(const void* A, long long lda, const void* B, long long ldb, int M, int N, int K,
                              const float* log_scale, int label0, const int* labels, void* part, int part_ld, int part0,
                              float* xlabel, void* stream) {
  if (!log_scale || !part || !xlabel || part_ld <= 0 || part0 < 0 || part0 + mmb_gemm_ce_num_parts(N) > part_ld ||
      (reinterpret_cast<uintptr_t>(part) & 15))
    return MMB_ERR_ARG;
  GemmArgs ce{};
  ce.ce_log_scale = log_scale; ce.ce_label0 = label0; ce.ce_labels = labels;
  ce.ce_part = reinterpret_cast<float4*>(part); ce.ce_part_ld = part_ld; ce.ce_part0 = part0; ce.ce_xlabel = xlabel;
  return gemm_dispatch(A, lda, 0, B, ldb, 0, nullptr, 0, nullptr, 0, M, N, K, EPI_CE_STATS, 0, 1.f, nullptr, nullptr, 0, 1, 0,
                       nullptr, &ce, stream);
}

extern "C" int mmb_gemm_ce_stats(const void* A, long long lda, const void* B, long long ldb, int M, int N, int K,
                                 const float* log_scale, int label0, void* part, int part_ld, int part0, float* xlabel,
                                 void* stream) {
  return gemm_ce_stats_impl(A, lda, B, ldb, M, N, K, log_scale, label0, nullptr, part, part_ld, part0, xlabel, stream);
}
// Same with an explicit label column per row (int32 [M]; a value outside [0, N) — e.g. an ignore_index — matches no
// column: xlabel[m] is then left untouched): Linear -> CrossEntropy heads over a vocabulary
// (models/coca/coca_model.py:443-454: captioning loss over the 49 408-entry vocabulary without a [B*76, V] logits tensor).
extern "C" int mmb_gemm_ce_stats_labels(const void* A, long long lda, const void* B, long long ldb, int M, int N, int K,
                                        const float* log_scale, const int* labels, void* part, int part_ld, int part0,
                                        float* xlabel, void* stream) {
  if (!labels) return MMB_ERR_ARG;
  return gemm_ce_stats_impl(A, lda, B, ldb, M, N, K, log_scale, 0, labels, part, part_ld, part0, xlabel, stream);
}

extern "C" int mmb_gemm_ce_grad(const void* A, long long lda, const void* B, long long ldb, int M, int N, int K,
                                const float* log_scale, int label0, int n_total, int rows_total, float smoothing,
                                float loss_weight, const float* lse_row, const float* row_w, const float* lse_col,
                                const float* col_w, int col_lo, int col_hi, void* dsims_bf16, long long ldd,
                                void* stream) {
  if (!log_scale || !lse_row || !dsims_bf16 || n_total <= 0 || rows_total <= 0) return MMB_ERR_ARG;
  GemmArgs ce{};
  ce.ce_log_scale = log_scale; ce.ce_label0 = label0; ce.ce_n_total = n_total; ce.ce_smoothing = smoothing;
  ce.ce_loss_weight = loss_weight; ce.ce_gs = loss_weight / (float)rows_total;
  ce.ce_lse_row = lse_row; ce.ce_row_w = row_w; ce.ce_lse_col = lse_col; ce.ce_col_w = col_w;
  ce.ce_col_lo = col_lo; ce.ce_col_hi = col_hi;
  return gemm_dispatch(A, lda, 0, B, ldb, 0, dsims_bf16, ldd, nullptr, 0, M, N, K, EPI_CE_GRAD, 0, 1.f, nullptr, nullptr, 0, 1,
                       0, nullptr, &ce, stream);
}
