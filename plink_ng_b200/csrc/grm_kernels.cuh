// grm_kernels.cuh - device kernels of the GRM path (CalcGrm, 2.0/plink2_matrix_calc.cc:4555).
//
// Replaces ExpandCenteredVarmaj + the dsyrk/dgemm accumulation (CalcGrmThread / CalcGrmPartThread,
// :4285-4327) and the CalcMissingMatrix popcount pass (:4404-4553) with ONE exact int8 tensor-core
// contraction per variant batch:
//
//   G_ij * obs_ij = sum_v z_iv z_jv,   z_v(g) = intercept_v + g * slope_v (0 for missing)   [PopulateRescaledDosage]
//                 = sum_v g_iv L1_v(g_jv) + m_iv L2_v(g_jv),   L1_v(g) = slope_v z_v(g),  L2_v(g) = intercept_v z_v(g)
//   obs_ij        = sum_v m_iv m_jv      (= M - miss_i - miss_j + bothmiss_ij, :4769-4788)
//
// g (ALT dosage 0/1/2, missing -> 0) and m (non-missing indicator) are exact small integers.  The
// real-valued per-variant 3-entry tables L1_v, L2_v are written in fixed point with scale 2^F
// (|L| 2^F < 2^38) and split into FIVE balanced base-256 digits (int8 in [-128,127]):
//   sum_v g_iv L_v(g_jv) = 2^-F * sum_k 256^k * (sum_v g_iv d_k,v(g_jv))     <- five exact int32 accumulators
// so the only error is the 2^-(F+1) rounding of each table entry: 40 significant bits relative to
// the largest |L| of the batch (DESIGN.md has the bound; measured < 1e-10 absolute on G).
//
// Tile = 128 rows (I side: planes g, m) x 80 cols (J side: 10 digit planes + m); accumulators D_0..D_4 and the
// obs counts.  The kernel itself is grm_ts_kernel.cuh.
#pragma once
#include "common.cuh"
#include "geno_expand.cuh"

namespace pl2 {

constexpr uint32_t kGrmTileCols = 80;
constexpr uint32_t kGrmSamplePad = 640;         // lcm(128, 80)
constexpr uint32_t kGrmLimbs = 5;
constexpr uint32_t kGrmFixedBits = 38;          // |L| * 2^F < 2^38
constexpr uint32_t kGrmPlanesJ = 2 * kGrmLimbs + 1;
constexpr uint32_t kGrmGroupsJ = kGrmTileCols / 16;  // 16-sample groups per J plane
constexpr uint32_t kGrmTileWords = kTileRows * kGrmTileCols;  // per-tile accumulator entries

// ---- per-variant digit tables, in the form the column-side expansion of grm_ts_kernel.cuh reads: for every chunk of
// 16 variants, digit plane p (0..4 = L1 digits, least significant first, 5..9 = L2 digits) and genotype code
// g (0..2) one 16-byte vector holding that digit of each variant of the chunk, variant v at byte SampleToPos(v % 16)
// (the K order of the operand rows).  Missing genotypes select no vector and give 0.  The m plane is constant.
// lvals[v] = {L1(0), L1(1), L1(2), L2(0), L2(1), L2(2)} as doubles (host-prepared, grm.cu).
constexpr uint32_t kGrmTabChunkBytes = 2 * kGrmLimbs * 3 * 16;  // 480 bytes per 16 variants
__host__ __device__ constexpr uint64_t grm_tab_offset(uint32_t v, uint32_t plane, uint32_t code) {
  return (static_cast<uint64_t>(v >> 4) * (2 * kGrmLimbs) + plane) * 48 + code * 16 + SampleToPos(v & 15u);
}

__global__ void grm_tables_kernel(const double* __restrict__ lvals, uint32_t variant_ct, uint32_t variant_ct_padded, double scale, uint8_t* __restrict__ tabk) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= variant_ct_padded) return;
#pragma unroll
  for (uint32_t which = 0; which < 2; ++which) {
#pragma unroll
    for (uint32_t g = 0; g < 3; ++g) {
      long long x = (v < variant_ct) ? __double2ll_rn(lvals[6ull * v + 3 * which + g] * scale) : 0;
#pragma unroll
      for (uint32_t k = 0; k < kGrmLimbs; ++k) {
        const long long d = ((x + 128) & 255) - 128;  // balanced base-256 digit in [-128, 127]
        x = (x - d) >> 8;
        tabk[grm_tab_offset(v, kGrmLimbs * which + k, g)] = static_cast<uint8_t>(d & 0xFF);
      }
    }
  }
}

// ---- finalisation: rows [r0, r1) of the lower triangle INCLUDING the diagonal into the reference's
// in-memory layout grm[(j - r0) * row_stride + i], i <= j (CalcGrm :4630, :4769-4788); optionally
// the per-pair observation counts as float (the .grm.N.bin payload, :4985-5019).
__global__ void __launch_bounds__(256)
grm_finalize_kernel(const double* __restrict__ acc_g, const int32_t* __restrict__ acc_obs, const uint32_t* __restrict__ tile_rt, const uint32_t* __restrict__ tile_tc, uint32_t sample_ct, uint32_t r0, uint32_t r1, uint64_t row_stride, int use_obs, double variant_ct_recip, double* __restrict__ out_g, float* __restrict__ out_obs) {
  __shared__ double s_g[16][kGrmTileCols + 1];
  __shared__ int32_t s_o[16][kGrmTileCols + 1];
  const uint32_t tile = blockIdx.x >> 3;
  const uint32_t sub = blockIdx.x & 7;
  const uint32_t row_base = tile_rt[tile] * kTileRows + sub * 16;
  if (row_base >= r1 || row_base + 16 <= r0) return;
  const uint32_t col_base = tile_tc[tile] * kGrmTileCols;
  if (col_base > row_base + 15) return;
  const uint32_t r = threadIdx.x & 15;
  for (uint32_t c = threadIdx.x >> 4; c < kGrmTileCols; c += 16) {
    const uint64_t off = static_cast<uint64_t>(tile) * kGrmTileWords + static_cast<uint64_t>(c) * kTileRows + sub * 16 + r;
    s_g[r][c] = acc_g[off];
    s_o[r][c] = acc_obs[off];
  }
  __syncthreads();
  for (uint32_t idx = threadIdx.x; idx < 16 * kGrmTileCols; idx += 256) {
    const uint32_t rr = idx / kGrmTileCols, cl = idx % kGrmTileCols;
    const uint32_t j = row_base + rr, i = col_base + cl;
    if (j < r0 || j >= r1 || j >= sample_ct || i > j) continue;
    const uint64_t o = static_cast<uint64_t>(j - r0) * row_stride + i;
    const double g = s_g[rr][cl];
    // reference: `/= u31tod(obs)` per entry, or `*= 1.0 / variant_ct` (:4769-4788)
    out_g[o] = use_obs ? (g / static_cast<double>(s_o[rr][cl])) : (g * variant_ct_recip);
    if (out_obs) out_obs[o] = static_cast<float>(s_o[rr][cl]);
  }
}

}  // namespace pl2
