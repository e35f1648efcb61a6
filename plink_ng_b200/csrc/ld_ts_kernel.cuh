// ld_ts_kernel.cuh - --indep-pairwise pair decisions on the int8 tensor pipe (wgmma, sm_90a).
//
// For every (second = a, first = b) variant pair within `band` positions the reference evaluates six exact
// integer sums over the founders (ComputeIndepPairwiseR2Components, 2.0/plink2_ld.cc:699-723: DotprodWords
// :235, SumSsqWords :317, SumSsqNmWords :578) and the r^2 test of :1085-1090.  With per-founder planes
//   nm = genotype non-missing, hom = genotype in {0,2}, x = +1 / 0 / -1 for genotype 0 / 1,missing / 2
// those sums are plain dot products over the founders:
//   nm12 = nm_a.nm_b   dot = x_a.x_b   ssq_b = nm_a.hom_b   sum_b = nm_a.x_b   ssq_a = hom_a.nm_b   sum_a = x_a.nm_b
// i.e. a banded (variants x variants) contraction over SAMPLES - the same shape as the KING kernel with the
// roles of the axes swapped, and here BOTH operands come straight from the variant-major 2-bit block: a
// variant's samples are contiguous in its PgrGet row, which is K-major for both wgmma operands.
//
// One CTA = 64 "second" variants (rows) x 64 "first" variants (columns), k-step = 32 founders, two warpgroups
// over the B planes [hom_b | nm_b | x_b] (N = 192), issuing the same shapes (ptxas serialises a wgmma under a
// branch):
//   warpgroup 0:  nm_a x [hom_b | nm_b] -> ssq_b, nm12 (N = 128);   nm_a x x_b  -> sum_b (N = 64)
//   warpgroup 1:  x_a  x [nm_b | x_b]   -> sum_a, dot  (N = 128);   hom_a x nm_b -> ssq_a (N = 64)
// 96 int32 accumulators per thread.  All founders are contracted inside one CTA, so nothing is accumulated in
// HBM: warpgroup 1 hands its three sums over through shared memory and warpgroup 0 turns the six sums of each
// pair into the 1-byte decision the host-side greedy walk looks up.
#pragma once

#include "common.cuh"
#include "geno_expand.cuh"
#include "wgmma.cuh"

namespace pl2 {

constexpr uint32_t kLdtRows = 64;                  // second variants per CTA
constexpr uint32_t kLdtCols = 64;                  // first variants per CTA
constexpr uint32_t kLdtThreads = 256;
constexpr uint32_t kLdtKs = 2;                     // k32 steps per stage (64 founders: the stage's sample padding)
constexpr uint32_t kLdtSbo = 2 * kLdtKs * kCoreBytes;   // 512: next group of 8 B rows
constexpr uint32_t kLdtBBytes = 3 * kLdtCols * 32 * kLdtKs;  // 12288
constexpr uint32_t kLdtABytes = kLdtRows * 8 * kLdtKs;       // 1024: [row][16 B]
constexpr uint32_t kLdtStageBytes = kLdtBBytes + kLdtABytes;
constexpr uint32_t kLdtXBytes = 3 * kLdtRows * kLdtCols * 4;  // warpgroup 1's sums for the epilogue
constexpr uint32_t kLdtSmemBytes = (2 * kLdtStageBytes > kLdtXBytes ? 2 * kLdtStageBytes : kLdtXBytes) + 128;

// raw: the staged block [row][pitch], row r = variant chunk_lo + r (rows are padded to a multiple of 64 with
// "missing"); sample_ct_padded: multiple of 64, padding founders coded missing (all planes 0).
// flags[(a - a_out0) * band + (a - b - 1)] = (cov12^2 > thresh * var1 * var2) for 0 < a - b <= band,
// a in [a_out0, a_out1), b >= chunk_lo; a, b are global variant indices.
static __global__ void __launch_bounds__(kLdtThreads, 1)
ld_ts_kernel(const uint8_t* __restrict__ raw, uint32_t pitch, uint32_t sample_ct_padded, uint32_t chunk_lo, uint32_t a_out0, uint32_t a_out1, uint32_t band, double thresh, uint8_t* __restrict__ flags) {
  // tile geometry (uniform per CTA); tiles without an in-band pair exit at once
  const uint32_t a_start = a_out0 + blockIdx.x * kLdtRows;                              // multiple of 64 (a_out0 is)
  const int64_t b_start_s = static_cast<int64_t>(a_start) + kLdtRows - kLdtCols - static_cast<int64_t>(kLdtCols) * blockIdx.y;
  if (b_start_s < static_cast<int64_t>(chunk_lo)) return;
  const uint32_t b_start = static_cast<uint32_t>(b_start_s);
  if (a_start > b_start + (kLdtCols - 1) && a_start - (b_start + kLdtCols - 1) > band) return;
  if (b_start >= a_start + kLdtRows - 1) return;                                        // no b < a in this tile

  extern __shared__ __align__(128) uint8_t smem_dyn[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 127) & ~static_cast<uintptr_t>(127));
  const uint32_t smem_base = static_cast<uint32_t>(__cvta_generic_to_shared(smem));
  const uint32_t tid = threadIdx.x, wg = tid >> 7, warp4 = (tid >> 5) & 3, lane = tid & 31, g = lane >> 2, c = lane & 3;
  const uint32_t stage_ct = sample_ct_padded / (32 * kLdtKs);
  const uint32_t thread_zero = tid * (sample_ct_padded >> 31);  // 0; keeps the plane tables in vector registers
  const uint32_t tab_nm = table_reg(kTabNonmiss, thread_zero), tab_hom = table_reg(kTabHom, thread_zero), tab_x = table_reg(kTabSgn, thread_zero);

  // staging: thread = (column variant, 16-founder word) of the stage; threads 0..63 also copy one row's 16 bytes
  const uint32_t bv = tid >> 2, bw = tid & 3;
  const uint8_t* b_src = raw + static_cast<uint64_t>(b_start - chunk_lo + bv) * pitch + 4 * bw;
  const uint8_t* a_src = raw + static_cast<uint64_t>(a_start - chunk_lo + (tid & 63)) * pitch;
  struct Pre {
    uint32_t w;
    uint4 a;
  };
  auto load_stage = [&](uint32_t st) -> Pre {
    Pre p;
    p.w = __ldg(reinterpret_cast<const uint32_t*>(b_src + st * 16));
    p.a = (tid < kLdtRows) ? __ldg(reinterpret_cast<const uint4*>(a_src + st * 16)) : make_uint4(0, 0, 0, 0);
    return p;
  };
  auto store_stage = [&](const Pre& p, uint32_t buf) {
    const uint32_t base = smem_base + buf * kLdtStageBytes;
    const Sel4 sel = make_selectors(p.w);
    const uint32_t tabs[3] = {tab_hom, tab_nm, tab_x};
#pragma unroll
    for (uint32_t pl = 0; pl < 3; ++pl) {
      const uint32_t row = pl * kLdtCols + bv;
      const uint4 v = expand16(tabs[pl], sel);
      asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(base + (row >> 3) * kLdtSbo + bw * kCoreBytes + (row & 7) * 16), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
    }
    if (tid < kLdtRows)
      asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(base + kLdtBBytes + tid * 16), "r"(p.a.x), "r"(p.a.y), "r"(p.a.z), "r"(p.a.w) : "memory");
  };

  int32_t d128[64], d64[32];
#pragma unroll
  for (uint32_t i = 0; i < 64; ++i) d128[i] = 0;
#pragma unroll
  for (uint32_t i = 0; i < 32; ++i) d64[i] = 0;
  const uint32_t tab_1 = wg ? tab_x : tab_nm, tab_2 = wg ? tab_hom : tab_nm;  // A planes of the N = 128 / N = 64 products
  const uint32_t off_1 = wg ? kLdtCols : 0, off_2 = wg ? kLdtCols : 2 * kLdtCols;  // first B row of each product
  const uint32_t r_lo = 16 * warp4 + g;

  {
    const Pre p0 = load_stage(0);
    store_stage(p0, 0);
  }
  for (uint32_t st = 0; st < stage_ct; ++st) {
    const uint32_t buf = st & 1;
    const bool more = st + 1 < stage_ct;
    Pre next;
    if (more) next = load_stage(st + 1);
    fence_proxy_async_smem();
    __syncthreads();  // stage st in shared memory; the other buffer's wgmmas have retired
    const uint32_t base = smem_base + buf * kLdtStageBytes;
    const uint64_t desc = make_wg_desc(base, kCoreBytes, kLdtSbo);
#pragma unroll
    for (uint32_t ks = 0; ks < kLdtKs; ++ks) {
      uint2 w_lo, w_hi;
      asm volatile("ld.shared.v2.b32 {%0,%1}, [%2];" : "=r"(w_lo.x), "=r"(w_lo.y) : "r"(base + kLdtBBytes + r_lo * 16 + ks * 8) : "memory");
      asm volatile("ld.shared.v2.b32 {%0,%1}, [%2];" : "=r"(w_hi.x), "=r"(w_hi.y) : "r"(base + kLdtBBytes + (r_lo + 8) * 16 + ks * 8) : "memory");
      const ASel sel = make_asel(w_lo, w_hi, c);
      uint32_t f1[4], f2[4];
      afrag(tab_1, sel, f1);
      afrag(tab_2, sel, f2);
      const uint64_t dk = desc + ((ks * 2 * kCoreBytes) >> 4);
      wgmma_fence();
      wgmma_s8_rs<128>(d128, f1, dk + (((off_1 / 8) * kLdtSbo) >> 4));
      wgmma_s8_rs<64>(d64, f2, dk + (((off_2 / 8) * kLdtSbo) >> 4));
      wgmma_commit();
      wgmma_wait<1>();
    }
    if (more) store_stage(next, buf ^ 1);
    wgmma_wait<0>();
  }

  // ---- epilogue: six sums per pair -> the r^2 decision byte
  __syncthreads();  // operand buffers are free
  int32_t* xs = reinterpret_cast<int32_t*>(smem);  // [3][64 rows][64 columns]: sum_a, dot, ssq_a
  if (wg == 1) {
#pragma unroll
    for (uint32_t j = 0; j < 8; ++j)
#pragma unroll
      for (uint32_t i = 0; i < 4; ++i) {
        const uint32_t col = 8 * j + 2 * c + (i & 1), row = r_lo + 8 * (i >> 1);
        xs[row * kLdtCols + col] = d128[4 * j + i];                               // sum_a = x_a . nm_b
        xs[kLdtRows * kLdtCols + row * kLdtCols + col] = d128[4 * (8 + j) + i];   // dot = x_a . x_b
        xs[2 * kLdtRows * kLdtCols + row * kLdtCols + col] = d64[4 * j + i];      // ssq_a = hom_a . nm_b
      }
  }
  __syncthreads();
  if (wg == 0) {
#pragma unroll
    for (uint32_t j = 0; j < 8; ++j)
#pragma unroll
      for (uint32_t i = 0; i < 4; ++i) {
        const uint32_t col = 8 * j + 2 * c + (i & 1), row = r_lo + 8 * (i >> 1);
        const uint32_t a = a_start + row, b = b_start + col;
        if (a >= a_out1 || b >= a || a - b > band) continue;
        const int64_t q_b = d128[4 * j + i], n12 = d128[4 * (8 + j) + i], s_b = d64[4 * j + i];  // first
        const int64_t s_a = xs[row * kLdtCols + col], dot = xs[kLdtRows * kLdtCols + row * kLdtCols + col], q_a = xs[2 * kLdtRows * kLdtCols + row * kLdtCols + col];
        // plink2_ld.cc:1085-1090; int64 -> double casts, unfused left-to-right multiplies
        const double cov12 = static_cast<double>(dot * n12 - s_b * s_a);
        const double var1 = static_cast<double>(q_b * n12 - s_b * s_b);
        const double var2 = static_cast<double>(q_a * n12 - s_a * s_a);
        const bool over = __dmul_rn(cov12, cov12) > __dmul_rn(__dmul_rn(thresh, var1), var2);
        flags[static_cast<uint64_t>(a - a_out0) * band + (a - b - 1)] = over ? 1 : 0;
      }
  }
}

}  // namespace pl2
