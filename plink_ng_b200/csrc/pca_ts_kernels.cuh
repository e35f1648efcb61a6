// pca_ts_kernels.cuh - the two skinny products of `--pca approx` (CalcPca approx branch,
// 2.0/plink2_matrix_calc.cc:5697-5941: CalcPcaXaThread :5243 / CalcPcaXtxaThread :5210 / CalcPcaXtbThread :5272)
// on the int8 tensor pipe (wgmma, sm_90a).
//
// Y is the M x N standardised genotype matrix (ExpandCenteredVarmaj, missing -> 0): y_vs = slope_v g_vs + icpt_v m_vs
// with g the ALT dosage (0/1/2, missing 0) and m the non-missing indicator - exact small integers.  The dense
// factor is fp64; per column it is scaled to 32-bit fixed point (|x| 2^F <= 2^30) and split into FOUR balanced
// base-256 digits, so every product is an exact int8 x int8 -> int32 contraction and the only rounding is the
// 2^-31-relative quantisation of the dense operand (the power iteration needs ~1e-6):
//
//   XA :  H[v][c]  = slope_v sum_s g_vs G[s][c] + icpt_v sum_s m_vs G[s][c]          (contract over samples)
//         A = {g, m} planes of 128 variants, read straight from the variant-major block (a variant's samples are
//         contiguous: K-major); B = digit planes of G;  2 wgmmas (N = 4 cg) per 32 samples;  epilogue recombines
//         digits in int64.
//   XtB:  O[s][c] += sum_v g_vs (slope_v H[v][c]) + m_vs (icpt_v H[v][c])           (contract over variants)
//         A = {g, m} planes of a 128-sample tile from the sample-major copy (as king_ts_kernel's row side);
//         B = digit planes of slope.H and of icpt.H (common per-column scale, so both wgmmas add into one
//         accumulator).
//
// The B operand needs no expansion: pca_digits_kernel writes it ONCE per pass in the K-major no-swizzle layout
// (8 columns x 16 K-bytes per core matrix), one contiguous 32 N-byte block per k-step, and the kernels stage it
// with cp.async.  K bytes are stored in the PRMT position order of the A side (geno_expand.cuh, wgmma.cuh).
// A thread holds accumulator columns 2 c, 2 c + 1 (mod 8) only, so the four digits d cg + col of a column meet in
// one thread when cg is a multiple of 8: every launch uses cg = kPcaCgMax (columns beyond the valid ones are 0).
#pragma once
#include "common.cuh"
#include "cp_async.cuh"
#include "geno_expand.cuh"
#include "wgmma.cuh"

namespace pl2 {

constexpr uint32_t kPcaDigits = 4;
constexpr uint32_t kPcaCgMax = 32;                      // columns per launch: N = 4 cg = 128 int32 accumulators per row
constexpr uint32_t kPcaNMax = kPcaDigits * kPcaCgMax;   // 128
constexpr uint32_t kPcaFixedBits = 30;                  // |x| 2^F <= 2^30 < the balanced 4-digit range (~2^31)

__host__ __device__ constexpr uint32_t pca_block_bytes(uint32_t n) { return 32 * n; }
// byte offset of (K byte k of the k-step, column n) inside a k-step block (K-major, LBO = 128, SBO = 256)
__host__ __device__ constexpr uint32_t pca_b_offset(uint32_t k, uint32_t n) {
  return (n >> 3) * 256 + (k >> 4) * kCoreBytes + (n & 7) * 16 + SampleToPos(k & 15u);
}

// ---- per-column scale: colmax[c] = max_r |src(r, c) * mul(r)| over one or two row multipliers -------------------
// src element (r, c) at src[r * rs + c * cs]; grid = (cg, row chunks); atomicMax on the bit pattern (values >= 0).
static __global__ void __launch_bounds__(256) pca_colmax_kernel(const double* __restrict__ src, uint64_t rs, uint64_t cs, uint32_t rows, const double* __restrict__ mul1, const double* __restrict__ mul2, unsigned long long* __restrict__ colmax_bits) {
  const uint32_t c = blockIdx.x;  // grid.x = number of VALID columns of the group
  double mx = 0.0;
  for (uint32_t r = blockIdx.y * blockDim.x + threadIdx.x; r < rows; r += gridDim.y * blockDim.x) {
    const double x = src[static_cast<uint64_t>(r) * rs + static_cast<uint64_t>(c) * cs];
    double a = fabs(mul1 ? x * mul1[r] : x);
    if (mul2) a = fmax(a, fabs(x * mul2[r]));
    mx = fmax(mx, a);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xFFFFFFFFu, mx, o));
  if ((threadIdx.x & 31) == 0 && mx > 0.0) atomicMax(&colmax_bits[c], static_cast<unsigned long long>(__double_as_longlong(mx)));
}

// scale[c] = 2^F with |x| 2^F <= 2^30; inv_scale[c] = 2^-F (both exact powers of two); all-zero column: 1
static __global__ void pca_scales_kernel(const unsigned long long* __restrict__ colmax_bits, uint32_t cg, double* __restrict__ scale, double* __restrict__ inv_scale) {
  const uint32_t c = threadIdx.x;
  if (c >= cg) return;
  const double mx = __longlong_as_double(static_cast<long long>(colmax_bits[c]));
  int f = 0;
  if (mx > 0.0) {
    int e;
    frexp(mx, &e);  // mx = m 2^e, m in [0.5, 1)
    f = static_cast<int>(kPcaFixedBits) - e;
  }
  scale[c] = ldexp(1.0, f);
  inv_scale[c] = ldexp(1.0, -f);
}

// ---- fp64 -> four balanced base-256 digit planes in the canonical k-step blocks --------------------------------
// out1 (and out2 when mul2 != nullptr): [rows_padded / 32][32 * 4 cg] bytes; rows >= `rows` are zero.
// thread = (row, column); grid.x = rows_padded / 64 (two k-steps per CTA), 64 x cg threads in strides.
// pass 0 encodes rn(y 2^F); pass 1 encodes the residual (y 2^F - rn(y 2^F)) 2^30 (exact in fp64), so the two passes
// together carry 60 bits below the column maximum - more than the fp64 operand the reference's dgemm reads.
constexpr double kPcaPass1Scale = 1073741824.0;  // 2^30
static __global__ void __launch_bounds__(256) pca_digits_kernel(const double* __restrict__ src, uint64_t rs, uint64_t cs, uint32_t rows, uint32_t cg, uint32_t cols_valid, const double* __restrict__ mul1, const double* __restrict__ mul2, const double* __restrict__ scale, uint8_t* __restrict__ out1, uint8_t* __restrict__ out2, int pass) {
  const uint32_t n_total = kPcaDigits * cg;
  const uint32_t blk = pca_block_bytes(n_total);
  for (uint32_t idx = threadIdx.x; idx < 64 * cg; idx += blockDim.x) {
    const uint32_t rl = idx % 64, c = idx / 64;   // consecutive threads = consecutive rows (coalesced for rs == 1)
    const uint32_t r = blockIdx.x * 64 + rl;
    double x = 0.0;
    if (r < rows && c < cols_valid) x = src[static_cast<uint64_t>(r) * rs + static_cast<uint64_t>(c) * cs];  // columns padding the group to a multiple of 4 are zero
    const uint64_t base = static_cast<uint64_t>(r >> 5) * blk;
    const uint32_t k = r & 31;
    const double sc = scale[c];
#pragma unroll
    for (int which = 0; which < 2; ++which) {
      uint8_t* out = which ? out2 : out1;
      if (!out) continue;
      const double* mul = which ? mul2 : mul1;
      const double y = (mul && r < rows) ? x * mul[r] : x;
      const double ys = y * sc;  // exact: sc is a power of two
      long long v = __double2ll_rn(ys);
      if (pass) v = __double2ll_rn((ys - static_cast<double>(v)) * kPcaPass1Scale);  // |residual| <= 0.5 -> |v| <= 2^29
#pragma unroll
      for (uint32_t d = 0; d < kPcaDigits; ++d) {
        const long long dig = ((v + 128) & 255) - 128;  // balanced digit in [-128, 127]
        v = (v - dig) >> 8;
        out[base + pca_b_offset(k, d * cg + c)] = static_cast<uint8_t>(static_cast<int8_t>(dig));
      }
    }
  }
}

// ================================================================================================================
// Both products: 2 warpgroups x 64 rows, N = kPcaNMax, one stage = 4 k-steps staged with cp.async into a double
// buffer [row words][B blocks], one __syncthreads per stage.
// ================================================================================================================
constexpr uint32_t kPcaThreads = 256;
constexpr uint32_t kPcaStageK = 4;                          // k-steps per stage
constexpr uint32_t kPcaABytes = kPcaStageK * 128 * 8;       // 4096: 128 rows x 4 k-steps x 8 B
constexpr uint32_t kPcaBlk = pca_block_bytes(kPcaNMax);     // 4096

// selectors of this thread's A fragment rows (r, r + 8) for one k-step; word (row, k-step j) at
// a_words + row * row_stride + j * ks_stride
__device__ __forceinline__ ASel pca_asel(uint32_t a_words, uint32_t row_stride, uint32_t ks_stride, uint32_t j, uint32_t r, uint32_t c) {
  uint2 w_lo, w_hi;
  asm volatile("ld.shared.v2.b32 {%0,%1}, [%2];" : "=r"(w_lo.x), "=r"(w_lo.y) : "r"(a_words + r * row_stride + j * ks_stride) : "memory");
  asm volatile("ld.shared.v2.b32 {%0,%1}, [%2];" : "=r"(w_hi.x), "=r"(w_hi.y) : "r"(a_words + (r + 8) * row_stride + j * ks_stride) : "memory");
  return make_asel(w_lo, w_hi, c);
}

// ================================================================================================================
// XA: H[v][c] for 128 variants per CTA (warpgroup w: variants v0 + 64 w ..), accumulators D_g, D_m in registers.
// Row words come from the variant-major block: a stage is 32 contiguous bytes (128 samples) of each variant.
// ================================================================================================================
constexpr uint32_t kPxaStage = kPcaABytes + kPcaStageK * kPcaBlk;
constexpr uint32_t kPxaSmemBytes = 2 * kPxaStage + 128;

static __global__ void __launch_bounds__(kPcaThreads, 1)
pca_xa_wg_kernel(const uint8_t* __restrict__ raw /* [variant][pitch] */, uint32_t pitch, uint32_t sample_ct_padded /* multiple of 128 */, uint32_t variant_ct, const uint8_t* __restrict__ gdig /* [samples / 32][32 N] */, uint32_t cols_valid,
                 const double* __restrict__ slope, const double* __restrict__ icpt, const double* __restrict__ inv_scale /* [kPcaCgMax] */, double* __restrict__ h /* column-major, ld = h_ld, first column = this group's */, uint64_t h_ld,
                 double post_scale /* 1, or 2^-30 for the residual pass */, int accumulate /* add to h instead of overwriting */) {
  extern __shared__ __align__(128) uint8_t smem_dyn[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 127) & ~static_cast<uintptr_t>(127));
  const uint32_t smem_base = static_cast<uint32_t>(__cvta_generic_to_shared(smem));
  const uint32_t tid = threadIdx.x, wg = tid >> 7, warp4 = (tid >> 5) & 3, lane = tid & 31, g = lane >> 2, c = lane & 3;
  const uint32_t v0 = blockIdx.x * 128;
  const uint32_t stage_ct = sample_ct_padded / (32 * kPcaStageK);
  const uint32_t thread_zero = tid * (sample_ct_padded >> 31);
  const uint32_t tab_g = table_reg(kTabDosage, thread_zero), tab_m = table_reg(kTabNonmiss, thread_zero);
  auto issue = [&](uint32_t st) {
    uint8_t* dst = smem + (st & 1) * kPxaStage;
    {  // row words: [variant][32 B]; thread = (variant, 16-byte half)
      const uint32_t v = tid >> 1, hf = tid & 1;
      cp_async16(dst + v * 32 + 16 * hf, raw + static_cast<uint64_t>(v0 + v) * pitch + st * (kPcaStageK * 8) + 16 * hf);
    }
    const uint8_t* src = gdig + static_cast<uint64_t>(st) * kPcaStageK * kPcaBlk;
    for (uint32_t i = tid; i < kPcaStageK * kPcaBlk / 16; i += kPcaThreads) cp_async16(dst + kPcaABytes + 16 * i, src + 16 * i);
    cp_async_commit();
  };

  int32_t dg[kPcaNMax / 2], dm[kPcaNMax / 2];
#pragma unroll
  for (uint32_t i = 0; i < kPcaNMax / 2; ++i) dg[i] = dm[i] = 0;
  const uint32_t r = 64 * wg + 16 * warp4 + g;
  issue(0);
  for (uint32_t st = 0; st < stage_ct; ++st) {
    if (st + 1 < stage_ct) {
      issue(st + 1);  // the other buffer: its wgmmas retired (wait<0>) before the barrier that ended stage st - 1
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    fence_proxy_async_smem();
    __syncthreads();
    const uint32_t base = smem_base + (st & 1) * kPxaStage;
    const uint64_t desc = make_wg_desc(base + kPcaABytes, kCoreBytes, 256);
#pragma unroll
    for (uint32_t j = 0; j < kPcaStageK; ++j) {
      const ASel sel = pca_asel(base, 32, 8, j, r, c);
      uint32_t fg[4], fm[4];
      afrag(tab_g, sel, fg);
      afrag(tab_m, sel, fm);
      const uint64_t dj = desc + ((j * kPcaBlk) >> 4);
      wgmma_fence();
      wgmma_s8_rs<kPcaNMax>(dg, fg, dj);  // sum_s g G
      wgmma_s8_rs<kPcaNMax>(dm, fm, dj);  // sum_s m G
      wgmma_commit();
      wgmma_wait<1>();
    }
    wgmma_wait<0>();
    __syncthreads();  // every warpgroup is done with this buffer before the next stage's copies into it
  }

  // ---- epilogue: digits -> int64 -> fp64, H[v][col] = (slope_v S_g + icpt_v S_m) 2^-F_col
#pragma unroll
  for (uint32_t rh = 0; rh < 2; ++rh) {
    const uint32_t v = v0 + r + 8 * rh;
    if (v >= variant_ct) continue;
    const double sl = slope[v], ic = icpt[v];
#pragma unroll
    for (uint32_t j = 0; j < kPcaCgMax / 8; ++j) {  // column col = 8 j + 2 c + e, digit d at accumulator column d cg + col
#pragma unroll
      for (uint32_t e = 0; e < 2; ++e) {
        long long sg = 0, sm = 0;
#pragma unroll
        for (int d = kPcaDigits - 1; d >= 0; --d) {
          const uint32_t reg = 4 * (d * (kPcaCgMax / 8) + j) + 2 * rh + e;
          sg = sg * 256 + dg[reg];
          sm = sm * 256 + dm[reg];
        }
        const uint32_t col = 8 * j + 2 * c + e;
        if (col < cols_valid) {
          double* dst = &h[static_cast<uint64_t>(col) * h_ld + v];
          const double val = (sl * static_cast<double>(sg) + ic * static_cast<double>(sm)) * (inv_scale[col] * post_scale);
          *dst = accumulate ? (*dst + val) : val;
        }
      }
    }
  }
}

// ================================================================================================================
// XtB: partial[split][s][c] = sum over this CTA's variants of g (slope H) + m (icpt H) for 128 samples per CTA
// (warpgroup w: samples 64 w ..).  Row words: the sample-major copy ([row tile][k-step][128][8 B]).
// ================================================================================================================
constexpr uint32_t kPxtStage = kPcaABytes + 2 * kPcaStageK * kPcaBlk;   // [row words][slope.H blocks][icpt.H blocks]
constexpr uint32_t kPxtSmemBytes = 2 * kPxtStage + 128;

static __global__ void __launch_bounds__(kPcaThreads, 1)
pca_xtb_wg_kernel(const uint8_t* __restrict__ raw_i /* [row tile][kstep_total][128][8 B] */, uint32_t kstep_total, uint32_t ksteps_per_split /* multiple of 4 */, uint32_t sample_ct, const uint8_t* __restrict__ hs_dig, const uint8_t* __restrict__ hi_dig /* [variants / 32][32 N] */,
                  const double* __restrict__ inv_scale /* [kPcaCgMax] */, double* __restrict__ partial /* [split][sample_ct_padded][kPcaCgMax] */, uint32_t sample_ct_padded) {
  extern __shared__ __align__(128) uint8_t smem_dyn[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 127) & ~static_cast<uintptr_t>(127));
  const uint32_t smem_base = static_cast<uint32_t>(__cvta_generic_to_shared(smem));
  const uint32_t tid = threadIdx.x, wg = tid >> 7, warp4 = (tid >> 5) & 3, lane = tid & 31, g = lane >> 2, c = lane & 3;
  const uint32_t rt = blockIdx.x;
  const uint32_t ks_begin = blockIdx.y * ksteps_per_split;
  const uint32_t ks_end = min(kstep_total, ks_begin + ksteps_per_split);
  const uint32_t stage_ct = ks_end > ks_begin ? (ks_end - ks_begin) / kPcaStageK : 0;  // kstep_total is a multiple of 4
  const uint32_t thread_zero = tid * (kstep_total >> 31);
  const uint32_t tab_g = table_reg(kTabDosage, thread_zero), tab_m = table_reg(kTabNonmiss, thread_zero);
  auto issue = [&](uint32_t st) {
    uint8_t* dst = smem + (st & 1) * kPxtStage;
    const uint64_t ks0 = ks_begin + st * kPcaStageK;
    const uint8_t* a_src = raw_i + (static_cast<uint64_t>(rt) * kstep_total + ks0) * 1024;
    cp_async16(dst + 16 * tid, a_src + 16 * tid);  // 4 KB = 256 x 16 B
    for (uint32_t i = tid; i < 2 * kPcaStageK * kPcaBlk / 16; i += kPcaThreads) {
      const uint32_t which = i / (kPcaStageK * kPcaBlk / 16), o = 16 * (i % (kPcaStageK * kPcaBlk / 16));
      cp_async16(dst + kPcaABytes + which * (kPcaStageK * kPcaBlk) + o, (which ? hi_dig : hs_dig) + ks0 * kPcaBlk + o);
    }
    cp_async_commit();
  };

  int32_t acc[kPcaNMax / 2];
#pragma unroll
  for (uint32_t i = 0; i < kPcaNMax / 2; ++i) acc[i] = 0;
  const uint32_t r = 64 * wg + 16 * warp4 + g;
  if (stage_ct) issue(0);
  for (uint32_t st = 0; st < stage_ct; ++st) {
    if (st + 1 < stage_ct) {
      issue(st + 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    fence_proxy_async_smem();
    __syncthreads();
    const uint32_t base = smem_base + (st & 1) * kPxtStage;
    const uint64_t desc_s = make_wg_desc(base + kPcaABytes, kCoreBytes, 256);
    const uint64_t desc_i = desc_s + ((kPcaStageK * kPcaBlk) >> 4);
#pragma unroll
    for (uint32_t j = 0; j < kPcaStageK; ++j) {
      const ASel sel = pca_asel(base, 8, 1024, j, r, c);
      uint32_t fg[4], fm[4];
      afrag(tab_g, sel, fg);
      afrag(tab_m, sel, fm);
      wgmma_fence();
      wgmma_s8_rs<kPcaNMax>(acc, fg, desc_s + ((j * kPcaBlk) >> 4));  // g x slope.H
      wgmma_s8_rs<kPcaNMax>(acc, fm, desc_i + ((j * kPcaBlk) >> 4));  // m x icpt.H
      wgmma_commit();
      wgmma_wait<1>();
    }
    wgmma_wait<0>();
    __syncthreads();
  }

  // ---- epilogue: digits -> fp64 partial sums
  if (!stage_ct) return;
#pragma unroll
  for (uint32_t rh = 0; rh < 2; ++rh) {
    const uint32_t s = 128 * rt + r + 8 * rh;
    if (s >= sample_ct_padded) continue;
    double* out = partial + (static_cast<uint64_t>(blockIdx.y) * sample_ct_padded + s) * kPcaCgMax;
#pragma unroll
    for (uint32_t j = 0; j < kPcaCgMax / 8; ++j) {
#pragma unroll
      for (uint32_t e = 0; e < 2; ++e) {
        long long sum = 0;
#pragma unroll
        for (int d = kPcaDigits - 1; d >= 0; --d) sum = sum * 256 + acc[4 * (d * (kPcaCgMax / 8) + j) + 2 * rh + e];
        const uint32_t col = 8 * j + 2 * c + e;
        out[col] = (s < sample_ct) ? static_cast<double>(sum) * inv_scale[col] : 0.0;
      }
    }
  }
}

// out(s, c) += scale * sum_split partial[split][s][c], fixed summation order (bit-reproducible)
static __global__ void __launch_bounds__(256) pca_xtb_reduce_kernel(const double* __restrict__ partial, uint32_t splits, uint32_t sample_ct, uint32_t sample_ct_padded, uint32_t cg, uint32_t cols_valid, double scale, double* __restrict__ out, uint64_t out_rs, uint64_t out_cs) {
  const uint64_t idx = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<uint64_t>(sample_ct) * cg) return;
  const uint32_t s = static_cast<uint32_t>(idx / cg), c = static_cast<uint32_t>(idx % cg);
  if (c >= cols_valid) return;
  double acc = 0.0;
  for (uint32_t k = 0; k < splits; ++k) acc += partial[(static_cast<uint64_t>(k) * sample_ct_padded + s) * cg + c];
  out[static_cast<uint64_t>(s) * out_rs + static_cast<uint64_t>(c) * out_cs] += acc * scale;
}

static __global__ void scale_kernel(double* __restrict__ x, uint64_t n, double s) {
  const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) x[i] *= s;
}

}  // namespace pl2
