// grm_ts_kernel.cuh - GRM contraction on the int8 tensor pipe (wgmma, sm_90a).  Same math, digit tables and
// accumulator semantics as grm_kernels.cuh, which documents the fixed-point digit decomposition:
//   D_l += g_I x d1_l,J + m_I x d2_l,J   (l = 0..4),   obs += m_I x m_J.
//
// One CTA = 64 rows (half of a 128-row tile) x 80 columns, two warpgroups with int32 accumulators in registers:
//   warpgroup 0: D_0, D_1, D_2;  warpgroup 1: D_3, D_4, obs (+ g x a zero plane, so that both warpgroups issue
//   the same six wgmmas per k32 step: a wgmma under a branch is serialised).
// Row side (A): planes g, m expanded by each thread straight into its fragment registers from the sample-major
// copy (wgmma.cuh).  Column side (B): 11 planes of the 80 column samples in the K-major no-swizzle layout in shared
// memory, one 64-variant stage ahead (double buffer).  A K-major row holds 16 variants of one sample, each with its
// own digit table, so a byte cannot come from one PRMT table as on the row side: the stage's tables are kept as
// three 16-byte vectors per (16-variant chunk, plane) - the digit for genotype 0, 1, 2 of each variant, in the K
// order of the fragments - and a row is (t0 & mask0) | (t1 & mask1) | (t2 & mask2) with byte masks of the codes.
#pragma once

#include "common.cuh"
#include "geno_expand.cuh"
#include "geno_tile.cuh"
#include "grm_kernels.cuh"
#include "wgmma.cuh"

namespace pl2 {

static_assert(kGrmTileCols == kTsCols && kGrmSamplePad == kTsSamplePad, "GRM shares the KING tiling");
constexpr uint32_t kGwKs = 2;                                        // k32 steps per stage (64 variants)
constexpr uint32_t kGwThreads = 256;
constexpr uint32_t kGwSbo = 2 * kGwKs * kCoreBytes;                  // 512: next group of 8 B rows
constexpr uint32_t kGwZeroPlane = kGrmPlanesJ;                       // plane 11: zeros
constexpr uint32_t kGwRowsB = (kGrmPlanesJ + 1) * kGrmTileCols;      // 960 B rows: planes 0..11 stacked along N
constexpr uint32_t kGwBBytes = kGwRowsB * 32 * kGwKs;                // 61440
constexpr uint32_t kGwABytes = kGwKs * 64 * 8;                       // 1024
constexpr uint32_t kGwTabBytes = (32 * kGwKs / 16) * kGrmTabChunkBytes;  // 1920
constexpr uint32_t kGwStageBytes = kGwBBytes + kGwABytes + kGwTabBytes;
constexpr uint32_t kGwSmemBytes = 2 * kGwStageBytes + 128;
constexpr uint32_t kGwItems = kGrmTileCols * 2 * kGwKs;              // (column sample, 16-variant chunk) per stage
static_assert(kGwSmemBytes <= 232448, "exceeds the 227 KB shared-memory opt-in limit");
static_assert(kGwTabBytes % 16 == 0, "staging granularity");

template <int N>
__device__ __forceinline__ void grm_acc_zero(int32_t (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) d[i] = 0;
}

// raw_t: sample-major copy of the whole padded block; tabk: grm_tables_kernel output.  Grid: 2 CTAs per tile.
__global__ void __launch_bounds__(kGwThreads, 1)
grm_wg_kernel(const uint8_t* __restrict__ raw_t, uint32_t variant_ct_padded /* multiple of 256 */, const uint8_t* __restrict__ tabk, double inv_scale, const uint32_t* __restrict__ tile_order, const uint32_t* __restrict__ tile_rt, const uint32_t* __restrict__ tile_tc, double* __restrict__ acc_g, int32_t* __restrict__ acc_obs) {
  extern __shared__ __align__(128) uint8_t smem_dyn[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 127) & ~static_cast<uintptr_t>(127));
  const uint32_t smem_base = static_cast<uint32_t>(__cvta_generic_to_shared(smem));
  const uint32_t tid = threadIdx.x, wg = tid >> 7, warp4 = (tid >> 5) & 3, lane = tid & 31, g = lane >> 2, c = lane & 3;
  const uint32_t tile = tile_order[blockIdx.x >> 1];
  const uint32_t half = blockIdx.x & 1;
  const uint32_t rt = tile_rt[tile], ct = tile_tc[tile];
  const uint32_t kstep_ct = variant_ct_padded / 32;
  const uint32_t stage_ct = kstep_ct / kGwKs;
  const uint32_t thread_zero = tid * (variant_ct_padded >> 31);
  const uint32_t tab_g = table_reg(kTabDosage, thread_zero), tab_m = table_reg(kTabNonmiss, thread_zero);
  const uint32_t mask0 = table_reg(0x000000FFu, thread_zero), mask1 = table_reg(0x0000FF00u, thread_zero), mask2 = table_reg(0x00FF0000u, thread_zero);

  // ---- staging of one stage: column words (registers), row words and tables (16-byte pieces)
  constexpr uint32_t kItemsPerThread = (kGwItems + kGwThreads - 1) / kGwThreads;
  struct Pre {
    uint32_t w[kItemsPerThread];
    uint2 a;
    uint4 t[(kGwTabBytes / 16 + kGwThreads - 1) / kGwThreads];
  };
  auto load_stage = [&](uint32_t st) -> Pre {
    Pre p;
#pragma unroll
    for (uint32_t q = 0; q < kItemsPerThread; ++q) {
      const uint32_t i = tid + q * kGwThreads;
      p.w[q] = 0xFFFFFFFFu;
      if (i < kGwItems) {
        const uint32_t n = i % kGrmTileCols, kc = i / kGrmTileCols;  // a warp shares its chunk: broadcast table reads
        const uint32_t s = kGrmTileCols * ct + n, ks = st * kGwKs + (kc >> 1);
        p.w[q] = __ldg(reinterpret_cast<const uint32_t*>(raw_t + (static_cast<uint64_t>(s >> 7) * kstep_ct + ks) * 1024 + (s & 127) * 8 + 4 * (kc & 1)));
      }
    }
    {  // row words: [k-step][64 rows][8 B]; thread = (k-step, row)
      const uint32_t ks = st * kGwKs + (tid >> 7), row = 64 * half + (tid & 63);
      p.a = (tid & 64) ? make_uint2(0, 0) : __ldg(reinterpret_cast<const uint2*>(raw_t + (static_cast<uint64_t>(rt) * kstep_ct + ks) * 1024 + row * 8));
    }
#pragma unroll
    for (uint32_t q = 0; q < sizeof(p.t) / 16; ++q) {
      const uint32_t i = tid + q * kGwThreads;
      if (i < kGwTabBytes / 16) p.t[q] = __ldg(reinterpret_cast<const uint4*>(tabk + static_cast<uint64_t>(st) * kGwTabBytes) + i);
    }
    return p;
  };
  auto sts128 = [](uint32_t addr, const uint4& v) { asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory"); };
  auto lds128 = [](uint32_t addr) -> uint4 {
    uint4 v;
    asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
    return v;
  };
  // part 1: row words and tables into shared memory (the tables feed part 2 of the same stage)
  auto store_stage_raw = [&](const Pre& p, uint32_t buf) {
    const uint32_t base = smem_base + buf * kGwStageBytes;
    if (!(tid & 64)) asm volatile("st.shared.v2.b32 [%0], {%1,%2};" ::"r"(base + kGwBBytes + (tid >> 7) * 512 + (tid & 63) * 8), "r"(p.a.x), "r"(p.a.y) : "memory");
#pragma unroll
    for (uint32_t q = 0; q < sizeof(p.t) / 16; ++q) {
      const uint32_t i = tid + q * kGwThreads;
      if (i < kGwTabBytes / 16) sts128(base + kGwBBytes + kGwABytes + 16 * i, p.t[q]);
    }
  };
  // part 2: column words -> 11 planes (needs the stage's tables in shared memory)
  auto store_stage_b = [&](const Pre& p, uint32_t buf) {
    const uint32_t base = smem_base + buf * kGwStageBytes;
    const uint32_t tabs = base + kGwBBytes + kGwABytes;
#pragma unroll
    for (uint32_t q = 0; q < kItemsPerThread; ++q) {
      const uint32_t i = tid + q * kGwThreads;
      if (i < kGwItems) {
        const uint32_t n = i % kGrmTileCols, kc = i / kGrmTileCols;
        const Sel4 sel = make_selectors(p.w[q]);
        const uint4 m0 = expand16(mask0, sel), m1 = expand16(mask1, sel), m2 = expand16(mask2, sel);
        const uint32_t dst = base + kc * kCoreBytes + (n & 7) * 16;
#pragma unroll
        for (uint32_t pl = 0; pl < 2 * kGrmLimbs; ++pl) {
          const uint32_t t = tabs + (kc * 2 * kGrmLimbs + pl) * 48;
          const uint4 t0 = lds128(t), t1 = lds128(t + 16), t2 = lds128(t + 32);
          uint4 v;
          v.x = (t0.x & m0.x) | (t1.x & m1.x) | (t2.x & m2.x);
          v.y = (t0.y & m0.y) | (t1.y & m1.y) | (t2.y & m2.y);
          v.z = (t0.z & m0.z) | (t1.z & m1.z) | (t2.z & m2.z);
          v.w = (t0.w & m0.w) | (t1.w & m1.w) | (t2.w & m2.w);
          const uint32_t row = pl * kGrmTileCols + n;
          sts128(dst + (row >> 3) * kGwSbo, v);
        }
        sts128(dst + ((2 * kGrmLimbs * kGrmTileCols + n) >> 3) * kGwSbo, expand16(tab_m, sel));  // plane 10: m
      }
    }
  };

  // warpgroup 0: D_0..D_2; warpgroup 1: D_3, D_4, obs
  int32_t da[kGrmTileCols / 2], db[kGrmTileCols / 2], dc[kGrmTileCols / 2];
  grm_acc_zero(da);
  grm_acc_zero(db);
  grm_acc_zero(dc);
  const uint32_t r_lo = 16 * warp4 + g;
  constexpr uint32_t kPlaneStep = (kGrmTileCols / 8) * kGwSbo;  // 5120 bytes between planes
  const uint32_t l0 = wg ? 3 : 0;                                // first digit of this warpgroup

  {
    constexpr uint32_t kZeroBytes = kGrmTileCols * 32 * kGwKs;
    for (uint32_t i = tid; i < 2 * kZeroBytes / 16; i += kGwThreads) {
      const uint32_t buf = i / (kZeroBytes / 16);
      sts128(smem_base + buf * kGwStageBytes + kGwZeroPlane * kZeroBytes + 16 * (i % (kZeroBytes / 16)), make_uint4(0, 0, 0, 0));
    }
    const Pre p0 = load_stage(0);
    store_stage_raw(p0, 0);
    __syncthreads();
    store_stage_b(p0, 0);
  }
  for (uint32_t st = 0; st < stage_ct; ++st) {
    const uint32_t buf = st & 1;
    const bool more = st + 1 < stage_ct;
    Pre next;
    if (more) next = load_stage(st + 1);
    fence_proxy_async_smem();
    __syncthreads();  // stage st in shared memory; the other buffer's wgmmas have retired
    if (more) store_stage_raw(next, buf ^ 1);
    const uint32_t base = smem_base + buf * kGwStageBytes;
    const uint64_t desc = make_wg_desc(base, kCoreBytes, kGwSbo);
#pragma unroll
    for (uint32_t ks = 0; ks < kGwKs; ++ks) {
      uint2 w_lo, w_hi;
      asm volatile("ld.shared.v2.b32 {%0,%1}, [%2];" : "=r"(w_lo.x), "=r"(w_lo.y) : "r"(base + kGwBBytes + ks * 512 + r_lo * 8) : "memory");
      asm volatile("ld.shared.v2.b32 {%0,%1}, [%2];" : "=r"(w_hi.x), "=r"(w_hi.y) : "r"(base + kGwBBytes + ks * 512 + (r_lo + 8) * 8) : "memory");
      const ASel sel = make_asel(w_lo, w_hi, c);
      uint32_t fg[4], fm[4];
      afrag(tab_g, sel, fg);
      afrag(tab_m, sel, fm);
      const uint64_t dk = desc + ((ks * 2 * kCoreBytes) >> 4);
      auto plane = [&](uint32_t pl) { return dk + ((pl * kPlaneStep) >> 4); };
      wgmma_fence();
      wgmma_s8_rs<kGrmTileCols>(da, fg, plane(l0));
      wgmma_s8_rs<kGrmTileCols>(da, fm, plane(kGrmLimbs + l0));
      wgmma_s8_rs<kGrmTileCols>(db, fg, plane(l0 + 1));
      wgmma_s8_rs<kGrmTileCols>(db, fm, plane(kGrmLimbs + l0 + 1));
      wgmma_s8_rs<kGrmTileCols>(dc, fg, plane(wg ? kGwZeroPlane : 2));
      wgmma_s8_rs<kGrmTileCols>(dc, fm, plane(wg ? 2 * kGrmLimbs : kGrmLimbs + 2));  // warpgroup 1: obs = m x m
      wgmma_commit();
      wgmma_wait<1>();
    }
    if (more) {
      __syncthreads();  // the next stage's tables are in shared memory
      store_stage_b(next, buf ^ 1);
    }
    wgmma_wait<0>();
  }

  // ---- epilogue: D = D_0 + 2^8 D_1 + ... + 2^32 D_4 in int64 (warpgroup 1 hands 2^24 D_3 + 2^32 D_4 over through
  // shared memory), then one fp64 add into acc_g and one int32 add into acc_obs per element
  __syncthreads();  // operand buffers are free
  long long* part = reinterpret_cast<long long*>(smem);  // [64 rows][80 columns]
  const uint32_t r = 64 * half + r_lo;
  if (wg == 1) {
#pragma unroll
    for (uint32_t j = 0; j < kGrmTileCols / 8; ++j)
#pragma unroll
      for (uint32_t i = 0; i < 4; ++i) {
        const uint32_t col = 8 * j + 2 * c + (i & 1), row = r_lo + 8 * (i >> 1);
        part[row * kGrmTileCols + col] = (static_cast<long long>(da[4 * j + i]) << 24) + (static_cast<long long>(db[4 * j + i]) << 32);
        int32_t* o = acc_obs + static_cast<uint64_t>(tile) * kGrmTileWords + static_cast<uint64_t>(col) * kTileRows + r + 8 * (i >> 1);
        *o += dc[4 * j + i];
      }
  }
  __syncthreads();
  if (wg == 0) {
#pragma unroll
    for (uint32_t j = 0; j < kGrmTileCols / 8; ++j)
#pragma unroll
      for (uint32_t i = 0; i < 4; ++i) {
        const uint32_t col = 8 * j + 2 * c + (i & 1), row = r_lo + 8 * (i >> 1);
        const long long tot = static_cast<long long>(da[4 * j + i]) + (static_cast<long long>(db[4 * j + i]) << 8) + (static_cast<long long>(dc[4 * j + i]) << 16) + part[row * kGrmTileCols + col];
        double* o = acc_g + static_cast<uint64_t>(tile) * kGrmTileWords + static_cast<uint64_t>(col) * kTileRows + r + 8 * (i >> 1);
        *o += static_cast<double>(tot) * inv_scale;
      }
  }
}

}  // namespace pl2
