// king_ts_kernel.cuh - KING pair counts on the int8 tensor pipe (wgmma, sm_90a).
//
//   D[r][c] += sum_v A_plane[r][v] * B_plane[c][v],  planes T (het), H (hom), S (+1 hom-REF / -1 hom-ALT),
// exact int32 sums, the raw accumulator semantics of king_kernels.cuh.  One CTA = 64 rows (half of a 128-row
// pair tile) x kCols columns, two warpgroups:
//   warpgroup 0:  T_I x T_J -> TT,  T_I x H_J -> TH,  S_I x S_J, columns [0, kS)
//   warpgroup 1:  H_I x T_J -> HT,  H_I x H_J -> HH,  S_I x S_J, columns [kCols - kS, kCols)
// so that each thread keeps ~100-120 int32 accumulators in registers for the whole variant loop (the 64 x 5 kCols
// accumulators of a half tile are 100-120 KB; a whole 128-row tile would not fit the register file).  Both
// warpgroups issue the same shapes (ptxas serialises a wgmma under a branch), so for 80 columns the S x S halves
// overlap by 16 columns and warpgroup 1 stores only its last 32.
//
// Both operands come from the sample-major copy of the staged block written by geno_tile_rows_kernel
// (raw_t[sample / 128][k-step][sample % 128][8 bytes = 32 variants]): K-major, which is what an 8-bit wgmma
// reads.  Row side (A): each thread expands only its own fragment bytes straight into registers (wgmma.cuh).
// Column side (B): all 256 threads expand the 3 planes of the kCols column samples into the K-major no-swizzle
// layout in shared memory, one 256-variant stage ahead of the tensor pipe (double buffer, one __syncthreads per
// stage); the row-side words of the stage are copied next to it.
#pragma once

#include "common.cuh"
#include "geno_expand.cuh"
#include "geno_tile.cuh"
#include "wgmma.cuh"

namespace pl2 {

constexpr uint32_t kTsAccCols = 5 * kTsCols;   // 400
constexpr uint32_t kTsTileAccWords = kTsAccCols * kTileRows;

constexpr uint32_t kKwKs = 8;                    // k32 steps per shared-memory stage (256 variants)
constexpr uint32_t kKwThreads = 256;             // two warpgroups
constexpr uint32_t kKwChunkBytes = 128;          // LBO: next 16-variant chunk (core matrix) of the same 8 samples
constexpr uint32_t kKwSbo = 2 * kKwKs * kKwChunkBytes;  // 2048: next group of 8 samples
constexpr uint32_t kKwABytes = kKwKs * 64 * 8;   // row-side words of one stage: [k-step][64 rows][8 B]

template <uint32_t kCols>
struct KingWgShape {
  static constexpr uint32_t kBBytes = 3 * kCols * 32 * kKwKs;  // planes T | H | S stacked along N
  static constexpr uint32_t kStageBytes = kBBytes + kKwABytes;
  static constexpr uint32_t kSmemBytes = 2 * kStageBytes + 128;
  static constexpr uint32_t kS = (kCols / 2 + 15) / 16 * 16;  // S x S columns per warpgroup (wgmma N: multiple of 16)
  static constexpr uint32_t kItems = kCols * kKwKs;             // (column sample, k-step) words per stage
  static constexpr uint32_t kItemsPerThread = (kItems + kKwThreads - 1) / kKwThreads;
  static_assert(kCols % 16 == 0 && 2 * kS >= kCols, "wgmma N");
  static_assert(kSmemBytes <= 232448, "exceeds the 227 KB shared-memory opt-in limit");
};

template <int N>
__device__ __forceinline__ void king_acc_add(int32_t* base, const int32_t (&d)[N / 2], uint32_t r, uint32_t c, int j0 = 0) {
  // base -> accumulator column 0 of this block, row 0 of the tile; fragment (j, i): column 8 j + 2 c + (i & 1),
  // row r + 8 (i >> 1); column groups j < j0 are skipped
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    if (j < j0) continue;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int32_t* p = base + static_cast<uint64_t>(8 * j + 2 * c + (i & 1)) * kTileRows + r + 8 * (i >> 1);
      *p += d[4 * j + i];
    }
  }
}

// raw_t: sample-major copy of the whole padded block (sample 0 at row tile 0); kstep_ct = variant_ct_padded / 32.
// Grid: 2 CTAs per tile (blockIdx.x & 1 = row half).
template <uint32_t kCols>
__global__ void __launch_bounds__(kKwThreads, 1)
king_wg_kernel(const uint8_t* __restrict__ raw_t, uint32_t variant_ct_padded /* multiple of 256 */, const uint32_t* __restrict__ tile_order, const uint32_t* __restrict__ tile_rt, const uint32_t* __restrict__ tile_tc, int32_t* __restrict__ raw_acc) {
  using S = KingWgShape<kCols>;
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t tid = threadIdx.x;
  const uint32_t wg = tid >> 7;
  const uint32_t warp4 = (tid >> 5) & 3;
  const uint32_t lane = tid & 31;
  const uint32_t g = lane >> 2, c = lane & 3;
  const uint32_t tile = tile_order[blockIdx.x >> 1];
  const uint32_t half = blockIdx.x & 1;
  const uint32_t rt = tile_rt[tile];
  const uint32_t ct = tile_tc[tile];
  const uint32_t kstep_ct = variant_ct_padded / 32;
  const uint32_t stage_ct = kstep_ct / kKwKs;
  const uint32_t smem_base = (static_cast<uint32_t>(__cvta_generic_to_shared(smem)) + 127u) & ~127u;

  const uint32_t thread_zero = tid * (variant_ct_padded >> 31);  // 0; keeps the plane tables in vector registers
  const uint32_t tab_t = table_reg(kTabHet, thread_zero), tab_h = table_reg(kTabHom, thread_zero), tab_s = table_reg(kTabSgn, thread_zero);

  // ---- staging: this thread's share of a stage (column-side words + one 16-byte piece of the row-side words)
  const uint8_t* a_src = raw_t + static_cast<uint64_t>(rt) * kstep_ct * 1024 + half * 512 + (tid >> 5) * 1024 + (tid & 31) * 16;
  // tid / 32 = k-step of the stage, (tid % 32) * 16 = byte of the 512-byte half row block
  struct Pre {
    uint2 w[S::kItemsPerThread];
    uint4 a;
  };
  auto load_stage = [&](uint32_t st) -> Pre {
    Pre p;
#pragma unroll
    for (uint32_t q = 0; q < S::kItemsPerThread; ++q) {
      const uint32_t i = tid + q * kKwThreads;
      p.w[q] = make_uint2(0xFFFFFFFFu, 0xFFFFFFFFu);
      if (i < S::kItems) {
        const uint32_t n = (i & 7) | (((i >> 3) % (kCols / 8)) << 3);
        const uint32_t ks = st * kKwKs + (i >> 3) / (kCols / 8);
        const uint32_t s = kCols * ct + n;
        p.w[q] = __ldg(reinterpret_cast<const uint2*>(raw_t + (static_cast<uint64_t>(s >> 7) * kstep_ct + ks) * 1024 + (s & 127) * 8));
      }
    }
    p.a = __ldg(reinterpret_cast<const uint4*>(a_src + static_cast<uint64_t>(st) * kKwKs * 1024));
    return p;
  };
  auto store_stage = [&](const Pre& p, uint32_t buf) {
    const uint32_t base = smem_base + buf * S::kStageBytes;
#pragma unroll
    for (uint32_t q = 0; q < S::kItemsPerThread; ++q) {
      const uint32_t i = tid + q * kKwThreads;
      if (i < S::kItems) {
        const uint32_t n = (i & 7) | (((i >> 3) % (kCols / 8)) << 3);
        const uint32_t ks = (i >> 3) / (kCols / 8);
        const uint32_t tabs[3] = {tab_t, tab_h, tab_s};
#pragma unroll
        for (uint32_t h = 0; h < 2; ++h) {
          const Sel4 sel = make_selectors(h ? p.w[q].y : p.w[q].x);
#pragma unroll
          for (uint32_t pl = 0; pl < 3; ++pl) {
            const uint32_t row = pl * kCols + n;
            const uint32_t addr = base + (row >> 3) * kKwSbo + (2 * ks + h) * kKwChunkBytes + (row & 7) * 16;
            const uint4 v = expand16(tabs[pl], sel);
            asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
          }
        }
      }
    }
    const uint32_t a_addr = base + S::kBBytes + tid * 16;
    asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(a_addr), "r"(p.a.x), "r"(p.a.y), "r"(p.a.z), "r"(p.a.w) : "memory");
  };

  int32_t acc_x[kCols / 2], acc_y[kCols / 2], acc_s[S::kS / 2];
#pragma unroll
  for (uint32_t i = 0; i < kCols / 2; ++i) acc_x[i] = acc_y[i] = 0;
#pragma unroll
  for (uint32_t i = 0; i < S::kS / 2; ++i) acc_s[i] = 0;
  const uint32_t s_first = wg ? kCols - S::kS : 0;  // first S x S column of this warpgroup

  const uint32_t tab_a = wg ? tab_h : tab_t;
  const uint32_t r_lo = 16 * warp4 + g;  // this thread's fragment rows r_lo, r_lo + 8 of the 64-row half

  {
    const Pre p0 = load_stage(0);
    store_stage(p0, 0);
  }
  for (uint32_t st = 0; st < stage_ct; ++st) {
    const uint32_t buf = st & 1;
    Pre next;
    const bool more = st + 1 < stage_ct;
    if (more) next = load_stage(st + 1);
    fence_proxy_async_smem();
    __syncthreads();  // stage st complete in shared memory; every wgmma of stage st - 1 (other buffer) has retired
    const uint32_t base = smem_base + buf * S::kStageBytes;
    const uint64_t desc_t = make_wg_desc(base, kKwChunkBytes, kKwSbo);
    constexpr uint32_t kPlaneStep = (kCols / 8) * kKwSbo;
#pragma unroll
    for (uint32_t ks = 0; ks < kKwKs; ++ks) {
      const uint32_t a_row = base + S::kBBytes + ks * 512;
      uint2 w_lo, w_hi;
      asm volatile("ld.shared.v2.b32 {%0,%1}, [%2];" : "=r"(w_lo.x), "=r"(w_lo.y) : "r"(a_row + r_lo * 8) : "memory");
      asm volatile("ld.shared.v2.b32 {%0,%1}, [%2];" : "=r"(w_hi.x), "=r"(w_hi.y) : "r"(a_row + (r_lo + 8) * 8) : "memory");
      const ASel sel = make_asel(w_lo, w_hi, c);
      uint32_t fa[4], fs[4];
      afrag(tab_a, sel, fa);
      afrag(tab_s, sel, fs);
      const uint64_t dk = desc_t + ((ks * 2 * kKwChunkBytes) >> 4);
      wgmma_fence();
      wgmma_s8_rs<kCols>(acc_x, fa, dk);                                   // x T_J
      wgmma_s8_rs<kCols>(acc_y, fa, dk + (kPlaneStep >> 4));               // x H_J
      wgmma_s8_rs<S::kS>(acc_s, fs, dk + ((2 * kPlaneStep + (s_first / 8) * kKwSbo) >> 4));
      wgmma_commit();
      wgmma_wait<1>();
      if (ks == kKwKs / 2 && more) store_stage(next, buf ^ 1);  // the other buffer: its wgmmas retired before the barrier
    }
    wgmma_wait<0>();
  }

  // ---- epilogue: registers -> raw accumulators (+=); rows are in natural sample order
  int32_t* acc_tile = raw_acc + static_cast<uint64_t>(tile) * (5ull * kCols * kTileRows);
  const uint32_t r = 64 * half + r_lo;
  king_acc_add<kCols>(acc_tile + static_cast<uint64_t>((wg ? 2 : 0) * kCols) * kTileRows, acc_x, r, c);  // TT | HT
  king_acc_add<kCols>(acc_tile + static_cast<uint64_t>((wg ? 3 : 1) * kCols) * kTileRows, acc_y, r, c);  // TH | HH
  // warpgroup 1 skips the columns warpgroup 0 already covers
  king_acc_add<S::kS>(acc_tile + static_cast<uint64_t>(4 * kCols + s_first) * kTileRows, acc_s, r, c, wg ? static_cast<int>((2 * S::kS - kCols) / 8) : 0);
}

}  // namespace pl2
