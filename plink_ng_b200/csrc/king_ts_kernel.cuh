// king_ts_kernel.cuh - KING pair counts on the tensor pipe (wgmma, sm_90a).
//
//   D[r][c] += sum_v A_plane[r][v] * B_plane[c][v],  planes T (het), H (hom), S (+1 hom-REF / -1 hom-ALT),
// exact int32 sums, the raw accumulator semantics of king_kernels.cuh.  Two kernels:
//   king_b1_kernel        the default (`tensor_ts`): binary AND-POPC wgmma on bit planes, one CTA per 128 x 64 pair
//                         tile (described below it)
//   king_wg_kernel<96>    the `tensor` algorithm, an independent int8 cross-check: two CTAs per 128 x 96 pair tile
//
// king_wg_kernel: one CTA = 64 rows (half of a 128-row pair tile) x kCols columns, three warpgroups:
//   warpgroup 0:  producer - stages the operands of the variant loop in a ring of shared-memory stages
//   warpgroup 1:  T_I x T_J -> TT,  T_I x H_J -> TH,  S_I x S_J, columns [0, kS)
//   warpgroup 2:  H_I x T_J -> HT,  H_I x H_J -> HH,  S_I x S_J, columns [kCols - kS, kCols)
// so that each consumer thread keeps ~100-120 int32 accumulators in registers for the whole variant loop (the
// 64 x 5 kCols accumulators of a half tile are 100-120 KB; a whole 128-row tile would not fit the register file).
// Both consumers issue the same shapes (ptxas serialises a wgmma under a branch), so where kCols / 2 is not a
// multiple of 16 the S x S halves overlap and warpgroup 2 stores only the columns warpgroup 1 does not cover.
//
// Both operands come from the sample-major copy of the staged block written by geno_tile_rows_kernel
// (raw_t[sample / 128][k-step][sample % 128][8 bytes = 32 variants]): K-major, which is what an 8-bit wgmma
// reads.  Column side (B): the producer loads the words of the kCols column samples one stage ahead in registers
// and expands them into the 3 planes, K-major no-swizzle layout; it copies the stage's row-side words next to
// them.  Row side (A): each consumer thread expands only its own fragment bytes from those words straight into
// registers (wgmma.cuh).  Each stage has a `full` mbarrier (the producer's 128 threads arrive after their
// stores) and an `empty` one (the consumers' 256 threads arrive once every wgmma reading the stage has
// retired), so the staging runs on its own warps while the consumers keep one wgmma group in flight across
// stage boundaries; nothing in the variant loop waits for the whole CTA.
#pragma once

#include "common.cuh"
#include "geno_expand.cuh"
#include "geno_tile.cuh"
#include "wgmma.cuh"

namespace pl2 {

constexpr uint32_t kKingTsTileAccWords = 5 * kKingTsCols * kTileRows;

constexpr uint32_t kKwProducerThreads = 128;  // warpgroup 0
constexpr uint32_t kKwConsumerThreads = 256;  // warpgroups 1, 2
constexpr uint32_t kKwThreads = kKwProducerThreads + kKwConsumerThreads;
constexpr uint32_t kKwChunkBytes = 128;       // LBO: next 16-variant chunk (core matrix) of the same 8 samples
constexpr uint32_t kKwSmemLimit = 232448;     // the 227 KB shared-memory opt-in

template <uint32_t kCols>
struct KingWgShape {
  // k32 steps per stage: 8 (256 variants) where three such stages fit the opt-in, else 4; both divide the
  // 256-variant padding unit
  static constexpr uint32_t stage_bytes(uint32_t ks) { return 3 * kCols * 32 * ks + ks * 64 * 8; }
  static constexpr uint32_t kKs = 3 * stage_bytes(8) + 256 <= kKwSmemLimit ? 8 : 4;
  static constexpr uint32_t kSbo = 2 * kKs * kKwChunkBytes;          // next group of 8 samples
  static constexpr uint32_t kBBytes = 3 * kCols * 32 * kKs;          // planes T | H | S stacked along N
  static constexpr uint32_t kABytes = kKs * 64 * 8;                  // row-side words: [k-step][64 rows][8 B]
  static constexpr uint32_t kStageBytes = kBBytes + kABytes;
  static constexpr uint32_t kStages = (kKwSmemLimit - 256) / kStageBytes < 4 ? (kKwSmemLimit - 256) / kStageBytes : 4;
  static constexpr uint32_t kSmemBytes = kStages * kStageBytes + 128 + 2 * kStages * 8;  // + alignment + mbarriers
  static constexpr uint32_t kS = (kCols / 2 + 15) / 16 * 16;  // S x S columns per consumer (wgmma N: multiple of 16)
  static constexpr uint32_t kItems = kCols * kKs;              // (column sample, k-step) words per stage
  static constexpr uint32_t kItemsPerThread = (kItems + kKwProducerThreads - 1) / kKwProducerThreads;
  static constexpr uint32_t kAPerThread = kABytes / 16 / kKwProducerThreads;  // 16-byte pieces of the row-side words
  static_assert(kCols % 16 == 0 && 2 * kS >= kCols, "wgmma N");
  static_assert(kStages >= 3, "the ring needs at least three stages");
  static_assert(kABytes % (16 * kKwProducerThreads) == 0, "row-side copy");
  static_assert(kSmemBytes <= kKwSmemLimit, "exceeds the 227 KB shared-memory opt-in limit");
};

// kRed = false: a load and a store per accumulator; true: one fire-and-forget `red.global.add.s32` instead, so the
// thread waits for no load round trip (integer addition is exact and order-free; the kernel boundary orders the
// reductions before anything that reads the counts)
template <int N, bool kRed = false>
__device__ __forceinline__ void king_acc_add(int32_t* base, const int32_t (&d)[N / 2], uint32_t r, uint32_t c, int j0 = 0) {
  // base -> accumulator column 0 of this block, row 0 of the tile; fragment (j, i): column 8 j + 2 c + (i & 1),
  // row r + 8 (i >> 1); column groups j < j0 are skipped
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    if (j < j0) continue;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int32_t* p = base + static_cast<uint64_t>(8 * j + 2 * c + (i & 1)) * kTileRows + r + 8 * (i >> 1);
      if constexpr (kRed) {
        asm volatile("red.global.add.s32 [%0], %1;" ::"l"(p), "r"(d[4 * j + i]) : "memory");
      } else {
        *p += d[4 * j + i];
      }
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
  const uint32_t tile = tile_order[blockIdx.x >> 1];
  const uint32_t half = blockIdx.x & 1;
  const uint32_t rt = tile_rt[tile];
  const uint32_t ct = tile_tc[tile];
  const uint32_t kstep_ct = variant_ct_padded / 32;
  const uint32_t stage_ct = kstep_ct / S::kKs;
  const uint32_t smem_base = (static_cast<uint32_t>(__cvta_generic_to_shared(smem)) + 127u) & ~127u;
  const uint32_t bar_full = smem_base + S::kStages * S::kStageBytes;  // full[s] = bar_full + 8 s
  const uint32_t bar_empty = bar_full + S::kStages * 8;               // empty[s] = bar_empty + 8 s
  if (tid == 0) {
    for (uint32_t s = 0; s < S::kStages; ++s) {
      mbar_init(bar_full + 8 * s, kKwProducerThreads);
      mbar_init(bar_empty + 8 * s, kKwConsumerThreads);
    }
  }
  __syncthreads();

  const uint32_t thread_zero = tid * (variant_ct_padded >> 31);  // 0; keeps the plane tables in vector registers
  const uint32_t tab_t = table_reg(kTabHet, thread_zero), tab_h = table_reg(kTabHom, thread_zero), tab_s = table_reg(kTabSgn, thread_zero);

  if (wg == 0) {
    // ---- producer: this thread's share of a stage (column-side words + 16-byte pieces of the row-side words)
    // Item i of a stage = (column sample n, k-step ks); its global word and its shared-memory rows move by a
    // whole stage from one stage to the next, so both offsets are computed once.
    const uint8_t* w_src[S::kItemsPerThread];
    uint32_t w_dst[S::kItemsPerThread];  // plane T, first 16 variants; H and S follow kCols rows apart
#pragma unroll
    for (uint32_t q = 0; q < S::kItemsPerThread; ++q) {
      const uint32_t i = tid + q * kKwProducerThreads;
      const uint32_t n = (i & 7) | (((i >> 3) % (kCols / 8)) << 3);
      const uint32_t ks = (i >> 3) / (kCols / 8);
      const uint32_t s = kCols * ct + n;
      w_src[q] = raw_t + (static_cast<uint64_t>(s >> 7) * kstep_ct + ks) * 1024 + (s & 127) * 8;
      w_dst[q] = (n >> 3) * S::kSbo + 2 * ks * kKwChunkBytes + (n & 7) * 16;
    }
    auto has_item = [&](uint32_t q) { return S::kItems % kKwProducerThreads == 0 || tid + q * kKwProducerThreads < S::kItems; };
    const uint8_t* a_src = raw_t + static_cast<uint64_t>(rt) * kstep_ct * 1024 + half * 512;
    struct Pre {
      uint2 w[S::kItemsPerThread];
      uint4 a[S::kAPerThread];
    };
    auto load_stage = [&](uint32_t st) -> Pre {
      Pre p;
      const uint64_t stage_off = static_cast<uint64_t>(st) * S::kKs * 1024;
#pragma unroll
      for (uint32_t q = 0; q < S::kItemsPerThread; ++q) {
        p.w[q] = make_uint2(0xFFFFFFFFu, 0xFFFFFFFFu);
        if (has_item(q)) p.w[q] = __ldg(reinterpret_cast<const uint2*>(w_src[q] + stage_off));
      }
#pragma unroll
      for (uint32_t q = 0; q < S::kAPerThread; ++q) {
        const uint32_t i = tid + q * kKwProducerThreads;  // i / 32 = k-step of the stage, (i % 32) * 16 = byte of the 512-byte half row block
        p.a[q] = __ldg(reinterpret_cast<const uint4*>(a_src + stage_off + (i >> 5) * 1024 + (i & 31) * 16));
      }
      return p;
    };
    auto store_stage = [&](const Pre& p, uint32_t base) {
      const uint32_t tabs[3] = {tab_t, tab_h, tab_s};
#pragma unroll
      for (uint32_t q = 0; q < S::kItemsPerThread; ++q) {
        if (has_item(q)) {
          const uint32_t addr = base + w_dst[q];
#pragma unroll
          for (uint32_t h = 0; h < 2; ++h) {
            const Sel4 sel = make_selectors(h ? p.w[q].y : p.w[q].x);
#pragma unroll
            for (uint32_t pl = 0; pl < 3; ++pl) {
              const uint4 v = expand16(tabs[pl], sel);
              asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(addr + pl * (kCols / 8) * S::kSbo + h * kKwChunkBytes), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
            }
          }
        }
      }
#pragma unroll
      for (uint32_t q = 0; q < S::kAPerThread; ++q) {
        const uint32_t a_addr = base + S::kBBytes + (tid + q * kKwProducerThreads) * 16;
        asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(a_addr), "r"(p.a[q].x), "r"(p.a[q].y), "r"(p.a[q].z), "r"(p.a[q].w) : "memory");
      }
    };

    // Words are loaded two stages ahead and issued after the previous stage's hand-off: the proxy fence (a
    // MEMBAR.ALL.CTA in SASS) waits for every memory access of this thread in flight, so loads issued just before
    // it would hold up the hand-off.  Near the end the last stage is loaded again; it is never stored twice.
    const uint32_t last = stage_ct - 1;
    Pre cur = load_stage(0), next = load_stage(last ? 1 : 0);
    uint32_t slot = 0, phase = 0;
    for (uint32_t st = 0; st < stage_ct; ++st) {
      // the first pass over the ring finds every slot free: parity 1 is the phase before a fresh barrier's first
      mbar_wait(bar_empty + 8 * slot, phase ^ 1);
      store_stage(cur, smem_base + slot * S::kStageBytes);
      fence_proxy_async_smem();  // this thread's st.shared -> visible to the consumers' wgmma operand fetch
      mbar_arrive(bar_full + 8 * slot);
      cur = next;
      next = load_stage(st + 2 < last ? st + 2 : last);
      if (++slot == S::kStages) slot = 0, phase ^= 1;
    }
    return;
  }

  // ---- consumers
  const uint32_t cw = wg - 1;  // 0: T_I rows, 1: H_I rows
  const uint32_t warp4 = (tid >> 5) & 3;
  const uint32_t lane = tid & 31;
  const uint32_t g = lane >> 2, c = lane & 3;
  int32_t acc_x[kCols / 2], acc_y[kCols / 2], acc_s[S::kS / 2];
#pragma unroll
  for (uint32_t i = 0; i < kCols / 2; ++i) acc_x[i] = acc_y[i] = 0;
#pragma unroll
  for (uint32_t i = 0; i < S::kS / 2; ++i) acc_s[i] = 0;
  const uint32_t s_first = cw ? kCols - S::kS : 0;  // first S x S column of this warpgroup

  const uint32_t tab_a = cw ? tab_h : tab_t;
  const uint32_t r_lo = 16 * warp4 + g;  // this thread's fragment rows r_lo, r_lo + 8 of the 64-row half

  uint32_t slot = 0, phase = 0, prev_slot = 0;
  for (uint32_t st = 0; st < stage_ct; ++st) {
    mbar_wait(bar_full + 8 * slot, phase);
    const uint32_t base = smem_base + slot * S::kStageBytes;
    const uint64_t desc_t = make_wg_desc(base, kKwChunkBytes, S::kSbo);
    constexpr uint32_t kPlaneStep = (kCols / 8) * S::kSbo;
#pragma unroll
    for (uint32_t ks = 0; ks < S::kKs; ++ks) {
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
      wgmma_s8_rs<S::kS>(acc_s, fs, dk + ((2 * kPlaneStep + (s_first / 8) * S::kSbo) >> 4));
      wgmma_commit();
      wgmma_wait<1>();
      // every group but the one just issued has retired, the previous stage's last one included: hand that slot back
      if (ks == 0 && st > 0) mbar_arrive(bar_empty + 8 * prev_slot);
    }
    prev_slot = slot;
    if (++slot == S::kStages) slot = 0, phase ^= 1;
  }
  wgmma_wait<0>();

  // ---- epilogue: registers -> raw accumulators (+=); rows are in natural sample order
  int32_t* acc_tile = raw_acc + static_cast<uint64_t>(tile) * (5ull * kCols * kTileRows);
  const uint32_t r = 64 * half + r_lo;
  king_acc_add<kCols>(acc_tile + static_cast<uint64_t>((cw ? 2 : 0) * kCols) * kTileRows, acc_x, r, c);  // TT | HT
  king_acc_add<kCols>(acc_tile + static_cast<uint64_t>((cw ? 3 : 1) * kCols) * kTileRows, acc_y, r, c);  // TH | HH
  // warpgroup 2 skips the columns warpgroup 1 already covers
  king_acc_add<S::kS>(acc_tile + static_cast<uint64_t>(4 * kCols + s_first) * kTileRows, acc_s, r, c, cw ? static_cast<int>((2 * S::kS - kCols) / 8) : 0);
}

// ---------------------------------------------------------------------------------------------------------------
// king_b1_kernel: the KING counts as AND-popcounts of bit planes on the binary tensor pipe (wgmma .b1 AND.POPC,
// m64nNk256).  From the low and high bits (lo, hi) of each 2-bit code:
//   T = lo & ~hi (het),  H = ~lo (hom),  R = ~lo & ~hi (hom-REF),  A = ~lo & hi (hom-ALT);
// missing data and padding (code 3) are zero in every plane.  The prep stream writes two copies of each staged block
// (geno_tile_rows_kernel<true>): the split sample-major copy (row side, {lo32, hi32} words) and the column planes,
// one 8 KB image per 64-sample column tile and k256 step, byte for byte what the B descriptor reads.  So the kernel
// is a pure bulk-copy -> wgmma pipeline.  One CTA = one whole 128 x 64 pair tile, three warpgroups:
//   warpgroup 0:  producer.  Thread 0 refills a slot of the ring as soon as the consumers have handed it back: the
//                 stage's row words and its plane images, bulk copies onto the slot's `full` mbarrier (tx count).
//   warpgroups 1, 2:  consumer c owns rows 64 c .. 64 c + 63.  Per k256 step it turns its own row words straight
//                 into fragment registers and issues   T_I x [T_J | H_J] (n128) -> TT | TH,
//                 H_I x [T_J | H_J] (n128) -> HT | HH,   R_I x A_J + A_I x R_J (n64, one accumulator) -> IBS0:
//                 160 int32 accumulators per thread, which fit once `setmaxnreg` moves registers from the producer
//                 (40) to the consumers (232).  The row words of the next k256 step are loaded while this step's
//                 group is being issued, so only LOP3s stand between a retired group and the next one.
// The epilogue writes SS = HH - 2 IBS0 (= the int8 form's S_I x S_J with S = R - A), so the raw accumulator layout
// {TT, TH, HT, HH, SS} is that of king_wg_kernel.  `empty` collects one arrival per consumer warp once
// `wgmma.wait_group 1` has retired the stage; one wgmma group stays in flight across stage boundaries.  A stage holds
// kKb1Ks k256 steps; the last one may be short (the block is padded to 256 variants only): its missing steps are not
// copied, and their row fragments are zero, so whatever the slot holds there adds nothing.
//
// kCluster = 2: the CTAs of a cluster run tiles (rt, ct) and (rt + 1, ct), which read the same plane images.  Each
// CTA copies its own row words and half of every plane image, multicast into both CTAs, so a tile still reads
// 12 KB from L2 per k256 step (8 KB of rows, 4 KB of planes).  A CTA's `full` barrier therefore also counts the
// partner's bytes, and a producer may refill a slot only once the consumers of both CTAs have released it: every
// consumer warp arrives on `empty` of both CTAs.  The tiles without a partner run with kCluster = 1.  The cluster
// barrier after the barrier set-up keeps copies and remote arrivals away from a barrier that is not yet initialised;
// the one before exit keeps a CTA alive while its partner may still copy into it or arrive on it.
// The epilogue adds the tile's counts with `red.global.add` (king_acc_add<.., true>): nothing waits for a load, and
// the consumers arrive on the exit barrier before it and wait after it, so the barrier's release fence does not wait
// for the reductions either.
constexpr uint32_t kKb1Ks = 2;       // k256 steps per stage
constexpr uint32_t kKb1Stages = 7;
constexpr uint32_t kKb1Sbo = 2 * kKwChunkBytes;                          // next group of 8 samples of a plane image
constexpr uint32_t kKb1PlaneBytes = (kKingTsCols / 8) * kKb1Sbo;         // one plane of the 64 column samples
constexpr uint32_t kKb1BStepBytes = 4 * kKb1PlaneBytes;                  // T | H | R | A of one k256 step
constexpr uint32_t kKb1SampleBytes = 64;                                 // one sample's words of one k256 step
constexpr uint32_t kKb1AStepBytes = kTileRows * kKb1SampleBytes;         // row words of one k256 step
constexpr uint32_t kKb1BBytes = kKb1Ks * kKb1BStepBytes;                 // [k256 step][plane image]
constexpr uint32_t kKb1ABytes = kKb1Ks * kKb1AStepBytes;                 // [k256 step][128 rows][64 B]
constexpr uint32_t kKb1StageBytes = kKb1BBytes + kKb1ABytes;
constexpr uint32_t kKb1SmemBytes = kKb1Stages * kKb1StageBytes + 128 + 2 * kKb1Stages * 8;  // + alignment + mbarriers
constexpr uint32_t kKb1ConsumerWarps = kKwConsumerThreads / 32;
static_assert(kKb1BStepBytes == kKingPlaneStepBytes, "plane image of geno_tile_rows_kernel<true>");
static_assert(kKb1SmemBytes <= kKwSmemLimit, "exceeds the 227 KB shared-memory opt-in limit");

// raw_t: split sample-major copy of the whole padded block (sample 0 at row tile 0),
// [sample / 128][k256 step][sample % 128][64 B], each 8-byte word {lo32, hi32} of 32 variants; planes: its plane
// images, [sample / 64][k256 step][8 KB] (geno_tile.cuh).  Grid: one CTA per tile, consecutive pairs of CTAs form a
// cluster when kCluster = 2 (tile_order lists the two tiles of a pair next to each other).
template <uint32_t kCluster>
__global__ void __launch_bounds__(kKwThreads, 1)
king_b1_kernel(const uint8_t* __restrict__ raw_t, const uint8_t* __restrict__ planes, uint32_t variant_ct_padded /* multiple of 256 */, const uint32_t* __restrict__ tile_order, const uint32_t* __restrict__ tile_rt, const uint32_t* __restrict__ tile_tc, int32_t* __restrict__ raw_acc) {
  static_assert(kCluster == 1 || kCluster == 2, "a tile pair at most");
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t tid = threadIdx.x;
  const uint32_t wg = tid >> 7;
  const uint32_t tile = tile_order[blockIdx.x];
  const uint32_t rt = tile_rt[tile];
  const uint32_t ct = tile_tc[tile];
  const uint32_t k256_ct = variant_ct_padded / 256;
  const uint32_t stage_ct = (k256_ct + kKb1Ks - 1) / kKb1Ks;
  // the same offset in every CTA of the cluster: multicast copies and remote arrivals address the partner with it
  const uint32_t smem_base = (static_cast<uint32_t>(__cvta_generic_to_shared(smem)) + 127u) & ~127u;
  const uint32_t bar_full = smem_base + kKb1Stages * kKb1StageBytes;  // full[s] = bar_full + 8 s
  const uint32_t bar_empty = bar_full + kKb1Stages * 8;
  if (tid == 0) {
    for (uint32_t s = 0; s < kKb1Stages; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, kCluster * kKb1ConsumerWarps);
    }
    mbar_init_fence();
  }
  // the partner copies into this CTA and arrives on its barriers only after they are initialised
  if constexpr (kCluster > 1) {
    cluster_sync();
  } else {
    __syncthreads();
  }

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (tid == 0) {
      // ---- producer: row words [k256 step][128 rows][64 B] of row tile rt, plane images of column tile ct
      const uint32_t rank = kCluster > 1 ? cluster_cta_rank() : 0;
      constexpr uint32_t kBPart = kKb1BStepBytes / kCluster;  // this CTA's part of each plane image
      const uint8_t* a_src = raw_t + static_cast<uint64_t>(rt) * k256_ct * kKb1AStepBytes;
      const uint8_t* b_src = planes + static_cast<uint64_t>(ct) * k256_ct * kKb1BStepBytes + rank * kBPart;
      for (uint32_t st = 0; st < stage_ct; ++st) {
        const uint32_t slot = st % kKb1Stages;
        // the first pass over the ring finds every slot free (parity 1 = the phase before a fresh barrier's first)
        const uint32_t parity = ((st / kKb1Stages) & 1) ^ 1;
        mbar_wait(bar_empty + 8 * slot, parity);
        const uint32_t base = smem_base + slot * kKb1StageBytes;
        const uint32_t bar = bar_full + 8 * slot;
        const uint32_t steps = min(kKb1Ks, k256_ct - st * kKb1Ks);
        const uint64_t k0 = static_cast<uint64_t>(st) * kKb1Ks;
        mbar_arrive_expect_tx(bar, steps * (kKb1AStepBytes + kKb1BStepBytes));
        bulk_copy_g2s(base + kKb1BBytes, a_src + k0 * kKb1AStepBytes, steps * kKb1AStepBytes, bar);
        if constexpr (kCluster > 1) {
          for (uint32_t j = 0; j < steps; ++j)
            bulk_copy_g2s_multicast(base + j * kKb1BStepBytes + rank * kBPart, b_src + (k0 + j) * kKb1BStepBytes, kBPart, bar, (1u << kCluster) - 1);
        } else {
          bulk_copy_g2s(base, b_src + k0 * kKb1BStepBytes, steps * kKb1BStepBytes, bar);
        }
      }
    }
    // the partner may still copy into this CTA and arrive on its barriers until it has passed the same point
    __syncwarp();
    if constexpr (kCluster > 1) cluster_sync();
    return;
  }

  // ---- consumers
  setmaxnreg_inc<232>();
  const uint32_t cw = wg - 1;
  const uint32_t warp4 = (tid >> 5) & 3;
  const uint32_t lane = tid & 31;
  const uint32_t g = lane >> 2, c = lane & 3;
  int32_t acc_t[kKingTsCols], acc_h[kKingTsCols], acc_i[kKingTsCols / 2];  // TT | TH, HT | HH, IBS0 (n128, n128, n64)
#pragma unroll
  for (uint32_t i = 0; i < kKingTsCols; ++i) acc_t[i] = acc_h[i] = 0;
#pragma unroll
  for (uint32_t i = 0; i < kKingTsCols / 2; ++i) acc_i[i] = 0;
  const uint32_t r_lo = 64 * cw + 16 * warp4 + g;  // this thread's fragment rows r_lo, r_lo + 8 of the tile

  // Fragment register q: row r_lo + 8 (q & 1), K bits 32 (c + 4 (q >> 1)) .. of the step = k32 step c + 4 (q >> 1).
  // Chunk c of a row's 64 bytes holds exactly k32 words c and c + 4, so a thread's words of a k256 step are two
  // LDS.128, one per row; a warp's 8 rows x 64 B are 512 contiguous bytes, 4 wavefronts without a conflict.
  // w[0] = {lo, hi of k32 word c, lo, hi of word c + 4} of row r_lo, w[1] the same of row r_lo + 8.
  uint4 w[2];
  auto load_words = [&](uint32_t base, uint32_t j) {
    const uint32_t a = base + kKb1BBytes + j * kKb1AStepBytes + r_lo * kKb1SampleBytes + 16 * c;
    asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(w[0].x), "=r"(w[0].y), "=r"(w[0].z), "=r"(w[0].w) : "r"(a) : "memory");
    asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(w[1].x), "=r"(w[1].y), "=r"(w[1].z), "=r"(w[1].w) : "r"(a + 8 * kKb1SampleBytes) : "memory");
  };
  // The words of step j + 1 are loaded right after step j's group is issued and before the wait that retires step
  // j - 1's group; the first step of the next stage only after that stage's `full` wait.  Every word load from a
  // slot has been consumed by the LOP3s of its step before the slot is handed back.
  uint32_t slot = 0, phase = 0, prev_slot = 0;
  mbar_wait(bar_full, 0);
  load_words(smem_base, 0);
  for (uint32_t st = 0; st < stage_ct; ++st) {
    const uint32_t base = smem_base + slot * kKb1StageBytes;
    const uint32_t steps = min(kKb1Ks, k256_ct - st * kKb1Ks);
    const uint32_t next_slot = slot + 1 == kKb1Stages ? 0 : slot + 1;
    const uint32_t next_phase = slot + 1 == kKb1Stages ? phase ^ 1 : phase;
    const uint64_t desc = make_wg_desc(base, kKwChunkBytes, kKb1Sbo);  // plane image of step j: + j * kKb1BStepBytes
#pragma unroll
    for (uint32_t j = 0; j < kKb1Ks; ++j) {
      const uint32_t lo[4] = {w[0].x, w[1].x, w[0].z, w[1].z}, hi[4] = {w[0].y, w[1].y, w[0].w, w[1].w};
      uint32_t ft[4], fh[4], fr[4], fa[4];
#pragma unroll
      for (uint32_t q = 0; q < 4; ++q) {
        ft[q] = lo[q] & ~hi[q];
        fh[q] = ~lo[q];
        fr[q] = ~(lo[q] | hi[q]);
        fa[q] = ~lo[q] & hi[q];
      }
      const uint64_t dk = desc + ((j * kKb1BStepBytes) >> 4);
      wgmma_fence();
      wgmma_b1_rs<2 * kKingTsCols>(acc_t, ft, dk);                               // x [T_J | H_J]
      wgmma_b1_rs<2 * kKingTsCols>(acc_h, fh, dk);                               // x [T_J | H_J]
      wgmma_b1_rs<kKingTsCols>(acc_i, fr, dk + ((3 * kKb1PlaneBytes) >> 4));     // R_I x A_J
      wgmma_b1_rs<kKingTsCols>(acc_i, fa, dk + ((2 * kKb1PlaneBytes) >> 4));     // + A_I x R_J
      wgmma_commit();
      if (j + 1 < kKb1Ks) {
        if (j + 1 < steps) {
          load_words(base, j + 1);
        } else {
          w[0] = w[1] = make_uint4(~0u, ~0u, ~0u, ~0u);  // missing step: code 3, zero planes
        }
      } else if (st + 1 < stage_ct) {
        mbar_wait(bar_full + 8 * next_slot, next_phase);
        load_words(smem_base + next_slot * kKb1StageBytes, 0);
      }
      wgmma_wait<1>();
      // every group but the one just issued has retired, the previous stage's last one included: hand that slot back,
      // to the producers of both CTAs of a cluster
      if (j == 0 && st > 0) {
        __syncwarp();
        if (lane == 0) {
          if constexpr (kCluster > 1) {
#pragma unroll
            for (uint32_t cta = 0; cta < kCluster; ++cta) mbar_arrive_cluster(bar_empty + 8 * prev_slot, cta);
          } else {
            mbar_arrive(bar_empty + 8 * prev_slot);
          }
        }
      }
    }
    prev_slot = slot;
    slot = next_slot, phase = next_phase;
  }
  // the exit barrier's arrive: this thread's last remote arrival is behind it, and its release (a fence of every
  // global access in flight) comes before the epilogue's reductions
  if constexpr (kCluster > 1) cluster_arrive();
  wgmma_wait<0>();
  wgmma_fence_operand(acc_t);
  wgmma_fence_operand(acc_h);
  wgmma_fence_operand(acc_i);

  // ---- epilogue: registers -> raw accumulators (red.global.add); rows are in natural sample order.  HH column
  // 8 j + .. sits in acc_h[32 + 4 j + i], the IBS0 of the same pair in acc_i[4 j + i]: SS = HH - 2 IBS0 in place.
#pragma unroll
  for (uint32_t i = 0; i < kKingTsCols / 2; ++i) acc_i[i] = acc_h[kKingTsCols / 2 + i] - 2 * acc_i[i];
  int32_t* acc_tile = raw_acc + static_cast<uint64_t>(tile) * kKingTsTileAccWords;
  king_acc_add<2 * kKingTsCols, true>(acc_tile, acc_t, r_lo, c);                                                   // TT | TH
  king_acc_add<2 * kKingTsCols, true>(acc_tile + static_cast<uint64_t>(2 * kKingTsCols) * kTileRows, acc_h, r_lo, c);  // HT | HH
  king_acc_add<kKingTsCols, true>(acc_tile + static_cast<uint64_t>(4 * kKingTsCols) * kTileRows, acc_i, r_lo, c);      // SS
  if constexpr (kCluster > 1) cluster_wait();
}

}  // namespace pl2
