// king_kernels.cuh - device kernels of the KING-robust pair-count path.
//
// Replaces the reference's IncrKing / IncrKingHomhom (2.0/plink2_matrix_calc.cc:1255-1334) and
// the SplitHomRef2hetUnsafeW + TransposeBitblock staging in front of it (:2055-2099).
//
// Device-resident accumulators ("raw tiles"): for every 128 x 96 pair tile, int32
//   raw[tile][q * 96 + c][r],  q in {TT, TH, HT, HH, SS},  r = row sample - 128*rt (larger index),
//   c = col sample - 96*tc (smaller index),
// with T = het indicator, H = hom indicator, S = +1 hom-REF / -1 hom-ALT:
//   TT = HETHET, TH = (row het, col hom) = HET2HOM1, HT = HET1HOM2, HH = HOMHOM,
//   SS = HH - 2*IBS0  (so IBS0 = (HH - SS) / 2, always an exact integer).
// Both algorithms (popcount and int8 wgmma) accumulate into the same layout, bit-identically.
#pragma once
#include "common.cuh"
#include "geno_expand.cuh"
#include "cp_async.cuh"

namespace pl2 {

// ---------------------------------------------------------------------------------------------
// Staging: force samples >= sample_ct and variant rows >= variant_ct of the padded raw block to
// "missing" (SetTrailingNyps, plink2_matrix_calc.cc:2060; zero-filled block tail, :2089-2099).
// raw: [variant_ct_padded][pitch bytes], pitch = sample_ct_padded / 4.
// ---------------------------------------------------------------------------------------------
__global__ void pad_genotypes_kernel(uint8_t* __restrict__ raw, uint32_t pitch, uint32_t sample_ct, uint32_t variant_ct, uint32_t variant_ct_padded) {
  const uint32_t v = blockIdx.x;
  if (v >= variant_ct_padded) return;
  uint8_t* row = raw + static_cast<uint64_t>(v) * pitch;
  if (v >= variant_ct) {
    for (uint32_t b = threadIdx.x; b < pitch; b += blockDim.x) row[b] = 0xFF;
    return;
  }
  const uint32_t first = sample_ct >> 2;
  const uint32_t rem = sample_ct & 3;
  for (uint32_t b = first + threadIdx.x; b < pitch; b += blockDim.x) {
    if (b == first && rem) {
      row[b] = row[b] | static_cast<uint8_t>(0xFFu << (2 * rem));
    } else {
      row[b] = 0xFF;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Popcount path, step 1: variant-major 2-bit -> sample-addressable bit planes
//   planes[p][kw][s], p in {hom, ref2het, het}, kw = 32-variant word index, s = sample.
// One warp transposes a 32-variant x 32-sample block with ballots (lane = variant on input,
// lane = sample on output); reads are 8-byte, writes 128-byte coalesced.
// Algorithmic bytes: N*M/4 read + 3*N*M/8 written.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) split_transpose_kernel(const uint8_t* __restrict__ raw, uint32_t pitch, uint32_t sample_ct_padded, uint32_t word_ct /* variant_ct_padded / 32 */, uint32_t* __restrict__ planes) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warp_in_block = threadIdx.x >> 5;
  const uint32_t sample_groups = sample_ct_padded >> 5;
  const uint64_t warp_global = static_cast<uint64_t>(blockIdx.x) * (blockDim.x >> 5) + warp_in_block;
  if (warp_global >= static_cast<uint64_t>(sample_groups) * word_ct) return;
  const uint32_t kw = static_cast<uint32_t>(warp_global / sample_groups);
  const uint32_t sg = static_cast<uint32_t>(warp_global % sample_groups);
  const uint64_t w = *reinterpret_cast<const uint64_t*>(raw + static_cast<uint64_t>(kw * 32 + lane) * pitch + static_cast<uint64_t>(sg) * 8);
  uint32_t my_hom = 0, my_r2h = 0, my_het = 0;
#pragma unroll
  for (uint32_t s = 0; s < 32; ++s) {
    const uint32_t code = static_cast<uint32_t>(w >> (2 * s)) & 3u;
    const uint32_t hom = __ballot_sync(0xFFFFFFFFu, (code & 1u) == 0u);
    const uint32_t r2h = __ballot_sync(0xFFFFFFFFu, (code & 2u) == 0u);
    const uint32_t het = __ballot_sync(0xFFFFFFFFu, code == 1u);
    if (lane == s) {
      my_hom = hom;
      my_r2h = r2h;
      my_het = het;
    }
  }
  const uint64_t plane_words = static_cast<uint64_t>(word_ct) * sample_ct_padded;
  const uint64_t off = static_cast<uint64_t>(kw) * sample_ct_padded + sg * 32 + lane;
  planes[off] = my_hom;
  planes[plane_words + off] = my_r2h;
  planes[2 * plane_words + off] = my_het;
}

// ---------------------------------------------------------------------------------------------
// Popcount path, step 2: the IncrKingHomhom inner loop (plink2_matrix_calc.cc:1309-1322) as a
// register-tiled kernel.  One CTA = half a pair tile (64 rows x 96 cols); each of 256 threads owns
// a 4 x 6 block of pairs (5 counters each) and walks the variant words staged in shared memory by
// cp.async double buffering.  Per pair and 32 variants: 5 LOP3 + 5 POPC + 5 IADD.
// ---------------------------------------------------------------------------------------------
constexpr uint32_t kPopcKw = 8;  // 32-variant words per smem chunk

__global__ void __launch_bounds__(256, 1)
king_popc_kernel(const uint32_t* __restrict__ planes, uint32_t sample_ct_padded, uint32_t word_ct, const uint32_t* __restrict__ tile_rt, const uint32_t* __restrict__ tile_tc, int32_t* __restrict__ raw_acc) {
  __shared__ __align__(16) uint32_t s_rows[2][3][kPopcKw][64];
  __shared__ __align__(16) uint32_t s_cols[2][3][kPopcKw][96];
  const uint32_t tile = blockIdx.x >> 1;
  const uint32_t half = blockIdx.x & 1;
  const uint32_t row0 = tile_rt[tile] * kTileRows + half * 64;
  const uint32_t col0 = tile_tc[tile] * kTileCols;
  const uint32_t tid = threadIdx.x;
  const uint32_t ry = tid >> 4;  // rows 4*ry .. 4*ry+3
  const uint32_t cx = tid & 15;  // cols 6*cx .. 6*cx+5
  const uint64_t plane_words = static_cast<uint64_t>(word_ct) * sample_ct_padded;

  uint32_t cnt[4][6][5];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 6; ++b)
#pragma unroll
      for (int q = 0; q < 5; ++q) cnt[a][b][q] = 0;

  const uint32_t chunk_ct = word_ct / kPopcKw;
  auto issue = [&](uint32_t chunk, uint32_t buf) {
    // rows: 3 planes x kPopcKw words x 64 samples = 384 x 16B; cols: 3 x kPopcKw x 96 = 576 x 16B
    for (uint32_t i = tid; i < 960; i += 256) {
      if (i < 384) {
        const uint32_t p = i / 128, rem = i % 128, kk = rem / 16, seg = rem % 16;
        const uint32_t* src = planes + p * plane_words + static_cast<uint64_t>(chunk * kPopcKw + kk) * sample_ct_padded + row0 + seg * 4;
        cp_async16(&s_rows[buf][p][kk][seg * 4], src);
      } else {
        const uint32_t j = i - 384;
        const uint32_t p = j / 192, rem = j % 192, kk = rem / 24, seg = rem % 24;
        const uint32_t* src = planes + p * plane_words + static_cast<uint64_t>(chunk * kPopcKw + kk) * sample_ct_padded + col0 + seg * 4;
        cp_async16(&s_cols[buf][p][kk][seg * 4], src);
      }
    }
    cp_async_commit();
  };

  if (chunk_ct) issue(0, 0);
  for (uint32_t chunk = 0; chunk < chunk_ct; ++chunk) {
    const uint32_t buf = chunk & 1;
    if (chunk + 1 < chunk_ct) {
      issue(chunk + 1, buf ^ 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
#pragma unroll 2
    for (uint32_t kk = 0; kk < kPopcKw; ++kk) {
      const uint4 rh = *reinterpret_cast<const uint4*>(&s_rows[buf][0][kk][4 * ry]);
      const uint4 rr = *reinterpret_cast<const uint4*>(&s_rows[buf][1][kk][4 * ry]);
      const uint4 rt = *reinterpret_cast<const uint4*>(&s_rows[buf][2][kk][4 * ry]);
      const uint32_t row_h[4] = {rh.x, rh.y, rh.z, rh.w};
      const uint32_t row_r[4] = {rr.x, rr.y, rr.z, rr.w};
      const uint32_t row_t[4] = {rt.x, rt.y, rt.z, rt.w};
      uint32_t col_h[6], col_r[6], col_t[6];
#pragma unroll
      for (int b = 0; b < 6; b += 2) {
        const uint2 ch = *reinterpret_cast<const uint2*>(&s_cols[buf][0][kk][6 * cx + b]);
        const uint2 cr = *reinterpret_cast<const uint2*>(&s_cols[buf][1][kk][6 * cx + b]);
        const uint2 ct = *reinterpret_cast<const uint2*>(&s_cols[buf][2][kk][6 * cx + b]);
        col_h[b] = ch.x; col_h[b + 1] = ch.y;
        col_r[b] = cr.x; col_r[b + 1] = cr.y;
        col_t[b] = ct.x; col_t[b + 1] = ct.y;
      }
#pragma unroll
      for (int a = 0; a < 4; ++a) {
#pragma unroll
        for (int b = 0; b < 6; ++b) {
          const uint32_t hh = row_h[a] & col_h[b];
          cnt[a][b][0] += __popc(row_t[a] & col_t[b]);           // TT
          cnt[a][b][1] += __popc(row_t[a] & col_h[b]);           // TH: row het, col hom
          cnt[a][b][2] += __popc(row_h[a] & col_t[b]);           // HT
          cnt[a][b][3] += __popc(hh);                            // HH
          cnt[a][b][4] += __popc((row_r[a] ^ col_r[b]) & hh);    // IBS0
        }
      }
    }
    __syncthreads();
  }

  int32_t* acc_tile = raw_acc + static_cast<uint64_t>(tile) * kKingTileAccWords;
#pragma unroll
  for (int b = 0; b < 6; ++b) {
#pragma unroll
    for (int q = 0; q < 5; ++q) {
      int4* p = reinterpret_cast<int4*>(acc_tile + static_cast<uint64_t>(q * kTileCols + 6 * cx + b) * kTileRows + half * 64 + 4 * ry);
      int4 v = *p;
      if (q < 4) {
        v.x += cnt[0][b][q]; v.y += cnt[1][b][q]; v.z += cnt[2][b][q]; v.w += cnt[3][b][q];
      } else {  // SS = HH - 2 * IBS0
        v.x += static_cast<int32_t>(cnt[0][b][3]) - 2 * static_cast<int32_t>(cnt[0][b][4]);
        v.y += static_cast<int32_t>(cnt[1][b][3]) - 2 * static_cast<int32_t>(cnt[1][b][4]);
        v.z += static_cast<int32_t>(cnt[2][b][3]) - 2 * static_cast<int32_t>(cnt[2][b][4]);
        v.w += static_cast<int32_t>(cnt[3][b][3]) - 2 * static_cast<int32_t>(cnt[3][b][4]);
      }
      *p = v;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Tensor path: the same five counts as exact contractions on the tensor pipe (binary AND-POPC or int8),
// king_b1_kernel (128 x 64 tiles, the default) and king_wg_kernel<kTileCols> (king_ts_kernel.cuh).
// ---------------------------------------------------------------------------------------------

// ---------------------------------------------------------------------------------------------
// Finalisation: raw tiles -> the reference's in-memory results for rows [out_row_start, out_row_end).
//   counts : uint32 [pair][5] = {IBS0, HETHET, HET2HOM1, HET1HOM2, HOMHOM} (plink2_matrix_calc.cc:864-868)
//   kinship: fp64 per pair (ComputeKinship, :1566-1573)
// pair order: for j in rows: for i in [0, min(j, col_end))  (:1545-1547; col_end = sample_ct for a full triangle).
// One CTA per (tile, 16-row sub-block): coalesced tile reads -> smem -> row-contiguous writes.
// ---------------------------------------------------------------------------------------------
// Pairs (j, i) with j < r and i < min(j, col_end): the strict lower triangle cut at column col_end.
__host__ __device__ inline uint64_t KingPairsBelow(uint64_t r, uint64_t col_end) {
  if (r <= col_end) return r ? r * (r - 1) / 2 : 0;
  return (col_end ? col_end * (col_end - 1) / 2 : 0) + (r - col_end) * col_end;
}

template <bool kKinship, uint32_t kCols>
__global__ void __launch_bounds__(256)
king_finalize_kernel(const int32_t* __restrict__ raw_acc, const uint32_t* __restrict__ tile_rt, const uint32_t* __restrict__ tile_tc, uint32_t sample_ct, uint32_t col_end, uint32_t out_row_start, uint32_t out_row_end, uint32_t* __restrict__ out_counts, double* __restrict__ out_kinship) {
  __shared__ int32_t s_acc[16][(5 * kCols) + 1];
  const uint32_t tile = blockIdx.x >> 3;
  const uint32_t sub = blockIdx.x & 7;
  const uint32_t rt = tile_rt[tile];
  const uint32_t tc = tile_tc[tile];
  const uint32_t row_base = rt * kTileRows + sub * 16;
  if (row_base >= out_row_end || row_base + 16 <= out_row_start) return;
  const uint32_t col_base = tc * kCols;
  if (col_base + 1 > row_base + 15) return;  // no strict-lower-triangle pair in this block
  const int32_t* acc_tile = raw_acc + static_cast<uint64_t>(tile) * (5 * kCols * kTileRows) + sub * 16;
  const uint32_t r = threadIdx.x & 15;
  for (uint32_t cidx = threadIdx.x >> 4; cidx < (5 * kCols); cidx += 16) {
    s_acc[r][cidx] = acc_tile[static_cast<uint64_t>(cidx) * kTileRows + r];
  }
  __syncthreads();
  const uint64_t tri_base = KingPairsBelow(out_row_start, col_end);
  for (uint32_t rr = 0; rr < 16; ++rr) {
    const uint32_t j = row_base + rr;
    if (j < out_row_start || j >= out_row_end || j >= sample_ct) continue;
    const uint64_t pair_row = KingPairsBelow(j, col_end) - tri_base;
    if (kKinship) {
      for (uint32_t cl = threadIdx.x; cl < kCols; cl += 256) {
        const uint32_t i = col_base + cl;
        if (i >= j || i >= col_end) continue;
        const int32_t tt = s_acc[rr][cl];
        const int32_t th = s_acc[rr][kCols + cl];
        const int32_t ht = s_acc[rr][2 * kCols + cl];
        const int32_t hh = s_acc[rr][3 * kCols + cl];
        const int32_t ss = s_acc[rr][4 * kCols + cl];
        const int64_t ibs0 = (hh - ss) >> 1;
        const int64_t het2hom1 = th, het1hom2 = ht;
        const int64_t smaller_het = tt + (het1hom2 < het2hom1 ? het1hom2 : het2hom1);
        out_kinship[pair_row + i] = 0.5 - static_cast<double>(4 * ibs0 + het1hom2 + het2hom1) / static_cast<double>(4 * smaller_het);
      }
    } else {
      for (uint32_t idx = threadIdx.x; idx < kCols * 5; idx += 256) {
        const uint32_t cl = idx / 5, q = idx % 5;
        const uint32_t i = col_base + cl;
        if (i >= j || i >= col_end) continue;
        uint32_t val;
        if (q == 0) {
          val = static_cast<uint32_t>((s_acc[rr][3 * kCols + cl] - s_acc[rr][4 * kCols + cl]) >> 1);  // IBS0
        } else if (q == 1) {
          val = static_cast<uint32_t>(s_acc[rr][cl]);  // HETHET = TT
        } else if (q == 2) {
          val = static_cast<uint32_t>(s_acc[rr][kCols + cl]);  // HET2HOM1 = TH
        } else if (q == 3) {
          val = static_cast<uint32_t>(s_acc[rr][2 * kCols + cl]);  // HET1HOM2 = HT
        } else {
          val = static_cast<uint32_t>(s_acc[rr][3 * kCols + cl]);  // HOMHOM = HH
        }
        out_counts[(pair_row + i) * 5 + q] = val;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// `--king-table-filter` on the device: append only the pairs of rows [row_start, row_end) and columns
// below col_end whose kinship is not below `min_kinship` (NaN is kept, as the reference's `kinship < filter` test does,
// 2.0/plink2_matrix_calc.cc:2296-2300).  At 100k samples the unfiltered table is 5e9 pairs = 100 GB of
// counts; relationship screening keeps a few thousand of them.  One CTA per tile, thread = tile row.
// Slots are handed out with an atomic counter, so the output order is arbitrary (the host sorts).
// ---------------------------------------------------------------------------------------------
template <uint32_t kCols>
__global__ void __launch_bounds__(kTileRows)
king_filter_kernel(const int32_t* __restrict__ raw_acc, const uint32_t* __restrict__ tile_rt, const uint32_t* __restrict__ tile_tc, uint32_t sample_ct, uint32_t col_end, uint32_t row_start, uint32_t row_end, double min_kinship, unsigned long long max_out,
                   unsigned long long* __restrict__ found, uint32_t* __restrict__ out_pairs, uint32_t* __restrict__ out_counts, double* __restrict__ out_kinship) {
  const uint32_t tile = blockIdx.x;
  const uint32_t j = tile_rt[tile] * kTileRows + threadIdx.x;
  const uint32_t col_base = tile_tc[tile] * kCols;
  if (j < row_start || j >= row_end || j >= sample_ct) return;
  const int32_t* acc = raw_acc + static_cast<uint64_t>(tile) * (5 * kCols * kTileRows) + threadIdx.x;
  for (uint32_t cl = 0; cl < kCols; ++cl) {
    const uint32_t i = col_base + cl;
    if (i >= j || i >= col_end) break;
    const int32_t tt = acc[static_cast<uint64_t>(cl) * kTileRows];
    const int32_t th = acc[static_cast<uint64_t>(kCols + cl) * kTileRows];
    const int32_t ht = acc[static_cast<uint64_t>(2 * kCols + cl) * kTileRows];
    const int32_t hh = acc[static_cast<uint64_t>(3 * kCols + cl) * kTileRows];
    const int32_t ss = acc[static_cast<uint64_t>(4 * kCols + cl) * kTileRows];
    const int64_t ibs0 = (hh - ss) >> 1;
    const int64_t het2hom1 = th, het1hom2 = ht;
    const int64_t smaller_het = tt + (het1hom2 < het2hom1 ? het1hom2 : het2hom1);
    const double kinship = 0.5 - static_cast<double>(4 * ibs0 + het1hom2 + het2hom1) / static_cast<double>(4 * smaller_het);
    if (kinship < min_kinship) continue;
    const unsigned long long slot = atomicAdd(found, 1ull);
    if (slot >= max_out) continue;
    out_pairs[2 * slot] = j;
    out_pairs[2 * slot + 1] = i;
    uint32_t* c = out_counts + 5 * slot;
    c[0] = static_cast<uint32_t>(ibs0);
    c[1] = static_cast<uint32_t>(tt);
    c[2] = static_cast<uint32_t>(th);
    c[3] = static_cast<uint32_t>(ht);
    c[4] = static_cast<uint32_t>(hh);
    out_kinship[slot] = kinship;
  }
}

}  // namespace pl2
