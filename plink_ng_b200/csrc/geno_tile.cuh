// geno_tile.cuh - sample-major re-tiling for the tensor kernels (king_ts_kernel.cuh, grm_ts_kernel.cuh,
// pca_ts_kernels.cuh): an 8-bit wgmma reads both operands K-major, i.e. the variants of one sample contiguous.
// Kernels are static (header is included by several translation units).
#pragma once
#include "common.cuh"

namespace pl2 {

// 128 x 80 pair tiles (the GRM tiling).
constexpr uint32_t kTsCols = 80;
constexpr uint32_t kTsSamplePad = 640;  // lcm(128, 80)
// 128 x 64 pair tiles (the default KING tiling); its blocks keep the 640-sample padding.
constexpr uint32_t kKingTsCols = 64;
static_assert(kTsSamplePad % 128 == 0 && kTsSamplePad % kKingTsCols == 0, "padded samples: whole row and column tiles");
// One plane image: the four bit planes T | H | R | A of one 64-sample column tile over one k256 step (king_b1_kernel).
constexpr uint32_t kKingPlaneStepBytes = 4 * kKingTsCols * 32;

// ---- operand re-tiling of the staged block raw[variant][pitch] (2-bit, variant-major) -------------
// kSplitBits = false (GRM, PCA and king_wg_kernel):
//   raw_i[row tile rt][k-step ks][row 0..127][8 bytes]   8 bytes = 32 variants of one sample, the 2-bit codes,
//   variant 32 k + v at bits 2 v, 2 v + 1 (the staged block's own form).
//   One CTA = 64 variants x 64 samples through a shared-memory byte tile.
// kSplitBits = true (the default KING path, king_b1_kernel):
//   raw_i[row tile rt][k256 step][row 0..127][64 bytes]   64 bytes = 256 variants of one sample as eight 8-byte words
//   {lo32, hi32}: bit v of lo32 is the low code bit of variant 32 k + v, bit v of hi32 its high bit (its bit planes are
//   single LOP3s of these halves).  The eight words of a k256 step are stored in the order of k32 words
//   0, 4, 1, 5, 2, 6, 3, 7, so 16-byte chunk c holds words c and c + 4: the two k32 steps that thread c of a quad
//   needs for its binary wgmma A fragment registers of one row.  Same size as the 2-bit form.
//   One CTA = 256 variants (one k256 step) x 64 samples, so each sample's 64-byte piece is written whole.
//   The same CTA also writes the plane image of its 64 samples (one column tile of the default KING kernel) and step:
//   planes[sample / 64][k256 step][plane T | H | R | A][sample % 64 / 8][core matrix h][sample % 8][16 B], with
//   T = lo & ~hi, H = ~lo, R = ~(lo | hi), A = ~lo & hi, core matrix h = k32 words 4 h .. 4 h + 3 as the 16-byte
//   little-endian image of their 32-bit words: the K-major, no-swizzle shared-memory layout of a wgmma B operand
//   (LBO 128 B, SBO 256 B), copied to shared memory as is.  Code 3 (missing, padding) is zero in every plane.
//   Twice the size of the split copy.
// Only samples [s_base, s_base + 64 * gridDim.y) are written (a job re-tiles its own row tiles only);
// row tile s_base / 128 is stored at index 0.
template <bool kSplitBits = false>
static __global__ void __launch_bounds__(256) geno_tile_rows_kernel(const uint8_t* __restrict__ raw, uint32_t pitch, uint32_t kstep_ct, uint32_t s_base, uint8_t* __restrict__ raw_i, uint8_t* __restrict__ planes = nullptr) {
  const uint32_t t = threadIdx.x;
  if constexpr (kSplitBits) {
    // codes[v][word ^ ((v >> 5) & 3)]: the 64 samples of variant v as four 32-bit words of 16 samples each.  The
    // XOR keeps both phases conflict-free: a warp stores 32 variants x 16 B contiguously, and in the read phase the
    // warp's four 16-byte chunks c read variant 32 c + i (or 32 (c + 4) + i) of the same 16-sample word, which the
    // XOR with c puts on four different banks (the eight samples of one chunk read the same word).
    __shared__ uint32_t codes[256][4];
    const uint32_t v0 = blockIdx.x * 256, s0 = s_base + blockIdx.y * 64;
    {
      const uint4 w = *reinterpret_cast<const uint4*>(raw + static_cast<uint64_t>(v0 + t) * pitch + s0 / 4);
      const uint32_t x = (t >> 5) & 3;
      const uint32_t w01[2] = {x & 1 ? w.y : w.x, x & 1 ? w.x : w.y}, w23[2] = {x & 1 ? w.w : w.z, x & 1 ? w.z : w.w};
      const uint4 o = x & 2 ? make_uint4(w23[0], w23[1], w01[0], w01[1]) : make_uint4(w01[0], w01[1], w23[0], w23[1]);
      *reinterpret_cast<uint4*>(&codes[t][0]) = o;
    }
    __syncthreads();
    // sample s0 + sl, chunk c: words c and c + 4 of the k256 step
    const uint32_t sl = t >> 2, c = t & 3;
    const uint32_t col = (sl >> 4) ^ c, sh = 2 * (sl & 15);
    uint32_t lo[2] = {0, 0}, hi[2] = {0, 0};
#pragma unroll
    for (uint32_t h = 0; h < 2; ++h) {
#pragma unroll
      for (uint32_t i = 0; i < 32; ++i) {
        const uint32_t code = codes[32 * (c + 4 * h) + i][col] >> sh;
        lo[h] |= (code & 1u) << i;
        hi[h] |= ((code >> 1) & 1u) << i;
      }
    }
    const uint32_t s = s0 + sl;
    *reinterpret_cast<uint4*>(raw_i + (static_cast<uint64_t>((s - s_base) >> 7) * (kstep_ct / 8) + blockIdx.x) * 8192 + (s & 127) * 64 + 16 * c) = make_uint4(lo[0], hi[0], lo[1], hi[1]);
    // word c of core matrix h is k32 word c + 4 h: a quad writes a sample's 16 bytes, a warp 8 samples' 128 bytes
    uint8_t* img = planes + (static_cast<uint64_t>((s - s_base) >> 6) * (kstep_ct / 8) + blockIdx.x) * kKingPlaneStepBytes + (sl >> 3) * 256 + (sl & 7) * 16 + 4 * c;
#pragma unroll
    for (uint32_t h = 0; h < 2; ++h) {
      const uint32_t pl[4] = {lo[h] & ~hi[h], ~lo[h], ~(lo[h] | hi[h]), ~lo[h] & hi[h]};
#pragma unroll
      for (uint32_t p = 0; p < 4; ++p) *reinterpret_cast<uint32_t*>(img + p * (kKingPlaneStepBytes / 4) + h * 128) = pl[p];
    }
  } else {
    __shared__ uint8_t tile[64][68];
    const uint32_t v0 = blockIdx.x * 64, s0 = s_base + blockIdx.y * 64;
    {
      const uint32_t v = t >> 2, sw = t & 3;
      const uint32_t w = *reinterpret_cast<const uint32_t*>(raw + static_cast<uint64_t>(v0 + v) * pitch + s0 / 4 + 4 * sw);
#pragma unroll
      for (uint32_t j = 0; j < 16; ++j) tile[v][16 * sw + j] = static_cast<uint8_t>((w >> (2 * j)) & 3u);
    }
    __syncthreads();
    {
      const uint32_t sl = t >> 2, vw = t & 3;
      uint32_t w = 0;
#pragma unroll
      for (uint32_t j = 0; j < 16; ++j) w |= static_cast<uint32_t>(tile[16 * vw + j][sl]) << (2 * j);
      const uint32_t s = s0 + sl, v = v0 + 16 * vw;
      *reinterpret_cast<uint32_t*>(raw_i + (static_cast<uint64_t>((s - s_base) >> 7) * kstep_ct + (v >> 5)) * 1024 + (s & 127) * 8 + 4 * ((v >> 4) & 1)) = w;
    }
  }
}

}  // namespace pl2
