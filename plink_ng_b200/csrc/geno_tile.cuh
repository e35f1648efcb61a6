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

// ---- operand re-tiling of the staged block raw[variant][pitch] (2-bit, variant-major) -------------
// Row side:  raw_i[row tile rt][k-step ks][row 0..127][8 bytes]   8 bytes = 32 variants of one sample
// One CTA = 64 variants x 64 samples through a shared-memory byte tile.
// Only samples [s_base, s_base + 64 * gridDim.y) are written (a job re-tiles its own row tiles only);
// row tile s_base / 128 is stored at index 0.
// The 8 bytes of a word hold, by kSplitBits:
//   false  the 2-bit codes, variant 32 k + v at bits 2 v, 2 v + 1 (the staged block's own form; GRM, PCA and
//          king_wg_kernel read this)
//   true   {lo32, hi32}: bit v of lo32 is the low code bit of variant 32 k + v, bit v of hi32 its high bit (the
//          default KING path, king_b1_kernel: its bit planes are single LOP3s of these halves)
template <bool kSplitBits = false>
static __global__ void __launch_bounds__(256) geno_tile_rows_kernel(const uint8_t* __restrict__ raw, uint32_t pitch, uint32_t kstep_ct, uint32_t s_base, uint8_t* __restrict__ raw_i) {
  __shared__ uint8_t tile[64][68];
  const uint32_t v0 = blockIdx.x * 64, s0 = s_base + blockIdx.y * 64;
  const uint32_t t = threadIdx.x;
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
    if constexpr (kSplitBits) {
      uint32_t lo = 0, hi = 0;
#pragma unroll
      for (uint32_t j = 0; j < 16; ++j) {
        const uint32_t code = tile[16 * vw + j][sl];
        lo |= (code & 1u) << j;
        hi |= (code >> 1) << j;
      }
      // lanes t, t ^ 1 hold the two 16-variant halves of one word: the even lane writes lo32, the odd one hi32
      const uint32_t odd = vw & 1;
      const uint32_t other = __shfl_xor_sync(0xFFFFFFFFu, odd ? lo : hi, 1);
      w = odd ? other | (hi << 16) : lo | (other << 16);
    } else {
#pragma unroll
      for (uint32_t j = 0; j < 16; ++j) w |= static_cast<uint32_t>(tile[16 * vw + j][sl]) << (2 * j);
    }
    const uint32_t s = s0 + sl, v = v0 + 16 * vw;
    *reinterpret_cast<uint32_t*>(raw_i + (static_cast<uint64_t>((s - s_base) >> 7) * kstep_ct + (v >> 5)) * 1024 + (s & 127) * 8 + 4 * ((v >> 4) & 1)) = w;
  }
}

}  // namespace pl2
