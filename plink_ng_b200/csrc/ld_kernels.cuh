// ld_kernels.cuh - small genotype kernels of the --indep-pairwise path, also used by GRM and approx PCA:
// per-variant genotype counts (allele frequencies, the load-time monomorphic rule) and the sample gather that
// re-stages the LD block for chrX / chrY / MT.  The r^2 pair decisions are ld_ts_kernel.cuh's; the greedy window
// walk (IndepPairwiseThread, 2.0/plink2_ld.cc:862-1109) runs on the host.
#pragma once
#include "common.cuh"

namespace pl2 {

// ---- per-variant genotype counts {hom-REF, het, hom-ALT, missing}: GenoarrCountFreqsUnsafe
// (2.0/include/pgenlib_misc.cc:702); one warp per variant over the padded raw block.
static __global__ void __launch_bounds__(256) geno_counts_kernel(const uint8_t* __restrict__ raw, uint32_t pitch, uint32_t sample_ct, uint32_t sample_ct_padded, uint32_t variant_ct, uint32_t* __restrict__ counts) {
  const uint32_t v = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const uint32_t lane = threadIdx.x & 31;
  if (v >= variant_ct) return;
  const uint64_t* row = reinterpret_cast<const uint64_t*>(raw + static_cast<uint64_t>(v) * pitch);
  const uint32_t words = pitch / 8;
  uint32_t n1 = 0, n2 = 0, n3 = 0;
  for (uint32_t w = lane; w < words; w += 32) {
    const uint64_t x = row[w];
    const uint64_t lo = x & 0x5555555555555555ull;
    const uint64_t hi = (x >> 1) & 0x5555555555555555ull;
    n1 += __popcll(lo & ~hi);
    n2 += __popcll(hi & ~lo);
    n3 += __popcll(lo & hi);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    n1 += __shfl_xor_sync(0xFFFFFFFFu, n1, o);
    n2 += __shfl_xor_sync(0xFFFFFFFFu, n2, o);
    n3 += __shfl_xor_sync(0xFFFFFFFFu, n3, o);
  }
  if (lane == 0) {
    n3 -= (sample_ct_padded - sample_ct);  // padding is coded "missing"
    counts[4ull * v + 0] = sample_ct - n1 - n2 - n3;
    counts[4ull * v + 1] = n1;
    counts[4ull * v + 2] = n2;
    counts[4ull * v + 3] = n3;
  }
}

// ---- sample gather for the sex-chromosome / haploid forms of the LD block (2.0/plink2_ld.cc:1356-1389):
// output sample t of every variant row = input sample (map[t] & 0x7FFFFFFF), with a het call turned into
// "missing" when bit 31 of map[t] is set (SetHetMissing).  A sample listed twice carries weight 2 in every sum
// of the pair sextuple, which is exactly how chrX counts nonmales (:982-998).  One thread per output byte.
static __global__ void __launch_bounds__(256) geno_gather_kernel(const uint8_t* __restrict__ in, uint64_t in_pitch, uint8_t* __restrict__ out, uint32_t out_pitch, const uint32_t* __restrict__ map, uint32_t out_sample_ct) {
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= out_pitch) return;
  const uint8_t* row = in + static_cast<uint64_t>(blockIdx.y) * in_pitch;
  uint32_t byte = 0;
#pragma unroll
  for (uint32_t q = 0; q < 4; ++q) {
    const uint32_t t = 4 * b + q;
    uint32_t code = 3;
    if (t < out_sample_ct) {
      const uint32_t mv = map[t], s = mv & 0x7FFFFFFFu;
      code = (row[s >> 2] >> (2 * (s & 3))) & 3;
      if ((mv >> 31) && code == 1) code = 3;
    }
    byte |= code << (2 * q);
  }
  out[static_cast<uint64_t>(blockIdx.y) * out_pitch + b] = static_cast<uint8_t>(byte);
}

}  // namespace pl2
