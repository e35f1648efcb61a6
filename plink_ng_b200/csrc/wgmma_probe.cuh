// wgmma_probe.cuh - self-tests and rate probes of the int8 and binary (AND-POPC) wgmma forms the tensor kernels
// use (A fragments in registers, B K-major no-swizzle in shared memory, wgmma.cuh).
#pragma once
#include <cstdint>

#include "wgmma.cuh"

namespace pl2 {

constexpr uint32_t kProbeN = 80, kProbeK = 64;

// One warpgroup: D[64][80] = A[64][64] x B[80][64]^T from row-major int8 images (a[m * K + k], b[n * K + k]).
// The A fragment is loaded in the register layout of wgmma.cuh; B is written in the K-major core-matrix
// layout (LBO = next 16-byte K chunk, SBO = next 8 rows) the kernels use.  d[m * N + n].
static __global__ void __launch_bounds__(128) wgmma_probe_kernel(const int8_t* __restrict__ a, const int8_t* __restrict__ b, int32_t* __restrict__ d) {
  __shared__ __align__(128) uint8_t sb[kProbeN * kProbeK];
  constexpr uint32_t kChunks = kProbeK / 16, kSbo = kChunks * 128;
  for (uint32_t i = threadIdx.x; i < kProbeN * kProbeK; i += 128) {
    const uint32_t n = i / kProbeK, k = i % kProbeK;
    sb[(n >> 3) * kSbo + (k >> 4) * 128 + (n & 7) * 16 + (k & 15)] = static_cast<uint8_t>(b[i]);
  }
  fence_proxy_async_smem();
  __syncthreads();
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, c = lane & 3;
  const uint32_t r = 16 * warp + g;
  int32_t acc[kProbeN / 2];
#pragma unroll
  for (uint32_t i = 0; i < kProbeN / 2; ++i) acc[i] = 0;
  const uint64_t desc = make_wg_desc(static_cast<uint32_t>(__cvta_generic_to_shared(sb)), 128, kSbo);
#pragma unroll
  for (uint32_t ks = 0; ks < kProbeK / 32; ++ks) {
    uint32_t fa[4];
    fa[0] = *reinterpret_cast<const uint32_t*>(a + r * kProbeK + 32 * ks + 4 * c);
    fa[1] = *reinterpret_cast<const uint32_t*>(a + (r + 8) * kProbeK + 32 * ks + 4 * c);
    fa[2] = *reinterpret_cast<const uint32_t*>(a + r * kProbeK + 32 * ks + 16 + 4 * c);
    fa[3] = *reinterpret_cast<const uint32_t*>(a + (r + 8) * kProbeK + 32 * ks + 16 + 4 * c);
    wgmma_fence();
    wgmma_s8_rs<kProbeN>(acc, fa, desc + ((ks * 256) >> 4));
    wgmma_commit();
  }
  wgmma_wait<0>();
#pragma unroll
  for (uint32_t j = 0; j < kProbeN / 8; ++j)
#pragma unroll
    for (uint32_t i = 0; i < 4; ++i) d[(r + 8 * (i >> 1)) * kProbeN + 8 * j + 2 * c + (i & 1)] = acc[4 * j + i];
}

// Rate probe: two warpgroups per SM issue back-to-back m64nNk32 int8 wgmmas on one shared-memory B tile.
template <int N>
static __global__ void __launch_bounds__(256, 1) wgmma_peak_kernel(uint32_t blocks, int32_t* __restrict__ sink) {
  __shared__ __align__(128) uint8_t sb[N * 32];
  for (uint32_t i = threadIdx.x; i < N * 32; i += 256) sb[i] = static_cast<uint8_t>(i * 7);
  fence_proxy_async_smem();
  __syncthreads();
  int32_t acc[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) acc[i] = 0;
  const uint32_t fa[4] = {threadIdx.x, threadIdx.x * 3u, threadIdx.x * 5u, threadIdx.x * 7u};
  const uint64_t desc = make_wg_desc(static_cast<uint32_t>(__cvta_generic_to_shared(sb)), 128, 256);
  for (uint32_t it = 0; it < blocks; ++it) {
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 32; ++k) wgmma_s8_rs<N>(acc, fa, desc);
    wgmma_commit();
    wgmma_wait<0>();
  }
  int32_t s = 0;
#pragma unroll
  for (int i = 0; i < N / 2; ++i) s ^= acc[i];
  if (s == 0x7FFFFFFF) sink[threadIdx.x] = s;  // keeps the loop alive
}

// Binary form: one warpgroup, D[64][kProbeB1N] = popc(A[64][kProbeB1K] AND B[kProbeB1N][kProbeB1K]) from bit images
// of 32-bit words (a[m * kProbeB1K / 32 + w], bit k % 32 of word k / 32 = K bit k).  The A fragment takes whole words
// (wgmma_b1_rs, wgmma.cuh); word w of B row n goes to bytes 4 (w % 4) .. of the 16-byte row of its core matrix.
constexpr uint32_t kProbeB1N = 64, kProbeB1K = 512;
static __global__ void __launch_bounds__(128) wgmma_b1_probe_kernel(const uint32_t* __restrict__ a, const uint32_t* __restrict__ b, int32_t* __restrict__ d) {
  constexpr uint32_t kWords = kProbeB1K / 32, kSbo = (kProbeB1K / 128) * 128;
  __shared__ __align__(128) uint32_t sb[kProbeB1N * kWords];
  for (uint32_t i = threadIdx.x; i < kProbeB1N * kWords; i += 128) {
    const uint32_t n = i / kWords, w = i % kWords;
    sb[((n >> 3) * kSbo + (w >> 2) * 128 + (n & 7) * 16 + (w & 3) * 4) / 4] = b[i];
  }
  fence_proxy_async_smem();
  __syncthreads();
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, c = lane & 3;
  const uint32_t r = 16 * warp + g;
  int32_t acc[kProbeB1N / 2];
#pragma unroll
  for (uint32_t i = 0; i < kProbeB1N / 2; ++i) acc[i] = 0;
  const uint64_t desc = make_wg_desc(static_cast<uint32_t>(__cvta_generic_to_shared(sb)), 128, kSbo);
#pragma unroll
  for (uint32_t ks = 0; ks < kProbeB1K / 256; ++ks) {
    uint32_t fa[4];
    fa[0] = a[r * kWords + 8 * ks + c];
    fa[1] = a[(r + 8) * kWords + 8 * ks + c];
    fa[2] = a[r * kWords + 8 * ks + 4 + c];
    fa[3] = a[(r + 8) * kWords + 8 * ks + 4 + c];
    wgmma_fence();
    wgmma_b1_rs<kProbeB1N>(acc, fa, desc + ((ks * 256) >> 4));
    wgmma_commit();
  }
  wgmma_wait<0>();
#pragma unroll
  for (uint32_t j = 0; j < kProbeB1N / 8; ++j)
#pragma unroll
    for (uint32_t i = 0; i < 4; ++i) d[(r + 8 * (i >> 1)) * kProbeB1N + 8 * j + 2 * c + (i & 1)] = acc[4 * j + i];
}

// Rate probe of the binary form: two warpgroups per SM issue back-to-back m64nNk256 AND-POPC wgmmas.
template <int N>
static __global__ void __launch_bounds__(256, 1) wgmma_b1_peak_kernel(uint32_t blocks, int32_t* __restrict__ sink) {
  __shared__ __align__(128) uint8_t sb[N * 32];
  for (uint32_t i = threadIdx.x; i < N * 32; i += 256) sb[i] = static_cast<uint8_t>(i * 7);
  fence_proxy_async_smem();
  __syncthreads();
  int32_t acc[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) acc[i] = 0;
  const uint32_t fa[4] = {threadIdx.x, threadIdx.x * 3u, threadIdx.x * 5u, threadIdx.x * 7u};
  const uint64_t desc = make_wg_desc(static_cast<uint32_t>(__cvta_generic_to_shared(sb)), 128, 256);
  for (uint32_t it = 0; it < blocks; ++it) {
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 32; ++k) wgmma_b1_rs<N>(acc, fa, desc);
    wgmma_commit();
    wgmma_wait<0>();
  }
  int32_t s = 0;
#pragma unroll
  for (int i = 0; i < N / 2; ++i) s ^= acc[i];
  if (s == 0x7FFFFFFF) sink[threadIdx.x] = s;  // keeps the loop alive
}

// Read-rate probe of the operand feed: one thread per CTA (one CTA per SM) keeps `chunks` bulk copies of kFeedChunk
// bytes (global -> shared, each onto its own mbarrier, the instruction king_b1_kernel feeds itself with) in flight and
// discards what arrives.  CTA b reads chunks b, b + gridDim.x, ... of a working set of ws_chunks chunks, wrapping
// around, `rounds` x `chunks` copies in all.
constexpr uint32_t kFeedChunk = 4096;
static __global__ void __launch_bounds__(32, 1) bulk_read_probe_kernel(const uint8_t* __restrict__ src, uint32_t ws_chunks, uint32_t chunks, uint32_t rounds) {
  extern __shared__ __align__(128) uint8_t smem[];
  if (threadIdx.x != 0) return;
  const uint32_t base = (static_cast<uint32_t>(__cvta_generic_to_shared(smem)) + 127u) & ~127u;
  const uint32_t bar = base + chunks * kFeedChunk;
  for (uint32_t i = 0; i < chunks; ++i) mbar_init(bar + 8 * i, 1);
  mbar_init_fence();
  uint32_t next = blockIdx.x % ws_chunks;
  auto issue = [&](uint32_t i) {
    mbar_arrive_expect_tx(bar + 8 * i, kFeedChunk);
    bulk_copy_g2s(base + i * kFeedChunk, src + static_cast<uint64_t>(next) * kFeedChunk, kFeedChunk, bar + 8 * i);
    next += gridDim.x;
    if (next >= ws_chunks) next %= ws_chunks;
  };
  for (uint32_t i = 0; i < chunks; ++i) issue(i);
  for (uint32_t r = 1; r < rounds; ++r)
    for (uint32_t i = 0; i < chunks; ++i) {
      mbar_wait(bar + 8 * i, (r - 1) & 1);
      issue(i);
    }
  for (uint32_t i = 0; i < chunks; ++i) mbar_wait(bar + 8 * i, (rounds - 1) & 1);
}

}  // namespace pl2
