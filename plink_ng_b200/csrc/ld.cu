// ld.cu - --indep-pairwise: genotype-count pass, banded r^2 decision kernel driver, and the
// host-side greedy window walk (function face of LdPrune/IndepPairwise, 2.0/plink2_ld.cc:2530, :1116).
#include <algorithm>
#include <cmath>
#include <vector>

#include "../../include/plink2_b200.h"
#include "common.cuh"
#include "ld_kernels.cuh"
#include "ld_ts_kernel.cuh"

using namespace pl2;

namespace {

constexpr double kSmallEpsilon = 1.0 / 17592186044416.0;  // 2^-44, 2.0/include/plink2_base.h kSmallEpsilon
constexpr uint32_t kLdChunkVariants = 16384;

constexpr const char* kOom = "insufficient device memory (%.2f GB requested)";

}  // namespace

extern "C" {

int pl2gpu_geno_counts(Pl2GpuCtx* ctx, const void* genovecs, uint64_t variant_stride_bytes, uint32_t sample_ct, uint32_t variant_ct, int src_is_device, uint32_t* counts_host) {
  if (!ctx || !sample_ct) {
    set_error("pl2gpu_geno_counts: bad arguments");
    return 1;
  }
  Ctx* c = &ctx->c;
  PL2_CUDA_OK(cudaSetDevice(c->device));
  GenoStage st;
  const uint32_t cap = std::min<uint32_t>(kMaxStageVariants, RoundUpU32(std::max(variant_ct, 1u), kVariantPad));
  PL2_TRY(StageAlloc(sample_ct, cap, &st));
  DevArray<uint32_t> d_counts;
  PL2_TRY(d_counts.alloc(4ull * cap, kOom, 16ull * cap / 1e9));
  const uint8_t* src = static_cast<const uint8_t*>(genovecs);
  int rc = 0;
  for (uint32_t done = 0; done < variant_ct && !rc; done += cap) {
    const uint32_t cur = std::min(cap, variant_ct - done);
    uint32_t padded;
    rc = StageUpload(c, &st, src + static_cast<uint64_t>(done) * variant_stride_bytes, variant_stride_bytes, cur, src_is_device, &padded);
    if (rc) break;
    geno_counts_kernel<<<DivUpU32(cur, 8), 256, 0, c->stream>>>(st.d_raw, st.pitch, st.sample_ct, st.sample_ct_padded, cur, d_counts);
    c->launches++;
    if (cudaMemcpyAsync(counts_host + 4ull * done, d_counts, 16ull * cur, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess || cudaStreamSynchronize(c->stream) != cudaSuccess) {
      set_error("pl2gpu_geno_counts: %s", cudaGetErrorString(cudaGetLastError()));
      rc = 1;
    }
  }
  return rc;
}

int pl2gpu_ld_band_flags(Pl2GpuCtx* ctx, const void* genovecs, uint64_t variant_stride_bytes, uint32_t founder_ct, uint32_t variant_ct, int src_is_device, uint32_t band, double prune_ld_thresh, uint8_t* flags_host) {
  if (!ctx || !founder_ct || !band) {
    set_error("pl2gpu_ld_band_flags: bad arguments");
    return 1;
  }
  Ctx* c = &ctx->c;
  PL2_CUDA_OK(cudaSetDevice(c->device));
  const uint32_t band_r = RoundUpU32(band, 64);
  const uint32_t rows_cap = kLdChunkVariants + band_r;
  // the copy of chunk k+1 (prep stream) overlaps the pair kernel of chunk k; flags come back through two device
  // buffers in the same rhythm
  StageRing ring;
  DevArray<uint8_t> d_flags[2];
  const uint64_t flag_bytes = static_cast<uint64_t>(kLdChunkVariants) * band;
  int rc = ring.alloc(c, founder_ct, rows_cap, 64);
  for (int b = 0; b < 2 && !rc; ++b) rc = d_flags[b].alloc(flag_bytes, kOom, flag_bytes / 1e9);
  if (!rc && cudaFuncSetAttribute(ld_ts_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kLdtSmemBytes) != cudaSuccess) {
    set_error("pl2gpu_ld_band_flags: %s", cudaGetErrorString(cudaGetLastError()));
    rc = 1;
  }
  const uint8_t* src = static_cast<const uint8_t*>(genovecs);
  struct Pending {
    uint32_t a0 = 0, a1 = 0;
    bool live = false;
  } pend[2];
  auto drain = [&](int b) -> int {  // flags of the chunk that used buffer b -> host
    if (!pend[b].live) return 0;
    pend[b].live = false;
    if (cudaMemcpyAsync(flags_host + static_cast<uint64_t>(pend[b].a0) * band, d_flags[b], static_cast<uint64_t>(pend[b].a1 - pend[b].a0) * band, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess ||
        cudaStreamSynchronize(c->stream) != cudaSuccess) {
      set_error("pl2gpu_ld_band_flags: %s", cudaGetErrorString(cudaGetLastError()));
      return 1;
    }
    return 0;
  };
  for (uint32_t a0 = 0; a0 < variant_ct && !rc; a0 += kLdChunkVariants) {
    const uint32_t a1 = std::min(variant_ct, a0 + kLdChunkVariants);
    const uint32_t lo = (a0 > band_r) ? (a0 - band_r) : 0;
    uint32_t b, padded;
    // drain(b): slot b is free again (its kernel has finished, its flags are on the host)
    rc = ring.acquire(src_is_device, &b) || drain(b) || ring.land(b, nullptr, src + static_cast<uint64_t>(lo) * variant_stride_bytes, variant_stride_bytes, a1 - lo, src_is_device) ||
         ring.pad(b, a1 - lo, true, 64, &padded) || ring.fence(b);
    if (rc) break;
    const GenoStage& st = ring.stage[b];
    ld_ts_kernel<<<dim3(DivUpU32(a1 - a0, kLdtRows), (kLdtRows - kLdtCols + band_r) / kLdtCols + 1), kLdtThreads, kLdtSmemBytes, c->stream>>>(st.d_raw, st.pitch, st.sample_ct_padded, lo, a0, a1, band, prune_ld_thresh, d_flags[b]);
    c->launches++;
    if (cudaGetLastError() != cudaSuccess) {
      set_error("pl2gpu_ld_band_flags: %s", cudaGetErrorString(cudaGetLastError()));
      rc = 1;
      break;
    }
    pend[b].a0 = a0;
    pend[b].a1 = a1;
    pend[b].live = true;
    // a host source may be reused by the caller only after the copy; chunks overlap by band_r rows, so wait here
    rc = ring.release_host_source(src_is_device);
  }
  for (uint32_t b = 0; b < 2; ++b) {
    if (!rc) rc = drain((ring.next + b) & 1);  // oldest pending first
  }
  cudaStreamSynchronize(c->stream);  // the ring and the flag buffers are freed on return
  cudaStreamSynchronize(c->copy_stream);
  return rc;
}

// ---------------------------------------------------------------------------------------------
// Function face.  `variant_ct` variants in file order (already restricted to the included set),
// `chr_codes[v]` = chromosome index (0 = unplaced -> never examined, plink2_ld.cc:2542),
// founders only.  removed_out[v]: 0 = kept (.prune.in), 1 = removed (.prune.out), 2 = unplaced.
// ---------------------------------------------------------------------------------------------
}  // extern "C"

namespace {

enum ChrClass { kDip = 0, kChrX = 1, kChrY = 2, kHap = 3 };
// human chromosome set: haploid_mask = X, Y, MT (2.0/plink2_common.cc:1979); XY (PAR) is diploid
ChrClass ClassOf(uint32_t chr_code) { return chr_code == 23 ? kChrX : chr_code == 24 ? kChrY : chr_code == 26 ? kHap : kDip; }

// subcontigs (LdPruneSubcontigSplitAll, plink2_ld.cc:2165-2268) and the widest window in variants
struct Sub {
  uint32_t first, len;
};
void PlanSubcontigs(uint32_t variant_ct, const uint32_t* chr_codes, const uint32_t* variant_bps, uint32_t window_size, int window_is_bp, std::vector<Sub>* subs_ptr, uint32_t* window_max_ptr) {
  std::vector<Sub>& subs = *subs_ptr;
  uint32_t window_max = 0;
  for (uint32_t s = 0; s < variant_ct;) {
    uint32_t e = s + 1;
    while (e < variant_ct && chr_codes[e] == chr_codes[s]) ++e;
    if (chr_codes[s] != 0 && e - s > 1) {
      if (!window_is_bp) {
        subs.push_back({s, e - s});
        window_max = std::max(window_max, std::min(e - s, window_size));
      } else {
        uint32_t first = s;
        for (uint32_t v = s + 1; v <= e; ++v) {
          const bool split = (v == e) || (variant_bps[v] >= window_size && variant_bps[v] - window_size > variant_bps[v - 1]);
          if (split) {
            if (v - first > 1) subs.push_back({first, v - first});
            first = v;
          }
        }
      }
    }
    s = e;
  }
  if (window_is_bp) {
    // widest window in variant count: for each variant, how many predecessors lie within window_size bp
    for (const Sub& sc : subs) {
      uint32_t lo = sc.first;
      for (uint32_t v = sc.first; v < sc.first + sc.len; ++v) {
        while (static_cast<uint64_t>(variant_bps[lo]) + window_size < variant_bps[v]) ++lo;
        window_max = std::max(window_max, v - lo + 1);
      }
    }
  }
  *window_max_ptr = window_max;
}

// rows [v0, v1) of the caller's block, gathered / het-masked per `map` into a dense device block
// out[v - v0][out_pitch] (PgrGet layout for out_sample_ct samples)
int GatherRun(Ctx* c, const uint8_t* src, uint64_t stride, uint32_t founder_ct, uint32_t v0, uint32_t v1, int src_is_device, const std::vector<uint32_t>& map, DevArray<uint8_t>* out, uint32_t* out_pitch_ptr) {
  const uint32_t out_ct = static_cast<uint32_t>(map.size());
  const uint32_t out_pitch = DivUpU32(std::max(out_ct, 1u), 32) * 8;
  *out_pitch_ptr = out_pitch;
  DevArray<uint32_t> d_map;
  DevArray<uint8_t> d_in;
  const uint64_t out_bytes = static_cast<uint64_t>(v1 - v0) * out_pitch;
  if (out->alloc(out_bytes, kOom, out_bytes / 1e9) || d_map.alloc(std::max(out_ct, 1u), kOom, 4ull * std::max(out_ct, 1u) / 1e9)) return 1;
  if (out_ct) PL2_CUDA_OK(cudaMemcpyAsync(d_map, map.data(), 4ull * out_ct, cudaMemcpyHostToDevice, c->stream));
  const uint32_t in_bytes = DivUpU32(founder_ct, 4);
  constexpr uint32_t kRows = 8192;
  if (!src_is_device && d_in.alloc(static_cast<uint64_t>(kRows) * in_bytes, kOom, static_cast<uint64_t>(kRows) * in_bytes / 1e9)) return 1;
  for (uint32_t r0 = v0; r0 < v1; r0 += kRows) {
    const uint32_t rows = std::min(kRows, v1 - r0);
    const uint8_t* in = src + static_cast<uint64_t>(r0) * stride;
    uint64_t in_pitch = stride;
    if (!src_is_device) {
      PL2_CUDA_OK(cudaMemcpy2DAsync(d_in, in_bytes, in, stride, in_bytes, rows, cudaMemcpyHostToDevice, c->stream));
      in = d_in;
      in_pitch = in_bytes;
    }
    geno_gather_kernel<<<dim3(DivUpU32(out_pitch, 256), rows), 256, 0, c->stream>>>(in, in_pitch, out->get() + static_cast<uint64_t>(r0 - v0) * out_pitch, out_pitch, d_map, out_ct);
    c->launches++;
    PL2_CUDA_OK(cudaGetLastError());
    if (!src_is_device) PL2_CUDA_OK(cudaStreamSynchronize(c->stream));  // d_in is reused by the next chunk
  }
  PL2_CUDA_OK(cudaStreamSynchronize(c->stream));
  return 0;
}

}  // namespace

extern "C" {

int pl2_indep_pairwise_ex(Pl2GpuCtx* ctx, const void* genovecs, uint64_t variant_stride_bytes, uint32_t founder_ct, uint32_t variant_ct, const uint32_t* chr_codes, const uint32_t* variant_bps, uint32_t window_size, uint32_t window_incr, double r2_thresh, int window_is_bp, const double* ref_freqs, const uint8_t* preferred, int src_is_device, const uint8_t* founder_sex, uint32_t flags_in, uint8_t* removed_out) {
  if (!ctx || !variant_ct || !removed_out || !chr_codes || (window_is_bp && !variant_bps)) {
    set_error("pl2_indep_pairwise: bad arguments");
    return 1;
  }
  if (window_size < 2 || !window_incr) {
    set_error("pl2_indep_pairwise: window size must be >= 2 and step >= 1");
    return 1;
  }
  Ctx* c = &ctx->c;
  PL2_CUDA_OK(cudaSetDevice(c->device));
  const uint8_t* src = static_cast<const uint8_t*>(genovecs);
  // chromosome runs by class: diploid runs go through the block as it is; chrX / chrY / MT runs are re-staged
  // (IndepPairwise loader, plink2_ld.cc:1356-1389): MT = every founder with hets -> missing; chrY = nonfemale
  // founders, hets -> missing; chrX = males (hets -> missing) once + nonmales twice (the reference adds the
  // nonmale-only sextuple twice to the male one, :982-998 / :1064-1078)
  std::vector<uint32_t> map_hap(founder_ct), map_y, map_y_raw, map_x, map_x_male_raw;
  for (uint32_t s = 0; s < founder_ct; ++s) {
    const uint32_t sex = founder_sex ? founder_sex[s] : 0;
    map_hap[s] = s | 0x80000000u;
    if (sex != 2) {
      map_y.push_back(s | 0x80000000u);
      map_y_raw.push_back(s);
    }
    if (sex == 1) {
      map_x.push_back(s | 0x80000000u);
      map_x_male_raw.push_back(s);
    }
  }
  const uint32_t male_ct = static_cast<uint32_t>(map_x.size());
  for (int rep = 0; rep < 2; ++rep)
    for (uint32_t s = 0; s < founder_ct; ++s)
      if (!(founder_sex && founder_sex[s] == 1)) map_x.push_back(s);
  // 1. genotype counts -> allele frequencies (ComputeAlleleFreqs, plink2_filter.cc:2113-2151; per-class counting
  //    rules of LoadAlleleAndGenoCountsThread, plink2_data.cc:2420-2690), major-allele frequencies
  //    (GetMajIdx/GetAlleleFreq, plink2_common.h:559-595) and the load-time monomorphic rule (plink2_ld.cc:902).
  std::vector<uint32_t> counts(4ull * variant_ct);
  PL2_TRY(pl2gpu_geno_counts(ctx, genovecs, variant_stride_bytes, founder_ct, variant_ct, src_is_device, counts.data()));
  std::vector<double> maj_freq(variant_ct);
  std::vector<uint8_t> mono(variant_ct);
  struct Run {
    uint32_t v0, v1;
    ChrClass cls;
  };
  std::vector<Run> runs;
  for (uint32_t s = 0; s < variant_ct;) {
    uint32_t e = s + 1;
    const ChrClass cls = ClassOf(chr_codes[s]);
    while (e < variant_ct && (cls == kDip ? ClassOf(chr_codes[e]) == kDip : chr_codes[e] == chr_codes[s])) ++e;
    runs.push_back({s, e, cls});
    s = e;
  }
  std::vector<DevArray<uint8_t>> run_blocks(runs.size());
  std::vector<uint32_t> run_pitch(runs.size(), 0), run_samples(runs.size(), founder_ct);
  std::vector<uint32_t> cls_counts, ld_counts;
  for (size_t ri = 0; ri < runs.size(); ++ri) {
    const Run& r = runs[ri];
    const uint32_t len = r.v1 - r.v0;
    ld_counts.assign(4ull * len, 0);
    if (r.cls != kDip) {
      const std::vector<uint32_t>& map_ld = r.cls == kChrX ? map_x : r.cls == kChrY ? map_y : map_hap;
      run_samples[ri] = static_cast<uint32_t>(map_ld.size());
      if (!map_ld.empty()) {
        PL2_TRY(GatherRun(c, src, variant_stride_bytes, founder_ct, r.v0, r.v1, src_is_device, map_ld, &run_blocks[ri], &run_pitch[ri]));
        PL2_TRY(pl2gpu_geno_counts(ctx, run_blocks[ri], run_pitch[ri], run_samples[ri], len, 1, ld_counts.data()));
      }
      const std::vector<uint32_t>* map_f = r.cls == kChrX ? &map_x_male_raw : r.cls == kChrY ? &map_y_raw : nullptr;
      cls_counts.assign(4ull * len, 0);
      if (map_f && !map_f->empty()) {
        DevArray<uint8_t> tmp;
        uint32_t tp = 0;
        PL2_TRY(GatherRun(c, src, variant_stride_bytes, founder_ct, r.v0, r.v1, src_is_device, *map_f, &tmp, &tp));
        PL2_TRY(pl2gpu_geno_counts(ctx, tmp, tp, static_cast<uint32_t>(map_f->size()), len, 1, cls_counts.data()));
      }
    }
    for (uint32_t v = r.v0; v < r.v1; ++v) {
      const uint32_t n0 = counts[4ull * v], n1 = counts[4ull * v + 1], n2 = counts[4ull * v + 2], n3 = counts[4ull * v + 3];
      const uint32_t* cc = &cls_counts[r.cls == kDip ? 0 : 4ull * (v - r.v0)];
      double ref_freq;
      if (ref_freqs && ref_freqs[v] == ref_freqs[v]) {  // NaN entry: compute from the block
        ref_freq = ref_freqs[v];
      } else if (r.cls == kChrX) {
        // nonmales count twice, a male het is half an ALT (plink2_data.cc:2642, :2685-2688)
        const uint64_t alt1 = 4ull * n2 + 2ull * n1 - 2ull * cc[2] - cc[1];
        const uint64_t wobs = (2ull * (founder_ct - n3) - male_ct + cc[3]) * 2;
        ref_freq = wobs ? (static_cast<double>(wobs - alt1) * (1.0 / static_cast<double>(wobs))) : 0.5;
      } else {
        const uint64_t a0 = r.cls == kChrY ? cc[0] : n0, a1 = r.cls == kChrY ? cc[1] : n1, a2 = r.cls == kChrY ? cc[2] : n2;
        const uint64_t tot = 2ull * (a0 + a1 + a2);
        ref_freq = tot ? (static_cast<double>(2ull * a0 + a1) * (1.0 / static_cast<double>(tot))) : 0.5;
      }
      double mf;
      if (ref_freq >= 0.5) {
        mf = ref_freq;
      } else {
        mf = 1.0 - ref_freq;
        if (mf < 0.0) mf = 0.0;
      }
      if (preferred && preferred[v]) mf -= 1.0;  // plink2_ld.cc:916-918
      maj_freq[v] = mf;
      // monomorphic at load (:902), on the (weighted) counts of the block the pair sums are taken over
      const uint32_t* lc = r.cls == kDip ? &counts[4ull * v] : &ld_counts[4ull * (v - r.v0)];
      const uint32_t p0 = lc[0], p2 = lc[2], nm = lc[0] + lc[1] + lc[2];
      mono[v] = ((!p0 && !p2) || p0 == nm || p2 == nm) ? 1 : 0;
    }
  }
  // 2. subcontigs and the widest window
  std::vector<Sub> subs;
  uint32_t window_max = 0;
  PlanSubcontigs(variant_ct, chr_codes, variant_bps, window_size, window_is_bp, &subs, &window_max);
  if (subs.empty()) {
    for (uint32_t v = 0; v < variant_ct; ++v) removed_out[v] = chr_codes[v] ? 0 : 2;
    return 0;
  }
  const uint32_t band = std::max(1u, window_max - 1);
  // 3. per-pair decisions on the GPU
  std::vector<uint8_t> flags(static_cast<uint64_t>(variant_ct) * band);
  const double thresh = r2_thresh * (1 + kSmallEpsilon);  // plink2_ld.cc:1255
  for (size_t ri = 0; ri < runs.size(); ++ri) {
    const Run& r = runs[ri];
    if (r.v1 - r.v0 < 2) continue;
    uint8_t* fl = flags.data() + static_cast<uint64_t>(r.v0) * band;
    if (r.cls == kDip) {
      PL2_TRY(pl2gpu_ld_band_flags(ctx, src + static_cast<uint64_t>(r.v0) * variant_stride_bytes, variant_stride_bytes, founder_ct, r.v1 - r.v0, src_is_device, band, thresh, fl));
    } else if (run_samples[ri]) {
      PL2_TRY(pl2gpu_ld_band_flags(ctx, run_blocks[ri], run_pitch[ri], run_samples[ri], r.v1 - r.v0, 1, band, thresh, fl));
      run_blocks[ri].reset();
    }
  }
  // 4. greedy window walk on the host
  return pl2_ld_prune_walk(variant_ct, chr_codes, variant_bps, window_size, window_incr, window_is_bp, maj_freq.data(), mono.data(), flags.data(), band, flags_in, removed_out);
}

int pl2_indep_pairwise(Pl2GpuCtx* ctx, const void* genovecs, uint64_t variant_stride_bytes, uint32_t founder_ct, uint32_t variant_ct, const uint32_t* chr_codes, const uint32_t* variant_bps, uint32_t window_size, uint32_t window_incr, double r2_thresh, int window_is_bp, const double* ref_freqs, const uint8_t* preferred, int src_is_device, uint8_t* removed_out) {
  return pl2_indep_pairwise_ex(ctx, genovecs, variant_stride_bytes, founder_ct, variant_ct, chr_codes, variant_bps, window_size, window_incr, r2_thresh, window_is_bp, ref_freqs, preferred, src_is_device, nullptr, 0, removed_out);
}

// ---- host half of the function face: the greedy window walk of IndepPairwiseThread over the per-pair decisions
// (flags[v * band + d - 1] for second = v, first = v - d), the load-time monomorphic marks and the major-allele
// frequencies.  No device work; exported so the walk can be checked on its own.
int pl2_ld_prune_walk(uint32_t variant_ct, const uint32_t* chr_codes, const uint32_t* variant_bps, uint32_t window_size, uint32_t window_incr, int window_is_bp, const double* maj_freq, const uint8_t* mono, const uint8_t* flags, uint32_t band, uint32_t flags_in, uint8_t* removed_out) {
  if (!variant_ct || !chr_codes || !maj_freq || !mono || !flags || !removed_out || (window_is_bp && !variant_bps) || window_size < 2 || !window_incr) {
    set_error("pl2_ld_prune_walk: bad arguments");
    return 1;
  }
  const bool plink1_order = (flags_in & kPl2LdPlink1Order) != 0;
  std::vector<Sub> subs;
  uint32_t window_max = 0;
  PlanSubcontigs(variant_ct, chr_codes, variant_bps, window_size, window_is_bp, &subs, &window_max);
  for (uint32_t v = 0; v < variant_ct; ++v) removed_out[v] = chr_codes[v] ? 0 : 2;
  if (subs.empty()) return 0;
  if (band + 1 < window_max) {
    set_error("pl2_ld_prune_walk: band %u is narrower than the widest window (%u variants)", band, window_max);
    return 1;
  }
  // greedy window walk per subcontig (IndepPairwiseThread default branch, plink2_ld.cc:862-1109;
  //    LdPruneNextSubcontig :605-633, LdPruneNextWindow :635-689)
  std::vector<uint32_t> win, first_unchecked;
  std::vector<uint8_t> win_removed;
  for (const Sub& sc : subs) {
    const uint32_t base = sc.first, L = sc.len;
    const uint32_t* bps = window_is_bp ? (variant_bps + base) : nullptr;
    uint32_t start = 0, next_end;
    if (bps) {
      const uint64_t bp_thresh = static_cast<uint64_t>(bps[0]) + window_size;
      uint32_t first_len = 1, idx = 0;
      while (true) {
        ++idx;
        if (!(bps[idx] <= bp_thresh)) break;
        if (!(++first_len < L)) break;
      }
      next_end = first_len;
    } else {
      next_end = std::min(L, window_size);
    }
    win.clear();
    win_removed.clear();
    if (plink1_order) first_unchecked.assign(L, 0);
    uint32_t winpos_split = 0;
    for (uint32_t cur = 0; cur < L; ++cur) {
      win.push_back(cur);
      if (mono[base + cur]) {
        win_removed.push_back(1);
        removed_out[base + cur] = 1;
      } else {
        win_removed.push_back(0);
        if (plink1_order) first_unchecked[cur] = cur + 1;  // :919-921
      }
      if (cur + 1 != next_end) continue;
      if (plink1_order) {
        // `--indep-order 1` (:931-1037): firsts in ascending order, each against the seconds it has not been
        // checked against yet; the sweep repeats while it removes something
        const uint32_t cur_tvidx = cur + 1, wsz = static_cast<uint32_t>(win.size());
        auto next_live = [&](uint32_t pos) {
          while (pos < wsz && win_removed[pos]) ++pos;
          return pos;
        };
        uint32_t removed_ct = 0;
        for (uint32_t r = 0; r < wsz; ++r) removed_ct += win_removed[r];
        for (;;) {
          const uint32_t prev_removed_ct = removed_ct;
          for (uint32_t fw = next_live(0); fw != wsz; fw = next_live(fw + 1)) {
            const uint32_t b = win[fw];
            const uint32_t fu = first_unchecked[b];
            if (fu == cur_tvidx) continue;
            uint32_t sw = next_live(fw + 1);
            while (sw != wsz && win[sw] < fu) sw = next_live(sw + 1);
            for (;; sw = next_live(sw + 1)) {
              if (sw == wsz) {
                first_unchecked[b] = cur_tvidx;
                break;
              }
              const uint32_t a = win[sw];
              if (flags[static_cast<uint64_t>(base + a) * band + (a - b - 1)]) {
                if (maj_freq[base + b] > maj_freq[base + a] * (1 + kSmallEpsilon)) {
                  win_removed[fw] = 1;
                  removed_out[base + b] = 1;
                } else {
                  win_removed[sw] = 1;
                  removed_out[base + a] = 1;
                  const uint32_t nx = next_live(sw + 1);
                  first_unchecked[b] = (nx != wsz) ? win[nx] : cur_tvidx;
                }
                ++removed_ct;
                break;
              }
            }
          }
          if (!(removed_ct > prev_removed_ct)) break;
        }
      }
      const uint32_t second_stop = plink1_order ? static_cast<uint32_t>(win.size()) : (winpos_split ? winpos_split : 1);
      for (uint32_t second_winpos = static_cast<uint32_t>(win.size()); second_winpos != second_stop;) {
        --second_winpos;
        const uint32_t a = base + win[second_winpos];
        const uint8_t* arow = flags + static_cast<uint64_t>(a) * band;
        for (uint32_t first_winpos = second_winpos; first_winpos;) {
          --first_winpos;
          if (win_removed[first_winpos]) continue;
          const uint32_t b = base + win[first_winpos];
          if (arow[a - b - 1]) {
            if (maj_freq[b] <= maj_freq[a] * (1 + kSmallEpsilon)) {
              win_removed[second_winpos] = 1;
              removed_out[a] = 1;
              break;
            }
            win_removed[first_winpos] = 1;
            removed_out[b] = 1;
          }
        }
      }
      if (next_end == L) break;
      if (bps) {
        const uint32_t min_bp = bps[next_end] - window_size;  // >= 0: bps[next_end] lies beyond the window
        uint32_t nstart = start, sbp;
        do {
          ++nstart;
          sbp = bps[nstart];
        } while (sbp < min_bp);
        const uint64_t end_thresh = static_cast<uint64_t>(sbp) + window_size;
        uint32_t e = next_end;
        while (true) {
          if (++e == L) break;
          if (!(bps[e] <= end_thresh)) break;
        }
        start = nstart;
        next_end = e;
      } else {
        start += window_incr;
        next_end = std::min(start + window_size, L);
      }
      uint32_t w = 0;
      for (uint32_t r = 0; r < win.size(); ++r) {
        if (!win_removed[r] && win[r] >= start) win[w++] = win[r];
      }
      win.resize(w);
      win_removed.assign(w, 0);
      winpos_split = w;
    }
  }
  return 0;
}

}  // extern "C"
