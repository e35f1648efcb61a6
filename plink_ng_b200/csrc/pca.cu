// pca.cu - `--pca approx` job (CalcPca approx branch, 2.0/plink2_matrix_calc.cc:5697-5941): the
// EIGENSOFT-style randomized range finder (Halko et al. 2011; Galinsky et al. 2016) on the resident
// 2-bit genotype matrix.  Gaussian start matrix is supplied by the caller (the host program
// reproduces the reference's SFMT / Box-Muller stream, host/sfmt.cc).
#include <algorithm>
#include <cmath>
#include <vector>

#include "../../include/plink2_b200.h"
#include "common.cuh"
#include "ld_kernels.cuh"    // geno_counts_kernel
#include "geno_tile.cuh"
#include "pca_ts_kernels.cuh"
#include "jacobi.cuh"
#include "dense_fp64.cuh"

using namespace pl2;

namespace {
constexpr double kSmallEpsilon = 1.0 / 17592186044416.0;

}  // namespace

struct Pl2PcaJob {
  Pl2GpuCtx* ctx = nullptr;
  uint32_t sample_ct = 0, sample_ct_padded = 0, pitch = 0;
  uint32_t variant_cap = 0, variant_ct = 0, pc_ct = 0;
  uint8_t* d_raw = nullptr;
  uint32_t* d_counts = nullptr;
  std::vector<uint32_t> h_counts;
  uint8_t* d_raw_i = nullptr;   // sample-major copy [row tile][k-step][128][8 B] of the whole matrix (geno_tile.cuh)
  double* d_slope = nullptr;    // per variant: inv_stdev (0 for skipped variants)
  double* d_icpt = nullptr;     // per variant: -2 alt_freq inv_stdev
  double* d_twof = nullptr;     // per variant: 2 alt_freq (the mean-imputation value of --variant-score)
  std::vector<double> h_slope, h_icpt, h_twof;
  uint32_t retiled_to = 0;      // variants [0, retiled_to) are in d_raw_i (multiple of 64)
  bool vscore_only = false;     // begun with pc_ct = 0: a --variant-score job (no approx-PCA requirements, see the header)
};

extern "C" {

int pl2gpu_pca_end(Pl2PcaJob* job);

static int PcaBeginImpl(Pl2GpuCtx* ctx, uint32_t sample_ct, uint32_t variant_ct_total, uint32_t pc_ct, bool shard, Pl2PcaJob** job_ptr) {
  *job_ptr = nullptr;
  if (!ctx || !sample_ct || !variant_ct_total || (!pc_ct && !shard)) {
    set_error("pl2gpu_pca_begin: bad arguments");
    return 1;
  }
  // the approx-PCA size requirements; a shard is judged at run time (PcaRunImpl), which leaves a --variant-score job
  // (pc_ct = 0) without any: VscoreReport scores any number of samples
  const uint64_t q = 2ull * pc_ct * (pc_ct + 1);
  if (q > variant_ct_total && !shard) {  // :5716-5719
    set_error("Too few variants to compute %u PCs with \"--pca approx\" (%llu required).", pc_ct, static_cast<unsigned long long>(q));
    return 2;
  }
  if (q > sample_ct && !shard) {
    set_error("pl2gpu_pca_begin: \"--pca approx\" with %u PCs needs at least %llu samples in this implementation (tall thin SVD)", pc_ct, static_cast<unsigned long long>(q));
    return 1;
  }
  PL2_CUDA_OK(cudaSetDevice(ctx->c.device));
  Pl2PcaJob* job = new Pl2PcaJob();
  job->ctx = ctx;
  job->sample_ct = sample_ct;
  job->sample_ct_padded = RoundUpU32(sample_ct, 128);
  job->pitch = job->sample_ct_padded / 4;
  job->variant_cap = RoundUpU32(variant_ct_total, 128);
  job->pc_ct = pc_ct;
  job->vscore_only = pc_ct == 0;
  if (cudaMalloc(&job->d_raw, static_cast<uint64_t>(job->variant_cap) * job->pitch) != cudaSuccess || cudaMalloc(&job->d_counts, 16ull * 65536) != cudaSuccess ||
      cudaMalloc(&job->d_raw_i, static_cast<uint64_t>(job->sample_ct_padded) * (job->variant_cap / 4)) != cudaSuccess || cudaMalloc(&job->d_slope, 8ull * job->variant_cap) != cudaSuccess ||
      cudaMalloc(&job->d_icpt, 8ull * job->variant_cap) != cudaSuccess || cudaMalloc(&job->d_twof, 8ull * job->variant_cap) != cudaSuccess) {
    cudaGetLastError();
    set_error("pl2gpu_pca_begin: insufficient device memory to keep %u x %u genotypes resident", variant_ct_total, sample_ct);
    pl2gpu_pca_end(job);
    return 1;
  }
  if (cudaMemsetAsync(job->d_slope, 0, 8ull * job->variant_cap, ctx->c.stream) != cudaSuccess || cudaMemsetAsync(job->d_icpt, 0, 8ull * job->variant_cap, ctx->c.stream) != cudaSuccess ||
      cudaFuncSetAttribute(pca_xa_wg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kPxaSmemBytes) != cudaSuccess ||
      cudaFuncSetAttribute(pca_xtb_wg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kPxtSmemBytes) != cudaSuccess) {
    if (!*get_error()) set_error("pl2gpu_pca_begin: %s", cudaGetErrorString(cudaGetLastError()));
    pl2gpu_pca_end(job);
    return 1;
  }
  *job_ptr = job;
  return 0;
}

int pl2gpu_pca_begin(Pl2GpuCtx* ctx, uint32_t sample_ct, uint32_t variant_ct_total, uint32_t pc_ct, Pl2PcaJob** job_ptr) { return PcaBeginImpl(ctx, sample_ct, variant_ct_total, pc_ct, false, job_ptr); }
int pl2gpu_pca_begin_shard(Pl2GpuCtx* ctx, uint32_t sample_ct, uint32_t shard_variant_ct, uint32_t pc_ct, Pl2PcaJob** job_ptr) { return PcaBeginImpl(ctx, sample_ct, shard_variant_ct, pc_ct, true, job_ptr); }

int pl2gpu_pca_add_variants(Pl2PcaJob* job, const void* genovecs, uint64_t variant_stride_bytes, uint32_t variant_ct, int src_is_device, const double* ref_freqs) {
  if (!job || job->variant_ct + static_cast<uint64_t>(variant_ct) > job->variant_cap) {
    set_error("pl2gpu_pca_add_variants: more variants than announced at pl2gpu_pca_begin");
    return 1;
  }
  Ctx* c = &job->ctx->c;
  PL2_CUDA_OK(cudaSetDevice(c->device));
  const uint8_t* src = static_cast<const uint8_t*>(genovecs);
  for (uint32_t done = 0; done < variant_ct;) {
    const uint32_t cur = std::min<uint32_t>(65536, variant_ct - done);
    uint8_t* dst = job->d_raw + static_cast<uint64_t>(job->variant_ct) * job->pitch;
    PL2_CUDA_OK(cudaMemcpy2DAsync(dst, job->pitch, src + static_cast<uint64_t>(done) * variant_stride_bytes, variant_stride_bytes, DivUpU32(job->sample_ct, 4), cur, src_is_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, c->stream));
    PL2_TRY(LaunchPadGenotypes(c, dst, job->pitch, job->sample_ct, cur, cur));
    geno_counts_kernel<<<DivUpU32(cur, 8), 256, 0, c->stream>>>(dst, job->pitch, job->sample_ct, job->sample_ct_padded, cur, job->d_counts);
    c->launches++;
    job->h_counts.resize(4ull * cur);
    PL2_CUDA_OK(cudaMemcpyAsync(job->h_counts.data(), job->d_counts, 16ull * cur, cudaMemcpyDeviceToHost, c->stream));
    PL2_CUDA_OK(cudaStreamSynchronize(c->stream));
    job->h_slope.assign(cur, 0.0);
    job->h_icpt.assign(cur, 0.0);
    job->h_twof.assign(cur, 0.0);
    for (uint32_t v = 0; v < cur; ++v) {
      const uint32_t n0 = job->h_counts[4ull * v], n1 = job->h_counts[4ull * v + 1], n2 = job->h_counts[4ull * v + 2];
      double ref_freq;
      if (ref_freqs && ref_freqs[done + v] == ref_freqs[done + v]) {  // NaN entry: compute from the block
        ref_freq = ref_freqs[done + v];
      } else {
        const uint64_t tot = 2ull * (static_cast<uint64_t>(n0) + n1 + n2);
        ref_freq = tot ? (static_cast<double>(2ull * n0 + n1) * (1.0 / static_cast<double>(tot))) : 0.5;
      }
      const double alt_freq = 1.0 - ref_freq;
      job->h_twof[v] = 2.0 * alt_freq;
      const double variance = 2 * ref_freq * alt_freq;
      if (!(variance > kSmallEpsilon)) {
        bool bad = n1 != 0;
        if (variance != variance) bad = bad || n0 || n2;
        else if (ref_freq > 0.5) bad = bad || n2;
        else bad = bad || n0;
        if (bad && !job->vscore_only) {  // CalcPca's consistency check (VscoreReport has none)
          set_error("pl2gpu_pca_add_variants: variant %u has zero-variance allele frequency %g but non-monomorphic genotypes (kPglRetDegenerateData)", job->variant_ct + v, ref_freq);
          return 2;
        }
        continue;
      }
      const double inv_stdev = 1.0 / sqrt(variance);
      job->h_slope[v] = inv_stdev;
      job->h_icpt[v] = -2 * alt_freq * inv_stdev;
    }
    PL2_CUDA_OK(cudaMemcpyAsync(job->d_slope + job->variant_ct, job->h_slope.data(), 8ull * cur, cudaMemcpyHostToDevice, c->stream));
    PL2_CUDA_OK(cudaMemcpyAsync(job->d_icpt + job->variant_ct, job->h_icpt.data(), 8ull * cur, cudaMemcpyHostToDevice, c->stream));
    PL2_CUDA_OK(cudaMemcpyAsync(job->d_twof + job->variant_ct, job->h_twof.data(), 8ull * cur, cudaMemcpyHostToDevice, c->stream));
    PL2_CUDA_OK(cudaStreamSynchronize(c->stream));
    job->variant_ct += cur;
    done += cur;
  }
  return 0;
}

}  // extern "C"

// ---- the two products on the int8 tensor pipe (pca_ts_kernels.cuh), shared by the run, --variant-score and
// pl2gpu_pca_products ----
// every dense operand goes through the tensor pipe twice: 30-bit fixed point, then the exact residual at another
// 30 bits (pca_digits_kernel pass 1) - 60 bits below the column maximum, so the passes lose nothing against the
// reference's fp64 dgemm (one 30-bit pass left the trailing, noise-level eigenvalues 2e-3 off)
constexpr int kPcaPasses = 2;
// The int32 digit accumulators of pca_xtb_wg_kernel gain at most 2 * 128 + 128 = 384 per variant (a dosage <= 2 and
// an indicator <= 1, each times a digit in [-128, 127]), 32 variants per k-step: a split of at most this many k-steps
// cannot overflow them.  An 80 GB card never holds a shard long enough for the cap to bind.
constexpr uint32_t kPcaXtbMaxKsteps = (0x7FFFFFFFu / (384u * 32u)) / 4 * 4;  // 174,760

// scratch of one job's products: digit planes, per-column scales, split-K partial sums of Y^T H
struct PcaTs {
  uint8_t *gdig = nullptr, *hs = nullptr, *hi = nullptr;
  double *scale = nullptr, *inv_scale = nullptr, *partial = nullptr;
  unsigned long long* colmax = nullptr;
  uint32_t splits = 0, ksteps_per_split = 0;
};

static void PcaTsFree(PcaTs* ts) {
  cudaFree(ts->gdig);
  cudaFree(ts->hs);
  cudaFree(ts->hi);
  cudaFree(ts->scale);
  cudaFree(ts->inv_scale);
  cudaFree(ts->colmax);
  cudaFree(ts->partial);
  *ts = PcaTs();
}

// xtb: also the slope.H / icpt.H digit planes and the split-K partial sums.  Split plan of Y^T H: about two CTAs per
// SM over the 128-sample row tiles, at least 64 k-steps (2,048 variants) per split, a whole number of 4-k-step stages
// per split, the last split short.
static int PcaTsAlloc(const Pl2PcaJob* job, bool xtb, PcaTs* ts) {
  const Ctx* c = &job->ctx->c;
  const uint32_t npad = job->sample_ct_padded, kstep_total = job->variant_cap / 32, tiles2 = npad / 128;
  uint32_t splits = std::max(1u, std::min(DivUpU32(2 * static_cast<uint32_t>(c->sm_count), tiles2), kstep_total / 64));
  ts->ksteps_per_split = std::min(kPcaXtbMaxKsteps, RoundUpU32(DivUpU32(kstep_total, splits), 4));
  ts->splits = DivUpU32(kstep_total, ts->ksteps_per_split);
  if (cudaMalloc(&ts->gdig, static_cast<uint64_t>(npad) * kPcaNMax) != cudaSuccess || cudaMalloc(&ts->scale, 8 * kPcaCgMax) != cudaSuccess || cudaMalloc(&ts->inv_scale, 8 * kPcaCgMax) != cudaSuccess ||
      cudaMalloc(&ts->colmax, 8 * kPcaCgMax) != cudaSuccess ||
      (xtb && (cudaMalloc(&ts->hs, static_cast<uint64_t>(job->variant_cap) * kPcaNMax) != cudaSuccess || cudaMalloc(&ts->hi, static_cast<uint64_t>(job->variant_cap) * kPcaNMax) != cudaSuccess ||
               cudaMalloc(&ts->partial, static_cast<uint64_t>(ts->splits) * npad * kPcaCgMax * 8) != cudaSuccess))) {
    cudaGetLastError();
    set_error("pl2gpu_pca: insufficient device memory for the digit planes");
    PcaTsFree(ts);
    return 1;
  }
  return 0;
}

// rows [variant_ct, variant_cap) must decode to "missing" in both layouts; sample_major: finish the sample-major copy
// (what Y^T H reads)
static int PcaFinishLayouts(Pl2PcaJob* job, bool sample_major) {
  Ctx* c = &job->ctx->c;
  const uint32_t m = job->variant_ct;
  if (job->variant_cap > m) PL2_TRY(LaunchPadGenotypes(c, job->d_raw + static_cast<uint64_t>(m) * job->pitch, job->pitch, job->sample_ct, 0, job->variant_cap - m));
  if (sample_major && job->retiled_to < job->variant_cap) {
    const uint32_t from = job->retiled_to;
    geno_tile_rows_kernel<<<dim3((job->variant_cap - from) / 64, job->sample_ct_padded / 64), 256, 0, c->stream>>>(job->d_raw + static_cast<uint64_t>(from) * job->pitch, job->pitch, job->variant_cap / 32, 0,
                                                                                                                 job->d_raw_i + static_cast<uint64_t>(from / 32) * 1024);
    c->launches++;
    job->retiled_to = job->variant_cap;
  }
  return 0;
}

// column group: up to kPcaCgMax columns (the columns past the valid ones are zero digits and never written)
static int PcaGroupScales(Ctx* c, PcaTs* ts, const double* src, uint64_t rs, uint64_t cs, uint32_t rows, uint32_t valid, const double* mul1, const double* mul2) {
  const int rc = cudaMemsetAsync(ts->colmax, 0, 8 * kPcaCgMax, c->stream) != cudaSuccess;
  pca_colmax_kernel<<<dim3(valid, std::min<uint32_t>(64, DivUpU32(rows, 256))), 256, 0, c->stream>>>(src, rs, cs, rows, mul1, mul2, ts->colmax);
  pca_scales_kernel<<<1, 64, 0, c->stream>>>(ts->colmax, kPcaCgMax, ts->scale, ts->inv_scale);
  c->launches += 2;
  return rc;
}

// H = Y G with y_vs = slope_v g_vs + icpt_v m_vs (the job's own per-variant arrays, or --variant-score's centring): G
// row-major (element (s, c) at g[s g_ld + c], sample_ct_padded rows, zero past sample_ct), H column-major (ld h_ld);
// cols columns
static int PcaLaunchXa(Pl2PcaJob* job, PcaTs* ts, const double* slope, const double* icpt, const double* g, uint32_t g_ld, double* h, uint64_t h_ld, uint32_t cols) {
  Ctx* c = &job->ctx->c;
  const uint32_t npad = job->sample_ct_padded;
  int rc = 0;
  for (uint32_t cc = 0; cc < cols; cc += kPcaCgMax) {
    const uint32_t valid = std::min(kPcaCgMax, cols - cc), cg = kPcaCgMax;
    rc |= PcaGroupScales(c, ts, g + cc, g_ld, 1, npad, valid, nullptr, nullptr);
    for (int pass = 0; pass < kPcaPasses; ++pass) {
      pca_digits_kernel<<<npad / 64, 256, 0, c->stream>>>(g + cc, g_ld, 1, npad, cg, valid, nullptr, nullptr, ts->scale, ts->gdig, nullptr, pass);
      pca_xa_wg_kernel<<<job->variant_cap / 128, kPcaThreads, kPxaSmemBytes, c->stream>>>(job->d_raw, job->pitch, npad, job->variant_ct, ts->gdig, valid, slope, icpt, ts->inv_scale, h + static_cast<uint64_t>(cc) * h_ld, h_ld,
                                                                                        pass ? 1.0 / kPcaPass1Scale : 1.0, pass);
      c->launches += 2;
    }
  }
  return rc;
}

// O += Y^T H: H column-major (ld h_ld, variant_ct rows), O element (s, c) at out[s out_rs + c out_cs]; cols columns.
// Needs the sample-major copy (PcaFinishLayouts) and the xtb scratch.
static int PcaLaunchXtb(Pl2PcaJob* job, PcaTs* ts, const double* h, uint64_t h_ld, uint32_t cols, double* out, uint64_t out_rs, uint64_t out_cs) {
  Ctx* c = &job->ctx->c;
  const uint32_t n = job->sample_ct, npad = job->sample_ct_padded, m = job->variant_ct;
  int rc = 0;
  for (uint32_t cc = 0; cc < cols; cc += kPcaCgMax) {
    const uint32_t valid = std::min(kPcaCgMax, cols - cc), cg = kPcaCgMax;
    const double* src = h + static_cast<uint64_t>(cc) * h_ld;
    rc |= PcaGroupScales(c, ts, src, 1, h_ld, m, valid, job->d_slope, job->d_icpt);
    for (int pass = 0; pass < kPcaPasses; ++pass) {
      pca_digits_kernel<<<job->variant_cap / 64, 256, 0, c->stream>>>(src, 1, h_ld, m, cg, valid, job->d_slope, job->d_icpt, ts->scale, ts->hs, ts->hi, pass);
      if (cudaMemsetAsync(ts->partial, 0, static_cast<uint64_t>(ts->splits) * npad * cg * 8, c->stream) != cudaSuccess) rc = 1;
      pca_xtb_wg_kernel<<<dim3(npad / 128, ts->splits), kPcaThreads, kPxtSmemBytes, c->stream>>>(job->d_raw_i, job->variant_cap / 32, ts->ksteps_per_split, n, ts->hs, ts->hi, ts->inv_scale, ts->partial, npad);
      pca_xtb_reduce_kernel<<<static_cast<uint32_t>(DivUpU64(static_cast<uint64_t>(n) * cg, 256)), 256, 0, c->stream>>>(ts->partial, ts->splits, n, npad, cg, valid, pass ? 1.0 / kPcaPass1Scale : 1.0,
                                                                                                                      out + static_cast<uint64_t>(cc) * out_cs, out_rs, out_cs);
      c->launches += 3;
    }
  }
  return rc;
}

// The run itself.  sharded:the job holds ONE variant shard of a world-size team (contexts joined by pl2gpu_comm_init;
// collective call).  Everything that contracts over variants is a partial sum on each rank and is completed by an
// in-place fp64 all-reduce (NCCL returns the same bits on every rank, so the replicated small steps stay in lockstep):
// G' = Y^T H per pass (N x 2k - the exchange SURVEY 8e names), the block Gram-Schmidt coefficients, B = Y^T Q.  The
// M x 2k block of each orthonormalisation pass is all-gathered (320 bytes per variant) and every rank runs the same
// Jacobi SVD on it, keeping its own rows.
static int PcaRunImpl(Pl2PcaJob* job, const double* g1_host, uint64_t total_variant_ct, bool sharded, double* eigvals_host, double* eigvecs_host) {
  if (!job || !g1_host || !job->pc_ct) {
    set_error("pl2gpu_pca_run: bad arguments (needs g1 and a job begun with pc_ct > 0)");
    return 1;
  }
  Ctx* c = &job->ctx->c;
  PL2_CUDA_OK(cudaSetDevice(c->device));
  const uint32_t n = job->sample_ct, npad = job->sample_ct_padded, m = job->variant_ct, k = job->pc_ct;
  const uint32_t c2 = 2 * k;
  const uint64_t q = static_cast<uint64_t>(c2) * (k + 1);
  const uint32_t world = sharded ? static_cast<uint32_t>(c->comm_world) : 1, rank = sharded ? static_cast<uint32_t>(c->comm_rank) : 0;
  if (sharded && (!c->comm || !m)) {
    set_error("pl2gpu_pca_run_sharded: needs a communicator on the context and a non-empty shard");
    return 1;
  }
  if (!sharded) total_variant_ct = m;
  if (q > total_variant_ct || q > n) {
    set_error("pl2gpu_pca_run: need 2k(k+1) = %llu <= min(variants %llu, samples %u)", static_cast<unsigned long long>(q), static_cast<unsigned long long>(total_variant_ct), n);
    return 1;
  }
  double *d_qq = nullptr, *d_u = nullptr, *d_g1 = nullptr, *d_g2 = nullptr, *d_b = nullptr, *d_gram = nullptr, *d_gram_u = nullptr, *d_gram_partial = nullptr, *d_colscale = nullptr;
  int rc = 1;
  const double m_recip = 1.0 / static_cast<double>(total_variant_ct);
  PL2_TRY(PcaFinishLayouts(job, true));
  PcaTs ts;
  PL2_TRY(PcaTsAlloc(job, true, &ts));
  int ts_rc = 0;
  // PL2_TIMING=1: phase times on stderr (stream-synchronising; development aid)
  const bool timing = getenv("PL2_TIMING") != nullptr;
  cudaEvent_t ev_t0 = nullptr, ev_t1 = nullptr;
  if (timing) {
    cudaEventCreate(&ev_t0);
    cudaEventCreate(&ev_t1);
    cudaEventRecord(ev_t0, c->stream);
  }
  auto mark = [&](const char* what) {
    if (!timing) return;
    cudaEventRecord(ev_t1, c->stream);
    cudaEventSynchronize(ev_t1);
    float ms = 0;
    cudaEventElapsedTime(&ms, ev_t0, ev_t1);
    fprintf(stderr, "[timing] pca_run %-34s %9.2f ms\n", what, ms);
    std::swap(ev_t0, ev_t1);
  };
  do {
    if (cudaMalloc(&d_qq, static_cast<uint64_t>(m) * q * 8) != cudaSuccess || cudaMalloc(&d_u, static_cast<uint64_t>(std::max(m, n)) * q * 8) != cudaSuccess || cudaMalloc(&d_g1, static_cast<uint64_t>(npad) * c2 * 8) != cudaSuccess ||
        cudaMalloc(&d_g2, static_cast<uint64_t>(npad) * c2 * 8) != cudaSuccess || cudaMalloc(&d_b, static_cast<uint64_t>(n) * q * 8) != cudaSuccess ) {
      cudaGetLastError();
      set_error("pl2gpu_pca_run: insufficient device memory for the %u x %llu Krylov matrix", m, static_cast<unsigned long long>(q));
      break;
    }
    if (cudaMemsetAsync(d_g1, 0, static_cast<uint64_t>(npad) * c2 * 8, c->stream) != cudaSuccess || cudaMemcpyAsync(d_g1, g1_host, static_cast<uint64_t>(n) * c2 * 8, cudaMemcpyHostToDevice, c->stream) != cudaSuccess) break;
    // k+1 projections; every H_t = Y G_t is kept side by side in qq (column-major M x q)   :5783-5855
    for (uint32_t iter = 0; iter <= k; ++iter) {
      double* h_t = d_qq + static_cast<uint64_t>(iter * c2) * m;
      ts_rc |= PcaLaunchXa(job, &ts, job->d_slope, job->d_icpt, d_g1, c2, h_t, m, c2);
      if (iter < k) {
        if (cudaMemsetAsync(d_g2, 0, static_cast<uint64_t>(npad) * c2 * 8, c->stream) != cudaSuccess) break;
        ts_rc |= PcaLaunchXtb(job, &ts, h_t, m, c2, d_g2, c2, 1);
        if (sharded && CommAllReduceSumF64(c, d_g2, static_cast<uint64_t>(npad) * c2, c->stream)) break;
        scale_kernel<<<static_cast<uint32_t>(DivUpU64(static_cast<uint64_t>(npad) * c2, 256)), 256, 0, c->stream>>>(d_g2, static_cast<uint64_t>(npad) * c2, m_recip);
        c->launches++;
        std::swap(d_g1, d_g2);
      }
    }
    if (cudaGetLastError() != cudaSuccess) {
      set_error("pl2gpu_pca_run: kernel launch failed");
      break;
    }
    mark("power iterations (Y.G / Yt.H)");
    // Orthonormal basis Q of the range of the Krylov matrix, built in place in qq   :5860 (the reference takes the left
    // singular vectors from dgesvd; only their span enters B = Y^T Q and everything after it).  Block classical
    // Gram-Schmidt over the k + 1 Krylov blocks, three projection passes per block (the blocks span 35 orders of
    // magnitude - two passes are not enough), each followed by a Jacobi SVD of the M x 2k residual whose unit left
    // singular vectors replace the block: O(M q^2) in all, what a one-sided Jacobi SVD of the whole M x q matrix costs
    // per sweep.  The structure PCs match the LAPACK-based restatement to 1e-13; the noise-level eigenvalues differ
    // from it by 1e-4..1e-3, because the Krylov matrix is numerically rank deficient and every method completes the
    // basis differently there.
    std::vector<double> s(q);
    const char* err = nullptr;
    double *d_c = nullptr, *d_cpart = nullptr, *d_wg = nullptr, *d_wf = nullptr, *d_uf = nullptr, *d_sizes = nullptr;
    uint64_t part_doubles = 1;
    for (uint32_t t = 1; t <= k; ++t) part_doubles = std::max(part_doubles, DgemmTNPartialDoubles(c, t * c2, c2, m));
    bool ok = cudaMalloc(&d_c, q * c2 * 8) == cudaSuccess && cudaMalloc(&d_cpart, part_doubles * 8) == cudaSuccess;
    // sharded: every rank learns the shard sizes (one all-reduce of a world-length vector), blocks are exchanged
    // in slots of the largest shard
    uint64_t m_pad = m;
    if (ok && sharded) {
      std::vector<double> sizes(world, 0.0);
      sizes[rank] = static_cast<double>(m);
      ok = cudaMalloc(&d_sizes, 8ull * world) == cudaSuccess && cudaMemcpyAsync(d_sizes, sizes.data(), 8ull * world, cudaMemcpyHostToDevice, c->stream) == cudaSuccess &&
           !CommAllReduceSumF64(c, d_sizes, world, c->stream) && cudaMemcpyAsync(sizes.data(), d_sizes, 8ull * world, cudaMemcpyDeviceToHost, c->stream) == cudaSuccess &&
           cudaStreamSynchronize(c->stream) == cudaSuccess;
      for (uint32_t r = 0; ok && r < world; ++r) m_pad = std::max<uint64_t>(m_pad, static_cast<uint64_t>(sizes[r]));
      const uint64_t blk = m_pad * c2 * 8;
      ok = ok && cudaMalloc(&d_wg, blk * world) == cudaSuccess && cudaMalloc(&d_wf, blk * world) == cudaSuccess && cudaMalloc(&d_uf, blk * world) == cudaSuccess;
    }
    const uint64_t m_full = m_pad * world;
    for (uint32_t t = 0; ok && t <= k; ++t) {
      double* w = d_qq + static_cast<uint64_t>(t) * c2 * m;
      const uint32_t prev = t * c2;
      for (int rep = 0; ok && rep < 3; ++rep) {
        if (prev) {
          ok = !DgemmTN(c, d_qq, m, prev, w, m, c2, m, d_cpart, d_c, prev) && !(sharded && CommAllReduceSumF64(c, d_c, static_cast<uint64_t>(prev) * c2, c->stream)) &&
               !DgemmNN(c, d_qq, m, m, prev, d_c, prev, c2, w, m, true, nullptr);
          if (!ok) break;
        }
        if (!sharded) {
          if (JacobiSvd(c, w, m, m, c2, c2, s.data(), d_u, m, nullptr, &err)) {
            ok = false;
            break;
          }
          ok = cudaMemcpyAsync(w, d_u, static_cast<uint64_t>(m) * c2 * 8, cudaMemcpyDeviceToDevice, c->stream) == cudaSuccess;
        } else {
          // my rows into my slot (zero-padded to m_pad), all-gather, repack to one column-major (world m_pad) x 2k
          // matrix, the same Jacobi SVD on every rank, my rows of the unit left singular vectors back into the block
          double* slot = d_wg + static_cast<uint64_t>(rank) * m_pad * c2;
          ok = cudaMemsetAsync(slot, 0, m_pad * c2 * 8, c->stream) == cudaSuccess &&
               cudaMemcpy2DAsync(slot, m_pad * 8, w, static_cast<uint64_t>(m) * 8, static_cast<uint64_t>(m) * 8, c2, cudaMemcpyDeviceToDevice, c->stream) == cudaSuccess &&
               !CommAllGatherInPlace(c, d_wg, m_pad * c2 * 8, c->stream);
          for (uint32_t r = 0; ok && r < world; ++r)
            ok = cudaMemcpy2DAsync(d_wf + static_cast<uint64_t>(r) * m_pad, m_full * 8, d_wg + static_cast<uint64_t>(r) * m_pad * c2, m_pad * 8, m_pad * 8, c2, cudaMemcpyDeviceToDevice, c->stream) == cudaSuccess;
          if (!ok) break;
          if (JacobiSvd(c, d_wf, m_full, static_cast<uint32_t>(m_full), c2, c2, s.data(), d_uf, m_full, nullptr, &err)) {
            ok = false;
            break;
          }
          ok = cudaMemcpy2DAsync(w, static_cast<uint64_t>(m) * 8, d_uf + static_cast<uint64_t>(rank) * m_pad, m_full * 8, static_cast<uint64_t>(m) * 8, c2, cudaMemcpyDeviceToDevice, c->stream) == cudaSuccess;
        }
      }
    }
    cudaFree(d_c);
    cudaFree(d_cpart);
    cudaFree(d_wg);
    cudaFree(d_wf);
    cudaFree(d_uf);
    cudaFree(d_sizes);
    if (!ok) {
      cudaGetLastError();
      if (!err && *get_error()) break;  // a collective already recorded its message
      set_error("Failed to orthonormalise the Krylov matrix (%s).", err ? err : "CUDA failure");
      break;
    }
    mark("orthonormal basis of the Krylov matrix (BCGS)");
    // B = Y^T Q (N x q, column-major)   :5870-5916
    if (cudaMemsetAsync(d_b, 0, static_cast<uint64_t>(n) * q * 8, c->stream) != cudaSuccess) break;
    ts_rc |= PcaLaunchXtb(job, &ts, d_qq, m, static_cast<uint32_t>(q), d_b, 1, n);
    if (sharded && CommAllReduceSumF64(c, d_b, static_cast<uint64_t>(n) * q, c->stream)) break;
    mark("B = Yt.Q");
    // Top-k left singular pairs of B (:5920, dgesvd in the reference).  Only the leading k of q are wanted and they
    // are the well-conditioned ones, so they come from the q x q Gram matrix: G = B^T B (fp64, fixed-order split
    // sums), eigenpairs of G by one-sided Jacobi on its columns (G V = V Lambda for a symmetric PSD matrix), then
    // U_k = B V_k Lambda_k^-1/2.  The relative error of sigma_i is eps (sigma_1 / sigma_i)^2 - 1e-14 here - and no
    // N x q Jacobi sweep over B is needed (1.2 s at N = 16,384, O(N q^2) per sweep).
    const uint32_t q32 = static_cast<uint32_t>(q);
    if (cudaMalloc(&d_gram, q * q * 8) != cudaSuccess || cudaMalloc(&d_gram_u, q * k * 8) != cudaSuccess || cudaMalloc(&d_gram_partial, DgemmTNPartialDoubles(c, q32, q32, n) * 8) != cudaSuccess ||
        cudaMalloc(&d_colscale, 8ull * k) != cudaSuccess) {
      cudaGetLastError();
      set_error("pl2gpu_pca_run: insufficient device memory for the %llu x %llu Gram matrix", static_cast<unsigned long long>(q), static_cast<unsigned long long>(q));
      break;
    }
    if (DgemmTN(c, d_b, n, q32, d_b, n, q32, n, d_gram_partial, d_gram, q)) break;
    if (JacobiSvd(c, d_gram, q, q32, q32, k, s.data(), d_gram_u, q, nullptr, &err)) {
      set_error("Failed to compute SVD of final matrix (%s).", err ? err : "?");
      break;
    }
    std::vector<double> inv_sigma(k);
    ok = true;
    for (uint32_t p = 0; p < k; ++p) {
      ok = ok && s[p] > 0.0;
      s[p] = sqrt(s[p]);  // eigenvalue of B^T B -> singular value of B
      inv_sigma[p] = ok ? 1.0 / s[p] : 0.0;
    }
    if (!ok) {
      set_error("Failed to compute SVD of final matrix (rank below the requested number of PCs).");
      break;
    }
    if (cudaMemcpyAsync(d_colscale, inv_sigma.data(), 8ull * k, cudaMemcpyHostToDevice, c->stream) != cudaSuccess) break;
    // d_u, the scratch of the basis construction, is free once B is formed (stream order): reuse it for U_k (N x k,
    // column-major)
    if (DgemmNN(c, d_b, n, n, q32, d_gram_u, q, k, d_u, n, false, d_colscale)) break;
    mark("top-k singular pairs of the N x q matrix B");
    // the context's stream is non-blocking: order the copy on it (a plain cudaMemcpy would not wait for the kernels)
    if (cudaMemcpyAsync(eigvecs_host, d_u, 8ull * k * n, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess || cudaStreamSynchronize(c->stream) != cudaSuccess) {
      set_error("pl2gpu_pca_run: %s", cudaGetErrorString(cudaGetLastError()));
      break;
    }
    for (uint32_t p = 0; p < k; ++p) eigvals_host[p] = s[p] * s[p] * m_recip;  // :5931
    rc = 0;
  } while (0);
  if (ev_t0) cudaEventDestroy(ev_t0);
  if (ev_t1) cudaEventDestroy(ev_t1);
  if (ts_rc && !rc) {
    set_error("pl2gpu_pca_run: a tensor-path launch failed");
    rc = 1;
  }
  PcaTsFree(&ts);
  cudaFree(d_gram);
  cudaFree(d_gram_u);
  cudaFree(d_gram_partial);
  cudaFree(d_colscale);
  cudaFree(d_qq);
  cudaFree(d_u);
  cudaFree(d_g1);
  cudaFree(d_g2);
  cudaFree(d_b);
  return rc;
}

extern "C" {

int pl2gpu_pca_run(Pl2PcaJob* job, const double* g1_host, double* eigvals_host, double* eigvecs_host) { return PcaRunImpl(job, g1_host, 0, false, eigvals_host, eigvecs_host); }

int pl2gpu_pca_run_sharded(Pl2PcaJob* job, const double* g1_host, uint64_t total_variant_ct, double* eigvals_host, double* eigvecs_host) {
  return PcaRunImpl(job, g1_host, total_variant_ct, true, eigvals_host, eigvecs_host);
}

int pl2gpu_pca_products(Pl2PcaJob* job, const double* g_host, uint32_t g_cols, double* yg_host, const double* h_host, uint32_t h_cols, double* yth_host) {
  if (!job || !job->variant_ct || (g_cols && (!g_host || !yg_host)) || (h_cols && (!h_host || !yth_host))) {
    set_error("pl2gpu_pca_products: bad arguments (needs a non-empty job)");
    return 1;
  }
  Ctx* c = &job->ctx->c;
  PL2_CUDA_OK(cudaSetDevice(c->device));
  const uint32_t n = job->sample_ct, npad = job->sample_ct_padded, m = job->variant_ct;
  PL2_TRY(PcaFinishLayouts(job, h_cols != 0));
  PcaTs ts;
  PL2_TRY(PcaTsAlloc(job, h_cols != 0, &ts));
  double *d_g = nullptr, *d_yg = nullptr, *d_h = nullptr, *d_yth = nullptr;
  int rc = 1;
  do {
    if (g_cols) {
      if (cudaMalloc(&d_g, static_cast<uint64_t>(npad) * g_cols * 8) != cudaSuccess || cudaMalloc(&d_yg, static_cast<uint64_t>(m) * g_cols * 8) != cudaSuccess) {
        cudaGetLastError();
        set_error("pl2gpu_pca_products: insufficient device memory for %u columns of Y G", g_cols);
        break;
      }
      if (cudaMemsetAsync(d_g, 0, static_cast<uint64_t>(npad) * g_cols * 8, c->stream) != cudaSuccess ||
          cudaMemcpyAsync(d_g, g_host, static_cast<uint64_t>(n) * g_cols * 8, cudaMemcpyHostToDevice, c->stream) != cudaSuccess || PcaLaunchXa(job, &ts, job->d_slope, job->d_icpt, d_g, g_cols, d_yg, m, g_cols) ||
          cudaMemcpyAsync(yg_host, d_yg, static_cast<uint64_t>(m) * g_cols * 8, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess) {
        set_error("pl2gpu_pca_products: Y G: %s", cudaGetErrorString(cudaGetLastError()));
        break;
      }
    }
    if (h_cols) {
      if (cudaMalloc(&d_h, static_cast<uint64_t>(m) * h_cols * 8) != cudaSuccess || cudaMalloc(&d_yth, static_cast<uint64_t>(n) * h_cols * 8) != cudaSuccess) {
        cudaGetLastError();
        set_error("pl2gpu_pca_products: insufficient device memory for %u columns of Y^T H", h_cols);
        break;
      }
      if (cudaMemcpyAsync(d_h, h_host, static_cast<uint64_t>(m) * h_cols * 8, cudaMemcpyHostToDevice, c->stream) != cudaSuccess ||
          cudaMemsetAsync(d_yth, 0, static_cast<uint64_t>(n) * h_cols * 8, c->stream) != cudaSuccess || PcaLaunchXtb(job, &ts, d_h, m, h_cols, d_yth, h_cols, 1) ||
          cudaMemcpyAsync(yth_host, d_yth, static_cast<uint64_t>(n) * h_cols * 8, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess) {
        set_error("pl2gpu_pca_products: Y^T H: %s", cudaGetErrorString(cudaGetLastError()));
        break;
      }
    }
    if (cudaStreamSynchronize(c->stream) != cudaSuccess || cudaGetLastError() != cudaSuccess) {
      set_error("pl2gpu_pca_products: %s", cudaGetErrorString(cudaGetLastError()));
      break;
    }
    rc = 0;
  } while (0);
  PcaTsFree(&ts);
  cudaFree(d_g);
  cudaFree(d_yg);
  cudaFree(d_h);
  cudaFree(d_yth);
  return rc;
}

// `--variant-score` (VscoreReport, 2.0/plink2_matrix_calc.cc:9274): per variant the dot product of sample weights with
// the ALT dosages, a missing call replaced by 2 x ALT frequency.  One H = Y W pass of the approx-PCA tile path does it:
// with Y the centred dosage (y = g - 2 f for a called genotype, 0 for a missing one: slope 1, intercept -2 f, whatever
// the variance - not the job's standardised matrix)
//   sum_s w_s dosage_vs  =  (Y W)_v + 2 f_v sum_s w_s .
static __global__ void __launch_bounds__(256) vscore_centre_kernel(const double* __restrict__ twof, uint32_t variant_ct, double* __restrict__ slope, double* __restrict__ icpt) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= variant_ct) return;
  slope[v] = 1.0;
  icpt[v] = -twof[v];
}

static __global__ void __launch_bounds__(256) vscore_finish_kernel(const double* __restrict__ h, uint64_t h_ld, uint32_t variant_ct, uint32_t cols, const double* __restrict__ twof, const double* __restrict__ wtot, double* __restrict__ out) {
  const uint64_t idx = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<uint64_t>(variant_ct) * cols) return;
  const uint32_t v = static_cast<uint32_t>(idx / cols), c = static_cast<uint32_t>(idx % cols);
  out[idx] = h[static_cast<uint64_t>(c) * h_ld + v] + twof[v] * wtot[c];
}

int pl2gpu_pca_vscore(Pl2PcaJob* job, const double* weights_host, uint32_t cols, double* out_host) {
  if (!job || !weights_host || !cols || !out_host || !job->variant_ct) {
    set_error("pl2gpu_pca_vscore: bad arguments (needs a non-empty job)");
    return 1;
  }
  Ctx* c = &job->ctx->c;
  PL2_CUDA_OK(cudaSetDevice(c->device));
  const uint32_t n = job->sample_ct, npad = job->sample_ct_padded, m = job->variant_ct;
  PL2_TRY(PcaFinishLayouts(job, false));
  PcaTs ts;
  PL2_TRY(PcaTsAlloc(job, false, &ts));
  double *d_w = nullptr, *d_h = nullptr, *d_wtot = nullptr, *d_out = nullptr, *d_slope = nullptr, *d_icpt = nullptr;
  int rc = 1;
  do {
    if (cudaMalloc(&d_w, static_cast<uint64_t>(npad) * cols * 8) != cudaSuccess || cudaMalloc(&d_h, static_cast<uint64_t>(m) * cols * 8) != cudaSuccess ||
        cudaMalloc(&d_wtot, 8ull * cols) != cudaSuccess || cudaMalloc(&d_out, static_cast<uint64_t>(m) * cols * 8) != cudaSuccess || cudaMalloc(&d_slope, 8ull * m) != cudaSuccess ||
        cudaMalloc(&d_icpt, 8ull * m) != cudaSuccess) {
      cudaGetLastError();
      set_error("pl2gpu_pca_vscore: insufficient device memory for %u score columns", cols);
      break;
    }
    std::vector<double> wtot(cols, 0.0);
    for (uint32_t s = 0; s < n; ++s)
      for (uint32_t cc = 0; cc < cols; ++cc) wtot[cc] += weights_host[static_cast<uint64_t>(s) * cols + cc];
    if (cudaMemsetAsync(d_w, 0, static_cast<uint64_t>(npad) * cols * 8, c->stream) != cudaSuccess || cudaMemcpyAsync(d_w, weights_host, static_cast<uint64_t>(n) * cols * 8, cudaMemcpyHostToDevice, c->stream) != cudaSuccess ||
        cudaMemcpyAsync(d_wtot, wtot.data(), 8ull * cols, cudaMemcpyHostToDevice, c->stream) != cudaSuccess)
      break;
    vscore_centre_kernel<<<DivUpU32(m, 256), 256, 0, c->stream>>>(job->d_twof, m, d_slope, d_icpt);
    c->launches++;
    if (PcaLaunchXa(job, &ts, d_slope, d_icpt, d_w, cols, d_h, m, cols) || cudaGetLastError() != cudaSuccess) {
      set_error("pl2gpu_pca_vscore: kernel launch failed");
      break;
    }
    vscore_finish_kernel<<<static_cast<uint32_t>(DivUpU64(static_cast<uint64_t>(m) * cols, 256)), 256, 0, c->stream>>>(d_h, m, m, cols, job->d_twof, d_wtot, d_out);
    c->launches++;
    if (cudaMemcpyAsync(out_host, d_out, static_cast<uint64_t>(m) * cols * 8, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess || cudaStreamSynchronize(c->stream) != cudaSuccess) {
      set_error("pl2gpu_pca_vscore: %s", cudaGetErrorString(cudaGetLastError()));
      break;
    }
    rc = 0;
  } while (0);
  PcaTsFree(&ts);
  cudaFree(d_w);
  cudaFree(d_h);
  cudaFree(d_wtot);
  cudaFree(d_out);
  cudaFree(d_slope);
  cudaFree(d_icpt);
  return rc;
}

int pl2gpu_pca_end(Pl2PcaJob* job) {
  if (!job) return 0;
  if (job->ctx) {
    cudaSetDevice(job->ctx->c.device);
    cudaStreamSynchronize(job->ctx->c.stream);
  }
  cudaFree(job->d_raw);
  cudaFree(job->d_raw_i);
  cudaFree(job->d_slope);
  cudaFree(job->d_icpt);
  cudaFree(job->d_twof);
  cudaFree(job->d_counts);
  cudaGetLastError();
  delete job;
  return 0;
}

}  // extern "C"
