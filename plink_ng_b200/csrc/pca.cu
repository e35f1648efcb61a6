// pca.cu - `--pca approx` job (CalcPca approx branch, 2.0/plink2_matrix_calc.cc:5697-5941): the
// EIGENSOFT-style randomized range finder (Halko et al. 2011; Galinsky et al. 2016) on the resident
// 2-bit genotype matrix.  Gaussian start matrix is supplied by the caller (the host program
// reproduces the reference's SFMT / Box-Muller stream, host/sfmt.cc).
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "../../include/plink2_b200.h"
#include "common.cuh"
#include "ld_kernels.cuh"    // geno_counts_kernel
#include "geno_tile.cuh"
#include "pca_kernels.cuh"
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
  double* d_ztab = nullptr;
  uint32_t* d_counts = nullptr;
  std::vector<double> h_ztab;
  std::vector<uint32_t> h_counts;
  // tensor path (default; PL2_PCA_ALGO=fp64 selects the CUDA-core kernels of pca_kernels.cuh as a cross-check)
  bool tensor = true;
  uint8_t* d_raw_i = nullptr;   // sample-major copy [row tile][k-step][128][8 B] of the whole matrix (geno_tile.cuh)
  double* d_slope = nullptr;    // per variant: inv_stdev (0 for skipped variants)
  double* d_icpt = nullptr;     // per variant: -2 alt_freq inv_stdev
  double* d_twof = nullptr;     // per variant: 2 alt_freq (the mean-imputation value of --variant-score)
  std::vector<double> h_slope, h_icpt, h_twof;
  uint32_t retiled_to = 0;      // variants [0, retiled_to) are in d_raw_i (multiple of 64)
};

extern "C" {

int pl2gpu_pca_end(Pl2PcaJob* job);

static int PcaBeginImpl(Pl2GpuCtx* ctx, uint32_t sample_ct, uint32_t variant_ct_total, uint32_t pc_ct, bool shard, Pl2PcaJob** job_ptr) {
  *job_ptr = nullptr;
  if (!ctx || !sample_ct || !variant_ct_total || !pc_ct) {
    set_error("pl2gpu_pca_begin: bad arguments");
    return 1;
  }
  const uint64_t q = 2ull * pc_ct * (pc_ct + 1);
  if (q > variant_ct_total && !shard) {  // :5716-5719 (a shard is judged on the total, at run time)
    set_error("Too few variants to compute %u PCs with \"--pca approx\" (%llu required).", pc_ct, static_cast<unsigned long long>(q));
    return 2;
  }
  if (q > sample_ct) {
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
  {
    const char* algo = getenv("PL2_PCA_ALGO");
    job->tensor = !(algo && !strcmp(algo, "fp64"));
  }
  if (cudaMalloc(&job->d_raw, static_cast<uint64_t>(job->variant_cap) * job->pitch) != cudaSuccess || cudaMalloc(&job->d_ztab, static_cast<uint64_t>(job->variant_cap) * 32) != cudaSuccess ||
      cudaMalloc(&job->d_counts, 16ull * 65536) != cudaSuccess ||
      (job->tensor && (cudaMalloc(&job->d_raw_i, static_cast<uint64_t>(job->sample_ct_padded) * (job->variant_cap / 4)) != cudaSuccess || cudaMalloc(&job->d_slope, 8ull * job->variant_cap) != cudaSuccess ||
                       cudaMalloc(&job->d_icpt, 8ull * job->variant_cap) != cudaSuccess || cudaMalloc(&job->d_twof, 8ull * job->variant_cap) != cudaSuccess))) {
    cudaGetLastError();
    set_error("pl2gpu_pca_begin: insufficient device memory to keep %u x %u genotypes resident", variant_ct_total, sample_ct);
    pl2gpu_pca_end(job);
    return 1;
  }
  if (job->tensor) {
    if (cudaMemsetAsync(job->d_slope, 0, 8ull * job->variant_cap, ctx->c.stream) != cudaSuccess || cudaMemsetAsync(job->d_icpt, 0, 8ull * job->variant_cap, ctx->c.stream) != cudaSuccess ||
        cudaFuncSetAttribute(pca_xa_wg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kPxaSmemBytes) != cudaSuccess ||
        cudaFuncSetAttribute(pca_xtb_wg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kPxtSmemBytes) != cudaSuccess) {
      if (!*get_error()) set_error("pl2gpu_pca_begin: %s", cudaGetErrorString(cudaGetLastError()));
      pl2gpu_pca_end(job);
      return 1;
    }
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
    job->h_ztab.assign(4ull * cur, 0.0);
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
        if (bad) {
          set_error("pl2gpu_pca_add_variants: variant %u has zero-variance allele frequency %g but non-monomorphic genotypes (kPglRetDegenerateData)", job->variant_ct + v, ref_freq);
          return 2;
        }
        continue;
      }
      const double inv_stdev = 1.0 / sqrt(variance);
      const double intercept = -2 * alt_freq * inv_stdev;
      double* z = &job->h_ztab[4ull * v];
      z[0] = intercept;
      z[1] = intercept + inv_stdev;
      z[2] = intercept + 2 * inv_stdev;
      job->h_slope[v] = inv_stdev;
      job->h_icpt[v] = intercept;
    }
    PL2_CUDA_OK(cudaMemcpyAsync(job->d_ztab + 4ull * job->variant_ct, job->h_ztab.data(), 32ull * cur, cudaMemcpyHostToDevice, c->stream));
    if (job->tensor) {
      PL2_CUDA_OK(cudaMemcpyAsync(job->d_slope + job->variant_ct, job->h_slope.data(), 8ull * cur, cudaMemcpyHostToDevice, c->stream));
      PL2_CUDA_OK(cudaMemcpyAsync(job->d_icpt + job->variant_ct, job->h_icpt.data(), 8ull * cur, cudaMemcpyHostToDevice, c->stream));
      PL2_CUDA_OK(cudaMemcpyAsync(job->d_twof + job->variant_ct, job->h_twof.data(), 8ull * cur, cudaMemcpyHostToDevice, c->stream));
    }
    PL2_CUDA_OK(cudaStreamSynchronize(c->stream));
    job->variant_ct += cur;
    done += cur;
  }
  return 0;
}

}  // extern "C"

// The run itself.  sharded: the job holds ONE variant shard of a world-size team (contexts joined by pl2gpu_comm_init;
// collective call).  Everything that contracts over variants is a partial sum on each rank and is completed by an
// in-place fp64 all-reduce (NCCL returns the same bits on every rank, so the replicated small steps stay in lockstep):
// G' = Y^T H per pass (N x 2k - the exchange SURVEY 8e names), the block Gram-Schmidt coefficients, B = Y^T Q.  The
// M x 2k block of each orthonormalisation pass is all-gathered (320 bytes per variant) and every rank runs the same
// Jacobi SVD on it, keeping its own rows.
static int PcaRunImpl(Pl2PcaJob* job, const double* g1_host, uint64_t total_variant_ct, bool sharded, double* eigvals_host, double* eigvecs_host) {
  if (!job || !g1_host) {
    set_error("pl2gpu_pca_run: bad arguments");
    return 1;
  }
  Ctx* c = &job->ctx->c;
  PL2_CUDA_OK(cudaSetDevice(c->device));
  const uint32_t n = job->sample_ct, npad = job->sample_ct_padded, m = job->variant_ct, k = job->pc_ct;
  const uint32_t c2 = 2 * k;
  const uint64_t q = static_cast<uint64_t>(c2) * (k + 1);
  const uint32_t world = sharded ? static_cast<uint32_t>(c->comm_world) : 1, rank = sharded ? static_cast<uint32_t>(c->comm_rank) : 0;
  if (sharded && (!c->comm || !job->tensor || !m)) {
    set_error("pl2gpu_pca_run_sharded: needs a communicator on the context, the tensor path and a non-empty shard");
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
  // ---- tensor path scratch (pca_ts_kernels.cuh): digit planes, per-column scales, split-K partial sums ----
  const bool tensor = job->tensor;
  uint8_t *d_gdig = nullptr, *d_hs = nullptr, *d_hi = nullptr;
  double *d_scale = nullptr, *d_inv_scale = nullptr, *d_partial = nullptr;
  unsigned long long* d_colmax = nullptr;
  const uint32_t kstep_total = job->variant_cap / 32;
  const uint32_t tiles2 = npad / 128;
  uint32_t splits = std::max(1u, std::min(DivUpU32(2 * static_cast<uint32_t>(c->sm_count), tiles2), kstep_total / 64));
  const uint32_t ksteps_per_split = RoundUpU32(DivUpU32(kstep_total, splits), 4);
  splits = DivUpU32(kstep_total, ksteps_per_split);
  int ts_rc = 0;
  if (tensor) {
    if (cudaMalloc(&d_gdig, static_cast<uint64_t>(npad) * kPcaNMax) != cudaSuccess || cudaMalloc(&d_hs, static_cast<uint64_t>(job->variant_cap) * kPcaNMax) != cudaSuccess ||
        cudaMalloc(&d_hi, static_cast<uint64_t>(job->variant_cap) * kPcaNMax) != cudaSuccess || cudaMalloc(&d_scale, 8 * kPcaCgMax) != cudaSuccess || cudaMalloc(&d_inv_scale, 8 * kPcaCgMax) != cudaSuccess ||
        cudaMalloc(&d_colmax, 8 * kPcaCgMax) != cudaSuccess || cudaMalloc(&d_partial, static_cast<uint64_t>(splits) * npad * kPcaCgMax * 8) != cudaSuccess) {
      cudaGetLastError();
      set_error("pl2gpu_pca_run: insufficient device memory for the digit planes");
      cudaFree(d_gdig); cudaFree(d_hs); cudaFree(d_hi); cudaFree(d_scale); cudaFree(d_inv_scale); cudaFree(d_colmax); cudaFree(d_partial);
      return 1;
    }
    // rows [variant_ct, variant_cap) must decode to "missing" in both layouts; finish the sample-major copy
    if (job->variant_cap > m) PL2_TRY(LaunchPadGenotypes(c, job->d_raw + static_cast<uint64_t>(m) * job->pitch, job->pitch, job->sample_ct, 0, job->variant_cap - m));
    if (job->retiled_to < job->variant_cap) {
      const uint32_t from = job->retiled_to;
      geno_tile_rows_kernel<<<dim3((job->variant_cap - from) / 64, npad / 64), 256, 0, c->stream>>>(job->d_raw + static_cast<uint64_t>(from) * job->pitch, job->pitch, kstep_total, 0, job->d_raw_i + static_cast<uint64_t>(from / 32) * 1024);
      c->launches++;
      job->retiled_to = job->variant_cap;
    }
  }
  // column group: up to 48 columns, padded to a multiple of 4 (the padding columns are zero digits and never written)
  auto group_scales = [&](const double* src, uint64_t rs, uint64_t cs, uint32_t rows, uint32_t valid, const double* mul1, const double* mul2) {
    if (cudaMemsetAsync(d_colmax, 0, 8 * kPcaCgMax, c->stream) != cudaSuccess) ts_rc = 1;
    pca_colmax_kernel<<<dim3(valid, std::min<uint32_t>(64, DivUpU32(rows, 256))), 256, 0, c->stream>>>(src, rs, cs, rows, mul1, mul2, d_colmax);
    pca_scales_kernel<<<1, 64, 0, c->stream>>>(d_colmax, kPcaCgMax, d_scale, d_inv_scale);
    c->launches += 2;
  };
  // every dense operand goes through the tensor pipe twice: 30-bit fixed point, then the exact residual at another
  // 30 bits (pca_digits_kernel pass 1) - 60 bits below the column maximum, so the passes lose nothing against the
  // reference's fp64 dgemm (one 30-bit pass left the trailing, noise-level eigenvalues 2e-3 off)
  constexpr int kPasses = 2;
  auto launch_xa_ts = [&](const double* g, uint32_t g_ld, double* hout, uint64_t h_ld, uint32_t hcol0, uint32_t cols_total) {
    for (uint32_t cc = 0; cc < cols_total; cc += kPcaCgMax) {
      const uint32_t valid = std::min(kPcaCgMax, cols_total - cc), cg = kPcaCgMax;
      group_scales(g + cc, g_ld, 1, npad, valid, nullptr, nullptr);
      for (int pass = 0; pass < kPasses; ++pass) {
        pca_digits_kernel<<<npad / 64, 256, 0, c->stream>>>(g + cc, g_ld, 1, npad, cg, valid, nullptr, nullptr, d_scale, d_gdig, nullptr, pass);
        pca_xa_wg_kernel<<<job->variant_cap / 128, kPcaThreads, kPxaSmemBytes, c->stream>>>(job->d_raw, job->pitch, npad, m, d_gdig, valid, job->d_slope, job->d_icpt, d_inv_scale, hout + static_cast<uint64_t>(hcol0 + cc) * h_ld, h_ld,
                                                                                          pass ? 1.0 / kPcaPass1Scale : 1.0, pass);
        c->launches += 2;
      }
    }
  };
  auto launch_xtb_ts = [&](const double* hin, uint64_t h_ld, uint32_t hcol0, uint32_t cols_total, double* out, uint64_t out_rs, uint64_t out_cs) {
    for (uint32_t cc = 0; cc < cols_total; cc += kPcaCgMax) {
      const uint32_t valid = std::min(kPcaCgMax, cols_total - cc), cg = kPcaCgMax;
      const double* src = hin + static_cast<uint64_t>(hcol0 + cc) * h_ld;
      group_scales(src, 1, h_ld, m, valid, job->d_slope, job->d_icpt);
      for (int pass = 0; pass < kPasses; ++pass) {
        pca_digits_kernel<<<job->variant_cap / 64, 256, 0, c->stream>>>(src, 1, h_ld, m, cg, valid, job->d_slope, job->d_icpt, d_scale, d_hs, d_hi, pass);
        if (cudaMemsetAsync(d_partial, 0, static_cast<uint64_t>(splits) * npad * cg * 8, c->stream) != cudaSuccess) ts_rc = 1;
        pca_xtb_wg_kernel<<<dim3(tiles2, splits), kPcaThreads, kPxtSmemBytes, c->stream>>>(job->d_raw_i, kstep_total, ksteps_per_split, n, d_hs, d_hi, d_inv_scale, d_partial, npad);
        pca_xtb_reduce_kernel<<<static_cast<uint32_t>(DivUpU64(static_cast<uint64_t>(n) * cg, 256)), 256, 0, c->stream>>>(d_partial, splits, n, npad, cg, valid, pass ? 1.0 / kPcaPass1Scale : 1.0, out + static_cast<uint64_t>(cc) * out_cs, out_rs, out_cs);
        c->launches += 3;
      }
    }
  };
  auto launch_xa_fp64 = [&](const double* g, uint32_t g_ld, double* hout, uint64_t h_ld, uint32_t hcol0, uint32_t cols_total) {
    for (uint32_t cc = 0; cc < cols_total; cc += kPcaColsMax) {
      const uint32_t cols = std::min(kPcaColsMax, cols_total - cc);
      pca_xa_kernel<<<DivUpU32(m, 128), 32 * DivUpU32(cols, 4), (128 * cols + 4) * 8, c->stream>>>(job->d_raw, job->pitch, npad, m, job->d_ztab, g + cc, g_ld, 0, cols, hout + static_cast<uint64_t>(hcol0 + cc) * h_ld, h_ld, 0);
      c->launches++;
    }
  };
  auto launch_xtb_fp64 = [&](const double* hin, uint64_t h_ld, uint32_t hcol0, uint32_t cols_total, double* out, uint64_t out_rs, uint64_t out_cs) {
    for (uint32_t cc = 0; cc < cols_total; cc += kPcaColsMax) {
      const uint32_t cols = std::min(kPcaColsMax, cols_total - cc);
      pca_xtb_kernel<<<DivUpU32(n, 128), 32 * DivUpU32(cols, 4), (128 * cols + 512) * 8, c->stream>>>(job->d_raw, job->pitch, n, m, job->d_ztab, hin + static_cast<uint64_t>(hcol0 + cc) * h_ld, h_ld, 0, 0, cols, out + static_cast<uint64_t>(cc) * out_cs, out_rs, out_cs);
      c->launches++;
    }
  };
  auto launch_xa = [&](const double* g, uint32_t g_ld, double* hout, uint64_t h_ld, uint32_t hcol0, uint32_t cols_total) {
    if (tensor) launch_xa_ts(g, g_ld, hout, h_ld, hcol0, cols_total);
    else launch_xa_fp64(g, g_ld, hout, h_ld, hcol0, cols_total);
  };
  auto launch_xtb = [&](const double* hin, uint64_t h_ld, uint32_t hcol0, uint32_t cols_total, double* out, uint64_t out_rs, uint64_t out_cs) {
    if (tensor) launch_xtb_ts(hin, h_ld, hcol0, cols_total, out, out_rs, out_cs);
    else launch_xtb_fp64(hin, h_ld, hcol0, cols_total, out, out_rs, out_cs);
  };
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
      launch_xa(d_g1, c2, d_qq, m, iter * c2, c2);
      if (iter < k) {
        if (cudaMemsetAsync(d_g2, 0, static_cast<uint64_t>(npad) * c2 * 8, c->stream) != cudaSuccess) break;
        launch_xtb(d_qq, m, iter * c2, c2, d_g2, c2, 1);
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
    // Orthonormal basis Q of the range of the Krylov matrix   :5860 (the reference takes the left singular vectors
    // from dgesvd; only their span enters B = Y^T Q and everything after it).
    //   Default: block classical Gram-Schmidt over the k + 1 Krylov blocks, three projection passes per block (the
    //   blocks span 35 orders of magnitude - two passes are not enough), each followed by a Jacobi SVD of the M x 2k
    //   residual whose unit left singular vectors replace the block.  O(M q^2) once instead of per Jacobi sweep.
    //   PL2_PCA_BASIS=jacobi: one-sided Jacobi SVD of the whole M x q matrix (jacobi.cuh), the round-1 form.
    //   Both give the structure PCs to 1e-13 of the LAPACK-based restatement and differ from it by 1e-4..1e-3 in the
    //   noise-level eigenvalues (tests/harness/pca_basis_compare.py): the Krylov matrix is numerically rank deficient
    //   and every method completes the basis differently there.
    std::vector<double> s(q);
    const char* err = nullptr;
    const char* basis_env = getenv("PL2_PCA_BASIS");
    const bool bcgs = sharded || !(basis_env && !strcmp(basis_env, "jacobi"));
    const double* d_basis = d_u;
    if (!bcgs) {
      if (JacobiSvd(c, d_qq, m, m, static_cast<uint32_t>(q), static_cast<uint32_t>(q), s.data(), d_u, m, nullptr, &err)) {
        set_error("Failed to compute SVD of Krylov matrix (%s).", err ? err : "?");
        break;
      }
    } else {
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
      d_basis = d_qq;
    }
    mark(bcgs ? "orthonormal basis of the Krylov matrix (BCGS)" : "SVD of the M x q Krylov matrix");
    // B = Y^T Q (N x q, column-major)   :5870-5916
    if (cudaMemsetAsync(d_b, 0, static_cast<uint64_t>(n) * q * 8, c->stream) != cudaSuccess) break;
    launch_xtb(d_basis, m, 0, static_cast<uint32_t>(q), d_b, 1, n);
    if (sharded && CommAllReduceSumF64(c, d_b, static_cast<uint64_t>(n) * q, c->stream)) break;
    mark("B = Yt.Q");
    // Top-k left singular pairs of B (:5920, dgesvd in the reference).  Only the leading k of q are wanted and they
    // are the well-conditioned ones, so they come from the q x q Gram matrix: G = B^T B (fp64, fixed-order split
    // sums), eigenpairs of G by one-sided Jacobi on its columns (G V = V Lambda for a symmetric PSD matrix), then
    // U_k = B V_k Lambda_k^-1/2.  The relative error of sigma_i is eps (sigma_1 / sigma_i)^2 - 1e-14 here - and the
    // N x q Jacobi sweep over B (1.2 s at N = 16,384, O(N q^2) per sweep) is gone.  PL2_PCA_FINAL=jacobi keeps it.
    const char* final_env = getenv("PL2_PCA_FINAL");
    if (final_env && !strcmp(final_env, "jacobi")) {
      // Q (d_u) is dead once B is formed (stream order): reuse it for the left singular vectors of B
      if (JacobiSvd(c, d_b, n, n, static_cast<uint32_t>(q), k, s.data(), d_u, n, nullptr, &err)) {
        set_error("Failed to compute SVD of final matrix (%s).", err ? err : "?");
        break;
      }
    } else {
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
      bool ok = true;
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
      // Q (d_u) is dead once B is formed (stream order): reuse it for U_k (N x k, column-major)
      if (DgemmNN(c, d_b, n, n, q32, d_gram_u, q, k, d_u, n, false, d_colscale)) break;
    }
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
  cudaFree(d_gdig);
  cudaFree(d_hs);
  cudaFree(d_hi);
  cudaFree(d_scale);
  cudaFree(d_inv_scale);
  cudaFree(d_colmax);
  cudaFree(d_partial);
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

// `--variant-score` (VscoreReport, 2.0/plink2_matrix_calc.cc:9274): per variant the dot product of sample weights with
// the ALT dosages, a missing call replaced by 2 x ALT frequency.  One H = Y W pass of the approx-PCA tile path does it:
// with Y the standardised matrix (y = (g - 2 f) / sd for a called genotype, 0 for a missing one)
//   sum_s w_s dosage_vs  =  (Y W)_v sd_v + 2 f_v sum_s w_s ,
// so the int8 tensor kernel runs unchanged and a small epilogue un-standardises (variants without variance: 2 f W).
static __global__ void __launch_bounds__(256) vscore_finish_kernel(const double* __restrict__ h, uint64_t h_ld, uint32_t variant_ct, uint32_t cols, const double* __restrict__ slope, const double* __restrict__ twof, const double* __restrict__ wtot, double* __restrict__ out) {
  const uint64_t idx = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<uint64_t>(variant_ct) * cols) return;
  const uint32_t v = static_cast<uint32_t>(idx / cols), c = static_cast<uint32_t>(idx % cols);
  const double sl = slope[v];
  out[idx] = (sl != 0.0 ? h[static_cast<uint64_t>(c) * h_ld + v] / sl : 0.0) + twof[v] * wtot[c];
}

int pl2gpu_pca_vscore(Pl2PcaJob* job, const double* weights_host, uint32_t cols, double* out_host) {
  if (!job || !weights_host || !cols || !out_host || !job->tensor || !job->variant_ct) {
    set_error("pl2gpu_pca_vscore: bad arguments (needs a non-empty tensor-path job)");
    return 1;
  }
  Ctx* c = &job->ctx->c;
  PL2_CUDA_OK(cudaSetDevice(c->device));
  const uint32_t n = job->sample_ct, npad = job->sample_ct_padded, m = job->variant_ct;
  uint8_t* d_gdig = nullptr;
  double *d_scale = nullptr, *d_inv_scale = nullptr, *d_w = nullptr, *d_h = nullptr, *d_wtot = nullptr, *d_out = nullptr;
  unsigned long long* d_colmax = nullptr;
  int rc = 1;
  do {
    if (cudaMalloc(&d_gdig, static_cast<uint64_t>(npad) * kPcaNMax) != cudaSuccess || cudaMalloc(&d_scale, 8 * kPcaCgMax) != cudaSuccess || cudaMalloc(&d_inv_scale, 8 * kPcaCgMax) != cudaSuccess ||
        cudaMalloc(&d_colmax, 8 * kPcaCgMax) != cudaSuccess || cudaMalloc(&d_w, static_cast<uint64_t>(npad) * cols * 8) != cudaSuccess || cudaMalloc(&d_h, static_cast<uint64_t>(m) * cols * 8) != cudaSuccess ||
        cudaMalloc(&d_wtot, 8ull * cols) != cudaSuccess || cudaMalloc(&d_out, static_cast<uint64_t>(m) * cols * 8) != cudaSuccess) {
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
    // rows [variant_ct, variant_cap) must decode to "missing"
    if (job->variant_cap > m && LaunchPadGenotypes(c, job->d_raw + static_cast<uint64_t>(m) * job->pitch, job->pitch, job->sample_ct, 0, job->variant_cap - m)) break;
    bool ok = true;
    for (uint32_t cc = 0; ok && cc < cols; cc += kPcaCgMax) {
      const uint32_t valid = std::min(kPcaCgMax, cols - cc), cg = kPcaCgMax;
      ok = cudaMemsetAsync(d_colmax, 0, 8 * kPcaCgMax, c->stream) == cudaSuccess;
      pca_colmax_kernel<<<dim3(valid, std::min<uint32_t>(64, DivUpU32(npad, 256))), 256, 0, c->stream>>>(d_w + cc, cols, 1, npad, nullptr, nullptr, d_colmax);
      pca_scales_kernel<<<1, 64, 0, c->stream>>>(d_colmax, kPcaCgMax, d_scale, d_inv_scale);
      c->launches += 2;
      for (int pass = 0; pass < 2; ++pass) {
        pca_digits_kernel<<<npad / 64, 256, 0, c->stream>>>(d_w + cc, cols, 1, npad, cg, valid, nullptr, nullptr, d_scale, d_gdig, nullptr, pass);
        pca_xa_wg_kernel<<<job->variant_cap / 128, kPcaThreads, kPxaSmemBytes, c->stream>>>(job->d_raw, job->pitch, npad, m, d_gdig, valid, job->d_slope, job->d_icpt, d_inv_scale, d_h + static_cast<uint64_t>(cc) * m, m,
                                                                                          pass ? 1.0 / kPcaPass1Scale : 1.0, pass);
        c->launches += 2;
      }
      ok = ok && cudaGetLastError() == cudaSuccess;
    }
    if (!ok) {
      set_error("pl2gpu_pca_vscore: kernel launch failed");
      break;
    }
    vscore_finish_kernel<<<static_cast<uint32_t>(DivUpU64(static_cast<uint64_t>(m) * cols, 256)), 256, 0, c->stream>>>(d_h, m, m, cols, job->d_slope, job->d_twof, d_wtot, d_out);
    c->launches++;
    if (cudaMemcpyAsync(out_host, d_out, static_cast<uint64_t>(m) * cols * 8, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess || cudaStreamSynchronize(c->stream) != cudaSuccess) {
      set_error("pl2gpu_pca_vscore: %s", cudaGetErrorString(cudaGetLastError()));
      break;
    }
    rc = 0;
  } while (0);
  cudaFree(d_gdig);
  cudaFree(d_scale);
  cudaFree(d_inv_scale);
  cudaFree(d_colmax);
  cudaFree(d_w);
  cudaFree(d_h);
  cudaFree(d_wtot);
  cudaFree(d_out);
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
  cudaFree(job->d_ztab);
  cudaFree(job->d_counts);
  cudaGetLastError();
  delete job;
  return 0;
}

}  // extern "C"
