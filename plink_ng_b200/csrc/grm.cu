// grm.cu - GRM job driver (kernel face of CalcGrm, 2.0/plink2_matrix_calc.cc:4555-5182).
#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <vector>


#include "../../include/plink2_b200.h"
#include "common.cuh"
#include "grm_kernels.cuh"
#include "grm_ts_kernel.cuh"
#include "jacobi.cuh"
#include "eig_krylov.cuh"
#include "ld_kernels.cuh"  // geno_counts_kernel

using namespace pl2;

namespace {
constexpr double kSmallEpsilon = 1.0 / 17592186044416.0;  // 2^-44
}

struct Pl2GrmJob {
  explicit Pl2GrmJob(Pl2GpuCtx* x) : ctx(x) {}
  ~Pl2GrmJob() {  // the kernels and copies that use the buffers finish before they are freed
    cudaSetDevice(ctx->c.device);
    cudaStreamSynchronize(ctx->c.stream);
    cudaStreamSynchronize(ctx->c.copy_stream);
  }
  Pl2GpuCtx* ctx;
  uint32_t sample_ct = 0, row_start = 0, row_end = 0;
  int flags = 0;
  TileList tiles;
  StageRing ring;  // genotype counts, digit tables and row re-tiling of each slot also run on the prep stream
  DevArray<uint8_t> d_raw_i[2];  // sample-major copy of the staged block (geno_tile.cuh)
  DevArray<uint8_t> d_tab[2];    // digit tables (grm_tables_kernel)
  DevArray<double> d_lvals[2];
  DevArray<uint32_t> d_counts[2];
  PinnedArray<double> h_lvals[2];
  PinnedArray<uint32_t> h_counts[2];
  DevArray<double> d_acc_g;
  DevArray<int32_t> d_acc_obs;
  DevArray<double> d_out_stage;
  uint64_t out_stage_bytes = 0;
  uint64_t variants_added = 0;
  uint64_t variants_with_missing = 0;
};

extern "C" {

int pl2gpu_grm_begin(Pl2GpuCtx* ctx, uint32_t sample_ct, uint32_t row_start, uint32_t row_end, int flags, Pl2GrmJob** job_ptr) {
  *job_ptr = nullptr;
  if (!ctx || !sample_ct || row_end > sample_ct || row_start > row_end) {  // empty range: a rank that only takes part in the all-gathers
    set_error("pl2gpu_grm_begin: bad row range [%u,%u) for %u samples", row_start, row_end, sample_ct);
    return 1;
  }
  PL2_CUDA_OK(cudaSetDevice(ctx->c.device));
  PL2_CUDA_OK(cudaFuncSetAttribute(grm_wg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kGwSmemBytes));
  std::unique_ptr<Pl2GrmJob, int (*)(Pl2GrmJob*)> job(new Pl2GrmJob(ctx), pl2gpu_grm_end);
  job->sample_ct = sample_ct;
  job->row_start = row_start;
  job->row_end = row_end;
  job->flags = flags;
  PL2_TRY(BuildTileList(row_start, row_end, true, &job->tiles, kGrmTileCols));
  const uint64_t words = static_cast<uint64_t>(job->tiles.tile_ct) * kGrmTileWords;
  job->out_stage_bytes = 256ull << 20;
  PL2_TRY(job->ring.alloc(&ctx->c, sample_ct, kMaxStageVariants, kGrmSamplePad));
  const uint64_t cap = job->ring.stage[0].variant_cap;
  const uint64_t raw_i_bytes = static_cast<uint64_t>(job->ring.stage[0].sample_ct_padded) * (cap / 4);
  const char* oom = "pl2gpu_grm_begin: insufficient device memory for %u pair tiles (%.1f GB of accumulators); narrow the row range";
  const uint32_t tile_ct = job->tiles.tile_ct;
  const double acc_gb = words * 12 / 1e9;
  for (int b = 0; b < 2; ++b) {
    if (job->d_raw_i[b].alloc(raw_i_bytes ? raw_i_bytes : 16, oom, tile_ct, acc_gb) || job->d_tab[b].alloc(cap / 16 * kGrmTabChunkBytes, oom, tile_ct, acc_gb) || job->d_lvals[b].alloc(cap * 6, oom, tile_ct, acc_gb) ||
        job->d_counts[b].alloc(cap * 4, oom, tile_ct, acc_gb) || job->h_lvals[b].alloc(cap * 6, oom, tile_ct, acc_gb) || job->h_counts[b].alloc(cap * 4, oom, tile_ct, acc_gb))
      return 1;
  }
  if (job->d_acc_g.alloc(words + 1, oom, tile_ct, acc_gb) || job->d_acc_obs.alloc(words + 1, oom, tile_ct, acc_gb) || job->d_out_stage.alloc(job->out_stage_bytes / 8, oom, tile_ct, acc_gb)) return 1;
  if (cudaMemsetAsync(job->d_acc_g, 0, words * 8, ctx->c.stream) != cudaSuccess || cudaMemsetAsync(job->d_acc_obs, 0, words * 4, ctx->c.stream) != cudaSuccess) {
    set_error("pl2gpu_grm_begin: memset failed");
    return 1;
  }
  *job_ptr = job.release();
  return 0;
}

// One staged batch: ring slot b rows [0, cur) hold the (already sample-padded when !pad_valid_rows) genotypes.
// Counts -> per-variant lookup values (host, a few microseconds per thousand variants) -> fixed-point digit
// tables, row re-tiling, tensor kernel.  ref_freqs: this batch's REF frequencies or nullptr.
static int GrmPrepAndLaunch(Pl2GrmJob* job, uint32_t b, uint32_t cur, bool pad_valid_rows, const double* ref_freqs) {
  Ctx* c = &job->ctx->c;
  cudaStream_t prep = c->copy_stream;
  const GenoStage& st = job->ring.stage[b];
  const bool cov = (job->flags & kPl2GrmCov) != 0;
  uint32_t padded;
  PL2_TRY(job->ring.pad(b, cur, pad_valid_rows, kVariantPad, &padded));
  // genotype counts of the batch: missingness presence, the zero-variance consistency check
  // (ExpandCenteredVarmaj :3844-3868) and, when the caller passes no frequencies, ComputeAlleleFreqs.
  geno_counts_kernel<<<DivUpU32(cur, 8), 256, 0, prep>>>(st.d_raw, st.pitch, st.sample_ct, st.sample_ct_padded, cur, job->d_counts[b]);
  c->launches++;
  uint32_t* h_counts = job->h_counts[b];
  double* h_lvals = job->h_lvals[b];
  PL2_CUDA_OK(cudaMemcpyAsync(h_counts, job->d_counts[b], 16ull * cur, cudaMemcpyDeviceToHost, prep));
  PL2_CUDA_OK(cudaStreamSynchronize(prep));  // the prep stream only: the previous batch's tensor kernel keeps running
  memset(h_lvals, 0, 48ull * cur);
  double max_l = 0.0;
  for (uint32_t v = 0; v < cur; ++v) {
    const uint32_t n0 = h_counts[4ull * v], n1 = h_counts[4ull * v + 1], n2 = h_counts[4ull * v + 2], n3 = h_counts[4ull * v + 3];
    if (n3) job->variants_with_missing++;
    double ref_freq;
    if (ref_freqs && ref_freqs[v] == ref_freqs[v]) {  // NaN entry: compute this variant's frequency from the block
      ref_freq = ref_freqs[v];
    } else {
      const uint64_t tot = 2ull * (static_cast<uint64_t>(n0) + n1 + n2);
      ref_freq = tot ? (static_cast<double>(2ull * n0 + n1) * (1.0 / static_cast<double>(tot))) : 0.5;
    }
    const double alt_freq = 1.0 - ref_freq;
    double inv_stdev;
    if (!cov) {
      const double variance = 2 * ref_freq * alt_freq;
      if (!(variance > kSmallEpsilon)) {
        // reference errors out unless the variant really is monomorphic for the expected allele
        bool bad = n1 != 0;
        if (variance != variance) {
          bad = bad || n0 || n2;
        } else if (ref_freq > 0.5) {
          bad = bad || n2;
        } else {
          bad = bad || n0;
        }
        if (bad) {
          set_error("pl2gpu_grm_add_variants: variant %llu has zero-variance allele frequency %g but non-monomorphic genotypes (kPglRetDegenerateData, plink2_matrix_calc.cc:3844-3868)", static_cast<unsigned long long>(job->variants_added + v), ref_freq);
          return 2;
        }
        continue;  // all-zero column
      }
      inv_stdev = 1.0 / sqrt(variance);
    } else {
      inv_stdev = 1.0;
    }
    // PopulateRescaledDosage lookup table (plink2_common.cc:323-330)
    const double slope = inv_stdev;
    const double intercept = -2 * alt_freq * inv_stdev;
    const double z[3] = {intercept, intercept + slope, intercept + 2 * slope};
    double* lv = &h_lvals[6ull * v];
    for (int g = 0; g < 3; ++g) {
      lv[g] = slope * z[g];          // multiplies the other sample's dosage g
      lv[3 + g] = intercept * z[g];  // multiplies the other sample's non-missing indicator
      max_l = std::max(max_l, std::max(fabs(lv[g]), fabs(lv[3 + g])));
    }
  }
  // fixed-point scale: |L| * 2^F < 2^38 so five balanced base-256 digits always suffice
  int f_bits = 0;
  if (max_l > 0.0) {
    int e;
    frexp(max_l, &e);  // max_l = m * 2^e, m in [0.5, 1)
    f_bits = static_cast<int>(kGrmFixedBits) - e;
  }
  const double scale = ldexp(1.0, f_bits), inv_scale = ldexp(1.0, -f_bits);
  PL2_CUDA_OK(cudaMemcpyAsync(job->d_lvals[b], h_lvals, 48ull * cur, cudaMemcpyHostToDevice, prep));
  grm_tables_kernel<<<DivUpU32(padded, 128), 128, 0, prep>>>(job->d_lvals[b], cur, padded, scale, job->d_tab[b]);
  c->launches++;
  if (job->tiles.tile_ct) {
    geno_tile_rows_kernel<<<dim3(padded / 64, st.sample_ct_padded / 64), 256, 0, prep>>>(st.d_raw, st.pitch, padded / 32, 0, job->d_raw_i[b]);
    c->launches++;
    PL2_CUDA_OK(cudaGetLastError());
    PL2_TRY(job->ring.fence(b));
    grm_wg_kernel<<<2 * job->tiles.tile_ct, kGwThreads, kGwSmemBytes, c->stream>>>(job->d_raw_i[b], padded, job->d_tab[b], inv_scale, job->tiles.d_tile_order, job->tiles.d_tile_rt, job->tiles.d_tile_tc, job->d_acc_g, job->d_acc_obs);
    c->launches++;
    PL2_CUDA_OK(cudaGetLastError());
  }
  return job->ring.mark_busy(b, job->tiles.tile_ct ? c->stream : prep);
}

int pl2gpu_grm_add_variants(Pl2GrmJob* job, const void* genovecs, uint64_t variant_stride_bytes, uint32_t variant_ct, int src_is_device, const double* ref_freqs) {
  if (!job) {
    set_error("pl2gpu_grm_add_variants: null job");
    return 1;
  }
  Ctx* c = &job->ctx->c;
  PL2_CUDA_OK(cudaSetDevice(c->device));
  if (variant_stride_bytes < DivUpU32(job->sample_ct, 4)) {
    set_error("pl2gpu_grm_add_variants: variant stride too small");
    return 1;
  }
  const uint8_t* src = static_cast<const uint8_t*>(genovecs);
  for (uint32_t done = 0; done < variant_ct;) {
    const uint32_t cur = std::min(job->ring.stage[0].variant_cap, variant_ct - done);
    uint32_t b;
    PL2_TRY(job->ring.acquire(src_is_device, &b));
    PL2_TRY(job->ring.land(b, nullptr, src + static_cast<uint64_t>(done) * variant_stride_bytes, variant_stride_bytes, cur, src_is_device));
    // GrmPrepAndLaunch synchronises the prep stream (it needs the counts on the host), so a host source has been
    // consumed when it returns; the tensor kernel keeps running
    const int rc = GrmPrepAndLaunch(job, b, cur, true, ref_freqs ? ref_freqs + done : nullptr);
    if (rc) return rc;
    job->variants_added += cur;
    done += cur;
  }
  return 0;
}

int pl2gpu_grm_add_variants_sharded(Pl2GrmJob* job, const void* slice, uint64_t variant_stride_bytes, uint32_t slice_variant_ct, uint32_t batch_variant_ct, int src_is_device, const double* ref_freqs) {
  if (!job || !job->ctx->c.comm) {
    set_error("pl2gpu_grm_add_variants_sharded: %s", job ? "no communicator attached to the context (pl2gpu_comm_init)" : "null job");
    return 1;
  }
  Ctx* c = &job->ctx->c;
  PL2_CUDA_OK(cudaSetDevice(c->device));
  const uint64_t total64 = static_cast<uint64_t>(slice_variant_ct) * c->comm_world;
  if (!slice_variant_ct || total64 > job->ring.stage[0].variant_cap || !batch_variant_ct || batch_variant_ct > total64) {
    set_error("pl2gpu_grm_add_variants_sharded: bad slice (%u variants x %d ranks, batch %u, stage capacity %u)", slice_variant_ct, c->comm_world, batch_variant_ct, job->ring.stage[0].variant_cap);
    return 1;
  }
  if (variant_stride_bytes < DivUpU32(job->sample_ct, 4)) {
    set_error("pl2gpu_grm_add_variants_sharded: variant stride too small");
    return 1;
  }
  uint32_t b;
  PL2_TRY(job->ring.acquire(src_is_device, &b));
  PL2_TRY(job->ring.land_slice(b, slice, variant_stride_bytes, slice_variant_ct, src_is_device));
  // only the first batch_variant_ct rows of the gathered tile are real variants (the last slice of a file is
  // topped up with filler rows); the rest is overwritten with "missing" by the tail padding
  const int rc = GrmPrepAndLaunch(job, b, batch_variant_ct, false, ref_freqs);
  if (rc) return rc;
  job->variants_added += batch_variant_ct;
  return 0;
}

int pl2gpu_grm_get_rows(Pl2GrmJob* job, uint32_t r0, uint32_t r1, double* dst_grm, float* dst_obs, uint64_t row_stride, int dst_is_device) {
  if (!job) {
    set_error("pl2gpu_grm_get_rows: null job");
    return 1;
  }
  if (r0 < job->row_start || r1 > job->row_end || r0 > r1 || row_stride < r1) {
    set_error("pl2gpu_grm_get_rows: rows [%u,%u) (stride %llu) outside the job's [%u,%u)", r0, r1, static_cast<unsigned long long>(row_stride), job->row_start, job->row_end);
    return 1;
  }
  Ctx* c = &job->ctx->c;
  PL2_CUDA_OK(cudaSetDevice(c->device));
  const bool meanimpute = (job->flags & kPl2GrmMeanimpute) != 0;
  const int use_obs = (!meanimpute && job->variants_with_missing) ? 1 : 0;  // CalcGrm :4756-4768
  const double recip = job->variants_added ? 1.0 / static_cast<double>(job->variants_added) : 0.0;
  const uint64_t per_row = row_stride * (dst_obs ? 12 : 8);
  uint32_t cur0 = r0;
  while (cur0 < r1) {
    uint32_t cur1;
    double* d_g;
    float* d_o = nullptr;
    if (dst_is_device) {
      cur1 = r1;
      d_g = dst_grm + static_cast<uint64_t>(cur0 - r0) * row_stride;
      if (dst_obs) d_o = dst_obs + static_cast<uint64_t>(cur0 - r0) * row_stride;
    } else {
      const uint64_t max_rows = job->out_stage_bytes / per_row;
      if (!max_rows) {
        set_error("pl2gpu_grm_get_rows: a single row exceeds the staging buffer");
        return 1;
      }
      cur1 = static_cast<uint32_t>(std::min<uint64_t>(r1, cur0 + max_rows));
      d_g = job->d_out_stage;
      if (dst_obs) d_o = reinterpret_cast<float*>(d_g + static_cast<uint64_t>(cur1 - cur0) * row_stride);
      PL2_CUDA_OK(cudaMemsetAsync(job->d_out_stage, 0, static_cast<uint64_t>(cur1 - cur0) * per_row, c->stream));
    }
    const uint32_t rt_a = cur0 / kTileRows - job->tiles.row_tile_first;
    const uint32_t rt_b = (cur1 - 1) / kTileRows - job->tiles.row_tile_first;
    const uint32_t tile_a = job->tiles.h_rowtile_offset[rt_a];
    const uint32_t tile_b = job->tiles.h_rowtile_offset[rt_b + 1];
    if (tile_b > tile_a) {
      grm_finalize_kernel<<<(tile_b - tile_a) * 8, 256, 0, c->stream>>>(job->d_acc_g + static_cast<uint64_t>(tile_a) * kGrmTileWords, job->d_acc_obs + static_cast<uint64_t>(tile_a) * kGrmTileWords, job->tiles.d_tile_rt + tile_a, job->tiles.d_tile_tc + tile_a,
                                                                              job->sample_ct, cur0, cur1, row_stride, use_obs, recip, d_g, d_o);
      c->launches++;
      PL2_CUDA_OK(cudaGetLastError());
    }
    if (!dst_is_device) {
      const uint64_t n = static_cast<uint64_t>(cur1 - cur0) * row_stride;
      PL2_CUDA_OK(cudaMemcpyAsync(dst_grm + static_cast<uint64_t>(cur0 - r0) * row_stride, d_g, n * 8, cudaMemcpyDeviceToHost, c->stream));
      if (dst_obs) PL2_CUDA_OK(cudaMemcpyAsync(dst_obs + static_cast<uint64_t>(cur0 - r0) * row_stride, d_o, n * 4, cudaMemcpyDeviceToHost, c->stream));
      PL2_CUDA_OK(cudaStreamSynchronize(c->stream));
    }
    cur0 = cur1;
  }
  return 0;
}

uint64_t pl2gpu_grm_variants_added(Pl2GrmJob* job) { return job ? job->variants_added : 0; }

}  // extern "C" (reopened below)

// ---- dense symmetric helpers for the exact-PCA eigensolve (jacobi.cuh) ----
namespace {
// get_rows fills the row-major lower triangle (= column-major upper); mirror it.
__global__ void symmetrize_kernel(double* __restrict__ a, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y;
  if (i < n && i > j) a[static_cast<uint64_t>(j) * n + i] = a[static_cast<uint64_t>(i) * n + j];
}
// per column: Gershgorin excess sum_{i != j} |a_ij| - a_jj, or NaN when the column holds a non-finite entry
__global__ void gershgorin_kernel(const double* __restrict__ a, uint32_t n, double* __restrict__ excess) {
  __shared__ double red[8];
  const uint32_t j = blockIdx.x;
  double sum = 0.0;
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
    const double v = a[static_cast<uint64_t>(j) * n + i];
    sum += (i == j) ? -v : fabs(v);  // NaN / inf propagate
  }
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xFFFFFFFFu, sum, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (uint32_t w = 0; w < blockDim.x / 32; ++w) t += red[w];
    excess[j] = t;
  }
}
__global__ void add_diagonal_kernel(double* __restrict__ a, uint32_t n, double mu) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[static_cast<uint64_t>(i) * n + i] += mu;
}
}  // namespace

extern "C" {

int pl2gpu_grm_eigen_topk(Pl2GrmJob* job, uint32_t pc_ct, double* eigvals_host, double* eigvecs_host) {
  if (!job || !pc_ct) {
    set_error("pl2gpu_grm_eigen_topk: bad arguments");
    return 1;
  }
  const uint32_t n = job->sample_ct;
  if (job->row_start != 0 || job->row_end != n) {
    set_error("pl2gpu_grm_eigen_topk: needs the whole matrix (rows [0,%u)), job holds [%u,%u)", n, job->row_start, job->row_end);
    return 1;
  }
  if (pc_ct > n) {
    set_error("pl2gpu_grm_eigen_topk: %u PCs requested from %u samples", pc_ct, n);
    return 1;
  }
  if (n > 46340) {  // same int32 n^2 limit as the reference's non-ILP64 LAPACK build (:5943-5948)
    set_error("pl2gpu_grm_eigen_topk: exact PCA is limited to 46340 samples; use --pca approx");
    return 1;
  }
  Ctx* c = &job->ctx->c;
  PL2_CUDA_OK(cudaSetDevice(c->device));
  // Top eigenpairs of the symmetric GRM by one-sided Jacobi on the shifted matrix G + mu I (mu = the
  // Gershgorin bound that makes it positive semi-definite, so singular values = eigenvalues + mu in
  // the same order and the unit columns of (G + mu I) V are the eigenvectors).  Replaces dsyevr (:5943-6039).
  DevArray<double> d_a, d_u, d_ex;
  const char* oom = "pl2gpu_grm_eigen_topk: insufficient device memory for a dense %u x %u matrix";
  if (d_a.alloc(static_cast<uint64_t>(n) * n, oom, n, n) || d_u.alloc(static_cast<uint64_t>(n) * pc_ct, oom, n, n) || d_ex.alloc(n, oom, n, n)) return 1;
  if (cudaMemsetAsync(d_a, 0, static_cast<uint64_t>(n) * n * 8, c->stream) != cudaSuccess) return 1;
  PL2_TRY(pl2gpu_grm_get_rows(job, 0, n, d_a, nullptr, n, 1));  // row-major lower triangle == column-major upper
  symmetrize_kernel<<<dim3(DivUpU32(n, 256), n), 256, 0, c->stream>>>(d_a, n);
  gershgorin_kernel<<<n, 256, 0, c->stream>>>(d_a, n, d_ex);
  c->launches += 2;
  std::vector<double> ex(n);
  if (cudaMemcpyAsync(ex.data(), d_ex, 8ull * n, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess || cudaStreamSynchronize(c->stream) != cudaSuccess) {
    set_error("pl2gpu_grm_eigen_topk: %s", cudaGetErrorString(cudaGetLastError()));
    return 1;
  }
  double mu = 0.0;
  bool finite = true;
  for (uint32_t j = 0; j < n; ++j) {
    finite = finite && std::isfinite(ex[j]);
    mu = std::max(mu, ex[j]);
  }
  if (!finite) {
    set_error("pl2gpu_grm_eigen_topk: GRM contains missing values (a sample pair has no jointly observed variant)");
    return 1;
  }
  // Small matrices: one-sided Jacobi on G + mu I (all eigenpairs, O(N^3) per sweep).  Beyond 2,048 samples - or with
  // PL2_EIGEN=krylov - the leading pairs come from a restarted block Krylov iteration on G itself (eig_krylov.cuh):
  // (2p + 1)(k + 8) N^2 MACs per restart instead of N^3 per sweep.  PL2_EIGEN=jacobi forces the dense form.
  const char* eig_env = getenv("PL2_EIGEN");
  const bool krylov = pc_ct + 8 <= n / 6 && ((eig_env && !strcmp(eig_env, "krylov")) || (!(eig_env && !strcmp(eig_env, "jacobi")) && n > 2048));
  std::vector<double> sigma(pc_ct);
  const char* err = nullptr;
  if (krylov) {
    uint32_t restarts = 0;
    if (SymEigTopKKrylov(c, d_a, n, pc_ct, sigma.data(), d_u, &restarts, &err)) {
      set_error("pl2gpu_grm_eigen_topk: eigendecomposition failed (%s)", err ? err : "?");
      return 1;
    }
    if (getenv("PL2_TIMING")) fprintf(stderr, "[timing]   eigen: block Krylov, %u restarts\n", restarts);
    mu = 0.0;
  } else {
    if (mu > 0.0) {
      add_diagonal_kernel<<<DivUpU32(n, 256), 256, 0, c->stream>>>(d_a, n, mu);
      c->launches++;
    }
    uint32_t sweeps = 0;
    if (JacobiSvd(c, d_a, n, n, n, pc_ct, sigma.data(), d_u, n, &sweeps, &err)) {
      set_error("pl2gpu_grm_eigen_topk: eigendecomposition failed (%s)", err ? err : "?");
      return 1;
    }
  }
  if (cudaMemcpyAsync(eigvecs_host, d_u, 8ull * pc_ct * n, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess || cudaStreamSynchronize(c->stream) != cudaSuccess) {
    set_error("pl2gpu_grm_eigen_topk: %s", cudaGetErrorString(cudaGetLastError()));
    return 1;
  }
  for (uint32_t k = 0; k < pc_ct; ++k) eigvals_host[k] = sigma[k] - mu;  // descending (:6024-6039)
  return 0;
}

int pl2gpu_grm_end(Pl2GrmJob* job) {
  if (!job) return 0;
  delete job;
  cudaGetLastError();
  return 0;
}

}  // extern "C"
