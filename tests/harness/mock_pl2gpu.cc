// mock_pl2gpu.cc - TEST INFRASTRUCTURE, never shipped and never linked into the product: a CPU stand-in for the few
// libpl2gpu entry points the `--indep-pairwise` / `--freq`-style host drivers call, injected with LD_PRELOAD so that
// the HOST ORCHESTRATION of plink2_b200 (filter view -> founder decode, chromosome runs spread over several device
// workers, relatedness-prune chaining with frozen allele frequencies) can be exercised in the CPU-only container.
// Like oracle/, it restates the reference's arithmetic (ComputeIndepPairwiseR2Components + the r^2 test,
// 2.0/plink2_ld.cc:699-723, :1085-1090; genotype counts) in plain loops; the greedy window walk is NOT restated - the
// real, exported pl2_ld_prune_walk of libpl2gpu.so (host code) is called.  Autosomal (diploid) chromosomes only.
// Build: g++ -O2 -std=c++17 -ffp-contract=off -shared -fPIC -o mock_pl2gpu.so mock_pl2gpu.cc
// PL2_MOCK_DEVICES = number of devices to report; PL2_MOCK_LOG = file that receives one line per entry-point call.
// Multi-GPU (--gpus): a communicator is a shared block in host memory; the *_add_variants_sharded calls all-gather
// every rank's slice into it at rank x slice and each rank then adds the whole gathered block, as NCCL would.
#include <cmath>
#include <condition_variable>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

struct MockComm;
struct Pl2GpuCtx {
  int device;
  MockComm* comm = nullptr;
  int rank = 0;
};

extern "C" int pl2_ld_prune_walk(uint32_t variant_ct, const uint32_t* chr_codes, const uint32_t* variant_bps, uint32_t window_size, uint32_t window_incr, int window_is_bp, const double* maj_freq, const uint8_t* mono,
                                 const uint8_t* pair_flags, uint32_t band, uint32_t flags, uint8_t* removed_out);

namespace {
thread_local std::string t_err;
std::mutex g_log_mu;
void Log(const char* fmt, int a, unsigned b) {
  const char* path = getenv("PL2_MOCK_LOG");
  if (!path) return;
  std::lock_guard<std::mutex> lock(g_log_mu);
  if (FILE* f = fopen(path, "a")) {
    fprintf(f, fmt, a, b);
    fclose(f);
  }
}
inline uint32_t Code(const uint8_t* row, uint32_t s) { return (row[s >> 2] >> (2 * (s & 3))) & 3; }
}  // namespace

struct MockComm {
  std::mutex mu;
  std::condition_variable cv;
  int world = 0;
  int arrived = 0;  // ranks whose slice has landed in this round
  int unread = 0;   // ranks still to copy out the previous round's block
  uint64_t round = 0;
  std::vector<uint8_t> block;
};
namespace {
// All-gather of equal-sized slices: rank r's bytes land at r x slice_bytes of the shared block; every rank waits until
// all `world` slices have landed and returns a copy of the whole block.  A new round starts only after every rank
// has copied out the previous one.
std::vector<uint8_t> AllGather(Pl2GpuCtx* ctx, const void* slice, uint64_t slice_bytes) {
  MockComm* c = ctx->comm;
  std::unique_lock<std::mutex> lock(c->mu);
  c->cv.wait(lock, [&] { return c->unread == 0; });
  if (!c->arrived) c->block.assign(static_cast<size_t>(c->world) * slice_bytes, 0);
  memcpy(&c->block[static_cast<size_t>(ctx->rank) * slice_bytes], slice, slice_bytes);
  const uint64_t round = c->round;
  if (++c->arrived == c->world) {
    c->arrived = 0;
    c->unread = c->world;
    ++c->round;
    c->cv.notify_all();
  } else {
    c->cv.wait(lock, [&] { return c->round != round; });
  }
  std::vector<uint8_t> out = c->block;
  if (--c->unread == 0) c->cv.notify_all();
  return out;
}
}  // namespace

extern "C" {

int pl2gpu_device_count(void) {
  const char* e = getenv("PL2_MOCK_DEVICES");
  return e ? atoi(e) : 1;
}
const char* pl2gpu_last_error(void) { return t_err.c_str(); }
int pl2gpu_ctx_create(int device_idx, Pl2GpuCtx** ctx_ptr) {
  if (device_idx < 0 || device_idx >= pl2gpu_device_count()) {
    t_err = "mock: no such device";
    return 1;
  }
  *ctx_ptr = new Pl2GpuCtx{device_idx};
  Log("ctx_create device=%d n=%u\n", device_idx, 0);
  return 0;
}
int pl2gpu_ctx_destroy(Pl2GpuCtx* ctx) {
  delete ctx;
  return 0;
}
// the id carries the address of a fresh communicator; every rank's pl2gpu_comm_init joins it
int pl2gpu_comm_unique_id(uint8_t* id_out) {
  MockComm* c = new MockComm;
  memset(id_out, 0, 128);
  memcpy(id_out, &c, sizeof(c));
  return 0;
}
int pl2gpu_comm_init(Pl2GpuCtx* ctx, int rank, int world, const uint8_t* id) {
  MockComm* c;
  memcpy(&c, id, sizeof(c));
  {
    std::lock_guard<std::mutex> lock(c->mu);
    c->world = world;
  }
  ctx->comm = c;
  ctx->rank = rank;
  Log("comm_init device=%d rank=%u\n", ctx->device, static_cast<unsigned>(rank));
  return 0;
}
int pl2gpu_comm_destroy(Pl2GpuCtx*) { return 0; }
int pl2gpu_ctx_synchronize(Pl2GpuCtx*) { return 0; }
int pl2gpu_host_alloc(uint64_t bytes, void** ptr) {
  *ptr = malloc(bytes ? bytes : 1);
  return *ptr ? 0 : 1;
}
int pl2gpu_host_free(void* ptr) {
  free(ptr);
  return 0;
}

int pl2gpu_geno_counts(Pl2GpuCtx* ctx, const void* genovecs, uint64_t stride, uint32_t sample_ct, uint32_t variant_ct, int, uint32_t* counts) {
  Log("geno_counts device=%d variants=%u\n", ctx->device, variant_ct);
  for (uint32_t v = 0; v < variant_ct; ++v) {
    const uint8_t* row = static_cast<const uint8_t*>(genovecs) + v * stride;
    uint32_t c[4] = {0, 0, 0, 0};
    for (uint32_t s = 0; s < sample_ct; ++s) ++c[Code(row, s)];
    memcpy(counts + 4ull * v, c, sizeof(c));
  }
  return 0;
}

// ---- KING pair counts (IncrKing, 2.0/plink2_matrix_calc.cc:1255-1295): the job keeps the variants it was given and counts on
// request.  counts[pair][5] = IBS0, HETHET, HET2HOM1, HET1HOM2, HOMHOM for pair (j, i), i < j, rows j in reference order.
}  // extern "C"
struct Pl2KingJob {
  uint32_t n, r0, r1;
  std::vector<uint8_t> codes;  // [variant][sample]
  uint64_t variants = 0;
  Pl2GpuCtx* ctx = nullptr;
};
namespace {
void PairCounts(const Pl2KingJob* job, uint32_t j, uint32_t i, uint32_t* c5) {
  uint32_t c[5] = {0, 0, 0, 0, 0};
  for (uint64_t v = 0; v < job->variants; ++v) {
    const uint8_t gi = job->codes[v * job->n + i], gj = job->codes[v * job->n + j];
    const bool hi = gi == 0 || gi == 2, hj = gj == 0 || gj == 2, ti = gi == 1, tj = gj == 1;
    c[0] += hi && hj && gi != gj;
    c[1] += ti && tj;
    c[2] += hi && tj;  // sample 2 (= j, the larger index) het, sample 1 hom
    c[3] += hj && ti;
    c[4] += hi && hj;
  }
  memcpy(c5, c, sizeof(c));
}
double Kinship(const uint32_t* c) {
  const double num = 4.0 * c[0] + c[3] + c[2], den = 4.0 * (c[1] + static_cast<double>(c[2] < c[3] ? c[2] : c[3]));
  return 0.5 - num / den;
}
}  // namespace
extern "C" {
int pl2gpu_ctx_mem_info(Pl2GpuCtx*, uint64_t* free_bytes, uint64_t* total_bytes) {
  const char* e = getenv("PL2_MOCK_MEM_MIB");
  const uint64_t mib = e ? strtoull(e, nullptr, 10) : 81920;
  *free_bytes = *total_bytes = mib << 20;
  return 0;
}
uint64_t pl2gpu_king_mem_required(uint32_t sample_ct, uint32_t row_start, uint32_t row_end, uint32_t) {
  return 2048ull * (static_cast<uint64_t>(row_end) * (row_end - 1) / 2 - static_cast<uint64_t>(row_start) * (row_start ? row_start - 1 : 0) / 2) + 4096ull * sample_ct;
}
int pl2gpu_king_begin_ex(Pl2GpuCtx* ctx, uint32_t sample_ct, uint32_t row_start, uint32_t row_end, int, uint32_t, Pl2KingJob** job_ptr) {
  Log("king_begin device=%d rows=%u\n", ctx->device, row_end - row_start);
  *job_ptr = new Pl2KingJob{sample_ct, row_start, row_end, {}, 0, ctx};
  return 0;
}
int pl2gpu_king_begin(Pl2GpuCtx* ctx, uint32_t sample_ct, uint32_t row_start, uint32_t row_end, int algo, Pl2KingJob** job_ptr) { return pl2gpu_king_begin_ex(ctx, sample_ct, row_start, row_end, algo, 0, job_ptr); }
int pl2gpu_king_add_variants(Pl2KingJob* job, const void* genovecs, uint64_t stride, uint32_t variant_ct, int) {
  for (uint32_t v = 0; v < variant_ct; ++v) {
    const uint8_t* row = static_cast<const uint8_t*>(genovecs) + v * stride;
    for (uint32_t s = 0; s < job->n; ++s) job->codes.push_back(static_cast<uint8_t>(Code(row, s)));
  }
  job->variants += variant_ct;
  return 0;
}
int pl2gpu_king_add_variants_sharded(Pl2KingJob* job, const void* slice, uint64_t stride, uint32_t slice_variant_ct, int src) {
  const std::vector<uint8_t> block = AllGather(job->ctx, slice, stride * slice_variant_ct);
  return pl2gpu_king_add_variants(job, block.data(), stride, static_cast<uint32_t>(block.size() / stride), src);
}
int pl2gpu_king_get_counts(Pl2KingJob* job, uint32_t out_row_start, uint32_t out_row_end, uint32_t* dst, int) {
  for (uint32_t j = out_row_start; j < out_row_end; ++j)
    for (uint32_t i = 0; i < j; ++i, dst += 5) PairCounts(job, j, i, dst);
  return 0;
}
int pl2gpu_king_get_kinship(Pl2KingJob* job, uint32_t out_row_start, uint32_t out_row_end, double* dst, int) {
  for (uint32_t j = out_row_start; j < out_row_end; ++j) {
    for (uint32_t i = 0; i < j; ++i) {
      uint32_t c[5];
      PairCounts(job, j, i, c);
      *dst++ = Kinship(c);
    }
  }
  return 0;
}
int pl2gpu_king_get_filtered(Pl2KingJob* job, uint32_t r0, uint32_t r1, double min_kinship, uint64_t max_out, uint32_t* pairs_out, uint32_t* counts_out, double* kinship_out, uint64_t* n_found) {
  uint64_t k = 0;
  for (uint32_t j = r0; j < r1; ++j) {
    for (uint32_t i = 0; i < j; ++i) {
      uint32_t c[5];
      PairCounts(job, j, i, c);
      const double kin = Kinship(c);
      if (kin < min_kinship) continue;
      if (k < max_out) {
        pairs_out[2 * k] = j;
        pairs_out[2 * k + 1] = i;
        memcpy(counts_out + 5 * k, c, sizeof(c));
        kinship_out[k] = kin;
      }
      ++k;
    }
  }
  *n_found = k;
  return 0;
}
uint64_t pl2gpu_king_variants_added(Pl2KingJob* job) { return job->variants; }
int pl2gpu_king_end(Pl2KingJob* job) {
  delete job;
  return 0;
}

// ---- GRM job (ExpandCenteredVarmaj + CalcGrm, 2.0/plink2_matrix_calc.cc:3839-3886, :4285, :4769-4788): variants kept as
// codes + REF frequency; values computed on request in plain fp64 loops.  eigen_topk: cyclic Jacobi on the full matrix.
}  // extern "C"
struct Pl2GrmJob {
  uint32_t n, r0, r1;
  int flags;
  std::vector<uint8_t> codes;   // [variant][sample]
  std::vector<double> ref_freq;  // per variant
  uint64_t variants = 0;
  Pl2GpuCtx* ctx = nullptr;
};
namespace {
void GrmMatrix(const Pl2GrmJob* job, std::vector<double>* g, std::vector<double>* obs) {
  const uint32_t n = job->n;
  const bool meanimpute = job->flags & 1, cov = job->flags & 2;
  g->assign(static_cast<size_t>(n) * n, 0.0);
  obs->assign(static_cast<size_t>(n) * n, 0.0);
  std::vector<double> z(n);
  std::vector<uint8_t> nm(n);
  for (uint64_t v = 0; v < job->variants; ++v) {
    const uint8_t* c = &job->codes[v * n];
    const double f = job->ref_freq[v], alt2 = 2.0 * (1.0 - f);
    const double var = 2.0 * f * (1.0 - f);
    const double inv_sd = cov ? 1.0 : (var > 0.0 ? 1.0 / sqrt(var) : 0.0);
    for (uint32_t s = 0; s < n; ++s) {
      nm[s] = c[s] != 3;
      z[s] = nm[s] ? (static_cast<double>(c[s]) - alt2) * inv_sd : 0.0;
      if (!cov && var <= 0.0) z[s] = 0.0;
    }
    for (uint32_t j = 0; j < n; ++j)
      for (uint32_t i = 0; i <= j; ++i) {
        (*g)[static_cast<size_t>(j) * n + i] += z[j] * z[i];
        (*obs)[static_cast<size_t>(j) * n + i] += nm[j] && nm[i];
      }
  }
  for (uint32_t j = 0; j < n; ++j)
    for (uint32_t i = 0; i <= j; ++i) {
      const double d = meanimpute ? static_cast<double>(job->variants) : (*obs)[static_cast<size_t>(j) * n + i];
      (*g)[static_cast<size_t>(j) * n + i] /= d;
    }
}
}  // namespace
extern "C" {
int pl2gpu_grm_begin(Pl2GpuCtx* ctx, uint32_t sample_ct, uint32_t row_start, uint32_t row_end, int flags, Pl2GrmJob** job_ptr) {
  Log("grm_begin device=%d rows=%u\n", ctx->device, row_end - row_start);
  *job_ptr = new Pl2GrmJob{sample_ct, row_start, row_end, flags, {}, {}, 0, ctx};
  return 0;
}
int pl2gpu_grm_add_variants(Pl2GrmJob* job, const void* genovecs, uint64_t stride, uint32_t variant_ct, int, const double* ref_freqs) {
  for (uint32_t v = 0; v < variant_ct; ++v) {
    const uint8_t* row = static_cast<const uint8_t*>(genovecs) + v * stride;
    uint64_t c[4] = {0, 0, 0, 0};
    for (uint32_t s = 0; s < job->n; ++s) {
      const uint32_t g = Code(row, s);
      ++c[g];
      job->codes.push_back(static_cast<uint8_t>(g));
    }
    const uint64_t tot = 2 * (c[0] + c[1] + c[2]);
    double f = tot ? static_cast<double>(2 * c[0] + c[1]) * (1.0 / static_cast<double>(tot)) : 0.5;
    if (ref_freqs && ref_freqs[v] == ref_freqs[v]) f = ref_freqs[v];
    job->ref_freq.push_back(f);
  }
  job->variants += variant_ct;
  return 0;
}
// the gathered block's first batch_variant_ct rows are the batch; the filler behind them is ignored
int pl2gpu_grm_add_variants_sharded(Pl2GrmJob* job, const void* slice, uint64_t stride, uint32_t slice_variant_ct, uint32_t batch_variant_ct, int src, const double* ref_freqs) {
  const std::vector<uint8_t> block = AllGather(job->ctx, slice, stride * slice_variant_ct);
  return pl2gpu_grm_add_variants(job, block.data(), stride, batch_variant_ct, src, ref_freqs);
}
int pl2gpu_grm_get_rows(Pl2GrmJob* job, uint32_t r0, uint32_t r1, double* dst_grm, float* dst_obs, uint64_t row_stride, int) {
  std::vector<double> g, obs;
  GrmMatrix(job, &g, &obs);
  for (uint32_t j = r0; j < r1; ++j)
    for (uint32_t i = 0; i <= j; ++i) {
      dst_grm[static_cast<uint64_t>(j - r0) * row_stride + i] = g[static_cast<size_t>(j) * job->n + i];
      if (dst_obs) dst_obs[static_cast<uint64_t>(j - r0) * row_stride + i] = static_cast<float>(obs[static_cast<size_t>(j) * job->n + i]);
    }
  return 0;
}
uint64_t pl2gpu_grm_variants_added(Pl2GrmJob* job) { return job->variants; }
int pl2gpu_grm_eigen_topk(Pl2GrmJob* job, uint32_t pc_ct, double* eigvals_host, double* eigvecs_host) {
  const uint32_t n = job->n;
  std::vector<double> a, obs;
  GrmMatrix(job, &a, &obs);
  for (uint32_t j = 0; j < n; ++j)
    for (uint32_t i = 0; i < j; ++i) a[static_cast<size_t>(i) * n + j] = a[static_cast<size_t>(j) * n + i];
  std::vector<double> vmat(static_cast<size_t>(n) * n, 0.0);
  for (uint32_t k = 0; k < n; ++k) vmat[static_cast<size_t>(k) * n + k] = 1.0;
  for (int sweep = 0; sweep < 60; ++sweep) {
    double off = 0.0;
    for (uint32_t p = 0; p < n; ++p)
      for (uint32_t q = p + 1; q < n; ++q) off += a[static_cast<size_t>(p) * n + q] * a[static_cast<size_t>(p) * n + q];
    if (off < 1e-26) break;
    for (uint32_t p = 0; p < n; ++p) {
      for (uint32_t q = p + 1; q < n; ++q) {
        const double apq = a[static_cast<size_t>(p) * n + q];
        if (apq == 0.0) continue;
        const double theta = (a[static_cast<size_t>(q) * n + q] - a[static_cast<size_t>(p) * n + p]) / (2.0 * apq);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0)), cs = 1.0 / sqrt(t * t + 1.0), sn = t * cs;
        for (uint32_t k = 0; k < n; ++k) {
          const double akp = a[static_cast<size_t>(k) * n + p], akq = a[static_cast<size_t>(k) * n + q];
          a[static_cast<size_t>(k) * n + p] = cs * akp - sn * akq;
          a[static_cast<size_t>(k) * n + q] = sn * akp + cs * akq;
        }
        for (uint32_t k = 0; k < n; ++k) {
          const double apk = a[static_cast<size_t>(p) * n + k], aqk = a[static_cast<size_t>(q) * n + k];
          a[static_cast<size_t>(p) * n + k] = cs * apk - sn * aqk;
          a[static_cast<size_t>(q) * n + k] = sn * apk + cs * aqk;
        }
        for (uint32_t k = 0; k < n; ++k) {
          const double vkp = vmat[static_cast<size_t>(k) * n + p], vkq = vmat[static_cast<size_t>(k) * n + q];
          vmat[static_cast<size_t>(k) * n + p] = cs * vkp - sn * vkq;
          vmat[static_cast<size_t>(k) * n + q] = sn * vkp + cs * vkq;
        }
      }
    }
  }
  std::vector<uint32_t> order(n);
  for (uint32_t k = 0; k < n; ++k) order[k] = k;
  for (uint32_t x = 0; x < n; ++x)
    for (uint32_t y = x + 1; y < n; ++y)
      if (a[static_cast<size_t>(order[y]) * n + order[y]] > a[static_cast<size_t>(order[x]) * n + order[x]]) std::swap(order[x], order[y]);
  for (uint32_t pc = 0; pc < pc_ct; ++pc) {
    eigvals_host[pc] = a[static_cast<size_t>(order[pc]) * n + order[pc]];
    for (uint32_t s = 0; s < n; ++s) eigvecs_host[static_cast<size_t>(pc) * n + s] = vmat[static_cast<size_t>(s) * n + order[pc]];
  }
  return 0;
}
int pl2gpu_grm_end(Pl2GrmJob* job) {
  delete job;
  return 0;
}

// ---- --score accumulation (contract in include/plink2_b200.h): per entry a 4-entry weight table and packed dosages
}  // extern "C"
struct Pl2ScoreJob {
  uint32_t n;
  std::vector<double> sums;
  std::vector<uint64_t> dosage;
  std::vector<uint32_t> missing;
};
extern "C" {
int pl2gpu_score_begin(Pl2GpuCtx* ctx, uint32_t sample_ct, Pl2ScoreJob** job_ptr) {
  Log("score_begin device=%d n=%u\n", ctx->device, sample_ct);
  *job_ptr = new Pl2ScoreJob{sample_ct, std::vector<double>(sample_ct, 0.0), std::vector<uint64_t>(sample_ct, 0), std::vector<uint32_t>(sample_ct, 0)};
  return 0;
}
int pl2gpu_score_add_variants(Pl2ScoreJob* job, const void* genovecs, uint64_t stride, uint32_t variant_ct, int, const double* weights4, const uint8_t* named_dosages) {
  for (uint32_t e = 0; e < variant_ct; ++e) {
    const uint8_t* row = static_cast<const uint8_t*>(genovecs) + e * stride;
    for (uint32_t s = 0; s < job->n; ++s) {
      const uint32_t g = Code(row, s);
      job->sums[s] += weights4[4ull * e + g];
      if (g == 3) ++job->missing[s];
      else job->dosage[s] += (named_dosages[e] >> (2 * g)) & 3;
    }
  }
  return 0;
}
int pl2gpu_score_get(Pl2ScoreJob* job, double* score_sums, uint64_t* named_dosage_sums, uint32_t* missing_cts) {
  memcpy(score_sums, job->sums.data(), job->n * sizeof(double));
  memcpy(named_dosage_sums, job->dosage.data(), job->n * sizeof(uint64_t));
  memcpy(missing_cts, job->missing.data(), job->n * sizeof(uint32_t));
  return 0;
}
int pl2gpu_score_end(Pl2ScoreJob* job) {
  delete job;
  return 0;
}

// ---- --variant-score on a "PCA job": only begin / add_variants / vscore / end are provided (no approx-PCA stand-in)
}  // extern "C"
struct Pl2PcaJob {
  uint32_t n;
  std::vector<uint8_t> codes;
  std::vector<double> alt_freq;
  uint64_t variants = 0;
};
struct Pl2KingPairJob {
  Pl2KingJob king;
  std::vector<uint32_t> pairs;
};
extern "C" {
int pl2gpu_pca_begin_shard(Pl2GpuCtx* ctx, uint32_t sample_ct, uint32_t, uint32_t, Pl2PcaJob** job_ptr) {
  Log("pca_begin device=%d n=%u\n", ctx->device, sample_ct);
  *job_ptr = new Pl2PcaJob{sample_ct, {}, {}, 0};
  return 0;
}
int pl2gpu_pca_add_variants(Pl2PcaJob* job, const void* genovecs, uint64_t stride, uint32_t variant_ct, int, const double* ref_freqs) {
  for (uint32_t v = 0; v < variant_ct; ++v) {
    const uint8_t* row = static_cast<const uint8_t*>(genovecs) + v * stride;
    uint64_t c[4] = {0, 0, 0, 0};
    for (uint32_t s = 0; s < job->n; ++s) {
      const uint32_t g = Code(row, s);
      ++c[g];
      job->codes.push_back(static_cast<uint8_t>(g));
    }
    const uint64_t tot = 2 * (c[0] + c[1] + c[2]);
    double f = tot ? static_cast<double>(2 * c[0] + c[1]) * (1.0 / static_cast<double>(tot)) : 0.5;
    if (ref_freqs && ref_freqs[v] == ref_freqs[v]) f = ref_freqs[v];
    job->alt_freq.push_back(1.0 - f);
  }
  job->variants += variant_ct;
  return 0;
}
int pl2gpu_pca_vscore(Pl2PcaJob* job, const double* weights_host, uint32_t cols, double* out_host) {
  for (uint64_t v = 0; v < job->variants; ++v) {
    for (uint32_t c = 0; c < cols; ++c) {
      double acc = 0.0;
      for (uint32_t s = 0; s < job->n; ++s) {
        const uint8_t g = job->codes[v * job->n + s];
        acc += weights_host[static_cast<size_t>(s) * cols + c] * (g == 3 ? 2.0 * job->alt_freq[v] : static_cast<double>(g));
      }
      out_host[v * cols + c] = acc;
    }
  }
  return 0;
}
int pl2gpu_pca_end(Pl2PcaJob* job) {
  delete job;
  return 0;
}
// ---- pair-list KING (--king-table-subset, rel-check): counts for the listed pairs {j, i} only
int pl2gpu_king_pairs_begin(Pl2GpuCtx* ctx, uint32_t sample_ct, const uint32_t* pairs_host, uint64_t pair_ct, Pl2KingPairJob** job_ptr) {
  Log("king_pairs_begin device=%d pairs=%u\n", ctx->device, static_cast<unsigned>(pair_ct));
  *job_ptr = new Pl2KingPairJob{Pl2KingJob{sample_ct, 0, sample_ct, {}, 0}, std::vector<uint32_t>(pairs_host, pairs_host + 2 * pair_ct)};
  return 0;
}
int pl2gpu_king_pairs_add_variants(Pl2KingPairJob* job, const void* genovecs, uint64_t stride, uint32_t variant_ct, int src) { return pl2gpu_king_add_variants(&job->king, genovecs, stride, variant_ct, src); }
int pl2gpu_king_pairs_get_counts(Pl2KingPairJob* job, uint64_t pair_start, uint64_t pair_end, uint32_t* dst, int) {
  for (uint64_t k = pair_start; k < pair_end; ++k, dst += 5) {
    const uint32_t a = job->pairs[2 * k], b = job->pairs[2 * k + 1];
    PairCounts(&job->king, b, a, dst);  // "1" = the first listed sample, "2" = the second (no reordering by index)
  }
  return 0;
}
int pl2gpu_king_pairs_end(Pl2KingPairJob* job) {
  delete job;
  return 0;
}

// pair-decision band on its own (the screening pass of --r2-unphased): flags[v * band + d - 1] = cov^2 > t var1 var2
// for second = v, first = v - d, exact integer sextuple over samples non-missing in both (plink2_ld.cc:699-723)
int pl2gpu_ld_band_flags(Pl2GpuCtx* ctx, const void* genovecs, uint64_t stride, uint32_t founder_ct, uint32_t variant_ct, int, uint32_t band, double thresh, uint8_t* flags_host) {
  Log("ld_band_flags device=%d variants=%u\n", ctx->device, variant_ct);
  const uint32_t n = founder_ct, m = variant_ct;
  std::vector<int8_t> x(static_cast<size_t>(m) * n), nm(static_cast<size_t>(m) * n);
  for (uint32_t v = 0; v < m; ++v) {
    const uint8_t* row = static_cast<const uint8_t*>(genovecs) + v * stride;
    for (uint32_t s = 0; s < n; ++s) {
      const uint32_t g = Code(row, s);
      x[static_cast<size_t>(v) * n + s] = g == 0 ? 1 : (g == 2 ? -1 : 0);
      nm[static_cast<size_t>(v) * n + s] = g != 3;
    }
  }
  memset(flags_host, 0, static_cast<size_t>(m) * band);
  for (uint32_t v = 1; v < m; ++v) {
    for (uint32_t d = 1; d <= band && d <= v; ++d) {
      const uint32_t b = v - d;
      const int8_t *xa = &x[static_cast<size_t>(v) * n], *na = &nm[static_cast<size_t>(v) * n], *xb = &x[static_cast<size_t>(b) * n], *nb = &nm[static_cast<size_t>(b) * n];
      int64_t nm_ct = 0, dot = 0, s_b = 0, q_b = 0, s_a = 0, q_a = 0;
      for (uint32_t s = 0; s < n; ++s) {
        nm_ct += nb[s] * na[s];
        dot += xb[s] * xa[s];
        s_b += xb[s] * na[s];
        q_b += xb[s] * xb[s] * na[s];
        s_a += nb[s] * xa[s];
        q_a += nb[s] * xa[s] * xa[s];
      }
      const double cov12 = static_cast<double>(dot * nm_ct - s_b * s_a);
      const double var1 = static_cast<double>(q_b * nm_ct - s_b * s_b), var2 = static_cast<double>(q_a * nm_ct - s_a * s_a);
      flags_host[static_cast<size_t>(v) * band + d - 1] = cov12 * cov12 > thresh * var1 * var2;
    }
  }
  return 0;
}

int pl2_indep_pairwise_ex(Pl2GpuCtx* ctx, const void* genovecs, uint64_t stride, uint32_t founder_ct, uint32_t variant_ct, const uint32_t* chr_codes, const uint32_t* variant_bps, uint32_t window_size, uint32_t window_incr,
                          double r2_thresh, int window_is_bp, const double* ref_freqs, const uint8_t* preferred, int, const uint8_t*, uint32_t flags_in, uint8_t* removed_out) {
  Log("indep_pairwise device=%d variants=%u\n", ctx->device, variant_ct);
  for (uint32_t v = 0; v < variant_ct; ++v) {
    if (chr_codes[v] == 0 || chr_codes[v] == 23 || chr_codes[v] == 24 || chr_codes[v] == 26) {  // the diploid class of ld.cu's ClassOf
      t_err = "mock: diploid chromosomes only";
      return 1;
    }
  }
  if (window_is_bp) {
    t_err = "mock: variant-count windows only";
    return 1;
  }
  const uint32_t n = founder_ct, m = variant_ct;
  std::vector<int8_t> x(static_cast<size_t>(m) * n), nm(static_cast<size_t>(m) * n);
  std::vector<double> maj(m);
  std::vector<uint8_t> mono(m);
  for (uint32_t v = 0; v < m; ++v) {
    const uint8_t* row = static_cast<const uint8_t*>(genovecs) + v * stride;
    uint64_t c[4] = {0, 0, 0, 0};
    for (uint32_t s = 0; s < n; ++s) {
      const uint32_t g = Code(row, s);
      ++c[g];
      x[static_cast<size_t>(v) * n + s] = g == 0 ? 1 : (g == 2 ? -1 : 0);
      nm[static_cast<size_t>(v) * n + s] = g != 3;
    }
    const uint64_t tot = 2 * (c[0] + c[1] + c[2]);
    double f = tot ? static_cast<double>(2 * c[0] + c[1]) * (1.0 / static_cast<double>(tot)) : 0.5;
    if (ref_freqs && ref_freqs[v] == ref_freqs[v]) f = ref_freqs[v];
    maj[v] = (f < 0.5 ? 1.0 - f : f) - ((preferred && preferred[v]) ? 1.0 : 0.0);
    const uint64_t nmc = c[0] + c[1] + c[2];
    mono[v] = (c[0] == 0 && c[2] == 0) || c[0] == nmc || c[2] == nmc;  // plink2_ld.cc:902
  }
  const uint32_t band = window_size - 1;
  const double thr = r2_thresh * (1.0 + 1.0 / 17592186044416.0);
  std::vector<uint8_t> flags(static_cast<size_t>(m) * band, 0);
  for (uint32_t v = 1; v < m; ++v) {
    for (uint32_t d = 1; d <= band && d <= v; ++d) {
      const uint32_t b = v - d;  // first
      if (chr_codes[b] != chr_codes[v]) break;
      const int8_t *xa = &x[static_cast<size_t>(v) * n], *na = &nm[static_cast<size_t>(v) * n], *xb = &x[static_cast<size_t>(b) * n], *nb = &nm[static_cast<size_t>(b) * n];
      int64_t nm_ct = 0, dot = 0, s_b = 0, q_b = 0, s_a = 0, q_a = 0;
      for (uint32_t s = 0; s < n; ++s) {
        nm_ct += nb[s] * na[s];
        dot += xb[s] * xa[s];
        s_b += xb[s] * na[s];
        q_b += xb[s] * xb[s] * na[s];
        s_a += nb[s] * xa[s];
        q_a += nb[s] * xa[s] * xa[s];
      }
      const double cov12 = static_cast<double>(dot * nm_ct - s_b * s_a);
      const double var1 = static_cast<double>(q_b * nm_ct - s_b * s_b), var2 = static_cast<double>(q_a * nm_ct - s_a * s_a);
      flags[static_cast<size_t>(v) * band + d - 1] = cov12 * cov12 > thr * var1 * var2;
    }
  }
  return pl2_ld_prune_walk(m, chr_codes, variant_bps, window_size, window_incr, 0, maj.data(), mono.data(), flags.data(), band, flags_in, removed_out);
}

}  // extern "C"
