// Test-only stand-in for the `--score` job of libpl2gpu with any number of coefficient columns
// (pl2gpu_score_begin_cols; contract in include/plink2_b200.h), as plain fp64 loops.  It is preloaded AHEAD of
// mock_pl2gpu.so (LD_PRELOAD="mock_score_cols.so mock_pl2gpu.so"), so its score_* symbols take the place of the
// one-column ones there while every other device entry point comes from mock_pl2gpu.so.  The product never loads it.
#include <cstdint>
#include <cstring>
#include <vector>

struct Pl2GpuCtx;
struct Pl2ScoreJob {
  uint32_t n, score_ct;
  std::vector<double> sums;  // [sample][score_ct]
  std::vector<uint64_t> dosage;
  std::vector<uint32_t> missing;
};

extern "C" {
int pl2gpu_score_begin_cols(Pl2GpuCtx*, uint32_t sample_ct, uint32_t score_ct, Pl2ScoreJob** job_ptr) {
  *job_ptr = new Pl2ScoreJob{sample_ct, score_ct, std::vector<double>(static_cast<size_t>(sample_ct) * score_ct, 0.0), std::vector<uint64_t>(sample_ct, 0), std::vector<uint32_t>(sample_ct, 0)};
  return 0;
}
int pl2gpu_score_begin(Pl2GpuCtx* ctx, uint32_t sample_ct, Pl2ScoreJob** job_ptr) { return pl2gpu_score_begin_cols(ctx, sample_ct, 1, job_ptr); }
int pl2gpu_score_add_variants(Pl2ScoreJob* job, const void* genovecs, uint64_t stride, uint32_t variant_ct, int, const double* weights4, const uint8_t* named_dosages) {
  const uint32_t sc = job->score_ct;
  for (uint32_t e = 0; e < variant_ct; ++e) {
    const uint8_t* row = static_cast<const uint8_t*>(genovecs) + e * stride;
    for (uint32_t s = 0; s < job->n; ++s) {
      const uint32_t g = (row[s >> 2] >> (2 * (s & 3))) & 3;
      for (uint32_t c = 0; c < sc; ++c) job->sums[static_cast<size_t>(s) * sc + c] += weights4[4ull * (static_cast<uint64_t>(e) * sc + c) + g];
      if (g == 3) ++job->missing[s];
      else job->dosage[s] += (named_dosages[e] >> (2 * g)) & 3;
    }
  }
  return 0;
}
int pl2gpu_score_get(Pl2ScoreJob* job, double* score_sums, uint64_t* named_dosage_sums, uint32_t* missing_cts) {
  memcpy(score_sums, job->sums.data(), job->sums.size() * sizeof(double));
  if (named_dosage_sums) memcpy(named_dosage_sums, job->dosage.data(), job->n * sizeof(uint64_t));
  if (missing_cts) memcpy(missing_cts, job->missing.data(), job->n * sizeof(uint32_t));
  return 0;
}
int pl2gpu_score_end(Pl2ScoreJob* job) {
  delete job;
  return 0;
}
}  // extern "C"
