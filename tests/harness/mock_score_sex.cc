// Test-only stand-in for the `--score` job of libpl2gpu with sex-dependent ploidy (pl2gpu_score_set_sex /
// _add_variants_ploidy / _get_ploidy) and any number of coefficient columns (contract in include/plink2_b200.h), as
// plain fp64 loops.  It is preloaded AHEAD of mock_pl2gpu.so (LD_PRELOAD="mock_score_sex.so mock_pl2gpu.so"), so its
// score_* symbols take the place of the ones there while every other device entry point comes from mock_pl2gpu.so.
// The product never loads it.
#include <cstdint>
#include <cstring>
#include <vector>

struct Pl2GpuCtx;
struct Pl2ScoreJob {
  uint32_t n, score_ct;
  std::vector<double> sums;    // [sample][score_ct]
  std::vector<uint64_t> hdos;  // half allele units
  std::vector<uint32_t> miss_dip, miss_hap;
  std::vector<uint8_t> sex;
};

extern "C" {
int pl2gpu_score_begin_cols(Pl2GpuCtx*, uint32_t sample_ct, uint32_t score_ct, Pl2ScoreJob** job_ptr) {
  *job_ptr = new Pl2ScoreJob{sample_ct, score_ct, std::vector<double>(static_cast<size_t>(sample_ct) * score_ct, 0.0), std::vector<uint64_t>(sample_ct, 0), std::vector<uint32_t>(sample_ct, 0), std::vector<uint32_t>(sample_ct, 0),
                             std::vector<uint8_t>(sample_ct, 0)};
  return 0;
}
int pl2gpu_score_begin(Pl2GpuCtx* ctx, uint32_t sample_ct, Pl2ScoreJob** job_ptr) { return pl2gpu_score_begin_cols(ctx, sample_ct, 1, job_ptr); }
int pl2gpu_score_set_sex(Pl2ScoreJob* job, const uint8_t* sample_sex) {
  job->sex.assign(sample_sex, sample_sex + job->n);
  return 0;
}
// classes: 0 diploid, 1 haploid for every sample, 2 chrY (females skipped, males haploid, unknown sex: diploid table,
// no dosage, haploid missing count), 3 chrX males haploid
int pl2gpu_score_add_variants_ploidy(Pl2ScoreJob* job, const void* genovecs, uint64_t stride, uint32_t variant_ct, int, const uint8_t* classes, const double* w_dip, const double* w_hap, const uint8_t* named_dosages) {
  const uint32_t sc = job->score_ct;
  for (uint32_t e = 0; e < variant_ct; ++e) {
    const uint8_t* row = static_cast<const uint8_t*>(genovecs) + e * stride;
    for (uint32_t s = 0; s < job->n; ++s) {
      const uint8_t pc = classes[e], sex = job->sex[s];
      if (pc == 2 && sex == 2) continue;
      const bool hap = pc == 1 || (pc == 2 && sex == 1) || (pc == 3 && sex == 1);
      const double* w = (hap ? w_hap : w_dip) + 4ull * static_cast<uint64_t>(e) * sc;
      const uint32_t g = (row[s >> 2] >> (2 * (s & 3))) & 3;
      for (uint32_t c = 0; c < sc; ++c) job->sums[static_cast<size_t>(s) * sc + c] += w[4 * c + g];
      if (g == 3) ++((hap || pc == 2) ? job->miss_hap : job->miss_dip)[s];
      else if (pc != 2 || hap) job->hdos[s] += ((named_dosages[e] >> (2 * g)) & 3) * (hap ? 1 : 2);
    }
  }
  return 0;
}
int pl2gpu_score_add_variants(Pl2ScoreJob* job, const void* genovecs, uint64_t stride, uint32_t variant_ct, int src_is_device, const double* weights4, const uint8_t* named_dosages) {
  const std::vector<uint8_t> classes(variant_ct, 0);
  return pl2gpu_score_add_variants_ploidy(job, genovecs, stride, variant_ct, src_is_device, classes.data(), weights4, nullptr, named_dosages);
}
int pl2gpu_score_get_ploidy(Pl2ScoreJob* job, double* score_sums, uint64_t* named_half_dosage_sums, uint32_t* missing_diploid_cts, uint32_t* missing_haploid_cts) {
  memcpy(score_sums, job->sums.data(), job->sums.size() * sizeof(double));
  if (named_half_dosage_sums) memcpy(named_half_dosage_sums, job->hdos.data(), job->n * sizeof(uint64_t));
  if (missing_diploid_cts) memcpy(missing_diploid_cts, job->miss_dip.data(), job->n * sizeof(uint32_t));
  if (missing_haploid_cts) memcpy(missing_haploid_cts, job->miss_hap.data(), job->n * sizeof(uint32_t));
  return 0;
}
int pl2gpu_score_get(Pl2ScoreJob* job, double* score_sums, uint64_t* named_dosage_sums, uint32_t* missing_cts) {
  memcpy(score_sums, job->sums.data(), job->sums.size() * sizeof(double));
  if (named_dosage_sums)
    for (uint32_t s = 0; s < job->n; ++s) named_dosage_sums[s] = job->hdos[s] / 2;
  if (missing_cts) memcpy(missing_cts, job->miss_dip.data(), job->n * sizeof(uint32_t));
  return 0;
}
int pl2gpu_score_end(Pl2ScoreJob* job) {
  delete job;
  return 0;
}
}  // extern "C"
