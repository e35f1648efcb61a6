// Test-only stand-in for the class-split `--score` job of libpl2gpu with shared rows (pl2gpu_score_begin_classes /
// _add_entries / _get_class, contract in include/plink2_b200.h), as plain fp64 loops: one accumulator set per class,
// each entry added to its class's set from the row it reads.  It is preloaded AHEAD of mock_pl2gpu.so
// (LD_PRELOAD="mock_score_list.so mock_pl2gpu.so") and defines every score_* symbol a --score-list run calls, so its
// job type is the only one such a run sees.  It counts the begin calls and rows added (PL2_MOCK_SCORE_LOG names a file
// that gets one line per begin call: "begin <class_ct>", and one per add call: "add <row_ct> <entry_ct>").  The product
// never loads it.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

struct Pl2GpuCtx;
struct Pl2ScoreJob {
  uint32_t n, score_ct, class_ct;
  std::vector<double> sums;    // [class][sample][score_ct]
  std::vector<uint64_t> hdos;  // [class][sample], half allele units
  std::vector<uint32_t> miss_dip, miss_hap;
  std::vector<uint8_t> sex;
};

namespace {
void Log(const char* what, uint32_t a, uint32_t b, bool two) {
  const char* path = getenv("PL2_MOCK_SCORE_LOG");
  if (!path) return;
  FILE* f = fopen(path, "a");
  if (!f) return;
  if (two) fprintf(f, "%s %u %u\n", what, a, b);
  else fprintf(f, "%s %u\n", what, a);
  fclose(f);
}
}  // namespace

extern "C" {
int pl2gpu_score_begin_classes(Pl2GpuCtx*, uint32_t sample_ct, uint32_t score_ct, uint32_t class_ct, Pl2ScoreJob** job_ptr) {
  const size_t nc = static_cast<size_t>(sample_ct) * class_ct;
  *job_ptr = new Pl2ScoreJob{sample_ct, score_ct, class_ct, std::vector<double>(nc * score_ct, 0.0), std::vector<uint64_t>(nc, 0), std::vector<uint32_t>(nc, 0), std::vector<uint32_t>(nc, 0), std::vector<uint8_t>(sample_ct, 0)};
  Log("begin", class_ct, 0, false);
  return 0;
}
int pl2gpu_score_set_sex(Pl2ScoreJob* job, const uint8_t* sample_sex) {
  job->sex.assign(sample_sex, sample_sex + job->n);
  return 0;
}
// ploidy classes: 0 diploid, 1 haploid for every sample, 2 chrY (females skipped, males haploid, unknown sex: diploid
// table, no dosage, haploid missing count), 3 chrX males haploid; NULL: every entry diploid
int pl2gpu_score_add_entries(Pl2ScoreJob* job, const void* genovecs, uint64_t stride, uint32_t row_ct, int, uint32_t entry_ct, const uint32_t* entry_rows, const uint32_t* entry_classes, const uint8_t* classes, const double* w_dip,
                             const double* w_hap, const uint8_t* named_dosages) {
  const uint32_t sc = job->score_ct;
  Log("add", row_ct, entry_ct, true);
  for (uint32_t e = 0; e < entry_ct; ++e) {
    if (entry_rows[e] >= row_ct || (e && entry_rows[e] < entry_rows[e - 1]) || entry_classes[e] >= job->class_ct) return 1;
    const uint8_t* row = static_cast<const uint8_t*>(genovecs) + entry_rows[e] * stride;
    const size_t o = static_cast<size_t>(entry_classes[e]) * job->n;
    const uint8_t pc = classes ? classes[e] : 0;
    for (uint32_t s = 0; s < job->n; ++s) {
      const uint8_t sex = job->sex[s];
      if (pc == 2 && sex == 2) continue;
      const bool hap = pc == 1 || (pc == 2 && sex == 1) || (pc == 3 && sex == 1);
      const double* w = (hap ? w_hap : w_dip) + 4ull * static_cast<uint64_t>(e) * sc;
      const uint32_t g = (row[s >> 2] >> (2 * (s & 3))) & 3;
      for (uint32_t c = 0; c < sc; ++c) job->sums[(o + s) * sc + c] += w[4 * c + g];
      if (g == 3) ++((hap || pc == 2) ? job->miss_hap : job->miss_dip)[o + s];
      else if (pc != 2 || hap) job->hdos[o + s] += ((named_dosages[e] >> (2 * g)) & 3) * (hap ? 1 : 2);
    }
  }
  return 0;
}
int pl2gpu_score_get_class(Pl2ScoreJob* job, uint32_t k, double* score_sums, uint64_t* named_half_dosage_sums, uint32_t* missing_diploid_cts, uint32_t* missing_haploid_cts) {
  const size_t o = static_cast<size_t>(k) * job->n;
  memcpy(score_sums, job->sums.data() + o * job->score_ct, static_cast<size_t>(job->n) * job->score_ct * sizeof(double));
  if (named_half_dosage_sums) memcpy(named_half_dosage_sums, job->hdos.data() + o, job->n * sizeof(uint64_t));
  if (missing_diploid_cts) memcpy(missing_diploid_cts, job->miss_dip.data() + o, job->n * sizeof(uint32_t));
  if (missing_haploid_cts) memcpy(missing_haploid_cts, job->miss_hap.data() + o, job->n * sizeof(uint32_t));
  return 0;
}
int pl2gpu_score_end(Pl2ScoreJob* job) {
  delete job;
  return 0;
}
}  // extern "C"
