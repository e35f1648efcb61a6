// plink2_b200 - host program: the plink2 command-line face of the pairwise-genotype commands
// (--make-king, --make-king-table, --king-cutoff, --make-grm-bin, --make-rel, --pca,
// --indep-pairwise) on top of the C-ABI GPU library (include/plink2_b200.h).
//
// Mirrors, per command, the reference's driver functions: flag semantics from 2.0/plink2.cc
// (:8462-8598 KING, :9099-9300 GRM, :7238-7312 --indep-pairwise, :10093 --parallel), execution
// order of Plink2Core (:2523-2670, :2925-2930: KING -> GRM -> PCA -> LD prune), output files of
// CalcKing / CalcGrm / LdPruneWrite.  File decoding, text formatting and the sequential graph /
// window logic run here on the host; every pairwise accumulation runs on the GPU - there is no
// CPU fallback and the program exits with kPglRetGpuFail-style status when the device is missing.
#include <immintrin.h>
#include <sched.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <unordered_map>
#include <chrono>
#include <cfloat>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <map>
#include <memory>
#include <ctime>
#include <string>
#include <thread>
#include <vector>

#include "../../../include/plink2_b200.h"
#include "dataset.h"
#include "filters.h"
#include "pca.h"
#include "ped_import.h"
#include "sfmt.h"
#include "text_util.h"

using namespace pl2host;

namespace {

// PglErr values used as process exit codes (2.0/include/plink2_base.h:358-387)
enum { kRetSuccess = 0, kRetNomem = 2, kRetOpenFail = 3, kRetReadFail = 4, kRetWriteFail = 5, kRetMalformedInput = 6, kRetInconsistentInput = 7, kRetInvalidCmdline = 8, kRetDegenerateData = 13, kRetGpuFail = 16, kRetNotYetSupported = 63 };

FILE* g_log = nullptr;
void logprintf(const char* fmt, ...) {
  char buf[4096];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  fputs(buf, stdout);
  fflush(stdout);
  if (g_log) fputs(buf, g_log);
}

// PL2_TIMING=1: phase timings on stderr (development aid; not part of the plink2 output contract)
struct PhaseClock {
  bool on = getenv("PL2_TIMING") != nullptr;
  std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now(), last = t0;
  void Mark(const char* what) {
    if (!on) return;
    const auto now = std::chrono::steady_clock::now();
    fprintf(stderr, "[timing] %-28s %8.3f s  (t = %.3f s)\n", what, std::chrono::duration<double>(now - last).count(), std::chrono::duration<double>(now - t0).count());
    last = now;
  }
  double Since(std::chrono::steady_clock::time_point t) const { return std::chrono::duration<double>(std::chrono::steady_clock::now() - t).count(); }
};
PhaseClock g_clock;

struct Cmd {
  std::string pgen, pvar, psam, out = "plink2";
  std::string ped, map;           // --ped + --map / --pedmap: legacy text fileset, converted to <out>-temporary.bed/.bim/.fam first
  bool keep_autoconv = false;     // --keep-autoconv: leave the converted fileset in place (as <out>.bed/.bim/.fam)
  uint32_t parallel_idx = 0, parallel_tot = 1;
  uint32_t threads = 0;
  uint64_t seed = 0;
  bool seed_given = false;
  int device = 0;
  uint32_t gpus = 1;            // --gpus: row-block split of the N x N jobs over this many devices (NCCL all-gather of each column tile)
  uint64_t gpu_memory_mib = 0;  // --gpu-memory / PL2_GPU_MEM_MIB: cap on the device memory a job may plan with (0 = what is free)
  // KING
  bool make_king = false, make_king_table = false;
  enum Shape { kTri, kSq, kSq0 } king_shape = kTri, rel_shape = kTri;
  enum Enc { kText, kBin, kBin4 } king_enc = kText, rel_enc = kText;
  bool king_counts = false, king_zs = false, king_table_zs = false, king_rel_check = false, grm_zs = false, rel_zs = false, freq_zs = false, freq_counts = false;
  bool col_fid_maybe = true, col_fid = false, col_id = true, col_sid_maybe = true, col_sid = false, col_nsnp = true, col_hethet = true, col_ibs0 = true, col_ibs1 = false, col_hamming = false, col_kinship = true;
  double king_table_filter = -DBL_MAX;
  double king_cutoff = -1;
  // GRM
  bool freq = false;                      // --freq
  std::string indep_preferred;            // --indep-preferred <file of variant IDs>
  std::string read_freq;                  // --read-freq <PLINK 2 --freq report>
  // --score <file> [i] [j] [k] [header | header-read] [no-mean-imputation] [zs] [ignore-dup-ids] [cols=]; with
  // --score-list, score_file names a list of score files (score_list)
  std::string score_file;
  bool score_list = false, score_ignore_dup_ids = false;
  uint32_t score_id_col = 1, score_allele_col = 2, score_coef_col = 3, score_numeric_params = 0;
  std::vector<uint32_t> score_col_nums;   // --score-col-nums: 1-based coefficient columns, increasing, no duplicates
  // --q-score-range <range file> <data file> [i] [j] ['header'] ['min']: variant IDs from column i, p-values from j
  std::string qsr_range_file, qsr_data_file;
  uint32_t qsr_id_col = 1, qsr_val_col = 2;
  bool qsr_header = false, qsr_min = false;
  std::vector<uint32_t> vscore_col_nums;  // --vscore-col-nums: 1-based weight columns, increasing, no duplicates
  bool score_header = false, score_header_read = false, score_no_meanimpute = false, score_zs = false, score_center = false, score_varstd = false, score_dominant = false, score_recessive = false, score_list_variants = false;
  bool sc_fid_maybe = true, sc_fid = false, sc_sid_maybe = true, sc_sid = false, sc_pheno1 = false, sc_phenos = true, sc_nallele = true, sc_denom = false, sc_dosagesum = true, sc_avgs = true, sc_sums = false;
  std::string vscore_file;                // --variant-score <file> ['zs'] ['cols=' chrom,pos,ref,alt,maybeprovref,provref,altfreq]
  uint32_t xchr_model = 2;                // --xchr-model {1,2}: chrX males haploid (1) or coded 0..2 like an autosome (2)
  bool xchr_model_given = false;
  bool vscore_zs = false, vs_chrom = true, vs_pos = true, vs_ref = true, vs_alt = true, vs_maybeprovref = true, vs_provref = false, vs_altfreq = false;
  std::string king_cutoff_table;          // --king-cutoff-table <.kin0 file> <threshold>
  double king_cutoff_table_thresh = -1;
  FilterSpec filters;                     // --keep / --remove / --keep-fam / --remove-fam / --extract / --exclude / --chr / --not-chr / --autosome[-xy]
  bool make_bed = false;                  // --make-bed: the filtered view as .bed/.bim/.fam (host-only)
  // --r2-unphased ['zs'] + --ld-window <#var+1> / --ld-window-kb <kb> / --ld-window-r2 <min> (plink2.cc:7908-7963, :11181-11204)
  bool r2_unphased = false, r2_zs = false;
  uint32_t ld_var_radius = 0x7fffffff, ld_bp_radius = 0xFFFFFFFFu;  // UINT32_MAX: --ld-window-kb not given (default 1000 kb)
  double ld_min_r2 = 2.0;                                             // 2.0: not given (default 0.2 (1 - 2^-44))
  std::string var_id_template;   // --set-all-var-ids / --set-missing-var-ids <template> ('@' chromosome, '#' bp, $r $a $1 $2 alleles)
  bool var_id_all = false;
  bool allow_extra_chr = false;  // --allow-extra-chr: unrecognised contig names are kept as autosome-like contigs
  bool nonfounders = false;  // --nonfounders: allele frequencies (and everything derived from them) from all samples, not founders only
  bool missing_report = false, missing_sample = true, missing_variant = true, missing_zs = false;  // --missing ['sample-only' | 'variant-only'] ['zs']
  bool write_snplist = false, write_samples = false;  // --write-snplist / --write-samples: the IDs that survived the filters
  bool make_pgen = false;                 // --make-pgen: the filtered view as fixed-width .pgen + .pvar + .psam (host-only)
  bool debug_founders_bed = false;        // --debug-founders-bed: .bed of the view's founders only (test hook for subset-of-view decoding)
  std::string king_cutoff_prefix;         // --king-cutoff <prefix of .king.id + triangular .king.bin> <threshold>
  double king_cutoff_prefix_thresh = -1;
  std::string king_table_subset;          // --king-table-subset <file> [kinship threshold]
  double king_table_subset_thresh = -DBL_MAX;
  std::vector<std::string> king_table_require;  // --king-table-require[-xor] <file...>: only pairs with >= 1 (-xor: exactly 1) listed sample
  bool king_table_require_xor = false;
  uint32_t king_table_require_flags = 0;        // how many of the two flags were given
  bool make_grm_sparse = false;            // --make-grm-sparse <cutoff>
  double grm_sparse_cutoff = -DBL_MAX;
  bool make_grm_bin = false, make_grm_list = false, make_rel = false, grm_cov = false, grm_meanimpute = false, grm_id_header = false;
  // PCA
  bool pca = false, pca_approx = false, pca_meanimpute = false;
  uint32_t pc_ct = 10;
  // LD
  bool indep_pairwise = false, indep_kb = false, bad_ld = false, indep_order1 = false;
  uint32_t indep_window = 0, indep_step = 1;
  double indep_r2 = 0;
};

bool ParseU32(const char* s, uint32_t* out) {
  char* e;
  const unsigned long v = strtoul(s, &e, 10);
  if (e == s || *e || v > 0xFFFFFFFFul) return false;
  *out = static_cast<uint32_t>(v);
  return true;
}
bool ParseDouble(const char* s, double* out) {
  char* e;
  *out = strtod(s, &e);
  return e != s && !*e;
}

int Usage(const char* msg) {
  logprintf("Error: %s\n", msg);
  return kRetInvalidCmdline;
}

// --score-col-nums / --vscore-col-nums (ParseNameRanges with positive integers, 2.0/plink2_cmdline.cc:2185-2330):
// comma-separated column numbers and a-b ranges (b > a) over one or more parameters.  The columns come back in
// increasing order, each once, whatever order they were given in and however the ranges overlap.
int ParseColNums(const std::string& flag, char** prm, int nparam, std::vector<uint32_t>* out) {
  std::vector<std::pair<std::string, std::string>> items;  // (start, end or "" for a single column)
  for (int k = 0; k < nparam; ++k) {
    const std::string a = prm[k];
    size_t pos = 0;
    while (pos < a.size()) {
      if (a[pos] == ',') {
        ++pos;
        continue;
      }
      size_t e = a.find(',', pos);
      if (e == std::string::npos) e = a.size();
      const std::string tok = a.substr(pos, e - pos);
      pos = e;
      const size_t dash = tok.find('-');
      if (dash == std::string::npos) {
        items.emplace_back(tok, "");
        continue;
      }
      if (dash == 0 || dash + 1 == tok.size() || tok.find('-', dash + 1) != std::string::npos) return Usage(("Invalid " + flag + " argument '" + a + "'.").c_str());
      items.emplace_back(tok.substr(0, dash), tok.substr(dash + 1));
    }
  }
  if (items.empty()) return Usage((flag + " requires at least one value.").c_str());
  // the same token twice is an error, before any is read as a number; overlapping ranges are not
  std::vector<std::string> seen;
  for (const auto& it : items) {
    for (const std::string* t : {&it.first, &it.second}) {
      if (t->empty()) continue;
      if (std::find(seen.begin(), seen.end(), *t) != seen.end()) return Usage(("Duplicate " + flag + " argument '" + *t + "'.").c_str());
      seen.push_back(*t);
    }
  }
  auto posint = [&](const std::string& t, uint32_t* v) {
    if (t.empty() || t.find_first_not_of("0123456789") != std::string::npos || t.size() > 10) return false;
    const uint64_t x = std::stoull(t);
    if (!x || x > 0x7ffffffe) return false;
    *v = static_cast<uint32_t>(x);
    return true;
  };
  std::vector<uint32_t> cols;
  for (const auto& it : items) {
    uint32_t a, b;
    if (!posint(it.first, &a)) return Usage(("Invalid " + flag + " argument '" + it.first + "'.").c_str());
    if (it.second.empty()) {
      cols.push_back(a);
      continue;
    }
    if (!posint(it.second, &b)) return Usage(("Invalid " + flag + " argument '" + it.second + "'.").c_str());
    if (b <= a) return Usage(("Invalid " + flag + " range '" + it.first + "-" + it.second + "'.").c_str());
    if (b - a > (1u << 24)) return Usage((flag + " range '" + it.first + "-" + it.second + "' names more columns than a line can hold.").c_str());
    for (uint32_t v = a; v <= b; ++v) cols.push_back(v);
  }
  std::sort(cols.begin(), cols.end());
  cols.erase(std::unique(cols.begin(), cols.end()), cols.end());
  *out = std::move(cols);
  return 0;
}

// --make-king-table cols= (default maybefid,id,maybesid,nsnp,hethet,ibs0,kinship; plink2_matrix_calc.h:60)
bool ParseKingCols(const std::string& spec, Cmd* c) {
  std::vector<std::string> toks;
  size_t i = 0;
  while (i <= spec.size()) {
    size_t j = spec.find(',', i);
    if (j == std::string::npos) j = spec.size();
    if (j > i) toks.push_back(spec.substr(i, j - i));
    i = j + 1;
  }
  if (toks.empty()) return false;
  const bool incremental = toks[0][0] == '+' || toks[0][0] == '-';
  if (!incremental) c->col_fid_maybe = c->col_fid = c->col_id = c->col_sid_maybe = c->col_sid = c->col_nsnp = c->col_hethet = c->col_ibs0 = c->col_ibs1 = c->col_hamming = c->col_kinship = false;
  for (std::string t : toks) {
    bool val = true;
    if (t[0] == '+' || t[0] == '-') {
      if (!incremental) return false;
      val = t[0] == '+';
      t = t.substr(1);
    } else if (incremental) {
      return false;
    }
    if (t == "maybefid") c->col_fid_maybe = val;
    else if (t == "fid") c->col_fid = val;
    else if (t == "id") c->col_id = val;
    else if (t == "maybesid") c->col_sid_maybe = val;
    else if (t == "sid") c->col_sid = val;
    else if (t == "nsnp") c->col_nsnp = val;
    else if (t == "hethet") c->col_hethet = val;
    else if (t == "ibs0") c->col_ibs0 = val;
    else if (t == "ibs1") c->col_ibs1 = val;
    else if (t == "ibs") c->col_hamming = val;
    else if (t == "kinship") c->col_kinship = val;
    else return false;
  }
  return true;
}

int ParseArgs(int argc, char** argv, Cmd* c) {
  std::string bfile, pfile, bed, bim, fam;
  bool pfile_vzs = false;
  for (int i = 1; i < argc;) {
    const std::string flag = argv[i];
    int j = i + 1;
    while (j < argc && !(argv[j][0] == '-' && argv[j][1] == '-')) ++j;
    const int nparam = j - i - 1;
    char** prm = argv + i + 1;
    auto need = [&](int lo, int hi) { return nparam >= lo && nparam <= hi; };
    if (flag == "--bfile") {
      if (!need(1, 1)) return Usage("--bfile requires a prefix.");
      bfile = prm[0];
    } else if (flag == "--pfile") {
      // 'vzs': the .pvar is Zstandard-compressed (<prefix>.pvar.zst), plink2.cc --pfile
      if (!need(1, 2) || (nparam == 2 && strcmp(prm[1], "vzs"))) return Usage("--pfile requires a prefix (optionally followed by 'vzs').");
      pfile = prm[0];
      pfile_vzs = nparam == 2;
    } else if (flag == "--bed" || flag == "--pgen") {
      if (!need(1, 1)) return Usage("--bed/--pgen requires a filename.");
      c->pgen = prm[0];
    } else if (flag == "--bim" || flag == "--pvar") {
      if (!need(1, 1)) return Usage("--bim/--pvar requires a filename.");
      c->pvar = prm[0];
    } else if (flag == "--fam" || flag == "--psam") {
      if (!need(1, 1)) return Usage("--fam/--psam requires a filename.");
      c->psam = prm[0];
    } else if (flag == "--ped" || flag == "--map") {
      if (!need(1, 1)) return Usage((flag + " requires a filename.").c_str());
      (flag == "--ped" ? c->ped : c->map) = prm[0];
    } else if (flag == "--pedmap") {
      if (!need(1, 1)) return Usage("--pedmap requires a prefix.");
      c->ped = std::string(prm[0]) + ".ped";
      c->map = std::string(prm[0]) + ".map";
    } else if (flag == "--keep-autoconv") {
      if (!need(0, 0)) return Usage("--keep-autoconv modifiers are not supported by plink2_b200.");
      c->keep_autoconv = true;
    } else if (flag == "--out") {
      if (!need(1, 1)) return Usage("--out requires a prefix.");
      c->out = prm[0];
    } else if (flag == "--threads") {
      if (!need(1, 1) || !ParseU32(prm[0], &c->threads)) return Usage("Invalid --threads argument.");
    } else if (flag == "--memory") {
      if (!need(1, 2)) return Usage("Invalid --memory argument.");  // host arena size: not used here
    } else if (flag == "--seed") {
      uint32_t s;
      if (!need(1, 1) || !ParseU32(prm[0], &s)) return Usage("Invalid --seed argument.");
      c->seed = s;
      c->seed_given = true;
    } else if (flag == "--gpus") {
      if (!need(1, 1) || !ParseU32(prm[0], &c->gpus) || !c->gpus || c->gpus > 64) return Usage("Invalid --gpus argument.");
    } else if (flag == "--gpu-memory") {
      // device-side analogue of --memory: the N x N accumulators are planned against this many MiB, which
      // forces the reference's multipass behaviour (CountTrianglePasses, plink2_matrix_calc.cc:216-255)
      uint32_t mib;
      if (!need(1, 1) || !ParseU32(prm[0], &mib) || !mib) return Usage("Invalid --gpu-memory argument.");
      c->gpu_memory_mib = mib;
    } else if (flag == "--gpu-device") {
      uint32_t d;
      if (!need(1, 1) || !ParseU32(prm[0], &d)) return Usage("Invalid --gpu-device argument.");
      c->device = static_cast<int>(d);
    } else if (flag == "--parallel") {
      if (!need(2, 2) || !ParseU32(prm[0], &c->parallel_idx) || !ParseU32(prm[1], &c->parallel_tot) || !c->parallel_idx || c->parallel_idx > c->parallel_tot) return Usage("Invalid --parallel arguments.");
      --c->parallel_idx;
    } else if (flag == "--make-king") {
      if (!need(0, 2)) return Usage("--make-king takes at most 2 arguments.");
      c->make_king = true;
      bool shape_set = false;
      for (int k = 0; k < nparam; ++k) {
        const std::string m = prm[k];
        if (m == "bin") c->king_enc = Cmd::kBin;
        else if (m == "bin4") c->king_enc = Cmd::kBin4;
        else if (m == "square") c->king_shape = Cmd::kSq, shape_set = true;
        else if (m == "square0") c->king_shape = Cmd::kSq0, shape_set = true;
        else if (m == "triangle") c->king_shape = Cmd::kTri, shape_set = true;
        else if (m == "zs") c->king_zs = true;
        else return Usage(("Invalid --make-king argument '" + m + "'.").c_str());
      }
      if (!shape_set) c->king_shape = (c->king_enc == Cmd::kText) ? Cmd::kTri : Cmd::kSq;  // plink2.cc:8521-8526
    } else if (flag == "--make-king-table") {
      c->make_king_table = true;
      for (int k = 0; k < nparam; ++k) {
        const std::string m = prm[k];
        if (m == "counts") c->king_counts = true;
        else if (m.compare(0, 5, "cols=") == 0) {
          if (!ParseKingCols(m.substr(5), c)) return Usage(("Invalid --make-king-table cols= argument '" + m + "'.").c_str());
        } else if (m == "zs") c->king_table_zs = true;
        else if (m == "rel-check") c->king_rel_check = true;
        else return Usage(("Invalid --make-king-table argument '" + m + "'.").c_str());
      }
    } else if (flag == "--king-table-filter") {
      if (!need(1, 1) || !ParseDouble(prm[0], &c->king_table_filter)) return Usage("Invalid --king-table-filter argument.");
    } else if (flag == "--king-table-subset") {
      if (!need(1, 2)) return Usage("--king-table-subset requires a filename and an optional kinship threshold.");
      c->king_table_subset = prm[0];
      if (nparam == 2 && !ParseDouble(prm[1], &c->king_table_subset_thresh)) return Usage("Invalid --king-table-subset threshold.");
    } else if (flag == "--king-table-require" || flag == "--king-table-require-xor") {
      if (nparam < 1) return Usage((flag + " requires at least one filename.").c_str());
      c->king_table_require.assign(prm, prm + nparam);
      c->king_table_require_xor = flag == "--king-table-require-xor";
      ++c->king_table_require_flags;
    } else if (flag == "--king-cutoff") {
      if (nparam == 2) {
        // plink2.cc:7671-7700: <prefix> <threshold> prunes from a matrix written earlier by --make-king bin[4] triangle
        c->king_cutoff_prefix = prm[0];
        if (!ParseDouble(prm[1], &c->king_cutoff_prefix_thresh) || c->king_cutoff_prefix_thresh < 0 || c->king_cutoff_prefix_thresh >= 0.5) return Usage((std::string("Invalid --king-cutoff[-table] argument '") + prm[1] + "'.").c_str());
      } else if (!need(1, 1) || !ParseDouble(prm[0], &c->king_cutoff) || c->king_cutoff < 0 || c->king_cutoff >= 0.5) return Usage("Invalid --king-cutoff argument.");
    } else if (flag == "--make-grm-sparse") {
      // <cutoff> ['cov'] ['meanimpute'] ['id-header']   (plink2.cc:9178-9226)
      if (!need(1, 5)) return Usage("--make-grm-sparse requires a relationship cutoff.");
      if (c->make_grm_bin) return Usage("--make-grm-sparse cannot be used with --make-grm-bin.");
      if (c->make_grm_list) return Usage("--make-grm-sparse cannot be used with --make-grm-list.");
      double dxx;
      if (!ParseDouble(prm[0], &dxx)) return Usage((std::string("Invalid --make-grm-sparse threshold '") + prm[0] + "'.").c_str());
      c->grm_sparse_cutoff = dxx * (1.0 - 1.0 / 17592186044416.0);
      c->make_grm_sparse = true;
      for (int k = 1; k < nparam; ++k) {
        const std::string m = prm[k];
        if (m == "cov") c->grm_cov = true;
        else if (m == "meanimpute") c->grm_meanimpute = true;
        else if (m == "id-header" || m == "idheader") c->grm_id_header = true;
        else if (m == "zs") c->grm_zs = true;
        else return Usage(("Invalid --make-grm-sparse argument '" + m + "'.").c_str());
      }
    } else if (flag == "--make-grm-bin" || flag == "--make-grm-list" || flag == "--make-rel") {
      if (c->make_grm_sparse) return Usage((flag + " cannot be used with --make-grm-sparse.").c_str());
      const bool is_rel = flag == "--make-rel";
      (is_rel ? c->make_rel : (flag == "--make-grm-list" ? c->make_grm_list : c->make_grm_bin)) = true;
      if (c->make_grm_bin && c->make_grm_list) return Usage("--make-grm-list cannot be used with --make-grm-bin.");
      bool shape_set = false;
      for (int k = 0; k < nparam; ++k) {
        const std::string m = prm[k];
        if (m == "cov") c->grm_cov = true;
        else if (m == "meanimpute") c->grm_meanimpute = true;
        else if (m == "id-header" && !is_rel) c->grm_id_header = true;
        else if (m == "zs" && flag == "--make-grm-list") c->grm_zs = true;
        else if (m == "zs" && is_rel) c->rel_zs = true;
        else if (is_rel && m == "bin") c->rel_enc = Cmd::kBin;
        else if (is_rel && m == "bin4") c->rel_enc = Cmd::kBin4;
        else if (is_rel && m == "square") c->rel_shape = Cmd::kSq, shape_set = true;
        else if (is_rel && m == "square0") c->rel_shape = Cmd::kSq0, shape_set = true;
        else if (is_rel && m == "triangle") c->rel_shape = Cmd::kTri, shape_set = true;
        else return Usage(("Invalid " + flag + " argument '" + m + "'.").c_str());
      }
      if (is_rel && !shape_set) c->rel_shape = (c->rel_enc == Cmd::kText) ? Cmd::kTri : Cmd::kSq;
    } else if (flag == "--pca") {
      c->pca = true;
      for (int k = 0; k < nparam; ++k) {
        const std::string m = prm[k];
        uint32_t v;
        if (m == "approx") c->pca_approx = true;
        else if (m == "meanimpute") c->pca_meanimpute = true;
        else if (ParseU32(m.c_str(), &v)) c->pc_ct = v;
        else return Usage(("Invalid or unsupported --pca argument '" + m + "'.").c_str());
      }
      if (c->pc_ct < 1 || c->pc_ct > 8000) return Usage("Invalid --pca PC count.");
    } else if (flag == "--freq") {
      for (int k = 0; k < nparam; ++k) {
        if (std::string(prm[k]) == "zs") c->freq_zs = true;
        else if (std::string(prm[k]) == "counts") c->freq_counts = true;
        else return Usage("--freq modifiers other than 'zs' and 'counts' (cols=, bins) are not supported by plink2_b200.");
      }
      c->freq = true;
    } else if (flag == "--score" || flag == "--score-list") {
      // plink2.cc --score / --score-list parsing (:11453-11570): filename, up to three 1-based column numbers, then
      // modifiers.  --score-list keeps the reference's wording for its refusals.
      const bool list = flag == "--score-list";
      if (nparam < 1) return Usage(list ? "--score-list requires a filename." : "--score requires a filename.");
      if (!c->score_file.empty() && list != c->score_list) return Usage("--score-list cannot be used with --score.");
      c->score_file = prm[0];
      c->score_list = list;
      if (list) c->sc_nallele = c->sc_dosagesum = false;  // kfScoreListColDefault: maybefid, maybesid, phenos, scoreavgs
      int k = 1;
      uint32_t nums[3], nnum = 0;
      while (k < nparam && nnum < 3 && ParseU32(prm[k], &nums[nnum]) && nums[nnum]) ++nnum, ++k;
      if (nnum >= 1) c->score_id_col = nums[0];
      c->score_allele_col = nnum >= 2 ? nums[1] : c->score_id_col + 1;
      c->score_coef_col = nnum >= 3 ? nums[2] : c->score_allele_col + 1;
      c->score_numeric_params = nnum;
      uint32_t model_bits = 0;  // center, variance-standardize, dominant, recessive
      for (; k < nparam; ++k) {
        const std::string m = prm[k];
        if (m == "header") c->score_header = true;
        else if (m == "header-read") c->score_header_read = true;
        else if (m == "no-mean-imputation") c->score_no_meanimpute = true;
        else if (m == "center") c->score_center = true, model_bits |= 1;
        else if (m == "variance-standardize") c->score_center = c->score_varstd = true, model_bits |= 2;
        else if (m == "dominant") c->score_dominant = true, model_bits |= 4;
        else if (m == "recessive") c->score_recessive = true, model_bits |= 8;
        else if (m == "list-variants") c->score_list_variants = true;
        else if (m == "zs") c->score_zs = true;
        else if (m == "ignore-dup-ids") c->score_ignore_dup_ids = true;
        else if (m.compare(0, 5, "cols=") == 0) {
          // column-set descriptor: a plain list replaces the default, +x / -x entries edit it
          const std::string spec = m.substr(5);
          const bool edit = !spec.empty() && (spec[0] == '+' || spec[0] == '-');
          if (!edit) c->sc_fid_maybe = c->sc_sid_maybe = c->sc_phenos = c->sc_nallele = c->sc_dosagesum = c->sc_avgs = false;
          size_t pos = 0;
          while (pos <= spec.size()) {
            size_t e = spec.find(',', pos);
            if (e == std::string::npos) e = spec.size();
            std::string tok = spec.substr(pos, e - pos);
            pos = e + 1;
            if (tok.empty()) continue;
            bool on = true;
            if (tok[0] == '+' || tok[0] == '-') {
              if (!edit) return Usage("Invalid --score cols= argument (mixing +/- entries with a plain list).");
              on = tok[0] == '+';
              tok = tok.substr(1);
            } else if (edit) {
              return Usage("Invalid --score cols= argument (mixing +/- entries with a plain list).");
            }
            if (tok == "maybefid") c->sc_fid_maybe = on;
            else if (tok == "fid") c->sc_fid = on;
            else if (tok == "maybesid") c->sc_sid_maybe = on;
            else if (tok == "sid") c->sc_sid = on;
            else if (tok == "pheno1") c->sc_pheno1 = on;
            else if (tok == "phenos") c->sc_phenos = on;
            else if (tok == "nallele") c->sc_nallele = on;
            else if (tok == "denom") c->sc_denom = on;
            else if (tok == "dosagesum") c->sc_dosagesum = on;
            else if (tok == "scoreavgs") c->sc_avgs = on;
            else if (tok == "scoresums") c->sc_sums = on;
            else return Usage(("Invalid --score cols= entry '" + tok + "'.").c_str());
          }
          if (list && (c->sc_nallele || c->sc_denom || c->sc_dosagesum)) return Usage("--score-list cannot be used with the nallele, denom, or dosagesum\ncolumn-sets.");
        } else if (list) {
          return Usage(("--score-list modifier '" + m + "' is not supported by plink2_b200 (supported: header, header-read, center, variance-standardize, dominant, recessive, no-mean-imputation, zs, ignore-dup-ids, cols=).").c_str());
        } else {
          return Usage(("--score modifier '" + m + "' is not supported by plink2_b200 (supported: header, header-read, center, variance-standardize, dominant, recessive, no-mean-imputation, list-variants, zs, ignore-dup-ids, cols=).").c_str());
        }
      }
      if (list) {
        if (c->score_header && c->score_header_read) return Usage("--score[-list] 'header' and 'header-read' modifiers cannot be used\ntogether.");
        if (model_bits & (model_bits - 1)) return Usage("--score[-list] 'dominant', 'recessive', 'center', and\n'variance-standardize' modifiers are mutually exclusive.");
        if (c->score_list_variants) return Usage("'list-variants[-zs]' modifier can only be used with --score, not\n--score-list.");
      }
      if (c->score_header && c->score_header_read) return Usage("--score 'header' and 'header-read' modifiers cannot be used together.");
      if ((c->score_dominant || c->score_recessive) && (c->score_center || (c->score_dominant && c->score_recessive))) return Usage("--score 'dominant' / 'recessive' cannot be combined with each other or with 'center' / 'variance-standardize'.");
    } else if (flag == "--q-score-range") {
      // plink2.cc:10746-10792
      if (nparam > 6) return Usage("--q-score-range accepts at most 6 arguments.");
      if (nparam < 2) return Usage("--q-score-range requires at least 2 arguments.");
      c->qsr_range_file = prm[0];
      c->qsr_data_file = prm[1];
      uint32_t cols[2] = {0, 0}, nnum = 0;
      for (int k = 2; k < nparam; ++k) {
        const std::string m = prm[k];
        if (m == "header") c->qsr_header = true;
        else if (m == "min") c->qsr_min = true;
        else {
          uint32_t v;
          if (!ParseU32(prm[k], &v) || !v || v > 0x3FFFFFFFu) return Usage(("Invalid --q-score-range argument '" + m + "'.").c_str());
          if (nnum == 2) return Usage("--q-score-range takes at most two numeric arguments.");
          cols[nnum] = v;
          if (nnum && cols[0] == cols[1]) return Usage("Identical --q-score-range column indexes.");
          ++nnum;
        }
      }
      if (nnum) c->qsr_id_col = cols[0];
      c->qsr_val_col = nnum == 2 ? cols[1] : c->qsr_id_col + 1;
    } else if (flag == "--score-col-nums" || flag == "--vscore-col-nums") {
      const bool vs = flag == "--vscore-col-nums";
      if (int rc = ParseColNums(flag, prm, nparam, vs ? &c->vscore_col_nums : &c->score_col_nums)) return rc;
    } else if (flag == "--xchr-model") {
      if (nparam != 1) return Usage("--xchr-model requires exactly one argument.");
      const std::string m = prm[0];
      if (m.size() != 1 || m[0] < '0' || m[0] > '2') return Usage(("Invalid --xchr-model argument '" + m + "'.").c_str());
      c->xchr_model = static_cast<uint32_t>(m[0] - '0');
      c->xchr_model_given = true;
    } else if (flag == "--variant-score" || flag == "--vscore") {
      if (nparam < 1) return Usage("--variant-score requires a filename.");
      c->vscore_file = prm[0];
      for (int k = 1; k < nparam; ++k) {
        const std::string m = prm[k];
        if (m == "zs") c->vscore_zs = true;
        else if (m.compare(0, 5, "cols=") == 0) {
          const std::string spec = m.substr(5);
          const bool edit = !spec.empty() && (spec[0] == '+' || spec[0] == '-');
          if (!edit) c->vs_chrom = c->vs_pos = c->vs_ref = c->vs_alt = c->vs_maybeprovref = false;
          size_t pos = 0;
          while (pos <= spec.size()) {
            size_t e = spec.find(',', pos);
            if (e == std::string::npos) e = spec.size();
            std::string tok = spec.substr(pos, e - pos);
            pos = e + 1;
            if (tok.empty()) continue;
            bool on = true;
            if (tok[0] == '+' || tok[0] == '-') {
              if (!edit) return Usage("Invalid --variant-score cols= argument (mixing +/- entries with a plain list).");
              on = tok[0] == '+';
              tok = tok.substr(1);
            } else if (edit) {
              return Usage("Invalid --variant-score cols= argument (mixing +/- entries with a plain list).");
            }
            if (tok == "chrom") c->vs_chrom = on;
            else if (tok == "pos") c->vs_pos = on;
            else if (tok == "ref") c->vs_ref = on;
            else if (tok == "alt" || tok == "alt1") c->vs_alt = on;
            else if (tok == "maybeprovref") c->vs_maybeprovref = on;
            else if (tok == "provref") c->vs_provref = on;
            else if (tok == "altfreq") c->vs_altfreq = on;
            else return Usage(("--variant-score cols= entry '" + tok + "' is not supported by plink2_b200 (supported: chrom, pos, ref, alt, maybeprovref, provref, altfreq).").c_str());
          }
        } else {
          return Usage(("--variant-score modifier '" + m + "' is not supported by plink2_b200 (supported: zs, cols=).").c_str());
        }
      }
    } else if (flag == "--keep" || flag == "--remove" || flag == "--keep-fam" || flag == "--remove-fam" || flag == "--extract" || flag == "--exclude") {
      // plink2.cc:7624, :10813, :5618, :5672: one or more files each
      if (nparam < 1) return Usage((flag + " requires at least one filename.").c_str());
      std::vector<std::string>& dst = flag == "--keep" ? c->filters.keep : flag == "--remove" ? c->filters.remove : flag == "--keep-fam" ? c->filters.keep_fam : flag == "--remove-fam" ? c->filters.remove_fam : flag == "--extract" ? c->filters.extract : c->filters.exclude;
      if ((flag == "--extract" || flag == "--exclude") && (!strcmp(prm[0], "range") || !strcmp(prm[0], "bed0") || !strcmp(prm[0], "bed1")) && nparam > 1) return Usage((flag + " " + prm[0] + " (positional ranges) is not supported by plink2_b200; list variant IDs instead.").c_str());
      for (int k = 0; k < nparam; ++k) dst.push_back(prm[k]);
    } else if (flag == "--chr" || flag == "--not-chr") {
      if (nparam < 1) return Usage((flag + " requires at least one chromosome code.").c_str());
      std::string perr;
      if (!ParseChrList(std::vector<std::string>(prm, prm + nparam), flag.c_str() + 2, flag == "--chr" ? &c->filters.chr_mask : &c->filters.not_chr_mask, &perr)) return Usage(perr.c_str());
    } else if (flag == "--autosome" || flag == "--autosome-xy" || flag == "--autosome-par") {
      if (!need(0, 0)) return Usage((flag + " takes no arguments.").c_str());
      (flag == "--autosome" ? c->filters.autosome : c->filters.autosome_xy) = true;
    } else if (flag == "--r2-unphased") {
      // table form only; matrix shapes / encodings, 'inter-chr', 'ref-based', cols= are not supported
      for (int k = 0; k < nparam; ++k) {
        if (!strcmp(prm[k], "zs")) c->r2_zs = true;
        else return Usage((std::string("--r2-unphased modifier '") + prm[k] + "' is not supported by plink2_b200 (supported: zs).").c_str());
      }
      c->r2_unphased = true;
    } else if (flag == "--ld-window") {
      uint32_t u;
      if (!need(1, 1) || !ParseU32(prm[0], &u) || u < 2) return Usage("Invalid --ld-window argument.");
      c->ld_var_radius = u - 1;
    } else if (flag == "--ld-window-kb") {
      double dxx;
      if (!need(1, 1) || !ParseDouble(prm[0], &dxx) || dxx < 0) return Usage("Invalid --ld-window-kb argument.");
      dxx *= 1000 * (1 + 1.0 / 17592186044416.0);
      c->ld_bp_radius = dxx > 2147483646 ? 2147483646u : static_cast<uint32_t>(static_cast<int32_t>(dxx));
    } else if (flag == "--ld-window-r2") {
      double dxx;
      if (!need(1, 1) || !ParseDouble(prm[0], &dxx) || dxx > 1.0) return Usage("Invalid --ld-window-r2 argument.");
      if (dxx > 0.0) dxx *= 1 - 1.0 / 17592186044416.0;
      c->ld_min_r2 = dxx;
    } else if (flag == "--set-all-var-ids" || flag == "--set-missing-var-ids") {
      if (!need(1, 1)) return Usage((flag + " requires a template string.").c_str());
      if (!c->var_id_template.empty()) return Usage("--set-all-var-ids cannot be used with --set-missing-var-ids in plink2_b200.");
      c->var_id_template = prm[0];
      c->var_id_all = flag == "--set-all-var-ids";
      if (c->var_id_template.find('@') == std::string::npos || c->var_id_template.find('#') == std::string::npos) return Usage((flag + " template must contain '@' (chromosome) and '#' (bp coordinate).").c_str());
    } else if (flag == "--allow-extra-chr") {
      if (!need(0, 1) || (nparam == 1 && strcmp(prm[0], "0"))) return Usage("Invalid --allow-extra-chr argument.");
      c->allow_extra_chr = true;
    } else if (flag == "--output-chr") {
      if (!need(1, 1) || !SetOutputChrStyle(prm[0])) return Usage("Invalid --output-chr argument (26, M, MT, chr26, chrM or chrMT).");
    } else if (flag == "--bp-space") {
      if (!need(1, 1) || !ParseU32(prm[0], &c->filters.min_bp_space) || !c->filters.min_bp_space) return Usage("Invalid --bp-space argument.");
    } else if (flag == "--max-alleles" || flag == "--min-alleles") {
      uint32_t u;
      if (!need(1, 1) || !ParseU32(prm[0], &u) || !u) return Usage(("Invalid " + flag + " argument.").c_str());
      (flag == "--max-alleles" ? c->filters.max_alleles : c->filters.min_alleles) = u;
    } else if (flag == "--snps-only") {
      if (!need(0, 1) || (nparam == 1 && strcmp(prm[0], "just-acgt"))) return Usage("Invalid --snps-only argument (only 'just-acgt' is accepted).");
      c->filters.snps_only = 1 + nparam;
    } else if (flag == "--from-bp" || flag == "--from-kb" || flag == "--from-mb" || flag == "--to-bp" || flag == "--to-kb" || flag == "--to-mb") {
      // plink2.cc:6221-6249, :11986-12014: lower bounds round up, upper bounds down, both with the 2^-44 guard
      const bool is_from = flag[2] == 'f';
      double dxx;
      if (!need(1, 1) || !ParseDouble(prm[0], &dxx)) return Usage(("Invalid " + flag + " argument.").c_str());
      const char unit = flag[flag.size() - 2];
      if (unit == 'k') dxx *= 1000;
      else if (unit == 'm') dxx *= 1000000;
      const double eps = 1.0 / 17592186044416.0;
      if (is_from) {
        if (c->filters.from_bp != -1) return Usage("Multiple --from-bp/-kb/-mb values.");
        if (dxx > 2147483646.0) return Usage("--from-bp/-kb/-mb argument too large.");
        c->filters.from_bp = dxx <= 0.0 ? 0 : 1 + static_cast<int32_t>(dxx * (1 - eps));
      } else {
        if (c->filters.to_bp != -1) return Usage("Multiple --to-bp/-kb/-mb values.");
        if (dxx < 0) return Usage("Negative --to-bp/-kb/-mb argument.");
        c->filters.to_bp = dxx >= 2147483646.0 ? 0x7ffffffe : static_cast<int32_t>(dxx * (1 + eps));
      }
    } else if (flag == "--missing") {
      for (int k = 0; k < nparam; ++k) {
        const std::string m = prm[k];
        if (m == "zs") c->missing_zs = true;
        else if (m == "sample-only") c->missing_variant = false;
        else if (m == "variant-only") c->missing_sample = false;
        else return Usage(("--missing modifier '" + m + "' is not supported by plink2_b200 (supported: sample-only, variant-only, zs).").c_str());
      }
      if (!c->missing_sample && !c->missing_variant) return Usage("--missing 'sample-only' and 'variant-only' cannot be used together.");
      c->missing_report = true;
    } else if (flag == "--write-snplist" || flag == "--write-samples") {
      if (!need(0, 0)) return Usage((flag + " modifiers are not supported by plink2_b200.").c_str());
      (flag == "--write-snplist" ? c->write_snplist : c->write_samples) = true;
    } else if (flag == "--nonfounders") {
      if (!need(0, 0)) return Usage("--nonfounders takes no arguments.");
      c->nonfounders = true;
    } else if (flag == "--keep-founders" || flag == "--keep-nonfounders") {
      if (!need(0, 0)) return Usage((flag + " takes no arguments.").c_str());
      if (c->filters.founders_only) return Usage("--keep-nonfounders cannot be used with --keep-founders.");
      c->filters.founders_only = flag == "--keep-founders" ? 1 : 2;
    } else if (flag == "--keep-males" || flag == "--keep-females" || flag == "--keep-nosex" || flag == "--remove-males" || flag == "--remove-females" || flag == "--remove-nosex") {
      // plink2.cc sex filters: keep-X excludes the other two classes, remove-X excludes X
      if (!need(0, 0)) return Usage((flag + " takes no arguments.").c_str());
      const bool keep = flag[2] == 'k';
      const std::string cls = flag.substr(keep ? 7 : 9);
      if (keep) {
        c->filters.excl_males = c->filters.excl_males || cls != "males";
        c->filters.excl_females = c->filters.excl_females || cls != "females";
        c->filters.excl_nosex = c->filters.excl_nosex || cls != "nosex";
      } else {
        (cls == "males" ? c->filters.excl_males : cls == "females" ? c->filters.excl_females : c->filters.excl_nosex) = true;
      }
    } else if (flag == "--mind" || flag == "--geno") {
      // [threshold], default 0.1 (plink2.cc:6487-6511); the 'dosage' / 'hh-missing' modifiers are not supported
      double thr = 0.1;
      if (!need(0, 1) || (nparam == 1 && (!ParseDouble(prm[0], &thr) || thr < 0.0 || thr > 1.0))) return Usage(("Invalid " + flag + " argument.").c_str());
      (flag == "--mind" ? c->filters.mind : c->filters.geno) = thr;
    } else if (flag == "--maf" || flag == "--max-maf") {
      double thr = 0.01;
      if (flag == "--max-maf" ? !need(1, 1) : !need(0, 1)) return Usage(("Invalid " + flag + " argument sequence.").c_str());
      if (nparam == 1 && (!ParseDouble(prm[0], &thr) || thr < 0.0 || thr > 1.0)) return Usage(("Invalid " + flag + " argument '" + prm[0] + "' (a number in [0, 1]; allele-selector suffixes are not supported).").c_str());
      (flag == "--maf" ? c->filters.min_maf : c->filters.max_maf) = thr;
    } else if (flag == "--mac" || flag == "--max-mac") {
      double cnt;
      if (!need(1, 1) || !ParseDouble(prm[0], &cnt) || cnt < 0.0 || cnt > 2147483646.0) return Usage(("Invalid " + flag + " argument.").c_str());
      // the reference compares allele "ddosages" (1/32768 units), so the thresholds are scaled the same way
      if (flag == "--mac") {  // rounded up (plink2.cc:8800-8807)
        const int32_t int_part = static_cast<int32_t>(cnt);
        const double frac = cnt - int_part;
        c->filters.min_mac = static_cast<uint64_t>(int_part) * 32768ull + (frac > 0.0 ? 1 + static_cast<uint64_t>(frac * (32768.0 * (1 - 1.0 / 17592186044416.0))) : 0);
      } else {
        c->filters.max_mac = static_cast<uint64_t>(static_cast<int64_t>(cnt * 32768.0));  // :8849
      }
    } else if (flag == "--debug-founders-bed") {
      c->debug_founders_bed = c->make_bed = true;
    } else if (flag == "--make-pgen") {
      if (!need(0, 0)) return Usage("--make-pgen modifiers are not supported by plink2_b200 (the output is always the uncompressed fixed-width mode).");
      c->make_pgen = true;
    } else if (flag == "--make-bed") {
      if (!need(0, 0)) return Usage("--make-bed modifiers are not supported by plink2_b200.");
      c->make_bed = true;
    } else if (flag == "--king-cutoff-table") {
      // plink2.cc:7665-7700
      if (!need(2, 2)) return Usage("--king-cutoff-table requires a filename and a kinship threshold.");
      c->king_cutoff_table = prm[0];
      if (!ParseDouble(prm[1], &c->king_cutoff_table_thresh) || c->king_cutoff_table_thresh < 0 || c->king_cutoff_table_thresh >= 0.5) return Usage("Invalid --king-cutoff-table threshold.");
    } else if (flag == "--read-freq") {
      if (!need(1, 1)) return Usage("--read-freq requires a filename.");
      c->read_freq = prm[0];
    } else if (flag == "--indep-preferred") {
      if (!need(1, 1)) return Usage("--indep-preferred requires a filename.");
      c->indep_preferred = prm[0];
    } else if (flag == "--indep-pairwise") {
      // <window size>['kb'] [step size (variant ct)] <r^2 threshold>   (plink2.cc:7238-7312)
      if (!need(2, 4)) return Usage("--indep-pairwise requires 2-4 arguments.");
      c->indep_pairwise = true;
      std::vector<std::string> p(prm, prm + nparam);
      std::string w = p[0];
      size_t next = 1;
      auto strip_kb = [&](std::string* s) {
        if (s->size() > 2 && (s->substr(s->size() - 2) == "kb" || s->substr(s->size() - 2) == "KB" || s->substr(s->size() - 2) == "Kb")) {
          s->resize(s->size() - 2);
          return true;
        }
        return false;
      };
      if (strip_kb(&w)) {
        c->indep_kb = true;
      } else if (next < p.size() && (p[next] == "kb" || p[next] == "KB")) {
        c->indep_kb = true;
        ++next;
      }
      double wd;
      if (!ParseDouble(w.c_str(), &wd) || wd < 0) return Usage("Invalid --indep-pairwise window size.");
      if (c->indep_kb) {
        wd *= 1000;
        if (wd > 2147483646) wd = 2147483646;
        c->indep_window = static_cast<uint32_t>(wd);
      } else {
        if (wd < 2 || wd != floor(wd)) return Usage("Invalid --indep-pairwise window size.");
        c->indep_window = static_cast<uint32_t>(wd);
      }
      const size_t remaining = p.size() - next;
      if (remaining == 2) {
        if (!ParseU32(p[next].c_str(), &c->indep_step) || !c->indep_step) return Usage("Invalid --indep-pairwise step size.");
        ++next;
      } else if (remaining != 1) {
        return Usage("Invalid --indep-pairwise argument sequence.");
      }
      if (c->indep_kb && c->indep_step != 1) return Usage("--indep-pairwise step size must be 1 when the window is in kilobase units.");
      if (!c->indep_kb && c->indep_step > c->indep_window) return Usage("--indep-pairwise step size cannot exceed the window size.");
      if (!ParseDouble(p[next].c_str(), &c->indep_r2) || c->indep_r2 < 0 || c->indep_r2 >= 1) return Usage("Invalid --indep-pairwise r^2 threshold.");
    } else if (flag == "--indep-order") {
      // plink2.cc:7325-7338: 1 = PLINK 1.x pruning order, 2 = default
      if (!need(1, 1)) return Usage("--indep-order requires one argument.");
      const std::string m = argv[i + 1];
      if (m == "1") c->indep_order1 = true;
      else if (m != "2") return Usage("Invalid --indep-order mode ('1' or '2' expected).");
    } else if (flag == "--bad-ld") {
      c->bad_ld = true;
    } else {
      return Usage(("Unrecognized or unsupported flag '" + flag + "' (plink2_b200 implements the KING / GRM / PCA / --indep-pairwise path only).").c_str());
    }
    i = j;
  }
  if (!bfile.empty()) {
    c->pgen = bfile + ".bed";
    c->pvar = bfile + ".bim";
    c->psam = bfile + ".fam";
  } else if (!pfile.empty()) {
    c->pgen = pfile + ".pgen";
    c->pvar = pfile + (pfile_vzs ? ".pvar.zst" : ".pvar");
    c->psam = pfile + ".psam";
  }
  if (!c->gpu_memory_mib) {
    const char* e = getenv("PL2_GPU_MEM_MIB");
    uint32_t mib;
    if (e && ParseU32(e, &mib)) c->gpu_memory_mib = mib;
  }
  if (!c->ped.empty() || !c->map.empty()) {
    if (c->ped.empty() || c->map.empty()) return Usage("--ped and --map must be used together (or use --pedmap <prefix>).");
    if (!c->pgen.empty() || !c->pvar.empty() || !c->psam.empty()) return Usage("--ped/--map cannot be combined with another input fileset.");
    const std::string prefix = c->out + (c->keep_autoconv ? "" : "-temporary");
    c->pgen = prefix + ".bed";
    c->pvar = prefix + ".bim";
    c->psam = prefix + ".fam";
  }
  if (c->pgen.empty() || c->pvar.empty() || c->psam.empty()) return Usage("No input dataset (--bfile / --pfile / --bed+--bim+--fam / --pgen+--pvar+--psam).");
  if (!c->indep_preferred.empty() && !c->indep_pairwise) return Usage("--indep-preferred must be used with --indep-pairwise.");
  // --score / --score-col-nums / --vscore-col-nums, in the reference's order (plink2.cc:11573-11582, :12566-12574,
  // :12955; column overlaps 2.0/plink2_matrix_calc.cc:7186-7234)
  if (!c->vscore_col_nums.empty() && c->vscore_file.empty()) return Usage("--vscore-col-nums must be used with --variant-score.");
  if (c->xchr_model_given && c->score_file.empty() && c->vscore_file.empty()) return Usage("--xchr-model must be used with --glm, --score[-list], or\n--variant-score.");
  if (c->xchr_model_given && c->xchr_model == 0) {
    logprintf("Error: --xchr-model 0 (skip chrX) is not supported by plink2_b200; use --not-chr X to leave chrX out.\n");
    return kRetNotYetSupported;
  }
  if (!c->qsr_range_file.empty() && c->score_file.empty()) return Usage("--q-score-range cannot be used without --score[-list].");
  if (!c->score_col_nums.empty()) {
    if (c->score_file.empty()) return Usage("--score-col-nums must be used with --score[-list].");
    if (c->score_numeric_params == 3) return Usage("--score-col-nums cannot be used when three numeric arguments are\nprovided to --score.");
    if (std::binary_search(c->score_col_nums.begin(), c->score_col_nums.end(), c->score_id_col)) return Usage("--score variant ID column index matches a coefficient column index.");
    if (std::binary_search(c->score_col_nums.begin(), c->score_col_nums.end(), c->score_allele_col)) return Usage("--score allele column index matches a coefficient column index.");
  } else if (!c->score_file.empty() && (c->score_id_col == c->score_allele_col || c->score_id_col == c->score_coef_col || c->score_allele_col == c->score_coef_col)) {
    return Usage("--score variant ID, allele and coefficient column numbers must be distinct.");
  }
  if (c->king_table_require_flags) {
    // the reference's checks (plink2.cc:7732-7750, :8467, :8571), in the order it meets them
    if (c->king_cutoff >= 0 || !c->king_cutoff_prefix.empty()) return Usage("--king-table-require[-xor] cannot be used with --king-cutoff.");
    if (c->king_table_require_flags > 1) return Usage("--king-table-require cannot be used with --king-table-require-xor.");
    if (c->make_king) return Usage("--make-king cannot be used with --king-table-subset or\n--king-table-require[-xor].");
    if (c->make_king_table && !c->col_id) return Usage("--king-table-require[-xor] requires --make-king-table cols= to include\nthe 'id' column set.");
  }
  if (c->pca) {
    // 2.0/plink2.cc:10207-10232
    if (c->pca_approx) {
      if (c->pc_ct > 100) return Usage("--pca approx does not support more than 100 PCs.");
    } else {
      if (c->parallel_tot != 1) return Usage("Non-approximate --pca cannot be used with --parallel.");
      if (c->make_rel || c->make_grm_bin || c->make_grm_list || c->make_grm_sparse) {
        if (c->grm_meanimpute != c->pca_meanimpute) return Usage("--make-rel/--make-grm-{bin,list,sparse} meanimpute setting must match\n--pca meanimpute setting.");
        if (c->grm_cov) return Usage("--make-rel/--make-grm-{bin,list,sparse} cannot be used to compute a\ncovariance matrix in the same run as non-approximate --pca.");
      }
    }
  }
  if (c->filters.from_bp != -1 || c->filters.to_bp != -1) {
    uint32_t named = 0;
    for (uint8_t f : c->filters.chr_mask) named += f;
    if (named != 1) return Usage("--from-bp/-kb/-mb and --to-bp/-kb/-mb must be used with --chr, and only one chromosome.");
    if (c->filters.from_bp != -1 && c->filters.to_bp != -1 && c->filters.from_bp > c->filters.to_bp) return Usage("--to-bp/-kb/-mb argument is smaller than --from-bp/-kb/-mb argument.");
  }
  if (!(c->make_king || c->make_king_table || c->king_cutoff >= 0 || c->make_grm_bin || c->make_grm_list || c->make_grm_sparse || c->make_rel || c->pca || c->indep_pairwise || c->freq || c->r2_unphased || c->make_bed || c->make_pgen || c->missing_report || c->write_snplist || c->write_samples || !c->king_cutoff_table.empty() || !c->king_cutoff_prefix.empty() || !c->score_file.empty() || !c->vscore_file.empty())) return Usage("No command given.");
  return 0;
}

// ParallelBounds / TriangleDivide (2.0/plink2_common.cc:4936-4961)
uint32_t TriangleDivide(int64_t cur_prod_x2, int32_t modif) {
  if (cur_prod_x2 == 0) return modif < 0 ? static_cast<uint32_t>(-modif) : 0;
  int64_t vv = static_cast<int64_t>(sqrt(static_cast<double>(cur_prod_x2)));
  while ((vv - 1) * (vv + modif - 1) >= cur_prod_x2) --vv;
  while (vv * (vv + modif) < cur_prod_x2) ++vv;
  return static_cast<uint32_t>(vv);
}
void ParallelBounds(uint32_t ct, int32_t start, uint32_t idx, uint32_t tot, uint32_t* b0, uint32_t* b1) {
  const int32_t modif = 1 - start * 2;
  const int64_t ct_tot = static_cast<int64_t>(ct) * (ct + modif);
  *b0 = TriangleDivide((ct_tot * idx) / tot, modif);
  *b1 = TriangleDivide((ct_tot * (idx + 1)) / tot, modif);
}

std::string PieceName(const std::string& base, const Cmd& c) { return c.parallel_tot == 1 ? base : base + "." + std::to_string(c.parallel_idx + 1); }

// sample ID text "[FID\t]IID[\tSID]" (CollapsedSampleFmtidInit, plink2_common.cc)
struct IdFmt {
  bool fid, sid;
};
IdFmt KingIdFmt(const Cmd& c, const SampleInfo& s) { return {c.col_fid || (c.col_fid_maybe && s.fid_present), c.col_sid || (c.col_sid_maybe && s.sid_present)}; }
std::string FmtId(const SampleInfo& s, uint32_t k, IdFmt f) {
  std::string r;
  if (f.fid) r += s.fid[k] + "\t";
  r += s.iid[k];
  if (f.sid) r += "\t" + s.sid[k];
  return r;
}

// WriteSampleIds: "#FID\tIID[\tSID]" header unless no_header
bool WriteIdFile(const std::string& path, const SampleInfo& s, const std::vector<uint32_t>& which, bool header) {
  OutFile f;
  if (!f.Open(path)) return false;
  if (header) {
    std::string h = "#";
    if (s.fid_present) h += "FID\t";
    h += "IID";
    if (s.sid_present) h += "\tSID";
    h += "\n";
    f.Puts(h.c_str());
  }
  for (uint32_t k : which) {
    std::string ln;
    if (s.fid_present) ln += s.fid[k] + "\t";
    ln += s.iid[k];
    if (s.sid_present) ln += "\t" + s.sid[k];
    ln += "\n";
    f.Puts(ln.c_str());
  }
  return f.Close();
}
bool WriteAllIds(const std::string& path, const SampleInfo& s, bool header) {
  std::vector<uint32_t> all(s.size());
  for (uint32_t k = 0; k < s.size(); ++k) all[k] = k;
  return WriteIdFile(path, s, all, header);
}

// ---- genotype block streaming: decode `idx` variants into a pinned host buffer ----
// host threads for genotype decoding: --threads if given, else min(affinity mask, cgroup CPU quota), at most 64
uint32_t g_decode_threads = 1;
uint32_t EffectiveHostThreads(uint32_t requested) {
  if (requested) return std::min<uint32_t>(requested, 256);
  uint32_t n = std::max(1u, std::thread::hardware_concurrency());
  cpu_set_t set;
  if (!sched_getaffinity(0, sizeof(set), &set)) n = std::max(1, CPU_COUNT(&set));
  if (FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
    char q[64];
    unsigned long long period = 0;
    if (fscanf(f, "%63s %llu", q, &period) == 2 && strcmp(q, "max") && period) {
      const unsigned long long quota = strtoull(q, nullptr, 10);
      if (quota) n = std::min<uint32_t>(n, static_cast<uint32_t>((quota + period - 1) / period));
    }
    fclose(f);
  }
  return std::max(1u, std::min(n, 64u));
}

struct BlockStreamer {
  Dataset* ds;
  const std::vector<uint32_t>* vidx;
  const uint64_t* sample_include = nullptr;  // null = all samples
  uint32_t sample_ct;
  uint32_t words;
  uint64_t* buf = nullptr;
  uint32_t cap;
  size_t pos = 0;
  uint32_t spare = 0;  // extra rows behind the block (filler for sharded uploads)
  uint32_t threads = 0;  // decode threads for this streamer (0: g_decode_threads)
  double decode_s = 0;  // time spent in Next
  BlockStreamer(Dataset* d, const std::vector<uint32_t>* v, uint32_t n_samples, uint32_t batch, uint32_t spare_rows = 0) : ds(d), vidx(v), sample_ct(n_samples), words(PgenReader::WordsFor(n_samples)), cap(batch), spare(spare_rows) {}
  ~BlockStreamer() { pl2gpu_host_free(buf); }
  bool Init() {
    void* p = nullptr;
    if (pl2gpu_host_alloc(static_cast<uint64_t>(cap + spare) * words * 8, &p)) return false;
    buf = static_cast<uint64_t*>(p);
    return true;
  }
  // returns number of variants decoded (0 at end), -1 on error.  Decoding is spread over the host threads this
  // process may use (--threads, else affinity mask / cgroup quota), like the reference's multithreaded block reads.
  int Next(std::string* err) {
    const uint32_t n = static_cast<uint32_t>(std::min<size_t>(cap, vidx->size() - pos));
    if (!n) return 0;
    const auto t = std::chrono::steady_clock::now();
    if (!ds->reader.GetBlock(vidx->data() + pos, n, sample_include, sample_ct, buf, words, threads ? threads : g_decode_threads, err)) return -1;
    decode_s += g_clock.Since(t);
    pos += n;
    return static_cast<int>(n);
  }
  void Rewind() { pos = 0; }
};

int GpuFail(const char* what) {
  logprintf("Error: %s: %s\n", what, pl2gpu_last_error());
  return kRetGpuFail;
}

// ------------------------------------------------------------------------------------------ multi-GPU team
// One context per device, one NCCL rank per context, all driven from this process (one host thread per rank for
// the collective calls).  ctx[0] is the caller's context.
struct GpuTeam {
  std::vector<Pl2GpuCtx*> ctx;
  ~GpuTeam() {
    if (ctx.size() > 1) pl2gpu_comm_destroy(ctx[0]);
    for (size_t g = 1; g < ctx.size(); ++g) pl2gpu_ctx_destroy(ctx[g]);
  }
  uint32_t size() const { return static_cast<uint32_t>(ctx.size()); }
};

// f(rank) on `g` host threads (rank 0 on the calling thread); returns the first nonzero return code and its
// pl2gpu_last_error() text (thread-local in the library, so it is captured inside the worker).
template <class F>
int ForEachRank(uint32_t g, F&& f, std::string* errtext) {
  std::vector<int> rc(g, 0);
  std::vector<std::string> msg(g);
  auto run = [&](uint32_t r) {
    rc[r] = f(r);
    if (rc[r]) msg[r] = pl2gpu_last_error();
  };
  std::vector<std::thread> th;
  for (uint32_t r = 1; r < g; ++r) th.emplace_back(run, r);
  run(0);
  for (auto& t : th) t.join();
  for (uint32_t r = 0; r < g; ++r) {
    if (rc[r]) {
      if (errtext) *errtext = msg[r];
      return rc[r];
    }
  }
  return 0;
}

// Contexts on devices first_device .. first_device + gpus - 1 joined in one communicator.  Returns 0, or a
// kRet* code after logging.
int TeamInit(Pl2GpuCtx* first, int first_device, uint32_t gpus, GpuTeam* team) {
  team->ctx.assign(1, first);
  if (gpus <= 1) return 0;
  if (pl2gpu_device_count() < first_device + static_cast<int>(gpus)) {
    logprintf("Error: --gpus %u needs devices %d..%d, but only %d CUDA device(s) are visible.\n", gpus, first_device, first_device + static_cast<int>(gpus) - 1, pl2gpu_device_count());
    return kRetGpuFail;
  }
  for (uint32_t g = 1; g < gpus; ++g) {
    Pl2GpuCtx* cx = nullptr;
    if (pl2gpu_ctx_create(first_device + static_cast<int>(g), &cx)) return GpuFail("pl2gpu_ctx_create");
    team->ctx.push_back(cx);
  }
  uint8_t id[PL2GPU_COMM_ID_BYTES];
  if (pl2gpu_comm_unique_id(id)) return GpuFail("pl2gpu_comm_unique_id");
  std::string err;
  if (ForEachRank(gpus, [&](uint32_t r) { return pl2gpu_comm_init(team->ctx[r], static_cast<int>(r), static_cast<int>(gpus), id); }, &err)) {
    logprintf("Error: pl2gpu_comm_init: %s\n", err.c_str());
    return kRetGpuFail;
  }
  return 0;
}

// Rows [r0, r1) of the lower triangle cut into `parts` contiguous blocks whose interior boundaries are multiples
// of the 128-row pair tile and which hold (nearly) the same number of 128 x 80 pair tiles - the unit the tensor
// kernels' time is proportional to.  Blocks may be empty when the range holds fewer row tiles than parts.
std::vector<uint32_t> TileAlignedBounds(uint32_t r0, uint32_t r1, uint32_t parts, bool include_diag) {
  std::vector<uint32_t> b(parts + 1, r1);
  b[0] = r0;
  if (parts <= 1 || r1 <= r0) return b;
  const uint32_t rt0 = r0 / 128, rt1 = (r1 + 127) / 128;
  std::vector<uint64_t> cum(1, 0);
  for (uint32_t rt = rt0; rt < rt1; ++rt) {
    const uint32_t row_end = std::min(r1, (rt + 1) * 128);
    const uint32_t cols = include_diag ? row_end : row_end - 1;
    cum.push_back(cum.back() + (cols + 79) / 80);
  }
  for (uint32_t k = 1; k < parts; ++k) {
    const double target = static_cast<double>(cum.back()) * k / parts;
    uint32_t best = 0;
    for (uint32_t t = 1; t < cum.size(); ++t) {
      if (fabs(static_cast<double>(cum[t]) - target) < fabs(static_cast<double>(cum[best]) - target)) best = t;
    }
    uint32_t row = std::min(r1, std::max(r0, (rt0 + best) * 128));
    b[k] = std::max(row, b[k - 1]);
  }
  return b;
}

// ------------------------------------------------------------------------------------------ relationship drivers
// Device jobs end (pl2gpu_*_end) when their owner goes out of scope.  An owner is declared after the GpuTeam whose
// context its job runs on, so that the job ends before the context is destroyed.
template <class J, int (*End)(J*)>
struct JobEnd {
  void operator()(J* job) const { End(job); }
};
using KingJob = std::unique_ptr<Pl2KingJob, JobEnd<Pl2KingJob, pl2gpu_king_end>>;
using KingPairJob = std::unique_ptr<Pl2KingPairJob, JobEnd<Pl2KingPairJob, pl2gpu_king_pairs_end>>;
using GrmJob = std::unique_ptr<Pl2GrmJob, JobEnd<Pl2GrmJob, pl2gpu_grm_end>>;
using PcaJob = std::unique_ptr<Pl2PcaJob, JobEnd<Pl2PcaJob, pl2gpu_pca_end>>;

// The variants KING and the GRM are computed over (KeptForRelationship); `what` names the calculation in the log.
int RelationshipVariants(const Dataset& ds, const char* what, std::vector<uint32_t>* vidx) {
  vidx->clear();
  uint32_t non_auto = 0;
  for (uint32_t v = 0; v < ds.variants.size(); ++v) {
    if (KeptForRelationship(ds.variants.chr_code[v])) vidx->push_back(v);
    else ++non_auto;
  }
  if (non_auto) logprintf("Excluding %u variant%s on non-autosomes from %s.\n", non_auto, non_auto == 1 ? "" : "s", what);
  if (vidx->empty()) {
    logprintf("Error: No variants remaining for %s.\n", what);
    return kRetDegenerateData;
  }
  return 0;
}

// f(got) for every block bs decodes from the start of its variant list; a decode error is logged and ends the stream
// with kRetMalformedInput.  f returns 0 or a kRet* code, which ends the stream too.
template <class F>
int StreamBlocks(BlockStreamer* bs, F&& f) {
  bs->Rewind();
  std::string err;
  for (;;) {
    const int got = bs->Next(&err);
    if (got < 0) {
      logprintf("\nError: %s\n", err.c_str());
      return kRetMalformedInput;
    }
    if (!got) return 0;
    const int rc = f(static_cast<uint32_t>(got));
    if (rc) return rc;
  }
}

// --gpus: device g adds rows [g * per, (g + 1) * per) of the decoded block through add(g, slice, per), one host thread
// per device, and the library all-gathers the column tile.  The filler rows that top the block up to per * G are
// all-missing and count nothing (bs has G spare rows behind the block).  Returns ForEachRank's code and error text.
template <class F>
int AddSharded(BlockStreamer* bs, uint32_t got, uint32_t G, F&& add, std::string* err) {
  const uint32_t per = (got + G - 1) / G;
  memset(bs->buf + static_cast<uint64_t>(got) * bs->words, 0xFF, static_cast<uint64_t>(per * G - got) * bs->words * 8);
  return ForEachRank(G, [&](uint32_t g) { return add(g, bs->buf + static_cast<uint64_t>(g) * per * bs->words, per); }, err);
}

// KING pass planning (CountTrianglePasses / NextTrianglePass, :216-255) for rows [r0, r1).  The budget is the least
// free device memory over `ctxs` less 10 %, capped by --gpu-memory.  Variants per staged block: the full 65,536 unless
// `block_copies` buffers of that size (the staged blocks and their device-side copies) would take more than a quarter
// of the budget; then halved until they fit.  Every pass is the largest row block from its start whose device memory,
// need(a, b, batch), fits the budget.  Returns 0 or a kRet* code after logging.
template <class Need>
int PlanKingPasses(const Cmd& c, const std::vector<Pl2GpuCtx*>& ctxs, const char* flagname, uint32_t n, uint32_t r0, uint32_t r1, uint32_t block_copies, Need&& need, uint32_t* batch, std::vector<uint32_t>* bounds) {
  uint64_t free_b = ~0ull;
  for (Pl2GpuCtx* cx : ctxs) {
    uint64_t f = 0, t = 0;
    if (pl2gpu_ctx_mem_info(cx, &f, &t)) return GpuFail("pl2gpu_ctx_mem_info");
    free_b = std::min(free_b, f);
  }
  uint64_t budget = free_b - free_b / 10;
  if (c.gpu_memory_mib && (c.gpu_memory_mib << 20) < budget) budget = c.gpu_memory_mib << 20;
  *batch = 65536;
  while (*batch > 2048 && static_cast<uint64_t>(block_copies) * *batch * ((n + 639) / 640 * 160) > budget / 4) *batch /= 2;
  auto fits = [&](uint32_t a, uint32_t b) { return need(a, b, *batch) <= budget; };
  bounds->assign(1, r0);
  while (bounds->back() < r1) {
    const uint32_t r = bounds->back();
    if (!fits(r, r + 1)) {
      logprintf("Error: Insufficient GPU memory for %s on %u samples.\n", flagname, n);
      return kRetNomem;
    }
    uint32_t lo = r + 1, hi = r1;
    while (lo < hi) {
      const uint32_t mid = lo + (hi - lo + 1) / 2;
      if (fits(r, mid)) lo = mid;
      else hi = mid - 1;
    }
    bounds->push_back(lo);
  }
  const uint32_t pass_ct = static_cast<uint32_t>(bounds->size() - 1);
  if (pass_ct > 1) logprintf("%s: %u passes over the variants (device accumulators planned against %llu MiB).\n", flagname, pass_ct, static_cast<unsigned long long>(budget >> 20));
  return 0;
}

// KING pairs (j, i) with i < min(j, col_end) over the rows j < r
uint64_t KingPairsBelow(uint64_t r, uint64_t col_end) { return r <= col_end ? (r ? r * (r - 1) / 2 : 0) : (col_end ? col_end * (col_end - 1) / 2 : 0) + (r - col_end) * col_end; }

// The pairs of rows [r0, r1) whose kinship is at least `threshold` (pl2gpu_king_get_filtered), the buffers grown until
// all of them fit: pair q is (pairs[2q], pairs[2q + 1]) with counts[5q..5q + 4] and kin[q], q < found.
int FetchKingFiltered(Pl2KingJob* job, uint32_t r0, uint32_t r1, double threshold, std::vector<uint32_t>* pairs, std::vector<uint32_t>* counts, std::vector<double>* kin, uint64_t* found) {
  uint64_t cap = 1ull << 22;
  for (;;) {
    pairs->resize(cap * 2);
    counts->resize(cap * 5);
    kin->resize(cap);
    if (pl2gpu_king_get_filtered(job, r0, r1, threshold, cap, pairs->data(), counts->data(), kin->data(), found)) return GpuFail("pl2gpu_king_get_filtered");
    if (*found <= cap) return 0;
    cap = *found;
  }
}

// Rows [r0, r1) of a KING job in chunks of at most ~512 MB of counts: f(c0, c1, pair_ct, counts) per chunk, counts =
// the chunk's counts[pair][5] in the library's pair order (KingPairsBelow), or unfetched when with_counts is false.
// f returns 0 or a kRet* code.
template <class F>
int ForEachKingCountChunk(Pl2KingJob* job, uint32_t r0, uint32_t r1, uint32_t col_end, bool with_counts, F&& f) {
  const uint64_t max_pairs = (512ull << 20) / 20;
  std::vector<uint32_t> counts;
  for (uint32_t c0 = r0; c0 < r1;) {
    uint32_t c1 = c0 + 1;
    while (c1 < r1 && KingPairsBelow(c1 + 1, col_end) - KingPairsBelow(c0, col_end) <= max_pairs) ++c1;
    const uint64_t pair_ct = KingPairsBelow(c1, col_end) - KingPairsBelow(c0, col_end);
    if (with_counts) {
      counts.resize(pair_ct * 5);
      if (pair_ct && pl2gpu_king_get_counts(job, c0, c1, counts.data(), 0)) return GpuFail("pl2gpu_king_get_counts");
    }
    const int rc = f(c0, c1, pair_ct, counts.data());
    if (rc) return rc;
    c0 = c1;
  }
  return 0;
}

// --make-king / --make-rel matrix writer (shapes triangle, square0, square; encodings text, bin4, bin) fed the rows of
// the lower triangle in order: Row(j, v, diag) with v[0..j-1] the values left of the diagonal.  `triangle` writes each
// row through its diagonal when tri_diag is set (REL), else without it (KING, whose triangle starts at row 1);
// square0 pads every row with zeros to n columns; square keeps the lower triangle with its diagonal, and Finish()
// writes the mirrored n x n matrix.
struct TriangleMatrixWriter {
  OutFile* f;
  uint32_t n;
  Cmd::Shape shape;
  Cmd::Enc enc;
  bool tri_diag;
  std::vector<double> full;  // square: row j at j * (j + 1) / 2
  std::vector<float> rowf;
  std::vector<double> rowd;
  TriangleMatrixWriter(OutFile* file, uint32_t n_samples, Cmd::Shape s, Cmd::Enc e, bool diag) : f(file), n(n_samples), shape(s), enc(e), tri_diag(diag), rowf(e == Cmd::kBin4 ? n : 0), rowd(e == Cmd::kBin ? n : 0) {
    if (shape == Cmd::kSq) full.resize(static_cast<uint64_t>(n) * (n + 1) / 2);
  }
  void Row(uint32_t j, const double* v, double diag) {
    if (shape == Cmd::kSq) {
      double* dst = &full[static_cast<uint64_t>(j) * (j + 1) / 2];
      memcpy(dst, v, sizeof(double) * j);
      dst[j] = diag;
    } else {
      Put(v, j, (shape == Cmd::kSq0 || tri_diag) ? &diag : nullptr, shape == Cmd::kSq0 ? n : j + tri_diag);
    }
  }
  void Finish() {
    if (shape != Cmd::kSq) return;
    std::vector<double> row(n);
    for (uint32_t j = 0; j < n; ++j) {
      for (uint32_t i = 0; i < n; ++i) row[i] = i <= j ? full[static_cast<uint64_t>(j) * (j + 1) / 2 + i] : full[static_cast<uint64_t>(i) * (i + 1) / 2 + j];
      Put(row.data(), n, nullptr, n);
    }
  }
  // one row of len values: v[0..nv-1], then *diag unless it is null, then zeros
  void Put(const double* v, uint32_t nv, const double* diag, uint32_t len) {
    if (!len) return;
    const uint32_t nd = nv + (diag != nullptr);
    if (enc == Cmd::kText) {
      char* w = f->Reserve(static_cast<size_t>(n) * 16 + 64);
      for (uint32_t i = 0; i < len; ++i) {
        w = dtoa_g(i < nv ? v[i] : (i < nd ? *diag : 0.0), w);
        *w++ = '\t';
      }
      w[-1] = '\n';
      f->Advance(w);
    } else if (enc == Cmd::kBin4) {
      for (uint32_t i = 0; i < nv; ++i) rowf[i] = static_cast<float>(v[i]);
      if (diag) rowf[nv] = static_cast<float>(*diag);
      std::fill(rowf.begin() + nd, rowf.begin() + len, 0.0f);
      f->Write(rowf.data(), sizeof(float) * len);
    } else {
      memcpy(rowd.data(), v, sizeof(double) * nv);
      if (diag) rowd[nv] = *diag;
      std::fill(rowd.begin() + nd, rowd.begin() + len, 0.0);
      f->Write(rowd.data(), sizeof(double) * len);
    }
  }
};

// ------------------------------------------------------------------------------------------ KING
// KinshipPruneDestructive (2.0/plink2_matrix_calc.cc:278-391): while edges remain, remove the
// partner of the first degree-1 vertex if any, else the first maximum-degree vertex.
void KinshipPrune(std::vector<uint64_t>* table_ptr, uint32_t n, std::vector<uint8_t>* removed) {
  std::vector<uint64_t>& tab = *table_ptr;
  const uint32_t wl = (n + 63) / 64;
  std::vector<uint32_t> degree(n, 0);
  std::vector<uint8_t> nz(n, 0);
  removed->assign(n, 0);
  uint32_t deg1 = 0, nz_ct = 0;
  for (uint32_t i = 0; i < n; ++i) {
    uint32_t d = 0;
    for (uint32_t w = 0; w < wl; ++w) d += static_cast<uint32_t>(__builtin_popcountll(tab[static_cast<uint64_t>(i) * wl + w]));
    if (d) {
      degree[i] = d;
      deg1 += d == 1;
      nz[i] = 1;
      ++nz_ct;
    }
  }
  auto first_set = [&](const uint64_t* row, uint32_t from) {
    for (uint32_t w = from / 64; w < wl; ++w) {
      uint64_t x = row[w];
      if (w == from / 64) x &= ~0ull << (from % 64);
      if (x) return w * 64 + static_cast<uint32_t>(__builtin_ctzll(x));
    }
    return n;
  };
  while (nz_ct) {
    uint32_t prune, cur_degree;
    if (deg1) {
      uint32_t u = 0;
      while (!(nz[u] && degree[u] == 1)) ++u;
      prune = first_set(&tab[static_cast<uint64_t>(u) * wl], 0);
      cur_degree = degree[prune];
    } else {
      prune = 0;
      cur_degree = 0;
      bool first = true;
      for (uint32_t u = 0; u < n; ++u) {
        if (!nz[u]) continue;
        if (first || degree[u] > cur_degree) {
          cur_degree = degree[u];
          prune = u;
          first = false;
        }
      }
    }
    const uint64_t col_mask = ~(1ull << (prune % 64));
    const uint64_t* row = &tab[static_cast<uint64_t>(prune) * wl];
    uint32_t u = 0;
    for (uint32_t p = 0; p < cur_degree; ++p, ++u) {
      u = first_set(row, u);
      const uint32_t nd = degree[u] - 1;
      if (!nd) {
        nz[u] = 0;
        --deg1;
        --nz_ct;
      } else {
        tab[static_cast<uint64_t>(u) * wl + prune / 64] &= col_mask;
        deg1 += nd == 1;
        degree[u] = nd;
      }
    }
    if (degree[prune] == 1) --deg1;
    (*removed)[prune] = 1;
    nz[prune] = 0;
    --nz_ct;
  }
}

inline double KinshipFromCounts(const uint32_t* c) {  // ComputeKinship, :1566-1573
  const int64_t ibs0 = c[0], hethet = c[1], het2hom1 = c[2], het1hom2 = c[3];
  const int64_t smaller = hethet + std::min(het1hom2, het2hom1);
  return 0.5 - static_cast<double>(4 * ibs0 + het1hom2 + het2hom1) / static_cast<double>(4 * smaller);
}

// AppendKingTableHeader (:1611-1652)
std::string KingTableHeader(const Cmd& c, const IdFmt& idf) {
  std::string h = "#";
  if (c.col_id) {
    if (idf.fid) h += "FID1\t";
    h += "IID1\t";
    if (idf.sid) h += "SID1\t";
    if (idf.fid) h += "FID2\t";
    h += "IID2\t";
    if (idf.sid) h += "SID2\t";
  }
  if (c.col_nsnp) h += "NSNP\t";
  if (c.col_hethet) h += "HETHET\t";
  if (c.col_ibs0) h += "IBS0\t";
  if (c.col_ibs1) h += "HET1_HOM2\tHET2_HOM1\t";
  if (c.col_hamming) h += "IBS\t";
  if (c.col_kinship) h += "KINSHIP\t";
  h.back() = '\n';
  return h;
}

// Opens this --parallel piece's --make-king-table output; the first piece writes the header.
bool OpenKingTable(const Cmd& c, const IdFmt& idf, OutFile* ftab, std::string* name) {
  *name = PieceName(c.out + ".kin0", c) + (c.king_table_zs ? ".zst" : "");
  if (!ftab->Open(*name, c.king_table_zs)) {
    logprintf("Error: Failed to open %s for writing.\n", name->c_str());
    return false;
  }
  if (!c.parallel_idx) ftab->Puts(KingTableHeader(c, idf).c_str());
  return true;
}

// The end of a pair-list or --king-table-require table of pair_ct pairs, `filtered` of them left out by
// --king-table-filter.
int CloseKingTable(const Cmd& c, OutFile* ftab, const std::string& name, size_t variant_ct, uint64_t pair_ct, uint64_t filtered) {
  if (!ftab->Close()) return kRetWriteFail;
  printf("\r");
  logprintf("--make-king-table: %u variant%s processed.\n", static_cast<uint32_t>(variant_ct), variant_ct == 1 ? "" : "s");
  logprintf("Results written to %s .\n", name.c_str());
  if (c.king_table_filter != -DBL_MAX) logprintf("--king-table-filter: %llu relationship%s reported (%llu filtered out).\n", static_cast<unsigned long long>(pair_ct - filtered), (pair_ct - filtered == 1) ? "" : "s", static_cast<unsigned long long>(filtered));
  return 0;
}

// One .kin0 line (:2285-2364 / :3705-3760): cc = {IBS0, HETHET, HET2HOM1, HET1HOM2, HOMHOM}.
// The reference's rare-variant pre-scan (CalcKingSparseThread, 2.0/plink2_matrix_calc.cc:904-1250; a variant is
// pre-scanned when its commonest genotype among hom-REF / hom-ALT covers all but row_end/33 of the pass's samples,
// KingMaxSparseCt :1654) reproduces dense counting in every pair case but one: where one sample carries the OTHER
// homozygote and its partner is missing, both branches add 1 to HOMHOM (:1086-1096, :1129-1139) although the pair
// is not jointly observed.  NSNP = HET1_HOM2 + HET2_HOM1 + HOMHOM + HETHET (:2315-2318) - and every proportion
// column, which divides by it - therefore comes out one higher per such variant than the dense count this
// program's kernels produce (178 of 251,594 rows at 4,096 x 65,536 --dummy data).  The .kin0 writer adds the same
// amount so that the table stays byte-identical; counts, kinship and the matrices are unaffected.
struct SparseNsnpFix {
  std::unordered_map<uint64_t, uint32_t> extra;  // (larger index << 32 | smaller index) -> pre-scanned variants with the (other-hom, missing) pattern
  void Scan(const uint64_t* buf, uint32_t variant_ct, uint32_t words, uint32_t s_ct, uint32_t r0, uint32_t r1, uint32_t threads) {
    if (s_ct < 66) return;  // max_sparse_ct = s_ct / 33 < 2: a pre-scanned variant cannot hold both rare genotypes
    threads = std::max(1u, std::min(threads, (variant_ct + 1023) / 1024));
    std::vector<std::vector<uint64_t>> found(threads);
    auto work = [&](uint32_t t) {
      const uint32_t v0 = static_cast<uint32_t>(static_cast<uint64_t>(variant_ct) * t / threads), v1 = static_cast<uint32_t>(static_cast<uint64_t>(variant_ct) * (t + 1) / threads);
      const uint32_t full_words = s_ct / 32, rem = s_ct % 32;
      const uint32_t min_common = s_ct - s_ct / 33;
      std::vector<uint32_t> oth, mis;
      for (uint32_t v = v0; v < v1; ++v) {
        const uint64_t* row = buf + static_cast<uint64_t>(v) * words;
        uint32_t n1 = 0, n2 = 0, n3 = 0;
        for (uint32_t w = 0; w < full_words + (rem ? 1 : 0); ++w) {
          uint64_t x = row[w];
          if (w == full_words) x &= (1ull << (2 * rem)) - 1;
          const uint64_t lo = x & 0x5555555555555555ull, hi = (x >> 1) & 0x5555555555555555ull;
          n1 += static_cast<uint32_t>(__builtin_popcountll(lo & ~hi));
          n2 += static_cast<uint32_t>(__builtin_popcountll(hi & ~lo));
          n3 += static_cast<uint32_t>(__builtin_popcountll(lo & hi));
        }
        const uint32_t n0 = s_ct - n1 - n2 - n3;
        uint32_t other_code;
        if (n0 >= min_common) other_code = 2;
        else if (n2 >= min_common) other_code = 0;
        else continue;
        if (!n3 || !(other_code == 2 ? n2 : n0)) continue;
        oth.clear();
        mis.clear();
        for (uint32_t w = 0; w < full_words + (rem ? 1 : 0); ++w) {
          uint64_t x = row[w];
          const uint32_t lim = (w == full_words) ? rem : 32;
          const uint64_t lo = x & 0x5555555555555555ull, hi = (x >> 1) & 0x5555555555555555ull;
          uint64_t m_bits = lo & hi, o_bits = (other_code == 2) ? (hi & ~lo) : (~(lo | hi) & 0x5555555555555555ull);
          if (lim < 32) {
            const uint64_t keep = (1ull << (2 * lim)) - 1;
            m_bits &= keep;
            o_bits &= keep;
          }
          for (; m_bits; m_bits &= m_bits - 1) mis.push_back(32 * w + static_cast<uint32_t>(__builtin_ctzll(m_bits)) / 2);
          for (; o_bits; o_bits &= o_bits - 1) oth.push_back(32 * w + static_cast<uint32_t>(__builtin_ctzll(o_bits)) / 2);
        }
        for (uint32_t o : oth) {
          for (uint32_t m : mis) {
            const uint32_t hi_s = std::max(o, m), lo_s = std::min(o, m);
            if (hi_s >= r0 && hi_s < r1) found[t].push_back((static_cast<uint64_t>(hi_s) << 32) | lo_s);
          }
        }
      }
    };
    std::vector<std::thread> th;
    for (uint32_t t = 1; t < threads; ++t) th.emplace_back(work, t);
    work(0);
    for (auto& x : th) x.join();
    for (auto& f : found)
      for (uint64_t k : f) ++extra[k];
  }
  uint32_t Get(uint32_t hi_s, uint32_t lo_s) const {
    if (extra.empty()) return 0;
    const auto it = extra.find((static_cast<uint64_t>(hi_s) << 32) | lo_s);
    return it == extra.end() ? 0 : it->second;
  }
};

void WriteKingTableRow(const Cmd& c, const std::string& id1, const std::string& id2, const uint32_t* cc, double kinship, OutFile* ftab, uint32_t nsnp_extra = 0) {
  const uint32_t ibs0 = cc[0], hethet = cc[1], het2hom1 = cc[2], het1hom2 = cc[3], homhom = cc[4];
  char* w = ftab->Reserve(id1.size() + id2.size() + 160);
  if (c.col_id) {
    memcpy(w, id1.data(), id1.size());
    w += id1.size();
    *w++ = '\t';
    memcpy(w, id2.data(), id2.size());
    w += id2.size();
    *w++ = '\t';
  }
  const uint32_t nonmiss = het1hom2 + het2hom1 + homhom + hethet + nsnp_extra;
  double recip = 0.0;
  if (c.col_nsnp) {
    w = u32toa(nonmiss, w);
    *w++ = '\t';
  }
  if (!c.king_counts) recip = 1.0 / static_cast<double>(nonmiss);
  auto put = [&](uint32_t v) {
    if (c.king_counts) w = u32toa(v, w);
    else w = dtoa_g(recip * static_cast<double>(v), w);
    *w++ = '\t';
  };
  if (c.col_hethet) put(hethet);
  if (c.col_ibs0) put(ibs0);
  if (c.col_ibs1) {
    put(het1hom2);
    put(het2hom1);
  }
  if (c.col_hamming) {
    const uint32_t hamming = 2 * ibs0 + het1hom2 + het2hom1;
    if (c.king_counts) w = u32toa(hamming, w);
    else w = dtoa_g(recip * 0.5 * static_cast<double>(hamming), w);
    *w++ = '\t';
  }
  if (c.col_kinship) {
    w = dtoa_g(kinship, w);
    *w++ = '\t';
  }
  w[-1] = '\n';
  ftab->Advance(w);
}

// `--make-king-table --king-table-subset <file> [thresh]` (CalcKingTableSubset, :3224; KingTableSubsetLoad,
// :2774): KING-robust for the pairs listed in a .kin0-style file, in file order, ID1 = first listed sample.
// PLINK 2's natural sort order (rules stated above strcmp_natural_scan_forward, 2.0/include/plink2_string.cc:375-392):
// letters compare as if capitalised; a run of digits that starts with a NONZERO digit at the same position in both
// strings compares by magnitude (zeros in front of it are ordinary characters, so "a01" < "a1" and "00" < "000");
// strings that differ only in capitalisation are ordered by ASCII at their first such difference.
int NaturalCompare(const std::string& a, const std::string& b) {
  auto up = [](unsigned char ch) { return (ch >= 'a' && ch <= 'z') ? static_cast<unsigned char>(ch - 32) : ch; };
  auto nz = [](unsigned char ch) { return ch >= '1' && ch <= '9'; };
  auto dg = [](unsigned char ch) { return ch >= '0' && ch <= '9'; };
  size_t i = 0, j = 0;
  int tie = 0;  // decided by the first capitalisation-only difference
  for (;;) {
    const unsigned char ca = i < a.size() ? static_cast<unsigned char>(a[i]) : 0, cb = j < b.size() ? static_cast<unsigned char>(b[j]) : 0;
    if (nz(ca) && nz(cb)) {
      size_t ea = i, eb = j;
      while (ea < a.size() && dg(static_cast<unsigned char>(a[ea]))) ++ea;
      while (eb < b.size() && dg(static_cast<unsigned char>(b[eb]))) ++eb;
      if (ea - i != eb - j) return (ea - i < eb - j) ? -1 : 1;
      const int cmp = a.compare(i, ea - i, b, j, eb - j);
      if (cmp) return cmp < 0 ? -1 : 1;
      i = ea;
      j = eb;
      continue;
    }
    if (!ca && !cb) return tie;
    if (ca != cb) {
      const unsigned char ua = up(ca), ub = up(cb);
      if (ua != ub) return ua < ub ? -1 : 1;
      if (!tie) tie = ca < cb ? -1 : 1;
    }
    ++i;
    ++j;
  }
}

// "--make-king-table rel-check" (GetRelCheckOrKTRequirePairs, 2.0/plink2_matrix_calc.cc:2975-3043): the samples in
// natural order of FID<tab>IID[<tab>SID]; inside every block of equal FID (equal up to capitalisation, see below) each
// sample is paired with all earlier ones, the later sample listed first.
// The sample indices in natural order of FID<tab>IID[<tab>SID] (the reference's nsorted_xidbox); *key_out gets the keys.
std::vector<uint32_t> NaturalSampleOrder(const SampleInfo& S, std::vector<std::string>* key_out = nullptr) {
  const uint32_t n = S.size();
  std::vector<std::string> key(n);
  for (uint32_t k = 0; k < n; ++k) {
    key[k] = S.fid[k] + "\t" + S.iid[k];
    if (S.sid_present) key[k] += "\t" + S.sid[k];
  }
  std::vector<uint32_t> ord(n);
  for (uint32_t k = 0; k < n; ++k) ord[k] = k;
  std::stable_sort(ord.begin(), ord.end(), [&](uint32_t x, uint32_t y) { return NaturalCompare(key[x], key[y]) < 0; });
  if (key_out) *key_out = std::move(key);
  return ord;
}

void RelCheckPairs(const SampleInfo& S, std::vector<uint32_t>* pairs) {
  const uint32_t n = S.size();
  std::vector<std::string> key;
  const std::vector<uint32_t> ord = NaturalSampleOrder(S, &key);
  for (uint32_t b0 = 0; b0 < n;) {
    // block end as the reference finds it (:3030-3042): the first sorted key not below "<FID of the block's first
    // entry> " in natural order - which also takes in FIDs that differ from it only in capitalisation
    const std::string bound = S.fid[ord[b0]] + " ";
    uint32_t b1 = b0 + 1;
    while (b1 < n && NaturalCompare(key[ord[b1]], bound) < 0) ++b1;
    for (uint32_t i1 = b0 + 1; i1 < b1; ++i1)
      for (uint32_t i2 = b0; i2 < i1; ++i2) {
        pairs->push_back(ord[i1]);
        pairs->push_back(ord[i2]);
      }
    b0 = b1;
  }
}

// --king-table-require[-xor] sample set (CalcKingTableSubset, 2.0/plink2_matrix_calc.cc:3248-3267): IDs read like --keep
// files, the lists of all files merged.
int LoadKingRequire(const Cmd& c, const SampleInfo& S, std::vector<uint8_t>* req) {
  std::string err;
  uint64_t dup_ct = 0;
  const int rc = MarkSampleIds(c.king_table_require, c.king_table_require_xor ? "king-table-require-xor" : "king-table-require", S, req, &dup_ct, &err);
  if (rc) {
    logprintf("Error: %s\n", err.c_str());
    return rc == 3 ? kRetOpenFail : kRetMalformedInput;
  }
  uint32_t ct = 0;
  for (uint8_t f : *req) ct += f;
  if (!ct) {
    logprintf("Error: No sample ID(s) in --king-table-require[-xor] file(s) are in the current\ndataset.\n");
    return kRetInconsistentInput;
  }
  if (c.king_table_require_xor && ct == S.size()) {
    logprintf("Error: All sample ID(s) in --king-table-require-xor file(s) are in the current\ndataset.\n");
    return kRetInconsistentInput;
  }
  logprintf("--king-table-require%s: %u sample ID%s loaded.\n", c.king_table_require_xor ? "-xor" : "", ct, ct == 1 ? "" : "s");
  return 0;
}

// A listed or rel-check pair is kept when it includes at least one required sample (-xor: exactly one), :2777-2779.
inline bool KingRequireKeeps(const Cmd& c, const std::vector<uint8_t>& req, uint32_t a, uint32_t b) {
  return c.king_table_require_xor ? req[a] != req[b] : (req[a] || req[b]);
}

int RunKingRequireDense(const Cmd& c, Dataset* ds, Pl2GpuCtx* ctx, const std::vector<uint32_t>& vidx, const std::vector<uint8_t>& req);

// rel_check: pairs of same-FID samples when there is no subset file.  Without a subset file or rel-check, the
// --king-table-require[-xor] pairs go to RunKingRequireDense instead of a pair list.
int RunKingSubset(const Cmd& c, Dataset* ds, Pl2GpuCtx* ctx, bool rel_check) {
  const SampleInfo& S = ds->samples;
  const uint32_t n = S.size();
  if (c.parallel_tot != 1) {
    logprintf("Error: %s with --parallel is not supported by plink2_b200 yet.\n", c.king_table_subset.empty() && !rel_check ? "--king-table-require[-xor]" : "--king-table-subset");
    return kRetNotYetSupported;
  }
  if (!c.king_table_require.empty() && c.gpus > 1) {
    logprintf("Error: --king-table-require[-xor] runs on one GPU; --gpus %u is not supported with it.\n", c.gpus);
    return kRetNotYetSupported;
  }
  if (n < 2) {
    logprintf("Error: --make-king-table requires at least 2 samples.\n");
    return kRetDegenerateData;
  }
  std::vector<uint32_t> vidx;
  const int vrc = RelationshipVariants(*ds, "KING-robust calculation", &vidx);
  if (vrc) return vrc;
  std::vector<uint8_t> req;
  if (!c.king_table_require.empty()) {
    const int rrc = LoadKingRequire(c, S, &req);
    if (rrc) return rrc;
    if (c.king_table_subset.empty() && !rel_check) return RunKingRequireDense(c, ds, ctx, vidx, req);
  }
  std::vector<uint32_t> pairs;
  if (c.king_table_subset.empty()) {
    RelCheckPairs(S, &pairs);  // rel-check without a subset file
    if (!req.empty()) {
      // the same pairs in the same order as GetRelCheckOrKTRequirePairs' require branch (:3045-3160)
      size_t w = 0;
      for (size_t p = 0; p < pairs.size(); p += 2) {
        if (!KingRequireKeeps(c, req, pairs[p], pairs[p + 1])) continue;
        pairs[w++] = pairs[p];
        pairs[w++] = pairs[p + 1];
      }
      pairs.resize(w);
    }
  } else {
  // ---- header (:3391-3452): [#FID1|FID] (ID1|IID1) [SID1] [FID2] (ID2|IID2) [SID2] ... [KINSHIP|Kinship]
  std::vector<std::string> lines;
  std::string rerr;
  if (!ReadLines(c.king_table_subset, &lines, &rerr)) {
    logprintf("Error: %s\n", rerr.c_str());
    return kRetOpenFail;
  }
  if (lines.empty()) {
    logprintf("Error: Empty --king-table-subset file.\n");
    return kRetMalformedInput;
  }
  std::vector<std::string> hd = SplitWs(lines[0]);
  auto bad_header = [&]() {
    logprintf("Error: Invalid header line in --king-table-subset file.\n");
    return kRetMalformedInput;
  };
  if (hd.empty()) return bad_header();
  size_t t = 0;
  bool fid_present = hd[0] == "#FID1" || hd[0] == "FID";
  std::string tok0 = hd[0];
  if (fid_present) {
    ++t;
    if (t >= hd.size()) return bad_header();
    tok0 = hd[t];
  } else {
    if (tok0.empty() || tok0[0] != '#') return bad_header();
    tok0 = tok0.substr(1);
  }
  if (tok0 != "ID1" && tok0 != "IID1") return bad_header();
  ++t;
  bool sid_cols = false;
  if (t < hd.size() && hd[t] == "SID1") {
    sid_cols = true;
    ++t;
  }
  if (fid_present) {
    if (t >= hd.size() || hd[t] != "FID2") return bad_header();
    ++t;
  }
  if (t >= hd.size() || (hd[t] != "ID2" && hd[t] != "IID2")) return bad_header();
  ++t;
  if (sid_cols) {
    if (t >= hd.size() || hd[t] != "SID2") return bad_header();
    ++t;
  }
  const size_t id_tokens = t;  // tokens of a data line before the first non-ID column
  size_t kinship_col = 0;
  double thresh = c.king_table_subset_thresh;
  if (thresh != -DBL_MAX) {
    thresh *= 1.0 - 1.0 / 17592186044416.0;  // kSmallEpsilon = 2^-44 (:3441)
    size_t k = t;
    for (; k < hd.size(); ++k)
      if (hd[k] == "KINSHIP" || hd[k] == "Kinship") break;
    if (k == hd.size()) {
      logprintf("Error: No kinship-coefficient column in --king-table-subset file.\n");
      return kRetInconsistentInput;
    }
    kinship_col = k;
  }
  // ---- sample lookup by FID<tab>IID.  A file without FID columns reads every ID with FID 0 (XidRead,
  // plink2_common.cc:1280-1284), so it only names samples whose own FID is 0 - the reference's behaviour, kept as is
  std::unordered_map<std::string, uint32_t> lookup;
  lookup.reserve(static_cast<size_t>(n) * 2);
  for (uint32_t k = 0; k < n; ++k) lookup.emplace(S.fid[k] + "\t" + S.iid[k], k);
  for (size_t li = 1; li < lines.size(); ++li) {
    const std::vector<std::string> f = SplitWs(lines[li]);
    if (f.empty()) continue;
    if (f.size() < id_tokens) {
      logprintf("Error: Line %zu of --king-table-subset file has fewer tokens than expected.\n", li + 1);
      return kRetMalformedInput;
    }
    size_t q = 0;
    std::string k1 = fid_present ? (f[q] + "\t" + f[q + 1]) : ("0\t" + f[q]);
    q += fid_present ? 2 : 1;
    if (sid_cols) ++q;
    std::string k2 = fid_present ? (f[q] + "\t" + f[q + 1]) : ("0\t" + f[q]);
    const auto i1 = lookup.find(k1), i2 = lookup.find(k2);
    if (i1 == lookup.end() || i2 == lookup.end()) continue;  // not loaded: skipped silently, as in the reference
    if (i1->second == i2->second) {
      logprintf("Error: Identical sample IDs on line %zu of --king-table-subset file.\n", li + 1);
      return kRetInconsistentInput;
    }
    if (!req.empty() && !KingRequireKeeps(c, req, i1->second, i2->second)) continue;
    if (thresh != -DBL_MAX) {
      if (f.size() <= kinship_col) {
        logprintf("Error: Line %zu of --king-table-subset file has fewer tokens than expected.\n", li + 1);
        return kRetMalformedInput;
      }
      double kv;
      if (!ParseDouble(f[kinship_col].c_str(), &kv)) continue;  // e.g. "nan": not a number -> line skipped
      if (kv < thresh) continue;
    }
    if (c.king_rel_check && S.fid[i1->second] != S.fid[i2->second]) continue;  // rel-check: same-FID pairs only
    pairs.push_back(i1->second);
    pairs.push_back(i2->second);
  }
  }  // subset file
  const uint64_t pair_ct = pairs.size() / 2;
  if (!pair_ct) {
    logprintf(c.king_table_subset.empty() ? "Error: No sample pairs with the same FID for --make-king-table rel-check.\n" : "Error: No valid pairs in --king-table-subset file.\n");
    return kRetInconsistentInput;
  }
  logprintf("%s: %llu pair%s loaded.\n", c.king_table_subset.empty() ? "--make-king-table rel-check" : "--king-table-subset", static_cast<unsigned long long>(pair_ct), pair_ct == 1 ? "" : "s");
  const IdFmt idf = KingIdFmt(c, S);
  std::string tab_name;
  OutFile ftab;
  if (!OpenKingTable(c, idf, &ftab, &tab_name)) return kRetOpenFail;
  Pl2KingPairJob* pair_job = nullptr;
  if (pl2gpu_king_pairs_begin(ctx, n, pairs.data(), pair_ct, &pair_job)) return GpuFail("pl2gpu_king_pairs_begin");
  const KingPairJob job(pair_job);
  BlockStreamer bs(ds, &vidx, n, 32768);
  if (!bs.Init()) return GpuFail("pl2gpu_host_alloc");
  uint32_t done = 0;
  const int src = StreamBlocks(&bs, [&](uint32_t got) -> int {
    if (pl2gpu_king_pairs_add_variants(job.get(), bs.buf, static_cast<uint64_t>(bs.words) * 8, got, 0)) return GpuFail("pl2gpu_king_pairs_add_variants");
    done += got;
    printf("\r--make-king-table pass 1: %u variants complete.", done);
    fflush(stdout);
    return 0;
  });
  if (src) return src;
  printf("\r--make-king-table pass 1: Writing...                   ");
  fflush(stdout);
  std::vector<uint32_t> counts;
  uint64_t filter_ct = 0;
  const uint64_t chunk = 8ull << 20;
  for (uint64_t p0 = 0; p0 < pair_ct; p0 += chunk) {
    const uint64_t p1 = std::min(pair_ct, p0 + chunk);
    counts.resize((p1 - p0) * 5);
    if (pl2gpu_king_pairs_get_counts(job.get(), p0, p1, counts.data(), 0)) return GpuFail("pl2gpu_king_pairs_get_counts");
    for (uint64_t p = p0; p < p1; ++p) {
      const uint32_t* cc = &counts[(p - p0) * 5];
      const double kinship = KinshipFromCounts(cc);
      if (c.king_table_filter != -DBL_MAX && kinship < c.king_table_filter) {
        ++filter_ct;
        continue;
      }
      WriteKingTableRow(c, FmtId(S, pairs[2 * p], idf), FmtId(S, pairs[2 * p + 1], idf), cc, kinship, &ftab);
    }
  }
  return CloseKingTable(c, &ftab, tab_name, vidx.size(), pair_ct, filter_ct);
}

// --king-table-require[-xor] without a pair list (GetRelCheckOrKTRequirePairs' require branch, :3045-3160): in natural
// sample order, row idx1 ascending, then idx2 < idx1 ascending, the pair (idx1, idx2) is written when it includes a
// required sample (-xor: exactly one).  Instead of listing those pairs, the device holds the samples in the order
// "non-required, then required" (each in index order): with n0 non-required samples the wanted pairs are exactly rows
// [n0, N) of the strict lower triangle over positions, cut at column n0 for -xor, so one mapped KING job computes them
// on the tensor tile path with work in proportion to r x N.  The results come back in positions, are oriented to the
// reference's row ("1" = the sample listed first) and sorted into its order on the host.  Without --king-table-filter
// every pair is held in host memory (28 bytes each) until the sort; with it only the qualifying pairs leave the device.
// NSNP is the dense count: CalcKingTableSubset has no rare-variant pre-scan.
int RunKingRequireDense(const Cmd& c, Dataset* ds, Pl2GpuCtx* ctx, const std::vector<uint32_t>& vidx, const std::vector<uint8_t>& req) {
  const SampleInfo& S = ds->samples;
  const uint32_t n = S.size();
  std::vector<uint32_t> order;
  order.reserve(n);
  for (uint32_t k = 0; k < n; ++k)
    if (!req[k]) order.push_back(k);
  const uint32_t n0 = static_cast<uint32_t>(order.size());
  for (uint32_t k = 0; k < n; ++k)
    if (req[k]) order.push_back(k);
  const uint32_t col_end = c.king_table_require_xor ? n0 : n;
  const uint64_t pair_ct = KingPairsBelow(n, col_end) - KingPairsBelow(n0, col_end);
  const bool filter = c.king_table_filter != -DBL_MAX;
  logprintf("--king-table-require%s: %llu pair%s on the device (rows %u-%u of the sample order with the required samples last).\n", c.king_table_require_xor ? "-xor" : "", static_cast<unsigned long long>(pair_ct), pair_ct == 1 ? "" : "s", n0, n - 1);
  if (!filter) logprintf("--king-table-require%s: the unfiltered table is sorted in host memory (%.1f MB) before it is written.\n", c.king_table_require_xor ? "-xor" : "", pair_ct * 28.0 / 1e6);
  std::vector<uint32_t> rank(n);
  {
    const std::vector<uint32_t> nat = NaturalSampleOrder(S);
    for (uint32_t r = 0; r < n; ++r) rank[nat[r]] = r;
  }
  // pass planning as in RunKing; each pass re-streams the variants
  uint32_t batch = 0;
  std::vector<uint32_t> bounds;
  const int prc = PlanKingPasses(c, {ctx}, "--make-king-table", n, n0, n, 5, [&](uint32_t a, uint32_t b, uint32_t bt) { return pl2gpu_king_mapped_mem_required(n, a, b, col_end, bt); }, &batch, &bounds);
  if (prc) return prc;
  const uint32_t pass_ct = static_cast<uint32_t>(bounds.size() - 1);
  struct Row {
    uint32_t r1, r2;  // natural-order ranks of the sample listed first (the larger) and second
    uint32_t cc[5];
  };
  std::vector<Row> rows;
  rows.reserve(filter ? 0 : pair_ct);
  // device pair (position pj, position pi < pj), counts with "1" = pi: listed first is the sample of larger rank
  auto add_row = [&](uint32_t pj, uint32_t pi, const uint32_t* cc) {
    const uint32_t sj = order[pj], si = order[pi];
    Row row;
    memcpy(row.cc, cc, 20);
    if (rank[sj] > rank[si]) {
      row.r1 = rank[sj];
      row.r2 = rank[si];
      std::swap(row.cc[2], row.cc[3]);  // "1" becomes the sample at the larger position
    } else {
      row.r1 = rank[si];
      row.r2 = rank[sj];
    }
    rows.push_back(row);
  };
  BlockStreamer bs(ds, &vidx, n, batch);
  if (!bs.Init()) return GpuFail("pl2gpu_host_alloc");
  for (uint32_t pass = 1; pass <= pass_ct; ++pass) {
    const uint32_t p0 = bounds[pass - 1], p1 = bounds[pass];
    Pl2KingJob* mapped_job = nullptr;
    if (pl2gpu_king_begin_mapped(ctx, n, order.data(), p0, p1, col_end, batch, &mapped_job)) return GpuFail("pl2gpu_king_begin_mapped");
    const KingJob job(mapped_job);
    uint32_t done = 0;
    int rc = StreamBlocks(&bs, [&](uint32_t got) -> int {
      if (pl2gpu_king_add_variants(job.get(), bs.buf, static_cast<uint64_t>(bs.words) * 8, got, 0)) return GpuFail("pl2gpu_king_add_variants");
      done += got;
      printf("\r--make-king-table pass %u/%u: %u variants complete.", pass, pass_ct, done);
      fflush(stdout);
      return 0;
    });
    if (rc) return rc;
    if (filter) {
      std::vector<uint32_t> fp, fc;
      std::vector<double> fk;
      uint64_t found = 0;
      rc = FetchKingFiltered(job.get(), p0, p1, c.king_table_filter, &fp, &fc, &fk, &found);
      if (rc) return rc;
      for (uint64_t q = 0; q < found; ++q) add_row(fp[2 * q], fp[2 * q + 1], &fc[5 * q]);
    } else {
      rc = ForEachKingCountChunk(job.get(), p0, p1, col_end, true, [&](uint32_t c0, uint32_t c1, uint64_t, const uint32_t* cc) {
        for (uint32_t pj = c0; pj < c1; ++pj)
          for (uint32_t pi = 0; pi < std::min(pj, col_end); ++pi, cc += 5) add_row(pj, pi, cc);
        return 0;
      });
      if (rc) return rc;
    }
  }
  printf("\r--make-king-table: Writing...                   ");
  fflush(stdout);
  std::sort(rows.begin(), rows.end(), [](const Row& a, const Row& b) { return a.r1 != b.r1 ? a.r1 < b.r1 : a.r2 < b.r2; });
  const IdFmt idf = KingIdFmt(c, S);
  std::string tab_name;
  OutFile ftab;
  if (!OpenKingTable(c, idf, &ftab, &tab_name)) return kRetOpenFail;
  {
    std::vector<uint32_t> by_rank(n);
    for (uint32_t k = 0; k < n; ++k) by_rank[rank[k]] = k;
    for (const Row& row : rows) WriteKingTableRow(c, FmtId(S, by_rank[row.r1], idf), FmtId(S, by_rank[row.r2], idf), row.cc, KinshipFromCounts(row.cc), &ftab);
  }
  return CloseKingTable(c, &ftab, tab_name, vidx.size(), pair_ct, pair_ct - rows.size());
}

int RunKing(const Cmd& c, Dataset* ds, Pl2GpuCtx* ctx, std::vector<uint8_t>* cutoff_removed) {
  const SampleInfo& S = ds->samples;
  const uint32_t n = S.size();
  const char* flagname = c.make_king ? "--make-king" : (c.make_king_table ? "--make-king-table" : "--king-cutoff");
  if (n < 2) {
    logprintf("Error: %s requires at least 2 samples.\n", flagname);
    return kRetDegenerateData;
  }
  std::vector<uint32_t> vidx;
  const int vrc = RelationshipVariants(*ds, "KING-robust calculation", &vidx);
  if (vrc) return vrc;
  uint32_t grand_r0, grand_r1;
  ParallelBounds(n, 1, c.parallel_idx, c.parallel_tot, &grand_r0, &grand_r1);
  const bool want_table = c.make_king_table;
  const bool want_matrix = c.make_king;
  if (want_matrix && c.king_shape == Cmd::kSq && c.parallel_tot != 1) {
    logprintf("Error: --make-king square output cannot be combined with --parallel; use square0 or triangle.\n");
    return kRetInvalidCmdline;
  }
  const uint32_t wl = (n + 63) / 64;
  std::vector<uint64_t> kin_table;
  if (c.king_cutoff >= 0) kin_table.assign(static_cast<uint64_t>(n) * wl, 0);

  OutFile fmat, ftab;
  std::string mat_name, tab_name;
  if (want_matrix) {
    const bool mat_zs = c.king_zs && c.king_enc == Cmd::kText;  // SetKingMatrixFname (:1576): text matrices only
    mat_name = PieceName(c.out + (c.king_enc == Cmd::kText ? ".king" : ".king.bin"), c) + (mat_zs ? ".zst" : "");
    if (!fmat.Open(mat_name, mat_zs)) {
      logprintf("Error: Failed to open %s for writing.\n", mat_name.c_str());
      return kRetOpenFail;
    }
  }
  const IdFmt idf = KingIdFmt(c, S);
  std::vector<std::string> fmtids;
  if (want_table) {
    if (!OpenKingTable(c, idf, &ftab, &tab_name)) return kRetOpenFail;
    fmtids.resize(n);
    for (uint32_t k = 0; k < n; ++k) fmtids[k] = FmtId(S, k, idf);
  }
  // the matrix's rows start at 1 (ParallelBounds with start 1); sample 0's row, the diagonal 0.5 alone, goes first
  // with the first --parallel piece (:2129-2132)
  TriangleMatrixWriter mat(&fmat, n, c.king_shape, c.king_enc, false);
  const double half = 0.5;
  if (want_matrix && !c.parallel_idx) mat.Row(0, &half, half);

  // multi-GPU team (--gpus): every pass's row block is cut into one tile-aligned slab per device
  GpuTeam team;
  {
    // not worth splitting tiny triangles: keep at least four 128-row tiles per device
    const uint32_t gpus_eff = std::max(1u, std::min(c.gpus, (grand_r1 - grand_r0) / 512));
    if (gpus_eff < c.gpus) logprintf("Note: --gpus %u reduced to %u for %u rows.\n", c.gpus, gpus_eff, grand_r1 - grand_r0);
    const int trc = TeamInit(ctx, c.device, gpus_eff, &team);
    if (trc) return trc;
  }
  const uint32_t G = team.size();
  // pass planning: every device holds the accumulators of its slab of the pass; the two staged blocks, their
  // sample-major copies and their column plane copies take 8 block sizes
  uint32_t batch = 0;
  std::vector<uint32_t> bounds;
  int rc = PlanKingPasses(c, team.ctx, flagname, n, grand_r0, grand_r1, 8, [&](uint32_t a, uint32_t b, uint32_t bt) {
    const std::vector<uint32_t> sb = TileAlignedBounds(a, b, G, false);
    uint64_t need = 0;
    for (uint32_t g = 0; g < G; ++g) {
      if (sb[g + 1] > sb[g]) need = std::max(need, pl2gpu_king_mem_required(n, sb[g], sb[g + 1], bt));
    }
    return need;
  }, &batch, &bounds);
  if (rc) return rc;
  const uint32_t pass_ct = static_cast<uint32_t>(bounds.size() - 1);
  BlockStreamer bs(ds, &vidx, n, batch, G);  // G spare rows: a sharded batch is topped up to a multiple of G
  if (!bs.Init()) return GpuFail("pl2gpu_host_alloc");
  // --make-king-table with --king-table-filter and nothing else to produce: filter on the device and fetch only the
  // surviving rows (the unfiltered table is 20 bytes x N^2/2)
  const bool device_filter = want_table && !want_matrix && c.king_cutoff < 0 && c.king_table_filter != -DBL_MAX;
  uint64_t filter_ct = 0;
  // NSNP compatibility with the reference's rare-variant pre-scan (SparseNsnpFix); only the table shows NSNP
  const bool nsnp_fix_on = want_table && (c.col_nsnp || !c.king_counts);
  SparseNsnpFix nsnp_fix;
  for (uint32_t pass = 1; pass <= pass_ct; ++pass) {
    const uint32_t pass_r0 = bounds[pass - 1], pass_r1 = bounds[pass];
    const std::vector<uint32_t> sbounds = TileAlignedBounds(pass_r0, pass_r1, G, false);
    std::vector<KingJob> jobs(G);
    for (uint32_t g = 0; g < G; ++g) {
      // an empty slab still takes part in the all-gathers (rank g of the communicator)
      Pl2KingJob* job = nullptr;
      if (pl2gpu_king_begin_ex(team.ctx[g], n, sbounds[g], sbounds[g + 1], kPl2KingAlgoAuto, batch, &job)) return GpuFail("pl2gpu_king_begin_ex");
      jobs[g].reset(job);
    }
    g_clock.Mark("king: begin (device alloc)");
    uint32_t done = 0;
    double t_add = 0;
    const double decode0 = bs.decode_s;
    rc = StreamBlocks(&bs, [&](uint32_t got) -> int {
      if (nsnp_fix_on) nsnp_fix.Scan(bs.buf, got, bs.words, grand_r1, pass_r0, pass_r1, g_decode_threads);
      const auto ta = std::chrono::steady_clock::now();
      if (G == 1) {
        if (pl2gpu_king_add_variants(jobs[0].get(), bs.buf, static_cast<uint64_t>(bs.words) * 8, got, 0)) return GpuFail("pl2gpu_king_add_variants");
      } else {
        std::string gerr;
        if (AddSharded(&bs, got, G, [&](uint32_t g, const uint64_t* slice, uint32_t per) { return pl2gpu_king_add_variants_sharded(jobs[g].get(), slice, static_cast<uint64_t>(bs.words) * 8, per, 0); }, &gerr)) {
          logprintf("\nError: pl2gpu_king_add_variants_sharded: %s\n", gerr.c_str());
          return kRetGpuFail;
        }
      }
      t_add += g_clock.Since(ta);
      done += got;
      printf("\r%s pass %u/%u: %u variants complete.", flagname, pass, pass_ct, done);
      fflush(stdout);
      return 0;
    });
    if (rc) return rc;
    printf("\r%s pass %u/%u: Writing...                   ", flagname, pass, pass_ct);
    fflush(stdout);
    if (g_clock.on) fprintf(stderr, "[timing]   decode (PgrGet) %.3f s, pl2gpu_king_add_variants %.3f s\n", bs.decode_s - decode0, t_add);
    g_clock.Mark("king: decode + add_variants");
    for (uint32_t g = 0; g < G; ++g) {
      Pl2KingJob* const job = jobs[g].get();
      const uint32_t row_start = sbounds[g], row_end = sbounds[g + 1];
      if (row_start >= row_end) continue;
      if (device_filter) {
        std::vector<uint32_t> fp, fc;
        std::vector<double> fk;
        uint64_t found = 0;
        rc = FetchKingFiltered(job, row_start, row_end, c.king_table_filter, &fp, &fc, &fk, &found);
        if (rc) return rc;
        for (uint64_t q = 0; q < found; ++q) WriteKingTableRow(c, fmtids[fp[2 * q]], fmtids[fp[2 * q + 1]], &fc[5 * q], fk[q], &ftab, nsnp_fix.Get(fp[2 * q], fp[2 * q + 1]));
        filter_ct += KingPairsBelow(row_end, n) - KingPairsBelow(row_start, n) - found;
        continue;
      }
      std::vector<double> kin;
      rc = ForEachKingCountChunk(job, row_start, row_end, n, want_table, [&](uint32_t c0, uint32_t c1, uint64_t pairs, const uint32_t* counts) {
        if (want_matrix || c.king_cutoff >= 0 || !want_table) {
          kin.resize(pairs);
          if (pairs && pl2gpu_king_get_kinship(job, c0, c1, kin.data(), 0)) return GpuFail("pl2gpu_king_get_kinship");
        }
        uint64_t p = 0;
        for (uint32_t j = c0; j < c1; ++j) {
          // --king-cutoff bit matrix (:2148-2151)
          if (c.king_cutoff >= 0) {
            for (uint32_t i = 0; i < j; ++i) {
              if (kin[p + i] > c.king_cutoff) {
                kin_table[static_cast<uint64_t>(j) * wl + i / 64] |= 1ull << (i % 64);
                kin_table[static_cast<uint64_t>(i) * wl + j / 64] |= 1ull << (j % 64);
              }
            }
          }
          if (want_matrix) mat.Row(j, &kin[p], half);
          if (want_table) {
            for (uint32_t i = 0; i < j; ++i) {
              const uint32_t* cc = &counts[(p + i) * 5];
              const double kinship = KinshipFromCounts(cc);
              if (c.king_table_filter != -DBL_MAX && kinship < c.king_table_filter) {
                ++filter_ct;
                continue;
              }
              WriteKingTableRow(c, fmtids[j], fmtids[i], cc, kinship, &ftab, nsnp_fix.Get(j, i));
            }
          }
          p += j;
        }
        return 0;
      });
      if (rc) return rc;
    }
    nsnp_fix.extra.clear();
    g_clock.Mark("king: fetch results + write");
    jobs.clear();
    g_clock.Mark("king: end (device free)");
  }
  if (want_matrix) mat.Finish();
  printf("\r                                              \r");
  logprintf("%s: %u variants processed.\n", flagname, static_cast<uint32_t>(vidx.size()));
  if (want_matrix) {
    if (!fmat.Close()) {
      logprintf("Error: File write failure.\n");
      return kRetWriteFail;
    }
    std::string idname = c.out + ".king.id";
    if (!c.parallel_idx) {
      if (!WriteAllIds(idname, S, true)) return kRetWriteFail;
      logprintf("Results written to %s and %s .\n", mat_name.c_str(), idname.c_str());
    } else {
      logprintf("Results written to %s .\n", mat_name.c_str());
    }
  }
  if (want_table) {
    if (!ftab.Close()) {
      logprintf("Error: File write failure.\n");
      return kRetWriteFail;
    }
    logprintf("Results written to %s .\n", tab_name.c_str());
    if (c.king_table_filter != -DBL_MAX) {
      const uint64_t tot = (static_cast<uint64_t>(grand_r1) * (grand_r1 - 1) - static_cast<uint64_t>(grand_r0) * (grand_r0 - 1)) / 2;
      logprintf("--king-table-filter: %llu relationship%s reported (%llu filtered out).\n", static_cast<unsigned long long>(tot - filter_ct), (tot - filter_ct == 1) ? "" : "s", static_cast<unsigned long long>(filter_ct));
    }
  }
  if (c.king_cutoff >= 0) {
    if (c.parallel_tot != 1) {
      logprintf("Error: --king-cutoff cannot be used with --parallel.\n");
      return kRetInvalidCmdline;
    }
    KinshipPrune(&kin_table, n, cutoff_removed);
    std::vector<uint32_t> in, out;
    for (uint32_t k = 0; k < n; ++k) ((*cutoff_removed)[k] ? out : in).push_back(k);
    const std::string in_name = c.out + ".king.cutoff.in.id", out_name = c.out + ".king.cutoff.out.id";
    if (!WriteIdFile(in_name, S, in, true) || !WriteIdFile(out_name, S, out, true)) return kRetWriteFail;
    logprintf("--king-cutoff: Excluded sample ID%s written to %s , and %u remaining sample ID%s written to %s .\n", out.size() == 1 ? "" : "s", out_name.c_str(), static_cast<uint32_t>(in.size()), in.size() == 1 ? "" : "s", in_name.c_str());
  }
  return 0;
}

// --king-cutoff-table (KingCutoffBatchTable, 2.0/plink2_matrix_calc.cc:643-862): the relatedness prune of --king-cutoff
// driven by a kinship table written earlier (.kin0: [#FID1] ID1|IID1 [SID1] [FID2] ID2|IID2 [SID2] ... KINSHIP).  Pairs
// whose kinship exceeds threshold (1 + 2^-44) become constraints; unknown IDs and non-numeric kinship cells are
// skipped.  Host-only work in the reference too - no device involved.
int RunKingCutoffTable(const Cmd& c, Dataset* ds, std::vector<uint8_t>* removed_out) {
  const SampleInfo& S = ds->samples;
  const uint32_t n = S.size();
  std::vector<std::string> lines;
  std::string err;
  if (!ReadLines(c.king_cutoff_table, &lines, &err)) {
    logprintf("Error: %s\n", err.c_str());
    return kRetOpenFail;
  }
  if (lines.empty() || lines[0].empty()) {
    logprintf("Error: Empty --king-cutoff-table file.\n");
    return kRetMalformedInput;
  }
  std::vector<std::string> h = SplitWs(lines[0]);
  size_t hi = 0;
  auto bad_header = []() {
    logprintf("Error: Invalid header line in --king-cutoff-table file.\n");
    return kRetMalformedInput;
  };
  const bool fid_present = h[0] == "#FID1" || h[0] == "FID";
  if (fid_present) {
    ++hi;
  } else {
    if (h[0].empty() || h[0][0] != '#') return bad_header();
    h[0] = h[0].substr(1);
  }
  if (hi >= h.size() || (h[hi] != "ID1" && h[hi] != "IID1")) return bad_header();
  ++hi;
  bool sid_col = false;
  if (hi < h.size() && h[hi] == "SID1") {
    sid_col = true;
    ++hi;
  }
  if (fid_present) {
    if (hi >= h.size() || h[hi] != "FID2") return bad_header();
    ++hi;
  }
  if (hi >= h.size() || (h[hi] != "ID2" && h[hi] != "IID2")) return bad_header();
  ++hi;
  if (sid_col) {
    if (hi >= h.size() || h[hi] != "SID2") return bad_header();
    ++hi;
  }
  size_t kin_col = hi;
  while (kin_col < h.size() && h[kin_col] != "KINSHIP" && h[kin_col] != "Kinship") ++kin_col;
  if (kin_col == h.size()) {
    logprintf("Error: No kinship-coefficient column in --king-cutoff-table file.\n");
    return kRetInconsistentInput;
  }
  const bool use_sid = sid_col && S.sid_present;
  auto key = [&](const std::string& fid, const std::string& iid, const std::string& sid) {
    std::string k = (fid_present ? fid : std::string("0")) + "\t" + iid;  // no FID column: FID 0 (XidRead, plink2_common.cc:1280)
    if (use_sid) k += "\t" + sid;
    return k;
  };
  // a file without FID columns therefore only names samples whose own FID is 0, as in the reference
  std::unordered_map<std::string, int64_t> by_key;
  by_key.reserve(static_cast<size_t>(n) * 2);
  for (uint32_t k = 0; k < n; ++k) {
    auto ins = by_key.emplace(S.fid[k] + "\t" + S.iid[k] + (use_sid ? "\t" + S.sid[k] : std::string()), k);
    if (!ins.second) ins.first->second = -1;
  }
  const uint32_t wl = (n + 63) / 64;
  std::vector<uint64_t> table(static_cast<uint64_t>(n) * wl, 0);
  const double thresh = c.king_cutoff_table_thresh * (1.0 + 1.0 / 17592186044416.0);
  const size_t ids_per_side = (fid_present ? 1 : 0) + 1 + (sid_col ? 1 : 0);
  uint64_t constraint_ct = 0;
  for (size_t li = 1; li < lines.size(); ++li) {
    if (lines[li].empty()) continue;
    const std::vector<std::string> t = SplitWs(lines[li]);
    if (t.size() <= kin_col) {
      logprintf("Error: Fewer tokens than expected on line %zu of %s .\n", li + 1, c.king_cutoff_table.c_str());
      return kRetMalformedInput;
    }
    int64_t idx[2];
    for (int side = 0; side < 2; ++side) {
      size_t p = side * ids_per_side;
      const std::string fid = fid_present ? t[p++] : std::string();
      const std::string iid = t[p++];
      const std::string sid = sid_col ? t[p++] : std::string();
      const auto it = by_key.find(key(fid, iid, sid));
      idx[side] = (it == by_key.end()) ? -1 : it->second;
    }
    if (idx[0] < 0 || idx[1] < 0) continue;
    if (idx[0] == idx[1]) {
      logprintf("Error: Identical sample IDs on line %zu of --king-cutoff-table file.\n", li + 1);
      return kRetInconsistentInput;
    }
    double kin;
    if (!ParseDouble(t[kin_col].c_str(), &kin)) continue;
    if (kin > thresh) {
      table[static_cast<uint64_t>(idx[0]) * wl + idx[1] / 64] |= 1ull << (idx[1] % 64);
      table[static_cast<uint64_t>(idx[1]) * wl + idx[0] / 64] |= 1ull << (idx[0] % 64);
      ++constraint_ct;
    }
  }
  logprintf("--king-cutoff-table: %llu constraint%s loaded.\n", static_cast<unsigned long long>(constraint_ct), constraint_ct == 1 ? "" : "s");
  std::vector<uint8_t>& removed = *removed_out;
  KinshipPrune(&table, n, &removed);
  std::vector<uint32_t> in, out;
  for (uint32_t k = 0; k < n; ++k) (removed[k] ? out : in).push_back(k);
  const std::string in_name = c.out + ".king.cutoff.in.id", out_name = c.out + ".king.cutoff.out.id";
  if (!WriteIdFile(in_name, S, in, true) || !WriteIdFile(out_name, S, out, true)) return kRetWriteFail;
  logprintf("--king-cutoff-table: Excluded sample ID%s written to %s , and %u remaining sample ID%s written to %s .\n", out.size() == 1 ? "" : "s", out_name.c_str(), static_cast<uint32_t>(in.size()), in.size() == 1 ? "" : "s", in_name.c_str());
  return 0;
}

// --king-cutoff <prefix> <threshold> (KingCutoffBatchBinary, 2.0/plink2_matrix_calc.cc:393-640): the relatedness
// prune driven by a matrix written earlier with `--make-king bin[4] triangle`.  <prefix>.king.id names the matrix rows
// (header #FID IID [SID] / #IID [SID], or headerless FID IID / IID lines).  Like the reference, lines whose ID is not
// loaded are dropped BEFORE rows are numbered (:441-460), so the .bin file has to be exactly the triangle over the
// matched IDs - in practice every listed ID must be loaded; loaded samples absent from the file carry no constraint.
// A file without a FID column only matches samples whose FID is 0 (XidRead, plink2_common.cc:1280-1284).
// <prefix>.king.bin holds row i's i leading entries,
// fp64 when the file size says so, else fp32 (compared against the threshold rounded to fp32, :566); a square file is
// refused.  Host-only in the reference too.
int RunKingCutoffBinary(const Cmd& c, Dataset* ds, std::vector<uint8_t>* removed_out) {
  const SampleInfo& S = ds->samples;
  const uint32_t n = S.size();
  const std::string id_name = c.king_cutoff_prefix + ".king.id", bin_name = c.king_cutoff_prefix + ".king.bin";
  std::vector<std::string> lines;
  std::string err;
  if (!ReadLines(id_name, &lines, &err)) {
    logprintf("Error: %s\n", err.c_str());
    return kRetOpenFail;
  }
  size_t li = 0;
  auto is_id_header = [](const std::string& l) { return l.compare(0, 4, "#FID") == 0 || l.compare(0, 4, "#IID") == 0; };
  while (li < lines.size() && (lines[li].empty() || (lines[li][0] == '#' && !is_id_header(lines[li])))) ++li;
  if (li == lines.size()) {
    logprintf("Error: Empty --king-cutoff ID file.\n");
    return kRetMalformedInput;
  }
  bool fid_col = true, sid_col = false, one_or_two = false;
  if (lines[li][0] == '#') {
    const std::vector<std::string> h = SplitWs(lines[li].substr(1));
    size_t t = 0;
    fid_col = h[0] == "FID";
    if (fid_col) ++t;
    if (t >= h.size() || h[t] != "IID") {
      logprintf("Error: No IID column on line %zu of --king-cutoff file.\n", li + 1);
      return kRetMalformedInput;
    }
    ++t;
    sid_col = t < h.size() && h[t] == "SID";
    ++li;
  } else {
    one_or_two = true;  // headerless: "FID IID" lines, or a lone IID (then FID is 0)
  }
  const bool use_sid = sid_col && S.sid_present;
  auto key = [&](const std::string& fid, const std::string& iid, const std::string& sid) {
    std::string k = (fid.empty() ? std::string("0") : fid) + "\t" + iid;
    if (use_sid) k += "\t" + sid;
    return k;
  };
  std::unordered_map<std::string, int64_t> by_key;
  by_key.reserve(static_cast<size_t>(n) * 2);
  for (uint32_t k = 0; k < n; ++k) {
    auto ins = by_key.emplace(key(S.fid[k], S.iid[k], S.sid[k]), k);
    if (!ins.second) ins.first->second = -1;
  }
  // king_to_sample[row of the matrix] = loaded sample index
  std::vector<int64_t> king_to_sample;
  std::vector<uint8_t> seen(n, 0);
  for (; li < lines.size(); ++li) {
    if (lines[li].empty()) continue;
    const std::vector<std::string> t = SplitWs(lines[li]);
    const size_t want = (fid_col && !one_or_two ? 2 : 1) + (sid_col ? 1 : 0);
    if (t.size() < want) {
      logprintf("Error: Fewer tokens than expected on line %zu of %s .\n", li + 1, id_name.c_str());
      return kRetMalformedInput;
    }
    size_t q = 0;
    std::string fid, iid, sid;
    if (one_or_two) {
      if (t.size() >= 2) {
        fid = t[0];
        iid = t[1];
      } else {
        fid = "0";
        iid = t[0];
      }
    } else {
      if (fid_col) fid = t[q++];
      iid = t[q++];
      if (sid_col) sid = t[q++];
    }
    const auto it = by_key.find(key(fid, iid, sid));
    if (it == by_key.end() || it->second < 0) continue;
    if (seen[it->second]) {
      logprintf("Error: Duplicate sample ID \"%s %s\" in %s .\n", fid.empty() ? "0" : fid.c_str(), iid.c_str(), id_name.c_str());
      return kRetMalformedInput;
    }
    seen[it->second] = 1;
    king_to_sample.push_back(it->second);
  }
  const uint64_t kn = king_to_sample.size();
  FILE* f = fopen(bin_name.c_str(), "rb");
  if (!f) {
    logprintf("Error: Failed to open %s : %s.\n", bin_name.c_str(), strerror(errno));
    return kRetOpenFail;
  }
  struct Closer {
    FILE* f;
    ~Closer() { fclose(f); }
  } closer{f};
  if (fseeko(f, 0, SEEK_END)) return kRetReadFail;
  const uint64_t fsize = static_cast<uint64_t>(ftello(f));
  const uint64_t tri = kn ? kn * (kn - 1) / 2 : 0;
  const bool is_double = fsize == tri * 8;
  if (!is_double && fsize != tri * 4) {
    if (fsize == kn * kn * 8 || fsize == kn * kn * 4) {
      logprintf("Error: --king-cutoff currently requires a *triangular* .bin file; the provided\nfile appears to be square.\n");
    } else {
      logprintf("Error: Invalid --king-cutoff .bin file size (expected %llu or %llu bytes).\n", static_cast<unsigned long long>(tri * 4), static_cast<unsigned long long>(tri * 8));
    }
    return kRetMalformedInput;
  }
  const uint32_t wl = (n + 63) / 64;
  std::vector<uint64_t> table(static_cast<uint64_t>(n) * wl, 0);
  const uint32_t esz = is_double ? 8 : 4;
  const float thresh_f = static_cast<float>(c.king_cutoff_prefix_thresh);
  const double thresh_d = c.king_cutoff_prefix_thresh;
  std::vector<unsigned char> row(kn * esz + 8);
  uint64_t constraint_ct = 0;
  rewind(f);
  for (uint64_t i = 1; i < kn; ++i) {
    if (fread(row.data(), i * esz, 1, f) != 1) {
      logprintf("Error: %s read failure.\n", bin_name.c_str());
      return kRetReadFail;
    }
    const uint64_t si = static_cast<uint64_t>(king_to_sample[i]);
    const float* rf = reinterpret_cast<const float*>(row.data());
    const double* rd = reinterpret_cast<const double*>(row.data());
    for (uint64_t j = 0; j < i; ++j) {
      if (is_double ? (rd[j] > thresh_d) : (rf[j] > thresh_f)) {
        const uint64_t sj = static_cast<uint64_t>(king_to_sample[j]);
        table[si * wl + sj / 64] |= 1ull << (sj % 64);
        table[sj * wl + si / 64] |= 1ull << (si % 64);
        ++constraint_ct;
      }
    }
  }
  logprintf("--king-cutoff: %llu constraint%s loaded.\n", static_cast<unsigned long long>(constraint_ct), constraint_ct == 1 ? "" : "s");
  std::vector<uint8_t>& removed = *removed_out;
  KinshipPrune(&table, n, &removed);
  std::vector<uint32_t> in, out;
  for (uint32_t k = 0; k < n; ++k) (removed[k] ? out : in).push_back(k);
  const std::string in_name = c.out + ".king.cutoff.in.id", out_name = c.out + ".king.cutoff.out.id";
  if (!WriteIdFile(in_name, S, in, true) || !WriteIdFile(out_name, S, out, true)) return kRetWriteFail;
  logprintf("--king-cutoff: Excluded sample ID%s written to %s , and %u remaining sample ID%s written to %s .\n", out.size() == 1 ? "" : "s", out_name.c_str(), static_cast<uint32_t>(in.size()), in.size() == 1 ? "" : "s", in_name.c_str());
  return 0;
}

// ------------------------------------------------------------------------------------------ GRM
// ComputeAlleleFreqs over founders (plink2.cc:2301, plink2_filter.cc:2113-2151).  Returns false
// when every sample is a founder (the library then derives the same numbers from each block).
// --read-freq (ReadAlleleFreqs, 2.0/plink2_filter.cc:2242-3300): the PLINK 2 --freq report form (ID, REF, ALT,
// ALT_FREQS columns), biallelic lines.  A line whose REF/ALT are the dataset's ALT/REF gives the dataset's REF
// frequency directly (:3187-3192); unknown IDs, foreign allele codes and nan entries are skipped with the reference's
// warning; OBS_CT is not consulted for frequency columns (:3170-3175).  Variants without an entry keep the
// frequency computed from the data.
int LoadReadFreq(const Cmd& c, Dataset* ds) {
  const VariantInfo& V = ds->variants;
  std::vector<std::string> lines;
  std::string err;
  if (!ReadLines(c.read_freq, &lines, &err)) {
    logprintf("Error: %s\n", err.c_str());
    return kRetOpenFail;
  }
  size_t li = 0;
  while (li < lines.size() && lines[li].size() >= 2 && lines[li][0] == '#' && lines[li][1] == '#') ++li;
  if (li == lines.size()) {
    logprintf("Error: Empty --read-freq file.\n");
    return kRetMalformedInput;
  }
  int col_id = -1, col_ref = -1, col_alt = -1, col_af = -1;
  {
    std::string h = lines[li];
    if (h.empty() || h[0] != '#') {
      logprintf("Error: Unrecognized header line in --read-freq file (plink2_b200 reads PLINK 2 --freq reports only).\n");
      return kRetMalformedInput;
    }
    const std::vector<std::string> hdr = SplitWs(h.substr(1));
    for (size_t k = 0; k < hdr.size(); ++k) {
      if (hdr[k] == "ID") col_id = static_cast<int>(k);
      else if (hdr[k] == "REF") col_ref = static_cast<int>(k);
      else if (hdr[k] == "ALT" || hdr[k] == "ALT1") col_alt = static_cast<int>(k);
      else if (hdr[k] == "ALT_FREQS" || hdr[k] == "ALT1_FREQ") col_af = static_cast<int>(k);
    }
    if (col_id < 0 || col_ref < 0 || col_alt < 0) {
      logprintf("Error: Missing column(s) in --read-freq file (ID, REF, ALT[1] required).\n");
      return kRetMalformedInput;
    }
    if (col_af < 0) {
      logprintf("Error: --read-freq files without an ALT_FREQS column (count / PLINK 1.x formats) are not supported by plink2_b200.\n");
      return kRetNotYetSupported;
    }
    ++li;
  }
  logprintf("--read-freq: PLINK 2 --freq file detected.\n");
  std::unordered_map<std::string, uint32_t> by_id;
  std::unordered_map<std::string, uint32_t> dup;
  by_id.reserve(static_cast<size_t>(V.size()) * 2);
  for (uint32_t v = 0; v < V.size(); ++v) {
    if (!by_id.emplace(V.id[v], v).second) dup.emplace(V.id[v], v);
  }
  ds->read_ref_freq.assign(V.size(), std::numeric_limits<double>::quiet_NaN());
  std::vector<uint8_t> seen(V.size(), 0);
  const int need_cols = std::max(std::max(col_id, col_ref), std::max(col_alt, col_af));
  uint64_t loaded = 0, skipped = 0;
  for (; li < lines.size(); ++li) {
    if (lines[li].empty()) continue;
    const std::vector<std::string> t = SplitWs(lines[li]);
    if (static_cast<int>(t.size()) <= need_cols) {
      logprintf("Error: Line %zu of --read-freq file has fewer tokens than expected.\n", li + 1);
      return kRetMalformedInput;
    }
    const auto it = by_id.find(t[col_id]);
    if (it == by_id.end()) {
      ++skipped;
      continue;
    }
    if (dup.count(t[col_id])) {
      logprintf("Error: --read-freq variant ID '%s' appears multiple times in main dataset.\n", t[col_id].c_str());
      return kRetMalformedInput;
    }
    const uint32_t v = it->second;
    if (seen[v]) {
      logprintf("Error: Variant ID '%s' appears multiple times in --read-freq file.\n", t[col_id].c_str());
      return kRetMalformedInput;
    }
    seen[v] = 1;
    const bool same = t[col_ref] == V.ref[v] && t[col_alt] == V.alt[v];
    const bool swapped = t[col_ref] == V.alt[v] && t[col_alt] == V.ref[v];
    double af;
    const std::string& afs = t[col_af];
    if (!ParseDouble(afs.c_str(), &af) || af != af) {
      if (afs == "nan" || afs == "NaN" || afs == "NA" || af != af) {
        ++skipped;
        continue;
      }
      logprintf("Error: Invalid frequencies/counts on line %zu of --read-freq file.\n", li + 1);
      return kRetMalformedInput;
    }
    if (!same && !swapped) {
      ++skipped;
      continue;
    }
    if (af < 0.0 || af > 1.0 * (1 + 1.0 / 17592186044416.0) / 0.99) {
      logprintf("Error: Invalid frequencies/counts on line %zu of --read-freq file.\n", li + 1);
      return kRetMalformedInput;
    }
    if (af > 1.0) af = 1.0;
    ds->read_ref_freq[v] = same ? (1.0 - af) : af;
    ++loaded;
  }
  logprintf("--read-freq: Frequencies for %llu variant%s loaded.\n", static_cast<unsigned long long>(loaded), loaded == 1 ? "" : "s");
  if (skipped) logprintf("Warning: %llu entr%s skipped due to missing variant IDs, mismatching allele codes, and/or zero observations.\n", static_cast<unsigned long long>(skipped), skipped == 1 ? "y" : "ies");
  return 0;
}

// loaded --read-freq values take precedence over the frequencies computed from the data; a NaN entry tells the
// library to compute that variant's frequency from the block it is given
bool ApplyReadFreq(const Dataset& ds, const std::vector<uint32_t>& vidx, std::vector<double>* ref_freqs, bool have_freqs) {
  if (ds.read_ref_freq.empty()) return have_freqs;
  if (!have_freqs) ref_freqs->assign(vidx.size(), std::numeric_limits<double>::quiet_NaN());
  for (size_t k = 0; k < vidx.size(); ++k) {
    const double f = ds.read_ref_freq[vidx[k]];
    if (f == f) (*ref_freqs)[k] = f;
  }
  return true;
}

bool FounderRefFreqs(Dataset* ds, Pl2GpuCtx* ctx, const std::vector<uint32_t>& vidx, std::vector<double>* ref_freqs, int* rc, bool force = false) {
  const SampleInfo& S = ds->samples;
  const uint32_t n = S.size();
  uint32_t founder_ct = 0;
  for (uint32_t k = 0; k < n; ++k) founder_ct += S.is_founder[k];
  *rc = 0;
  if (founder_ct == n && !force) return false;
  ref_freqs->assign(vidx.size(), 0.5);
  if (!founder_ct) return true;
  std::vector<uint64_t> inc((n + 63) / 64, 0);
  for (uint32_t k = 0; k < n; ++k)
    if (S.is_founder[k]) inc[k / 64] |= 1ull << (k % 64);
  BlockStreamer bs(ds, &vidx, founder_ct, 16384);
  if (founder_ct != n) bs.sample_include = inc.data();
  if (!bs.Init()) {
    *rc = GpuFail("pl2gpu_host_alloc");
    return true;
  }
  std::vector<uint32_t> counts(4ull * 16384);
  std::string err;
  size_t base = 0;
  for (;;) {
    const int got = bs.Next(&err);
    if (got < 0) {
      logprintf("Error: %s\n", err.c_str());
      *rc = kRetMalformedInput;
      return true;
    }
    if (!got) break;
    if (pl2gpu_geno_counts(ctx, bs.buf, static_cast<uint64_t>(bs.words) * 8, founder_ct, static_cast<uint32_t>(got), 0, counts.data())) {
      *rc = GpuFail("pl2gpu_geno_counts");
      return true;
    }
    for (int v = 0; v < got; ++v) {
      const uint64_t n0 = counts[4ull * v], n1 = counts[4ull * v + 1], n2 = counts[4ull * v + 2];
      const uint64_t tot = 2 * (n0 + n1 + n2);
      (*ref_freqs)[base + v] = tot ? static_cast<double>(2 * n0 + n1) * (1.0 / static_cast<double>(tot)) : 0.5;
    }
    base += static_cast<size_t>(got);
  }
  return true;
}

int RunGrm(const Cmd& c, Dataset* ds, Pl2GpuCtx* ctx, bool keep_for_pca, GrmJob* kept_job) {
  const SampleInfo& S = ds->samples;
  const uint32_t n = S.size();
  std::vector<uint32_t> vidx;
  const int vrc = RelationshipVariants(*ds, "GRM construction", &vidx);
  if (vrc) return vrc;
  uint32_t r0, r1;
  ParallelBounds(n, 0, c.parallel_idx, c.parallel_tot, &r0, &r1);
  std::vector<double> ref_freqs;
  int rc = 0;
  bool have_freqs = FounderRefFreqs(ds, ctx, vidx, &ref_freqs, &rc);
  if (rc) return rc;
  have_freqs = ApplyReadFreq(*ds, vidx, &ref_freqs, have_freqs);
  const int flags = (c.grm_cov ? kPl2GrmCov : 0) | ((c.grm_meanimpute || (keep_for_pca && c.pca_meanimpute && !c.make_grm_bin && !c.make_grm_list && !c.make_grm_sparse && !c.make_rel)) ? kPl2GrmMeanimpute : 0);
  // multi-GPU team (--gpus): rows [r0, r1) in one tile-aligned slab per device (CalcGrm's own row split is
  // TriangleFill2 over threads, 2.0/plink2_matrix_calc.cc:4596); exact --pca needs the whole matrix on one device
  GpuTeam team;
  {
    uint32_t gpus_eff = std::max(1u, std::min(c.gpus, (r1 - r0) / 512));
    if (keep_for_pca) gpus_eff = 1;
    if (gpus_eff < c.gpus) logprintf("Note: GRM computed on %u GPU%s (--gpus %u%s).\n", gpus_eff, gpus_eff == 1 ? "" : "s", c.gpus, keep_for_pca ? "; non-approximate --pca keeps the matrix on one device" : "");
    const int trc = TeamInit(ctx, c.device, gpus_eff, &team);
    if (trc) return trc;
  }
  const uint32_t G = team.size();
  const std::vector<uint32_t> sbounds = TileAlignedBounds(r0, r1, G, true);
  std::vector<GrmJob> jobs(G);
  for (uint32_t g = 0; g < G; ++g) {
    Pl2GrmJob* job = nullptr;
    if (pl2gpu_grm_begin(team.ctx[g], n, sbounds[g], sbounds[g + 1], flags, &job)) return GpuFail("pl2gpu_grm_begin");
    jobs[g].reset(job);
  }
  BlockStreamer bs(ds, &vidx, n, 32768, G);
  if (!bs.Init()) return GpuFail("pl2gpu_host_alloc");
  logprintf("Constructing GRM: ");
  size_t base = 0;
  rc = StreamBlocks(&bs, [&](uint32_t got) -> int {
    int arc;
    std::string gerr;
    const double* batch_freqs = have_freqs ? ref_freqs.data() + base : nullptr;
    if (G == 1) {
      arc = pl2gpu_grm_add_variants(jobs[0].get(), bs.buf, static_cast<uint64_t>(bs.words) * 8, got, 0, batch_freqs);
      if (arc) gerr = pl2gpu_last_error();
    } else {
      arc = AddSharded(&bs, got, G, [&](uint32_t g, const uint64_t* slice, uint32_t per) { return pl2gpu_grm_add_variants_sharded(jobs[g].get(), slice, static_cast<uint64_t>(bs.words) * 8, per, got, 0, batch_freqs); }, &gerr);
    }
    if (arc) {
      logprintf("\nError: %s\n", gerr.c_str());
      return arc == 2 ? kRetDegenerateData : kRetGpuFail;
    }
    base += got;
    printf("\rConstructing GRM: %u%%", static_cast<uint32_t>(base * 100 / vidx.size()));
    fflush(stdout);
    return 0;
  });
  if (rc) return rc;
  printf("\r");
  logprintf("Constructing GRM: done.\n");
  // writers: f(j, g, obs) for rows j of [r0, r1) in order, with row j's values and observation counts; fetched in
  // chunks of rows that never straddle two devices' slabs
  const uint64_t stride = r1;
  const uint64_t max_rows = std::max<uint64_t>(1, (384ull << 20) / (stride * 12));
  std::vector<double> g;
  std::vector<float> obs;
  auto for_each_row = [&](auto&& f) -> int {
    for (uint32_t a = r0, sg = 0; a < r1;) {
      while (a >= sbounds[sg + 1]) ++sg;
      const uint32_t b = static_cast<uint32_t>(std::min<uint64_t>(a + max_rows, sbounds[sg + 1]));
      g.assign(static_cast<uint64_t>(b - a) * stride, 0.0);
      obs.assign(static_cast<uint64_t>(b - a) * stride, 0.0f);
      if (pl2gpu_grm_get_rows(jobs[sg].get(), a, b, g.data(), obs.data(), stride, 0)) return GpuFail("pl2gpu_grm_get_rows");
      for (uint32_t j = a; j < b; ++j) f(j, &g[static_cast<uint64_t>(j - a) * stride], &obs[static_cast<uint64_t>(j - a) * stride]);
      a = b;
    }
    return 0;
  };
  // "<msg> ." in the log, with " , and IDs to <idname>" after the first --parallel piece has written that file
  auto report = [&](std::string msg, const std::string& idname, bool header) -> int {
    if (!c.parallel_idx) {
      if (!WriteAllIds(idname, S, header)) return kRetWriteFail;
      msg += " , and IDs to " + idname;
    }
    logprintf("%s .\n", msg.c_str());
    return 0;
  };
  const std::string piece = c.parallel_tot != 1 ? "component " : "";
  if (c.make_grm_bin) {
    const std::string gname = PieceName(c.out + ".grm.bin", c), nname = PieceName(c.out + ".grm.N.bin", c);
    OutFile fg, fn;
    if (!fg.Open(gname) || !fn.Open(nname)) return kRetOpenFail;
    TriangleMatrixWriter gmat(&fg, n, Cmd::kTri, Cmd::kBin4, true);
    rc = for_each_row([&](uint32_t j, const double* gr, const float* orow) {
      gmat.Row(j, gr, gr[j]);
      fn.Write(orow, sizeof(float) * (j + 1));
    });
    if (rc) return rc;
    if (!fg.Close() || !fn.Close()) return kRetWriteFail;
    rc = report("--make-grm-bin: GRM " + piece + "written to " + gname + " , observation counts to " + nname, c.out + ".grm.id", c.grm_id_header);
    if (rc) return rc;
  }
  if (c.make_grm_list) {
    // `.grm`: one line per pair i <= j, "j+1 <tab> i+1 <tab> observation count <tab> value" (2.0/plink2_matrix_calc.cc:5082-5106)
    const std::string gname = PieceName(c.out + ".grm", c) + (c.grm_zs ? ".zst" : "");
    OutFile fg;
    if (!fg.Open(gname, c.grm_zs)) return kRetOpenFail;
    std::string line;
    char num[64];
    rc = for_each_row([&](uint32_t j, const double* gr, const float* orow) {
      line.clear();
      for (uint32_t i = 0; i <= j; ++i) {
        line.append(num, u32toa(j + 1, num) - num);
        line.push_back('\t');
        line.append(num, u32toa(i + 1, num) - num);
        line.push_back('\t');
        line.append(num, u32toa(static_cast<uint32_t>(orow[i]), num) - num);
        line.push_back('\t');
        line.append(num, dtoa_g(gr[i], num) - num);
        line.push_back('\n');
      }
      fg.Write(line.data(), line.size());
    });
    if (rc) return rc;
    if (!fg.Close()) return kRetWriteFail;
    rc = report("--make-grm-list: GRM " + piece + "written to " + gname, c.out + ".grm.id", c.grm_id_header);
    if (rc) return rc;
  }
  if (c.make_grm_sparse) {
    // `.grm.sp` (GCTA sparse GRM): "j <tab> i <tab> value" (0-based, 8 significant digits) for every i <= j whose
    // value is not below the cutoff (2.0/plink2_matrix_calc.cc:5064-5081)
    const std::string gname = PieceName(c.out + ".grm.sp", c) + (c.grm_zs ? ".zst" : "");
    OutFile fg;
    if (!fg.Open(gname, c.grm_zs)) return kRetOpenFail;
    rc = for_each_row([&](uint32_t j, const double* gr, const float*) {
      for (uint32_t i = 0; i <= j; ++i) {
        if (gr[i] < c.grm_sparse_cutoff) continue;
        char* w = fg.Reserve(64);
        w = u32toa(j, w);
        *w++ = '\t';
        w = u32toa(i, w);
        *w++ = '\t';
        w = dtoa_g_p8(gr[i], w);
        *w++ = '\n';
        fg.Advance(w);
      }
    });
    if (rc) return rc;
    if (!fg.Close()) return kRetWriteFail;
    rc = report("--make-grm-sparse: GRM " + piece + "written to " + gname, c.out + ".grm.id", c.grm_id_header);
    if (rc) return rc;
  }
  if (c.make_rel) {
    const std::string base_name = c.out + (c.rel_enc == Cmd::kText ? ".rel" : ".rel.bin");
    const bool rel_zs = c.rel_zs && c.rel_enc == Cmd::kText;
    const std::string rname = PieceName(base_name, c) + (rel_zs ? ".zst" : "");
    if (c.rel_shape == Cmd::kSq && c.parallel_tot != 1) {
      logprintf("Error: --make-rel square output cannot be combined with --parallel; use square0 or triangle.\n");
      return kRetInvalidCmdline;
    }
    OutFile fr;
    if (!fr.Open(rname, rel_zs)) return kRetOpenFail;
    TriangleMatrixWriter mat(&fr, n, c.rel_shape, c.rel_enc, true);
    rc = for_each_row([&](uint32_t j, const double* gr, const float*) { mat.Row(j, gr, gr[j]); });
    if (rc) return rc;
    mat.Finish();
    if (!fr.Close()) return kRetWriteFail;
    rc = report("--make-rel: GRM " + piece + "written to " + rname, c.out + ".rel.id", true);
    if (rc) return rc;
  }
  if (keep_for_pca) *kept_job = std::move(jobs[0]);  // G == 1 in that case
  return 0;
}

// ------------------------------------------------------------------------------------------ PCA
int RunPca(const Cmd& c, Dataset* ds, Pl2GpuCtx* ctx, Pl2GrmJob* grm_job) {
  const SampleInfo& S = ds->samples;
  const uint32_t n = S.size();
  uint32_t pc_ct = c.pc_ct;
  if (pc_ct > n) {
    logprintf("Warning: calculating %u PCs, since there are only %u samples.\n", n, n);
    pc_ct = n;
  }
  std::vector<double> eigvals(pc_ct), eigvecs(static_cast<uint64_t>(pc_ct) * n);
  if (!c.pca_approx) {
    // exact: top eigenpairs of the GRM already accumulated on the device (CalcPca :5942-6040)
    logprintf("Extracting eigenvalue%s and eigenvector%s... ", pc_ct == 1 ? "" : "s", pc_ct == 1 ? "" : "s");
    if (pl2gpu_grm_eigen_topk(grm_job, pc_ct, eigvals.data(), eigvecs.data())) {
      logprintf("\n");
      return GpuFail("pl2gpu_grm_eigen_topk");
    }
    logprintf("done.\n");
  } else {
    // approx (:5697-5941)
    if (n <= 5000) logprintf("Warning: \"--pca approx\" is only recommended for analysis of >5000 samples.\n");
    std::vector<uint32_t> vidx;
    for (uint32_t v = 0; v < ds->variants.size(); ++v)
      if (KeptForRelationship(ds->variants.chr_code[v])) vidx.push_back(v);
    const uint64_t q = 2ull * pc_ct * (pc_ct + 1);
    if (q > vidx.size()) {
      logprintf("Error: Too few variants to compute %u PCs with \"--pca approx\" (%llu required).\n", pc_ct, static_cast<unsigned long long>(q));
      return kRetDegenerateData;
    }
    std::vector<double> ref_freqs;
    int rc = 0;
    bool have_freqs = FounderRefFreqs(ds, ctx, vidx, &ref_freqs, &rc);
    if (rc) return rc;
    have_freqs = ApplyReadFreq(*ds, vidx, &ref_freqs, have_freqs);
    // --gpus G: contiguous variant shards, one per device (sizes multiple of 128 so every shard tiles evenly); the
    // library completes the cross-shard sums with all-reduces (pl2gpu_pca_run_sharded)
    GpuTeam team;
    {
      const uint32_t gpus_eff = std::max(1u, std::min<uint32_t>(c.gpus, static_cast<uint32_t>(vidx.size() / std::max<uint64_t>(q, 4096))));
      if (gpus_eff < c.gpus) logprintf("Note: --pca approx on %u GPU%s (--gpus %u): too few variants per shard otherwise.\n", gpus_eff, gpus_eff == 1 ? "" : "s", c.gpus);
      const int trc = TeamInit(ctx, c.device, gpus_eff, &team);
      if (trc) return trc;
    }
    const uint32_t G = team.size();
    const uint32_t shard = static_cast<uint32_t>(((vidx.size() + G - 1) / G + 127) / 128 * 128);
    std::vector<PcaJob> jobs(G);
    for (uint32_t r = 0; r < G; ++r) {
      const size_t s0 = std::min<size_t>(vidx.size(), static_cast<size_t>(r) * shard), s1 = std::min<size_t>(vidx.size(), s0 + shard);
      if (s0 == s1) {
        logprintf("Error: --gpus %u leaves a device without variants.\n", G);
        return kRetInvalidCmdline;
      }
      Pl2PcaJob* job = nullptr;
      rc = G == 1 ? pl2gpu_pca_begin(team.ctx[r], n, static_cast<uint32_t>(vidx.size()), pc_ct, &job) : pl2gpu_pca_begin_shard(team.ctx[r], n, static_cast<uint32_t>(s1 - s0), pc_ct, &job);
      jobs[r].reset(job);
      if (rc) {
        logprintf("Error: %s\n", pl2gpu_last_error());
        return rc == 2 ? kRetDegenerateData : kRetGpuFail;
      }
      std::vector<uint32_t> sub(vidx.begin() + s0, vidx.begin() + s1);
      BlockStreamer bs(ds, &sub, n, 32768);
      if (!bs.Init()) return GpuFail("pl2gpu_host_alloc");
      std::string err;
      size_t base = s0;
      for (;;) {
        const int got = bs.Next(&err);
        if (got < 0) {
          logprintf("Error: %s\n", err.c_str());
          return kRetMalformedInput;
        }
        if (!got) break;
        const int arc = pl2gpu_pca_add_variants(jobs[r].get(), bs.buf, static_cast<uint64_t>(bs.words) * 8, static_cast<uint32_t>(got), 0, have_freqs ? ref_freqs.data() + base : nullptr);
        if (arc) {
          logprintf("Error: %s\n", pl2gpu_last_error());
          return arc == 2 ? kRetDegenerateData : kRetGpuFail;
        }
        base += static_cast<size_t>(got);
      }
    }
    // Gaussian start: the reference's main SFMT stream (seeded by --seed, else by time) sliced over
    // min(--threads, ceil(N*k / 262144)) Box-Muller streams (FillGaussianDArr, plink2_random.cc:89)
    Sfmt19937 rng;
    const uint32_t seed = c.seed_given ? static_cast<uint32_t>(c.seed) : static_cast<uint32_t>(time(nullptr));
    if (!c.seed_given) logprintf("Random number seed: %u\n", seed);
    rng.InitGenRand(seed);
    std::vector<double> g1(static_cast<uint64_t>(n) * 2 * pc_ct);
    FillGaussian(static_cast<uint64_t>(n) * pc_ct, c.threads ? c.threads : 1, &rng, g1.data());
    logprintf("Projecting random vectors, computing SVD of Krylov matrix, recovering top PCs... ");
    if (G == 1) {
      if (pl2gpu_pca_run(jobs[0].get(), g1.data(), eigvals.data(), eigvecs.data())) {
        logprintf("\nError: %s\n", pl2gpu_last_error());
        return kRetGpuFail;
      }
    } else {
      // collective: one host thread per rank; every rank returns the same result, rank 0's is kept
      std::vector<std::vector<double>> vals(G, std::vector<double>(pc_ct)), vecs(G);
      for (uint32_t r = 1; r < G; ++r) vecs[r].resize(static_cast<uint64_t>(pc_ct) * n);
      std::string errtext;
      const int prc = ForEachRank(G, [&](uint32_t r) { return pl2gpu_pca_run_sharded(jobs[r].get(), g1.data(), vidx.size(), r ? vals[r].data() : eigvals.data(), r ? vecs[r].data() : eigvecs.data()); }, &errtext);
      if (prc) {
        logprintf("\nError: %s\n", errtext.c_str());
        return kRetGpuFail;
      }
    }
    logprintf("done.\n");
  }
  if (!WriteEigen(c.out, S, pc_ct, eigvals.data(), eigvecs.data())) {
    logprintf("Error: File write failure.\n");
    return kRetWriteFail;
  }
  logprintf("--pca: Eigenvector%s written to %s.eigenvec , and eigenvalue%s written to %s.eigenval .\n", pc_ct == 1 ? "" : "s", c.out.c_str(), pc_ct == 1 ? "" : "s", c.out.c_str());
  return 0;
}

// ---------------------------------------------------------------------------------------- --score
// One phenotype column as the report prints it (LoadPsam typing, 2.0/plink2_psam.cc:58: every value in
// {-9, 0, 1, 2, NA} -> case/control with 0 / -9 / NA missing; other numbers -> quantitative with -9 / NA missing;
// anything non-numeric -> categorical).  A column without a single nonmissing value is not a phenotype
// ("No phenotype data present").
struct PhenoOut {
  std::string name;
  std::vector<std::string> text;  // per sample
  bool categorical = false;
};
bool TypePheno(const std::string& name, const std::vector<std::string>& tok, PhenoOut* out) {
  const size_t n = tok.size();
  std::vector<double> val(n, 0.0);
  std::vector<uint8_t> is_na(n, 0);
  bool numeric = true, binary = true;
  for (size_t k = 0; k < n && numeric; ++k) {
    const std::string& t = tok[k];
    if (t == "NA" || t == "nan" || t == "NaN" || t == "na") {
      is_na[k] = 1;
      continue;
    }
    double d;
    if (!ParseDouble(t.c_str(), &d)) {
      numeric = false;
      break;
    }
    val[k] = d;
    if (!(d == -9 || d == 0 || d == 1 || d == 2)) binary = false;
  }
  out->name = name;
  out->categorical = !numeric;
  out->text.assign(n, "NA");
  bool any = false;
  char buf[32];
  if (!numeric) {
    for (size_t k = 0; k < n; ++k) {
      const bool miss = tok[k] == "NA" || tok[k] == "NONE" || tok[k] == "nan";
      out->text[k] = miss ? "NONE" : tok[k];
      any = any || !miss;
    }
    return any;
  }
  for (size_t k = 0; k < n; ++k) {
    if (is_na[k] || val[k] == -9 || (binary && val[k] == 0)) continue;
    any = true;
    if (binary) {
      out->text[k] = val[k] == 1 ? "1" : "2";
    } else {
      *dtoa_g(val[k], buf) = '\0';
      out->text[k] = buf;
    }
  }
  return any;
}

std::vector<uint32_t> AllVariants(const Dataset& ds) {
  std::vector<uint32_t> vidx(ds.variants.size());
  for (uint32_t v = 0; v < vidx.size(); ++v) vidx[v] = v;
  return vidx;
}
int SexChrRefFreqs(Dataset* ds, Pl2GpuCtx* ctx, const std::vector<uint32_t>& vidx, std::vector<double>* ref_freqs);

// --q-score-range (ScoreReport, 2.0/plink2_matrix_calc.cc:6960-7170).  Range file: name, lower and upper bound per
// line; lines without two numeric bounds are skipped.  Data file: a variant ID and a p-value per line, from columns
// qsr_id_col / qsr_val_col.  Lines whose ID is not in the dataset, or is duplicated there, are skipped and counted; NA
// p-values are skipped silently.  A variant lies in a range when lb <= p <= ub.  Line numbers count nonempty lines.
struct QsrRange {
  std::string name;
  double lb, ub;
};
// the 'NA' / 'nan' tokens (any case) the reference tolerates as p-values (IsNanStr)
bool QsrNaToken(const std::string& t) {
  if (t.size() != 2 && t.size() != 3) return false;
  if ((t[0] | 0x20) != 'n' || (t[1] | 0x20) != 'a') return false;
  return t.size() == 2 || (t[2] | 0x20) == 'n';
}
int LoadQsr(const Cmd& c, const VariantInfo& V, const std::unordered_map<std::string, uint32_t>& by_id, const std::unordered_map<std::string, uint32_t>& dup, std::vector<QsrRange>* ranges, std::vector<double>* pval,
            std::vector<uint8_t>* seen) {
  std::vector<std::string> lines;
  std::string err;
  if (!ReadLines(c.qsr_range_file, &lines, &err)) {
    logprintf("Error: %s\n", err.c_str());
    return kRetOpenFail;
  }
  size_t line_idx = 0;
  for (const std::string& ln : lines) {
    const std::vector<std::string> t = SplitWs(ln);
    if (t.empty()) continue;
    ++line_idx;
    double lb, ub;
    if (t.size() < 3 || !ParseDouble(t[1].c_str(), &lb) || !ParseDouble(t[2].c_str(), &ub)) continue;
    if (lb > ub) {
      logprintf("Error: Upper bound < lower bound on line %zu of --q-score-range range file.\n", line_idx);
      return kRetMalformedInput;
    }
    ranges->push_back({t[0], lb, ub});
  }
  if (ranges->empty()) {
    logprintf("Error: Empty --q-score-range range file.\n");
    return kRetInconsistentInput;
  }
  lines.clear();
  if (!ReadLines(c.qsr_data_file, &lines, &err)) {
    logprintf("Error: %s\n", err.c_str());
    return kRetOpenFail;
  }
  pval->assign(V.size(), 0.0);
  seen->assign(V.size(), 0);
  line_idx = 0;
  bool header = c.qsr_header;
  uint64_t miss_ct = 0;
  uint32_t loaded = 0;
  const uint32_t need = std::max(c.qsr_id_col, c.qsr_val_col);
  for (const std::string& ln : lines) {
    const std::vector<std::string> t = SplitWs(ln);
    if (t.empty()) continue;
    ++line_idx;
    if (header) {
      header = false;
      continue;
    }
    if (t.size() < need) {
      logprintf("Error: Line %zu of --q-score-range data file has fewer tokens than expected.\n", line_idx);
      return kRetInconsistentInput;
    }
    const std::string& id = t[c.qsr_id_col - 1];
    const auto it = by_id.find(id);
    if (it == by_id.end() || dup.count(id)) {
      ++miss_ct;
      continue;
    }
    const std::string& val = t[c.qsr_val_col - 1];
    double p;
    if (QsrNaToken(val)) continue;
    if (!ParseDouble(val.c_str(), &p)) {
      logprintf("Error: Invalid value '%s' on line %zu of --q-score-range data file.\n", val.c_str(), line_idx);
      return kRetMalformedInput;
    }
    const uint32_t v = it->second;
    if ((*seen)[v]) {
      if (!c.qsr_min) {
        logprintf("Error: Duplicate variant ID '%s' in --q-score-range data file. (Add the 'min' modifier if this is a multiallelic variant that you want to use the minimum p-value for.)\n", id.c_str());
        return kRetMalformedInput;
      }
      if ((*pval)[v] <= p) continue;
    } else {
      ++loaded;
    }
    (*seen)[v] = 1;
    (*pval)[v] = p;
  }
  if (c.qsr_header && line_idx == 0) {
    logprintf("Error: Empty --q-score-range data file.\n");
    return kRetMalformedInput;
  }
  if (!loaded) {
    logprintf("Error: No valid entries in --q-score-range data file.\n");
    return kRetInconsistentInput;
  }
  logprintf("--q-score-range: %zu range%s and %u variant%s loaded.\n", ranges->size(), ranges->size() == 1 ? "" : "s", loaded, loaded == 1 ? "" : "s");
  if (miss_ct) logprintf("Warning: %llu line%s skipped in --q-score-range data file.\n", static_cast<unsigned long long>(miss_ct), miss_ct == 1 ? "" : "s");
  return 0;
}

// --score-list (ScoreListLoad, 2.0/plink2_matrix_calc.cc:6332): the first token of each line names a score file, as
// written; like the reference, the list ends at its first line without a token.
int LoadScoreList(const std::string& list, std::vector<std::string>* files) {
  std::vector<std::string> lines;
  std::string err;
  if (!ReadLines(list, &lines, &err)) {
    logprintf("Error: %s\n", err.c_str());
    return kRetOpenFail;
  }
  for (const std::string& ln : lines) {
    const std::vector<std::string> t = SplitWs(ln);
    if (t.empty()) break;
    files->push_back(t[0]);
  }
  if (files->empty()) {
    logprintf("Error: --score-list: %s is empty.\n", list.c_str());
    return kRetMalformedInput;
  }
  return 0;
}

// `--score` and `--score-list` (ScoreReport, 2.0/plink2_matrix_calc.cc:6892-9270) for hard calls: default report
// columns plus denom / scoresums, 'header' / 'header-read', 'no-mean-imputation', 'ignore-dup-ids', and any number of
// coefficient columns (--score-col-nums).  chrX, chrY and MT entries are scored with the reference's sex-dependent
// ploidy (--xchr-model 2: chrX like an autosome; 1: chrX males haploid).  The per-sample sums of every column come from
// one device pass (pl2gpu_score_*); the file parsing, allele matching, mean-imputation weights and the report are here.
// Each file of a --score-list has its own score columns and its own denominators (:7324, :8389): its entries form
// classes of their own, and a variant several files score is staged once and gathered once per entry on the device.
int RunScore(const Cmd& c, Dataset* ds, Pl2GpuCtx* ctx) {
  const SampleInfo& S = ds->samples;
  const VariantInfo& V = ds->variants;
  const uint32_t n = S.size();
  const char* flagname = c.score_list ? "--score-list" : "--score";
  std::vector<std::string> files;
  std::vector<std::string> lines;
  std::string err;
  if (c.score_list) {
    if (int rc = LoadScoreList(c.score_file, &files)) return rc;
  } else {
    files.push_back(c.score_file);
    if (!ReadLines(c.score_file, &lines, &err)) {
      logprintf("Error: %s\n", err.c_str());
      return kRetOpenFail;
    }
  }
  const uint32_t file_ct = static_cast<uint32_t>(files.size());
  std::unordered_map<std::string, uint32_t> by_id;
  std::unordered_map<std::string, uint32_t> dup;
  by_id.reserve(static_cast<size_t>(V.size()) * 2);
  for (uint32_t v = 0; v < V.size(); ++v)
    if (!by_id.emplace(V.id[v], v).second) dup.emplace(V.id[v], v);
  // --q-score-range: the ranges and the data file's p-values, read before the score file as the reference does
  const bool qsr = !c.qsr_range_file.empty();
  std::vector<QsrRange> ranges;
  std::vector<double> qsr_p;
  std::vector<uint8_t> qsr_seen;
  if (qsr) {
    if (int rc = LoadQsr(c, V, by_id, dup, &ranges, &qsr_p, &qsr_seen)) return rc;
  }
  struct Entry {
    uint32_t v;
    uint8_t aidx;  // 0 = REF named, 1 = ALT named
    size_t coef_row;  // coefficients at coefs[coef_row * score_ct ...]
    uint32_t file;    // index in the --score-list (0 for --score)
  };
  std::vector<Entry> entries;
  std::vector<double> coefs;
  std::vector<uint8_t> seen;
  const bool y_prohibited = !c.score_no_meanimpute && std::find(S.sex.begin(), S.sex.end(), 0) != S.sex.end();
  // coefficient columns in file order (1-based); without --score-col-nums the one column --score names
  const std::vector<uint32_t> score_cols = c.score_col_nums.empty() ? std::vector<uint32_t>{c.score_coef_col} : c.score_col_nums;
  const uint32_t score_ct = static_cast<uint32_t>(score_cols.size());
  const uint32_t need_cols = std::max({c.score_id_col, c.score_allele_col, score_cols.back()});
  // names, file by file: the header tokens with 'header-read', else SCORE1 .. by position in all the files' columns
  // (:7620-7672)
  std::vector<std::string> score_names(static_cast<size_t>(file_ct) * score_ct);
  for (size_t j = 0; j < score_names.size(); ++j) score_names[j] = "SCORE" + std::to_string(j + 1);
  std::vector<size_t> file_processed(file_ct, 0);
  for (uint32_t f = 0; f < file_ct; ++f) {
    const std::string& fname = files[f];
    // a --score file is described as such in messages, a --score-list file by its name (:8683)
    const std::string fdesc = c.score_list ? fname : "--score file";
    if (c.score_list) {
      lines.clear();
      if (!ReadLines(fname, &lines, &err)) {
        logprintf("Error: %s\n", err.c_str());
        return kRetOpenFail;
      }
      if (std::all_of(lines.begin(), lines.end(), [](const std::string& ln) { return SplitWs(ln).empty(); })) {
        logprintf("Error: --score-list: %s is empty.\n", fname.c_str());
        return kRetMalformedInput;
      }
    }
    seen.assign(2ull * V.size(), 0);
    uint64_t missing_id = 0, missing_allele = 0, dup_id = 0;
    const size_t file_first = entries.size();
    size_t li = 0;
    if ((c.score_header || c.score_header_read) && !lines.empty()) {
      if (c.score_header_read) {
        const std::vector<std::string> h = SplitWs(lines[0]);
        if (h.size() < need_cols) {
          logprintf("Error: Line 1 of %s has fewer tokens than expected.\n", fdesc.c_str());
          return kRetMalformedInput;
        }
        for (uint32_t j = 0; j < score_ct; ++j) score_names[static_cast<size_t>(f) * score_ct + j] = h[score_cols[j] - 1];
        // the reference checks the first file's names (:7655-7668)
        std::vector<std::string> sorted_names(score_names.begin(), score_names.begin() + score_ct);
        std::sort(sorted_names.begin(), sorted_names.end());
        if (f == 0 && std::adjacent_find(sorted_names.begin(), sorted_names.end()) != sorted_names.end()) {
          logprintf("Error: %s: Score IDs are not unique.\n", flagname);
          return kRetMalformedInput;
        }
      }
      li = 1;
    }
    for (; li < lines.size(); ++li) {
      if (lines[li].empty()) continue;
      const std::vector<std::string> t = SplitWs(lines[li]);
      if (t.empty()) continue;
      // the ID and allele tokens are needed first; the coefficients only on lines that are scored (:7712-7790)
      if (t.size() < std::max(c.score_id_col, c.score_allele_col)) {
        logprintf("Error: Line %zu of %s has fewer tokens than expected.\n", li + 1, fdesc.c_str());
        return kRetMalformedInput;
      }
      const std::string& id = t[c.score_id_col - 1];
      const auto it = by_id.find(id);
      if (it == by_id.end()) {
        ++missing_id;
        continue;
      }
      if (dup.count(id)) {
        if (!c.score_ignore_dup_ids) {
          logprintf("Error: %s variant ID '%s' appears multiple times in main dataset.\n", flagname, id.c_str());
          return kRetInconsistentInput;
        }
        ++dup_id;  // 'ignore-dup-ids' (:7724)
        continue;
      }
      const uint32_t v = it->second;
      const std::string& al = t[c.score_allele_col - 1];
      uint8_t aidx;
      if (al == V.ref[v]) aidx = 0;
      else if (al == V.alt[v]) aidx = 1;
      else {
        ++missing_allele;
        continue;
      }
      if (seen[2ull * v + aidx]) {
        logprintf("Error: %s: %s allele for variant '%s' appears multiple times in %s%s file.\n", flagname, aidx ? "ALT1" : "REF", id.c_str(), fname.c_str(), c.score_list ? "-list" : "");
        return kRetMalformedInput;
      }
      seen[2ull * v + aidx] = 1;
      if (t.size() < need_cols) {
        logprintf("Error: Line %zu of %s has fewer tokens than expected.\n", li + 1, fdesc.c_str());
        return kRetMalformedInput;
      }
      for (const uint32_t col : score_cols) {
        double coef;
        if (!ParseDouble(t[col - 1].c_str(), &coef)) {
          logprintf("Error: Line %zu of %s has an invalid coefficient.\n", li + 1, fdesc.c_str());
          return kRetMalformedInput;
        }
        coefs.push_back(coef);
      }
      // the reference's refusals for haploid chromosomes (:7794-7814)
      const uint32_t chr = V.chr_code[v];
      if ((chr == 23 || chr == 24 || chr == 26) && (c.score_dominant || c.score_recessive)) {
        logprintf("Error: --score[-list] 'dominant' and 'recessive' modifiers cannot be used with\nhaploid chromosomes.\n");
        return kRetInconsistentInput;
      }
      if ((chr == 23 || chr == 26) && c.score_varstd) {
        logprintf("Error: --score[-list] 'variance-standardize' cannot be used with chrX or MT.\n");
        return kRetInconsistentInput;
      }
      if (chr == 24 && y_prohibited) {
        logprintf("Error: When both chrY variants and unknown-sex samples are present,\n--score[-list] can only be run with the 'no-mean-imputation' modifier.\n");
        return kRetInconsistentInput;
      }
      entries.push_back({v, aidx, entries.size(), f});
    }
    if (!c.score_list) {
      if (missing_id || missing_allele) {
        logprintf("Warning: --score: %llu entr%s in %s %s skipped due to missing variant IDs, and %llu %s skipped due to mismatching allele codes.\n", static_cast<unsigned long long>(missing_id), missing_id == 1 ? "y" : "ies",
                  c.score_file.c_str(), missing_id == 1 ? "was" : "were", static_cast<unsigned long long>(missing_allele), missing_allele == 1 ? "was" : "were");
      }
    } else if (missing_id && missing_allele) {  // the reference's three forms (:8239-8280)
      logprintf("Warning: --score-list: %llu entr%s in %s %s skipped due to %s, and %llu %s skipped due to %s.\n", static_cast<unsigned long long>(missing_id), missing_id == 1 ? "y" : "ies", fname.c_str(), missing_id == 1 ? "was" : "were",
                missing_id == 1 ? "a missing variant ID" : "missing variant IDs", static_cast<unsigned long long>(missing_allele), missing_allele == 1 ? "was" : "were", missing_allele == 1 ? "a mismatching allele code" : "mismatching allele codes");
    } else if (missing_id || missing_allele) {
      const uint64_t ct = missing_id + missing_allele;
      logprintf("Warning: --score-list: %llu entr%s in %s %s skipped due to %s.\n", static_cast<unsigned long long>(ct), ct == 1 ? "y" : "ies", fname.c_str(), ct == 1 ? "was" : "were",
                missing_id ? (ct == 1 ? "a missing variant ID" : "missing variant IDs") : (ct == 1 ? "a mismatching allele code" : "mismatching allele codes"));
    }
    if (dup_id) {
      logprintf("Warning: %s: %llu entr%s in %s %s skipped since %s multiple times in the main dataset.\n", flagname, static_cast<unsigned long long>(dup_id), dup_id == 1 ? "y" : "ies", fname.c_str(), dup_id == 1 ? "was" : "were",
                dup_id == 1 ? "its variant ID appears" : "their variant IDs appear");
    }
    if (entries.size() == file_first) {
      if (c.score_list) logprintf("Error: --score-list: No valid variants in %s.\n", fname.c_str());
      else logprintf("Error: No valid variants in --score file.\n");
      return kRetDegenerateData;
    }
    file_processed[f] = entries.size() - file_first;
  }
  // <out>.sscore.vars lists the variants in score-file order, each once (:7790-7800)
  std::vector<uint32_t> file_order;
  if (c.score_list_variants) {
    std::vector<uint8_t> listed(V.size(), 0);
    for (const Entry& e : entries) {
      if (!listed[e.v]) {
        listed[e.v] = 1;
        file_order.push_back(e.v);
      }
    }
  }
  // device passes run in variant order (sums are order-independent up to fp64 rounding; the device adds in a fixed
  // order); a variant's entries stay in list order
  std::stable_sort(entries.begin(), entries.end(), [](const Entry& a, const Entry& b) { return a.v < b.v; });
  // classes: one per file, split further under --q-score-range into the entries whose variant lies in the same set of
  // ranges (numbered in variant order); each range of a file is the union of its classes.  Entries in no range are
  // dropped here.
  std::vector<uint32_t> entry_class(entries.size(), 0);  // per entry
  std::vector<uint32_t> class_file;                     // per class
  std::vector<std::vector<uint8_t>> class_ranges;      // per class: 1 for each range it lies in
  {
    std::map<std::pair<uint32_t, std::vector<uint8_t>>, uint32_t> class_of;
    std::vector<Entry> kept;
    std::vector<uint32_t> kept_class;
    for (const Entry& e : entries) {
      std::vector<uint8_t> in(ranges.size(), 0);
      if (qsr) {
        if (!qsr_seen[e.v]) continue;
        bool any = false;
        for (size_t r = 0; r < ranges.size(); ++r) {
          in[r] = !(qsr_p[e.v] < ranges[r].lb || qsr_p[e.v] > ranges[r].ub);
          any = any || in[r];
        }
        if (!any) continue;
      }
      const auto it = class_of.emplace(std::make_pair(e.file, in), static_cast<uint32_t>(class_ranges.size()));
      if (it.second) {
        class_ranges.push_back(in);
        class_file.push_back(e.file);
      }
      kept_class.push_back(it.first->second);
      kept.push_back(e);
    }
    entries.swap(kept);
    entry_class.swap(kept_class);
  }
  const uint32_t class_ct = std::max<uint32_t>(1, static_cast<uint32_t>(class_ranges.size()));
  const bool class_job = qsr || c.score_list;
  // staged rows: one per entry for --score (the rows are the entries), one per variant for --score-list
  std::vector<uint32_t> vidx, entry_row(entries.size());
  for (size_t k = 0; k < entries.size(); ++k) {
    if (!c.score_list || vidx.empty() || vidx.back() != entries[k].v) vidx.push_back(entries[k].v);
    entry_row[k] = static_cast<uint32_t>(vidx.size() - 1);
  }
  // named-allele frequencies for the mean imputation (per row): founders (ComputeAlleleFreqs), --read-freq values first
  std::vector<double> ref_freqs;
  {
    int rc = 0;
    bool have = FounderRefFreqs(ds, ctx, vidx, &ref_freqs, &rc, true);
    if (rc) return rc;
    if ((rc = SexChrRefFreqs(ds, ctx, vidx, &ref_freqs))) return rc;
    ApplyReadFreq(*ds, vidx, &ref_freqs, have);
  }
  // ploidy class of each entry (pl2gpu_score_add_variants_ploidy); a job with diploid entries only keeps the plain path
  auto ploidy_class = [&](uint32_t v) -> uint8_t {
    const uint32_t chr = V.chr_code[v];
    if (chr == 24) return kPl2ScoreChrY;
    if (chr == 26) return kPl2ScoreHaploidAll;
    return (chr == 23 && c.xchr_model == 1) ? kPl2ScoreChrXMaleHaploid : kPl2ScoreDiploid;
  };
  bool ploidy_job = false;
  for (const Entry& e : entries) ploidy_job = ploidy_job || ploidy_class(e.v) != kPl2ScoreDiploid;
  // class groups: the accumulators take class_ct x (8 score_ct + 24) bytes per padded sample.  When they do not all fit
  // the device budget (free memory less 10 %, capped by --gpu-memory) next to the job's staging buffers, consecutive
  // classes are scored in groups, one pass over the genotypes each.
  std::vector<uint32_t> group_start{0, class_ct};
  if (class_job && class_ct > 1) {
    uint64_t free_b = 0, total_b = 0;
    if (pl2gpu_ctx_mem_info(ctx, &free_b, &total_b)) return GpuFail("pl2gpu_ctx_mem_info");
    uint64_t budget = free_b - free_b / 10;
    if (c.gpu_memory_mib && (c.gpu_memory_mib << 20) < budget) budget = c.gpu_memory_mib << 20;
    const uint64_t np = (n + 63) / 64 * 64;
    const uint64_t staging = 2ull * 16384 * (np / 4) + np * 64 * (8ull * std::min(score_ct, 4u) + 12) + 16384ull * (64ull * score_ct + 5);
    const uint64_t per_class = np * (8ull * score_ct + 24);
    const uint64_t fit = budget > staging ? (budget - staging) / per_class : 0;
    if (fit < class_ct) {
      const uint32_t step = static_cast<uint32_t>(std::max<uint64_t>(fit, 1));
      group_start.assign(1, 0);
      for (uint32_t k = step; k < class_ct; k += step) group_start.push_back(k);
      group_start.push_back(class_ct);
      logprintf("%s: The accumulators of %u score classes do not fit in GPU memory together; scoring them in %zu passes over the genotypes.\n", flagname, class_ct, group_start.size() - 1);
    }
  }
  // per class: score sums [sample][score_ct], named-allele dosage sums in half allele units, diploid and haploid
  // missing calls (with the second entries of variants a file names by both alleles taken back out)
  std::vector<double> sums(static_cast<uint64_t>(class_ct) * n * score_ct);
  std::vector<uint64_t> hdos(static_cast<uint64_t>(class_ct) * n);
  std::vector<uint32_t> miss(static_cast<uint64_t>(class_ct) * n), miss_hap(static_cast<uint64_t>(class_ct) * n, 0);
  std::vector<int64_t> repeat_miss(static_cast<uint64_t>(class_ct) * n, 0), repeat_miss_hap(static_cast<uint64_t>(class_ct) * n, 0);  // [class][sample]
  for (size_t g = 0; g + 1 < group_start.size(); ++g) {
    const uint32_t k0 = group_start[g], k1 = group_start[g + 1];
    // this group's entries (in entry order) and the rows they read
    std::vector<size_t> gent;
    std::vector<uint32_t> gvidx, grow;  // staged variants; per group entry, its row among them
    for (size_t k = 0; k < entries.size(); ++k) {
      if (entry_class[k] < k0 || entry_class[k] >= k1) continue;
      if (gent.empty() || entry_row[k] != entry_row[gent.back()]) gvidx.push_back(entries[k].v);
      gent.push_back(k);
      grow.push_back(static_cast<uint32_t>(gvidx.size() - 1));
    }
    Pl2ScoreJob* job = nullptr;
    if (class_job) {
      if (pl2gpu_score_begin_classes(ctx, n, score_ct, k1 - k0, &job)) return GpuFail("pl2gpu_score_begin_classes");
    } else if (score_ct == 1) {  // the one-column job (same device work as pl2gpu_score_begin_cols with one column)
      if (pl2gpu_score_begin(ctx, n, &job)) return GpuFail("pl2gpu_score_begin");
    } else if (pl2gpu_score_begin_cols(ctx, n, score_ct, &job)) {
      return GpuFail("pl2gpu_score_begin_cols");
    }
    struct JobGuard {
      Pl2ScoreJob* j;
      ~JobGuard() { pl2gpu_score_end(j); }
    } guard{job};
    if (ploidy_job && pl2gpu_score_set_sex(job, S.sex.data())) return GpuFail("pl2gpu_score_set_sex");
    BlockStreamer bs(ds, &gvidx, n, 16384);
    if (!bs.Init()) return GpuFail("pl2gpu_host_alloc");
    std::vector<double> w4, w4h;  // diploid and haploid tables
    std::vector<uint8_t> d4, cls;
    std::vector<uint32_t> ecls, erow;
    size_t ge = 0;        // next group entry
    uint32_t row0 = 0;    // first row of the block
    for (;;) {
      const int got = bs.Next(&err);
      if (got < 0) {
        logprintf("Error: %s\n", err.c_str());
        return kRetMalformedInput;
      }
      if (!got) break;
      size_t ge_end = ge;
      while (ge_end < gent.size() && grow[ge_end] < row0 + static_cast<uint32_t>(got)) ++ge_end;
      const uint32_t ecnt = static_cast<uint32_t>(ge_end - ge);
      w4.resize(4ull * score_ct * ecnt);
      w4h.resize(4ull * score_ct * ecnt);
      d4.resize(ecnt);
      cls.resize(ecnt);
      ecls.resize(ecnt);
      erow.resize(ecnt);
      for (uint32_t k = 0; k < ecnt; ++k) {
        const size_t ei = gent[ge + k];
        const Entry& e = entries[ei];
        erow[k] = grow[ge + k] - row0;
        ecls[k] = entry_class[ei] - k0;
        const uint64_t cbase = static_cast<uint64_t>(entry_class[ei]) * n;
        const uint8_t pc = cls[k] = ploidy_class(e.v);
        const double rf = ref_freqs[entry_row[ei]];
        const double f_named = e.aidx ? (1.0 - rf) : rf;
        // genotype code = ALT allele count; named-allele dosage of codes 0, 1, 2.  The tables below do not depend on
        // the column; each column scales them by its coefficient.  'center' / 'variance-standardize'
        // (:8003-8033): dosage x slope + intercept with intercept = -p f slope and slope = 1 / sqrt(p / 2 x 2 f (1 - f))
        // (0 when the variance is not above 2^-44), p the variant's ploidy: 1 on chrY and MT, else 2 (chrX too, whatever
        // the model).  A missing call contributes (sample ploidy) f slope WITHOUT the intercept in the reference
        // (missing_effect, :6756-6762, :6795-6836) - kept, since the outputs are compared with its files.
        const uint32_t d0 = e.aidx ? 0 : 2, d2 = e.aidx ? 2 : 0;
        const bool haploid_variant = pc == kPl2ScoreChrY || pc == kPl2ScoreHaploidAll;
        double slope = 1.0, icpt = 0.0;
        if (c.score_center) {
          if (c.score_varstd) {
            const double variance = (haploid_variant ? 0.5 : 1.0) * (2.0 * f_named * (1.0 - f_named));
            if (!(variance > 1.0 / 17592186044416.0)) {
              slope = 0.0;  // the reference additionally insists that such a variant is monomorphic (:8013-8027); a weight of 0 scores it the same
            } else {
              slope = 1.0 / sqrt(variance);
            }
          }
          icpt = ((haploid_variant ? -1.0 : -2.0) * f_named) * slope;
        }
        // 'dominant' / 'recessive' (:6747-6762): copies -> min(copies, 1) / max(copies - 1, 0), a missing call -> ONE x f
        uint32_t e0 = d0, e1 = 1, e2 = d2;
        double miss_dosage = 2.0 * f_named;
        if (c.score_dominant) {
          e0 = d0 ? 1 : 0, e2 = d2 ? 1 : 0;
          miss_dosage = f_named;
        } else if (c.score_recessive) {
          e0 = d0 ? 1 : 0, e1 = 0, e2 = d2 ? 1 : 0;
          miss_dosage = f_named;
        }
        const double t0 = static_cast<double>(e0) * slope + icpt, t1 = static_cast<double>(e1) * slope + icpt, t2 = static_cast<double>(e2) * slope + icpt, t3 = miss_dosage * slope;
        // a haploid sample (chrY nonfemales, MT, chrX males under --xchr-model 1) holds half the dosage of each code
        const double h0 = (0.5 * e0) * slope + icpt, h1 = (0.5 * e1) * slope + icpt, h2 = (0.5 * e2) * slope + icpt, h3 = f_named * slope;
        for (uint32_t j = 0; j < score_ct; ++j) {
          const double coef = coefs[e.coef_row * score_ct + j];
          double* w = &w4[4ull * (static_cast<uint64_t>(k) * score_ct + j)];
          w[0] = coef * t0;
          w[1] = coef * t1;
          w[2] = coef * t2;
          w[3] = c.score_no_meanimpute ? 0.0 : coef * t3;
          if (pc == kPl2ScoreChrY) {  // the first table serves unknown-sex samples, whose chrY dosage the reference zeroes
            w[0] = w[1] = w[2] = coef * icpt;
            w[3] = c.score_no_meanimpute ? 0.0 : coef * h3;
          }
          double* wh = &w4h[4ull * (static_cast<uint64_t>(k) * score_ct + j)];
          wh[0] = coef * h0;
          wh[1] = coef * h1;
          wh[2] = coef * h2;
          wh[3] = c.score_no_meanimpute ? 0.0 : coef * h3;
        }
        d4[k] = static_cast<uint8_t>(e0 | (e1 << 2) | (e2 << 4));
        // a file that names both alleles of a variant (PC projection with allele weights): the device counts the missing
        // calls of both entries, the reference counts them once per variant and file (:7788), so the second entry's are
        // taken back out here, from the diploid or haploid count the sample's class put them in
        if (ei > 0 && entries[ei - 1].v == e.v && entry_class[ei - 1] == entry_class[ei]) {
          const uint64_t* row = bs.buf + static_cast<uint64_t>(erow[k]) * bs.words;
          for (uint32_t w = 0; w < bs.words; ++w) {
            uint64_t ms = row[w] & (row[w] >> 1) & 0x5555555555555555ull;
            if (32ull * (w + 1) > n) ms &= (1ull << (2 * (n - 32 * w))) - 1;
            for (; ms; ms &= ms - 1) {
              const uint32_t s = 32 * w + __builtin_ctzll(ms) / 2;
              const uint8_t sex = S.sex[s];
              if (pc == kPl2ScoreDiploid || (pc == kPl2ScoreChrXMaleHaploid && sex != 1)) --repeat_miss[cbase + s];
              else if (pc != kPl2ScoreChrY || sex != 2) --repeat_miss_hap[cbase + s];  // chrY females are not counted
            }
          }
        }
      }
      if (c.score_list) {
        if (pl2gpu_score_add_entries(job, bs.buf, static_cast<uint64_t>(bs.words) * 8, static_cast<uint32_t>(got), 0, ecnt, erow.data(), ecls.data(), ploidy_job ? cls.data() : nullptr, w4.data(), w4h.data(), d4.data()))
          return GpuFail("pl2gpu_score_add_entries");
      } else if (qsr) {  // one entry per row
        if (pl2gpu_score_add_variants_classes(job, bs.buf, static_cast<uint64_t>(bs.words) * 8, ecnt, 0, ecls.data(), ploidy_job ? cls.data() : nullptr, w4.data(), w4h.data(), d4.data()))
          return GpuFail("pl2gpu_score_add_variants_classes");
      } else if (ploidy_job) {
        if (pl2gpu_score_add_variants_ploidy(job, bs.buf, static_cast<uint64_t>(bs.words) * 8, ecnt, 0, cls.data(), w4.data(), w4h.data(), d4.data())) return GpuFail("pl2gpu_score_add_variants_ploidy");
      } else if (pl2gpu_score_add_variants(job, bs.buf, static_cast<uint64_t>(bs.words) * 8, ecnt, 0, w4.data(), d4.data())) {
        return GpuFail("pl2gpu_score_add_variants");
      }
      ge = ge_end;
      row0 += static_cast<uint32_t>(got);
    }
    if (class_job) {
      for (uint32_t k = k0; k < k1; ++k) {
        const uint64_t o = static_cast<uint64_t>(k) * n;
        if (pl2gpu_score_get_class(job, k - k0, sums.data() + o * score_ct, hdos.data() + o, miss.data() + o, miss_hap.data() + o)) return GpuFail("pl2gpu_score_get_class");
      }
    } else if (ploidy_job) {
      if (pl2gpu_score_get_ploidy(job, sums.data(), hdos.data(), miss.data(), miss_hap.data())) return GpuFail("pl2gpu_score_get_ploidy");
    } else {
      if (pl2gpu_score_get(job, sums.data(), hdos.data(), miss.data())) return GpuFail("pl2gpu_score_get");
      for (uint64_t& d : hdos) d *= 2;
    }
  }
  for (uint64_t k = 0; k < miss.size(); ++k) {
    miss[k] = static_cast<uint32_t>(miss[k] + repeat_miss[k]);
    miss_hap[k] = static_cast<uint32_t>(miss_hap[k] + repeat_miss_hap[k]);
  }
  if (c.score_list) {
    for (uint32_t f = 0; f < file_ct; ++f) logprintf("--score-list file %u/%u: %zu variant%s processed.\n", f + 1, file_ct, file_processed[f], file_processed[f] == 1 ? "" : "s");
  } else {
    logprintf("--score: %zu variant%s processed.\n", file_processed[0], file_processed[0] == 1 ? "" : "s");
  }
  if (c.score_list_variants) {
    OutFile fv;
    const std::string vname = c.out + ".sscore.vars";
    if (!fv.Open(vname)) return kRetOpenFail;
    for (const uint32_t v : file_order) {
      fv.Write(V.id[v].data(), V.id[v].size());
      fv.Puts("\n");
    }
    if (!fv.Close()) return kRetWriteFail;
    logprintf("Variant list written to %s .\n", vname.c_str());
  }
  // DENOM = base + nonfemale x chrY variants - male x chrX variants under --xchr-model 1 (:8581); base counts 2 per
  // diploid variant and 1 per MT variant.  Per class here; a range's terms are the sums over its classes (:8389).
  std::vector<uint32_t> denom_base(class_ct, 0), y_incr(class_ct, 0), x_decr(class_ct, 0);
  for (size_t k = 0; k < entries.size(); ++k) {
    if (k && entries[k - 1].v == entries[k].v && entry_class[k - 1] == entry_class[k]) continue;
    const uint8_t pc = ploidy_class(entries[k].v);
    const uint32_t cl = entry_class[k];
    denom_base[cl] += pc == kPl2ScoreHaploidAll ? 1 : pc == kPl2ScoreChrY ? 0 : 2;
    y_incr[cl] += pc == kPl2ScoreChrY;
    x_decr[cl] += pc == kPl2ScoreChrXMaleHaploid;
  }
  // report (:8470-8625)
  std::vector<PhenoOut> phenos;
  if (c.sc_phenos || c.sc_pheno1) {
    for (size_t pc = 0; pc < S.pheno_names.size(); ++pc) {
      PhenoOut po;
      if (TypePheno(S.pheno_names[pc], S.pheno_tokens[pc], &po)) phenos.push_back(std::move(po));
      if (!c.sc_phenos && !phenos.empty()) break;  // pheno1: first active phenotype only
    }
  }
  const IdFmt idf{c.sc_fid || (c.sc_fid_maybe && S.fid_present), c.sc_sid || (c.sc_sid_maybe && S.sid_present)};
  std::string hdr = "#";
  if (idf.fid) hdr += "FID\t";
  hdr += "IID";
  if (idf.sid) hdr += "\tSID";
  for (const PhenoOut& po : phenos) hdr += "\t" + po.name;
  if (c.sc_nallele) hdr += "\tALLELE_CT";
  if (c.sc_denom) hdr += "\tDENOM";
  if (c.sc_dosagesum) hdr += "\tNAMED_ALLELE_DOSAGE_SUM";
  // every file's _AVG columns, then every file's _SUM columns (:8520-8539, :8595-8612)
  if (c.sc_avgs)
    for (const std::string& nm : score_names) hdr += "\t" + nm + "_AVG";
  if (c.sc_sums)
    for (const std::string& nm : score_names) hdr += "\t" + nm + "_SUM";
  hdr += "\n";
  // one report: per file, the classes with in_report[class] set, added in ascending class order.  ALLELE_CT, DENOM and
  // NAMED_ALLELE_DOSAGE_SUM exist for --score only (one file).
  auto write_report = [&](const std::string& name, const std::vector<uint8_t>& in_report) -> int {
    std::vector<double> rs(static_cast<uint64_t>(file_ct) * n * score_ct, 0.0);  // [file][sample][score_ct]
    std::vector<uint64_t> rhdos(static_cast<uint64_t>(file_ct) * n, 0);
    std::vector<uint32_t> rmiss(static_cast<uint64_t>(file_ct) * n, 0), rmiss_hap(static_cast<uint64_t>(file_ct) * n, 0);
    std::vector<uint32_t> rbase(file_ct, 0), ry(file_ct, 0), rx(file_ct, 0);
    for (uint32_t k = 0; k < class_ct; ++k) {
      if (!in_report[k]) continue;
      const uint32_t f = class_file.empty() ? 0 : class_file[k];
      const uint64_t o = static_cast<uint64_t>(k) * n, fo = static_cast<uint64_t>(f) * n;
      for (uint64_t i = 0; i < static_cast<uint64_t>(n) * score_ct; ++i) rs[fo * score_ct + i] += sums[o * score_ct + i];
      for (uint32_t s = 0; s < n; ++s) {
        rhdos[fo + s] += hdos[o + s];
        rmiss[fo + s] += miss[o + s];
        rmiss_hap[fo + s] += miss_hap[o + s];
      }
      rbase[f] += denom_base[k];
      ry[f] += y_incr[k];
      rx[f] += x_decr[k];
    }
    OutFile out;
    if (!out.Open(name, c.score_zs)) return kRetOpenFail;
    out.Puts(hdr.c_str());
    char num[64];
    std::vector<uint32_t> denom(file_ct);
    for (uint32_t k = 0; k < n; ++k) {
      std::string row = FmtId(S, k, idf);
      for (const PhenoOut& po : phenos) row += "\t" + po.text[k];
      for (uint32_t f = 0; f < file_ct; ++f) {
        const uint64_t fk = static_cast<uint64_t>(f) * n + k;
        const uint32_t denom_full = rbase[f] + (S.sex[k] != 2 ? ry[f] : 0) - (S.sex[k] == 1 ? rx[f] : 0);
        const uint32_t nallele = denom_full - 2 * rmiss[fk] - rmiss_hap[fk];
        denom[f] = c.score_no_meanimpute ? nallele : denom_full;
        if (f) continue;
        if (c.sc_nallele) {
          *u32toa(nallele, num) = '\0';
          row += std::string("\t") + num;
        }
        if (c.sc_denom) {
          *u32toa(denom[0], num) = '\0';
          row += std::string("\t") + num;
        }
        if (c.sc_dosagesum) row += "\t" + std::to_string(rhdos[fk] / 2) + ((rhdos[fk] & 1) ? ".5" : "");
      }
      if (c.sc_avgs) {
        for (uint32_t f = 0; f < file_ct; ++f) {
          const double* ks = &rs[(static_cast<uint64_t>(f) * n + k) * score_ct];
          for (uint32_t j = 0; j < score_ct; ++j) {
            *dtoa_g(ks[j] * (1.0 / static_cast<double>(denom[f])), num) = '\0';
            row += std::string("\t") + num;
          }
        }
      }
      if (c.sc_sums) {
        for (uint32_t f = 0; f < file_ct; ++f) {
          const double* ks = &rs[(static_cast<uint64_t>(f) * n + k) * score_ct];
          for (uint32_t j = 0; j < score_ct; ++j) {
            *dtoa_g(ks[j], num) = '\0';
            row += std::string("\t") + num;
          }
        }
      }
      row += "\n";
      out.Write(row.data(), row.size());
    }
    return out.Close() ? 0 : kRetWriteFail;
  };
  const char* ext = c.score_zs ? ".sscore.zst" : ".sscore";
  if (!qsr) {
    const std::string name = c.out + ext;
    if (int rc = write_report(name, std::vector<uint8_t>(class_ct, 1))) return rc;
    logprintf("%s: Results written to %s .\n", flagname, name.c_str());
    return 0;
  }
  // one report per range, in range-file order; a range no entry lies in gets one of zero sums
  for (size_t r = 0; r < ranges.size(); ++r) {
    std::vector<uint8_t> in_report(class_ct, 0);
    for (uint32_t k = 0; k < class_ranges.size(); ++k) in_report[k] = class_ranges[k][r];
    if (int rc = write_report(c.out + "." + ranges[r].name + ext, in_report)) return rc;
  }
  logprintf("%s + --q-score-range: Results written to %s.<range name>%s .\n", flagname, c.out.c_str(), ext);
  return 0;
}

// `--variant-score` (VscoreReport, 2.0/plink2_matrix_calc.cc:9274-10100): sample weights from a file ([#FID] IID [SID]
// + named weight columns, or headerless FID IID + VSCORE1..), per variant the weighted sum of ALT dosages with a missing
// call replaced by 2 x ALT frequency.  The sums are one pass of the approx-PCA tensor tile path (pl2gpu_pca_vscore).
// chrY and MT dosages count half (slope 0.5), chrY only for males, and chrX males count half under --xchr-model 1
// (VscoreThread :8831-8868, :9158-9200): the product is linear in the weights, so those variants run as jobs of their
// own with the weight matrix rescaled or masked that way.
int RunVscore(const Cmd& c, Dataset* ds, Pl2GpuCtx* ctx) {
  const SampleInfo& S = ds->samples;
  const VariantInfo& V = ds->variants;
  const uint32_t n = S.size(), m = V.size();
  if (std::find(V.chr_code.begin(), V.chr_code.end(), 24u) != V.chr_code.end() && std::find(S.sex.begin(), S.sex.end(), 0) != S.sex.end()) {  // :9297-9301
    logprintf("Error: When chrY is present, --variant-score cannot be used with unknown-sex\nsamples.\n");
    return kRetInconsistentInput;
  }
  std::vector<std::string> lines;
  std::string err;
  if (!ReadLines(c.vscore_file, &lines, &err)) {
    logprintf("Error: %s\n", err.c_str());
    return kRetOpenFail;
  }
  size_t li = 0;
  while (li < lines.size() && lines[li].empty()) ++li;
  if (li == lines.size()) {
    logprintf("Error: Empty --variant-score file.\n");
    return kRetMalformedInput;
  }
  bool fid_col = true, sid_col = false;
  std::vector<std::string> names;
  size_t id_tokens = 2;
  const size_t first_line = li;
  if (lines[li][0] == '#') {
    const std::vector<std::string> h = SplitWs(lines[li].substr(1));
    size_t t = 0;
    fid_col = !h.empty() && h[0] == "FID";
    if (fid_col) ++t;
    if (t >= h.size() || h[t] != "IID") {
      logprintf("Error: Invalid header line in --variant-score file (#FID or #IID expected first).\n");
      return kRetMalformedInput;
    }
    ++t;
    if (t < h.size() && h[t] == "SID") {
      sid_col = true;
      ++t;
    }
    id_tokens = t;
    names.assign(h.begin() + t, h.end());
    ++li;
  } else {
    const size_t tok_ct = SplitWs(lines[li]).size();
    for (size_t k = 2; k < tok_ct; ++k) names.push_back("VSCORE" + std::to_string(k - 1));
  }
  if (names.empty()) {
    logprintf("Error: No score columns in --variant-score file.\n");
    return kRetMalformedInput;
  }
  // weight columns as token indices: all after the IDs, or those --vscore-col-nums selects (1-based over the whole
  // line; 2.0/plink2_matrix_calc.cc:9343-9384); a headerless file names them VSCORE1 .. by position in the selection
  std::vector<uint32_t> wcols;
  if (c.vscore_col_nums.empty()) {
    for (size_t k = 0; k < names.size(); ++k) wcols.push_back(static_cast<uint32_t>(id_tokens + k));
  } else {
    if (c.vscore_col_nums.back() > id_tokens + names.size()) {
      logprintf("Error: Line %zu of --variant-score file has fewer tokens than expected.\n", first_line + 1);
      return kRetInconsistentInput;
    }
    if (c.vscore_col_nums.front() <= id_tokens) {
      logprintf("Error: --vscore-col-nums argument overlaps with ID columns.\n");
      return kRetInconsistentInput;
    }
    std::vector<std::string> picked;
    for (const uint32_t col : c.vscore_col_nums) {
      wcols.push_back(col - 1);
      picked.push_back(li > first_line ? names[col - 1 - id_tokens] : "VSCORE" + std::to_string(picked.size() + 1));
    }
    names = std::move(picked);
  }
  const uint32_t cols = static_cast<uint32_t>(names.size());
  const size_t need_tokens = wcols.back() + 1;
  auto key = [&](const std::string& fid, const std::string& iid, const std::string& sid) {
    std::string k = (fid_col ? fid : std::string("0")) + "\t" + iid;  // no FID column: FID 0 (XidRead, plink2_common.cc:1280)
    if (sid_col && S.sid_present) k += "\t" + sid;
    return k;
  };
  std::unordered_map<std::string, int64_t> by_key;
  by_key.reserve(static_cast<size_t>(n) * 2);
  for (uint32_t k = 0; k < n; ++k) {
    auto ins = by_key.emplace(S.fid[k] + "\t" + S.iid[k] + ((sid_col && S.sid_present) ? "\t" + S.sid[k] : std::string()), k);
    if (!ins.second) ins.first->second = -1;
  }
  std::vector<double> w(static_cast<uint64_t>(n) * cols, 0.0);
  std::vector<uint8_t> seen(n, 0);
  uint64_t skipped = 0;
  uint32_t loaded = 0;
  for (; li < lines.size(); ++li) {
    if (lines[li].empty()) continue;
    const std::vector<std::string> t = SplitWs(lines[li]);
    if (t.size() < need_tokens) {
      logprintf("Error: Line %zu of --variant-score file has fewer tokens than expected.\n", li + 1);
      return kRetMalformedInput;
    }
    size_t q = 0;
    const std::string fid = fid_col ? t[q++] : std::string();
    const std::string iid = t[q++];
    const std::string sid = sid_col ? t[q++] : std::string();
    const auto it = by_key.find(key(fid, iid, sid));
    if (it == by_key.end() || it->second < 0) {
      ++skipped;
      continue;
    }
    const uint32_t sidx = static_cast<uint32_t>(it->second);
    if (seen[sidx]) {
      logprintf("Error: Sample ID on line %zu of --variant-score file appears more than once.\n", li + 1);
      return kRetMalformedInput;
    }
    seen[sidx] = 1;
    ++loaded;
    for (uint32_t cc = 0; cc < cols; ++cc) {
      double d;
      if (!ParseDouble(t[wcols[cc]].c_str(), &d) || d != d) {
        logprintf("Error: Invalid coefficient on line %zu of --variant-score file.\n", li + 1);
        return kRetMalformedInput;
      }
      w[static_cast<uint64_t>(sidx) * cols + cc] = d;
    }
  }
  if (skipped) logprintf("Warning: %llu line%s skipped in --variant-score file.\n", static_cast<unsigned long long>(skipped), skipped == 1 ? "" : "s");
  if (!loaded) {
    logprintf("Error: No valid entries in --variant-score file.\n");
    return kRetDegenerateData;
  }
  logprintf("--variant-score: %u score-vector%s loaded for %u sample%s.\n", cols, cols == 1 ? "" : "s", loaded, loaded == 1 ? "" : "s");
  const std::vector<uint32_t> vidx = AllVariants(*ds);
  std::vector<double> ref_freqs;
  int rc = 0;
  {
    const bool have = FounderRefFreqs(ds, ctx, vidx, &ref_freqs, &rc, true);
    if (rc) return rc;
    if ((rc = SexChrRefFreqs(ds, ctx, vidx, &ref_freqs))) return rc;
    ApplyReadFreq(*ds, vidx, &ref_freqs, have);
  }
  // variant classes by weight matrix: 0 as given (autosomes, XY, chrX under --xchr-model 2), 1 chrX under
  // --xchr-model 1 (male weights halved), 2 chrY (male weights halved, others zero), 3 MT (all weights halved)
  std::vector<uint32_t> cls_vidx[4];
  for (uint32_t v = 0; v < m; ++v) {
    const uint32_t chr = V.chr_code[v];
    cls_vidx[chr == 26 ? 3 : chr == 24 ? 2 : (chr == 23 && c.xchr_model == 1) ? 1 : 0].push_back(v);
  }
  std::vector<double> scores(static_cast<uint64_t>(m) * cols);
  for (int cl = 0; cl < 4; ++cl) {
    const std::vector<uint32_t>& list = cls_vidx[cl];
    if (list.empty()) continue;
    std::vector<double> wc(w);
    for (uint32_t k = 0; cl && k < n; ++k) {
      const double f = (cl == 3 || S.sex[k] == 1) ? 0.5 : cl == 2 ? 0.0 : 1.0;
      for (uint32_t cc = 0; cc < cols; ++cc) wc[static_cast<uint64_t>(k) * cols + cc] *= f;
    }
    // the matrix is kept resident in pieces that fit comfortably; every piece is one pl2gpu_pca job
    const uint32_t lm = static_cast<uint32_t>(list.size()), piece = 262144;
    for (uint32_t p0 = 0; p0 < lm; p0 += piece) {
      const uint32_t p1 = std::min(lm, p0 + piece);
      Pl2PcaJob* job = nullptr;
      if (pl2gpu_pca_begin_shard(ctx, n, p1 - p0, 0, &job)) return GpuFail("pl2gpu_pca_begin_shard");  // pc_ct 0: a --variant-score job
      struct Guard {
        Pl2PcaJob* j;
        ~Guard() { pl2gpu_pca_end(j); }
      } guard{job};
      std::vector<uint32_t> sub(list.begin() + p0, list.begin() + p1);
      std::vector<double> sub_freqs(sub.size());
      for (size_t k = 0; k < sub.size(); ++k) sub_freqs[k] = ref_freqs[sub[k]];
      BlockStreamer bs(ds, &sub, n, 32768);
      if (!bs.Init()) return GpuFail("pl2gpu_host_alloc");
      size_t base = 0;
      for (;;) {
        const int got = bs.Next(&err);
        if (got < 0) {
          logprintf("Error: %s\n", err.c_str());
          return kRetMalformedInput;
        }
        if (!got) break;
        const int arc = pl2gpu_pca_add_variants(job, bs.buf, static_cast<uint64_t>(bs.words) * 8, static_cast<uint32_t>(got), 0, sub_freqs.data() + base);
        if (arc) {
          logprintf("Error: %s\n", pl2gpu_last_error());
          return arc == 2 ? kRetDegenerateData : kRetGpuFail;
        }
        base += static_cast<size_t>(got);
      }
      std::vector<double> out(static_cast<uint64_t>(sub.size()) * cols);
      if (pl2gpu_pca_vscore(job, wc.data(), cols, out.data())) return GpuFail("pl2gpu_pca_vscore");
      for (size_t k = 0; k < sub.size(); ++k) std::copy_n(out.data() + k * cols, cols, scores.data() + static_cast<uint64_t>(sub[k]) * cols);
    }
  }
  // report (:9900-10060): #CHROM POS ID REF ALT [PROVISIONAL_REF?] [ALT_FREQ] <score names>
  const bool provref_col = c.vs_provref || (c.vs_maybeprovref && V.provisional_ref && c.vs_ref);
  const std::string name = c.out + (c.vscore_zs ? ".vscore.zst" : ".vscore");
  OutFile f;
  if (!f.Open(name, c.vscore_zs)) return kRetOpenFail;
  std::string hdr = "#";
  if (c.vs_chrom) hdr += "CHROM\t";
  if (c.vs_pos) hdr += "POS\t";
  hdr += "ID";
  if (c.vs_ref) hdr += "\tREF";
  if (c.vs_alt) hdr += "\tALT";
  if (provref_col) hdr += "\tPROVISIONAL_REF?";
  if (c.vs_altfreq) hdr += "\tALT_FREQ";
  for (const std::string& nm : names) hdr += "\t" + nm;
  hdr += "\n";
  f.Puts(hdr.c_str());
  char num[64];
  for (uint32_t v = 0; v < m; ++v) {
    std::string row;
    if (c.vs_chrom) row += ChrNameOut(V.chr_code[v], V.chr_name[v]) + "\t";
    if (c.vs_pos) row += std::to_string(V.bp[v]) + "\t";
    row += V.id[v];
    if (c.vs_ref) row += "\t" + V.ref[v];
    if (c.vs_alt) row += "\t" + V.alt[v];
    if (provref_col) row += V.provisional_ref ? "\tY" : "\tN";
    if (c.vs_altfreq) {
      *dtoa_g(1.0 - ref_freqs[v], num) = '\0';
      row += std::string("\t") + num;
    }
    for (uint32_t cc = 0; cc < cols; ++cc) {
      *dtoa_g(scores[static_cast<uint64_t>(v) * cols + cc], num) = '\0';
      row += std::string("\t") + num;
    }
    row += "\n";
    f.Write(row.data(), row.size());
  }
  if (!f.Close()) return kRetWriteFail;
  logprintf("--variant-score: Results written to %s .\n", name.c_str());
  return 0;
}

// ---------------------------------------------------------------------------------------- --freq
// `--freq` (WriteAlleleFreqs, 2.0/plink2_misc.cc:3573; counts from the LoadAlleleAndGenoCounts pass,
// 2.0/plink2.cc:2280): founder ALT allele frequencies of biallelic hard calls -> <out>.afreq.
// Founder allele "ddosage" totals per variant, in 1/32768 units as the reference accumulates them: alt_dd[v] / tot_dd[v]
// is the ALT frequency `--freq` prints and every later command consumes (allele_freqs, plink2.cc:2301).  Computed for
// the variants vidx (view indices); the outputs follow vidx's order.
int FounderAlleleDosages(Dataset* ds, Pl2GpuCtx* ctx, const std::vector<uint32_t>& vidx, std::vector<uint64_t>* alt_dd_out, std::vector<uint64_t>* tot_dd_out, bool all_samples = false) {
  const SampleInfo& S = ds->samples;
  const VariantInfo& V = ds->variants;
  const uint32_t n = S.size(), m = static_cast<uint32_t>(vidx.size());
  uint32_t founder_ct = 0, male_ct = 0, nonfemale_ct = 0;
  std::vector<uint64_t> inc((n + 63) / 64, 0), inc_male((n + 63) / 64, 0), inc_nonfemale((n + 63) / 64, 0);
  for (uint32_t k = 0; k < n; ++k) {
    if (S.is_founder[k] || all_samples) {  // --nonfounders: allele_ddosages over every sample (plink2.cc:2301)
      inc[k / 64] |= 1ull << (k % 64);
      ++founder_ct;
      if (S.sex[k] == 1) {
        inc_male[k / 64] |= 1ull << (k % 64);
        ++male_ct;
      }
      if (S.sex[k] != 2) {
        inc_nonfemale[k / 64] |= 1ull << (k % 64);
        ++nonfemale_ct;
      }
    }
  }
  if (!founder_ct) {
    logprintf("Error: No founders to estimate allele frequencies from.\n");
    return kRetDegenerateData;
  }
  // genotype counts on the device for a variant list over a sample subset (LoadAlleleAndGenoCountsThread's counting,
  // 2.0/plink2_data.cc:2304): all founders for every variant, founder males for chrX, nonfemale founders for chrY
  auto count_pass = [&](const std::vector<uint32_t>& vidx, const uint64_t* include, uint32_t sample_ct, std::vector<uint32_t>* out) -> int {
    out->assign(4ull * vidx.size(), 0);
    if (vidx.empty() || !sample_ct) return 0;
    BlockStreamer bs(ds, &vidx, sample_ct, 16384);
    if (sample_ct != n) bs.sample_include = include;
    if (!bs.Init()) return GpuFail("pl2gpu_host_alloc");
    std::string err;
    size_t base = 0;
    for (;;) {
      const int got = bs.Next(&err);
      if (got < 0) {
        logprintf("Error: %s\n", err.c_str());
        return kRetMalformedInput;
      }
      if (!got) break;
      if (pl2gpu_geno_counts(ctx, bs.buf, static_cast<uint64_t>(bs.words) * 8, sample_ct, static_cast<uint32_t>(got), 0, out->data() + 4ull * base)) return GpuFail("pl2gpu_geno_counts");
      base += static_cast<size_t>(got);
    }
    return 0;
  };
  std::vector<uint32_t> xv, yv;
  for (const uint32_t v : vidx) {
    if (V.chr_code[v] == 23) xv.push_back(v);
    else if (V.chr_code[v] == 24) yv.push_back(v);
  }
  std::vector<uint32_t> counts, xmale, ynonfemale;
  int rc = count_pass(vidx, inc.data(), founder_ct, &counts);
  if (!rc) rc = count_pass(xv, inc_male.data(), male_ct, &xmale);
  if (!rc) rc = count_pass(yv, inc_nonfemale.data(), nonfemale_ct, &ynonfemale);
  if (rc) return rc;
  alt_dd_out->assign(m, 0);
  tot_dd_out->assign(m, 0);
  size_t xi = 0, yi = 0;
  for (uint32_t k = 0; k < m; ++k) {
    const uint32_t v = vidx[k];
    const uint64_t n0 = counts[4ull * k], n1 = counts[4ull * k + 1], n2 = counts[4ull * k + 2], n3 = counts[4ull * k + 3];
    // allele "ddosages" in 1/32768 units, as the reference accumulates them (plink2_data.cc:2420-2690): diploid x2;
    // MT and chrY (nonfemale founders) haploid, a het counting half; chrX nonmales twice, males once
    uint64_t alt_dd, tot_dd;
    if (V.chr_code[v] == 23) {
      const uint32_t* mc = &xmale[4 * xi++];
      const uint64_t alt1 = 4 * n2 + 2 * n1 - 2ull * mc[2] - mc[1];
      const uint64_t wobs = (2 * (founder_ct - n3) - male_ct + mc[3]) * 2;
      alt_dd = alt1 * 16384ull;
      tot_dd = wobs * 16384ull;
    } else if (V.chr_code[v] == 24) {
      const uint32_t* yc = &ynonfemale[4 * yi++];
      alt_dd = (yc[1] + 2ull * yc[2]) * 16384ull;
      tot_dd = 2ull * (static_cast<uint64_t>(yc[0]) + yc[1] + yc[2]) * 16384ull;
    } else if (V.chr_code[v] == 26) {
      alt_dd = (n1 + 2 * n2) * 16384ull;
      tot_dd = 2 * (n0 + n1 + n2) * 16384ull;
    } else {
      alt_dd = (n1 + 2 * n2) * 32768ull;
      tot_dd = 2 * (n0 + n1 + n2) * 32768ull;
    }
    (*alt_dd_out)[k] = alt_dd;
    (*tot_dd_out)[k] = tot_dd;
  }
  return 0;
}

// --score / --variant-score: the REF frequencies of the chrX, chrY and MT variants among vidx from the per-class
// founder counting above (ComputeAlleleFreqs), written over FounderRefFreqs' all-diploid values; the other variants
// keep theirs.  Nothing to do without such variants, or without founders (FounderRefFreqs' 0.5 then stands).
int SexChrRefFreqs(Dataset* ds, Pl2GpuCtx* ctx, const std::vector<uint32_t>& vidx, std::vector<double>* ref_freqs) {
  const VariantInfo& V = ds->variants;
  std::vector<uint32_t> pos, sub;
  for (size_t k = 0; k < vidx.size(); ++k) {
    const uint32_t chr = V.chr_code[vidx[k]];
    if (chr == 23 || chr == 24 || chr == 26) {
      pos.push_back(static_cast<uint32_t>(k));
      sub.push_back(vidx[k]);
    }
  }
  const std::vector<uint8_t>& fo = ds->samples.is_founder;
  if (sub.empty() || std::find(fo.begin(), fo.end(), 1) == fo.end()) return 0;
  std::vector<uint64_t> alt_dd, tot_dd;
  if (const int rc = FounderAlleleDosages(ds, ctx, sub, &alt_dd, &tot_dd)) return rc;
  for (size_t k = 0; k < sub.size(); ++k) (*ref_freqs)[pos[k]] = tot_dd[k] ? static_cast<double>(tot_dd[k] - alt_dd[k]) * (1.0 / static_cast<double>(tot_dd[k])) : 0.5;
  return 0;
}

int RunFreq(const Cmd& c, Dataset* ds, Pl2GpuCtx* ctx) {
  const VariantInfo& V = ds->variants;
  const uint32_t m = V.size();
  if (ds->reader.nonref_flags_storage() == 3) {
    logprintf("Error: --freq on a .pgen with per-variant provisional-REF flags is not supported by plink2_b200 yet.\n");
    return kRetNotYetSupported;
  }
  std::vector<uint64_t> alt_dds, tot_dds;
  const int rc = FounderAlleleDosages(ds, ctx, AllVariants(*ds), &alt_dds, &tot_dds, c.nonfounders);
  if (rc) return rc;
  if (c.freq_counts && !c.nonfounders) {  // plink2.cc:2102
    for (uint8_t fo : ds->samples.is_founder) {
      if (!fo) {
        logprintf("Error: \"--freq counts\" specified, but with neither --ac-founders nor --nonfounders; and nonfounders are present.\n");
        return kRetInconsistentInput;
      }
    }
  }
  const std::string name = c.out + (c.freq_counts ? ".acount" : ".afreq") + (c.freq_zs ? ".zst" : "");
  OutFile f;
  if (!f.Open(name, c.freq_zs)) return kRetOpenFail;
  f.Puts((std::string("#CHROM\tID\tREF\tALT\t") + (V.provisional_ref ? "PROVISIONAL_REF?\t" : "") + (c.freq_counts ? "ALT_CTS" : "ALT_FREQS") + "\tOBS_CT\n").c_str());
  for (uint32_t v = 0; v < m; ++v) {
    const uint64_t alt_dd = alt_dds[v], tot_dd = tot_dds[v];
    const double recip = tot_dd ? 1.0 / static_cast<double>(tot_dd) : 0.0;
    char* w = f.Reserve(V.chr_name[v].size() + V.id[v].size() + V.ref[v].size() + V.alt[v].size() + 96);
    auto puts = [&](const std::string& t) {
      memcpy(w, t.data(), t.size());
      w += t.size();
      *w++ = '\t';
    };
    puts(ChrNameOut(V.chr_code[v], V.chr_name[v]));
    puts(V.id[v]);
    puts(V.ref[v]);
    puts(V.alt[v]);
    if (V.provisional_ref) {
      *w++ = 'Y';
      *w++ = '\t';
    }
    // 'counts': the allele dosage itself (1/32768 units -> alleles; halves appear for haploid hets)
    w = dtoa_g(c.freq_counts ? static_cast<double>(alt_dd) * (1.0 / 32768.0) : static_cast<double>(alt_dd) * recip, w);
    *w++ = '\t';
    w = u32toa(static_cast<uint32_t>(tot_dd / 32768ull), w);
    *w++ = '\n';
    f.Advance(w);
  }
  if (!f.Close()) return kRetWriteFail;
  logprintf("--freq%s: Allele %s (%s) written to %s .\n", c.freq_counts ? " counts" : "", c.freq_counts ? "counts" : "frequencies", c.nonfounders ? "all samples" : "founders only", name.c_str());
  return 0;
}

int RunLdPrune(const Cmd& c, Dataset* ds, Pl2GpuCtx* ctx) {
  const SampleInfo& S = ds->samples;
  const VariantInfo& V = ds->variants;
  const uint32_t n = S.size();
  // unique variant IDs (plink2_ld.cc:2590-2593)
  {
    std::vector<std::string> ids;
    for (uint32_t v = 0; v < V.size(); ++v)
      if (V.chr_code[v]) ids.push_back(V.id[v]);
    std::sort(ids.begin(), ids.end());
    for (size_t k = 1; k < ids.size(); ++k) {
      if (ids[k] == ids[k - 1]) {
        logprintf("Error: --indep-pairwise requires unique variant IDs ('%s' appears multiple times).\n", ids[k].c_str());
        return kRetInconsistentInput;
      }
    }
  }
  uint32_t founder_ct = 0;
  std::vector<uint64_t> inc((n + 63) / 64, 0);
  std::vector<uint8_t> founder_sex;  // chrX / chrY / MT handling needs it (plink2_ld.cc:1356-1389)
  for (uint32_t k = 0; k < n; ++k) {
    if (S.is_founder[k]) {
      inc[k / 64] |= 1ull << (k % 64);
      founder_sex.push_back(S.sex[k]);
      ++founder_ct;
    }
  }
  if (!founder_ct) {
    logprintf("Error: No founders left for --indep-pairwise.\n");
    return kRetDegenerateData;
  }
  const uint32_t m = V.size();
  const uint32_t words = PgenReader::WordsFor(founder_ct);
  // --indep-preferred (plink2_ld.cc:2577-2597, NondupIdLoad): variants whose ID is listed keep priority in
  // the pairwise victim choice (:916-918)
  std::vector<uint8_t> preferred;
  if (!c.indep_preferred.empty()) {
    std::vector<std::string> plines;
    std::string perr;
    if (!ReadLines(c.indep_preferred, &plines, &perr)) {
      logprintf("Error: %s\n", perr.c_str());
      return kRetOpenFail;
    }
    std::unordered_map<std::string, uint32_t> by_id;
    by_id.reserve(static_cast<size_t>(m) * 2);
    for (uint32_t v = 0; v < m; ++v)
      if (V.chr_code[v]) by_id.emplace(V.id[v], v);
    preferred.assign(m, 0);
    uint32_t pref_ct = 0;
    for (const std::string& ln : plines) {
      for (const std::string& tok : SplitWs(ln)) {
        const auto it = by_id.find(tok);
        if (it != by_id.end() && !preferred[it->second]) {
          preferred[it->second] = 1;
          ++pref_ct;
        }
      }
    }
    logprintf("--indep-preferred: %u variant%s loaded.\n", pref_ct, pref_ct == 1 ? "" : "s");
  }
  // Chromosomes are independent jobs (LdPruneSubcontigSplitAll never crosses one, plink2_ld.cc:2165-2268): each
  // contiguous chromosome run is staged in pinned host memory and handed to the function-face entry point on its own, so
  // the staging buffer and the decision matrix are O(largest chromosome), not O(genome).
  std::vector<uint8_t> removed(m, 0);
  struct ChrRun {
    uint32_t v0, v1;
  };
  std::vector<ChrRun> chr_runs;
  uint32_t longest = 0;
  for (uint32_t s0 = 0; s0 < m;) {
    uint32_t e = s0 + 1;
    while (e < m && V.chr_code[e] == V.chr_code[s0]) ++e;
    if (V.chr_code[s0] == 0) {
      for (uint32_t v = s0; v < e; ++v) removed[v] = 2;
    } else if (e - s0 >= 2) {
      chr_runs.push_back({s0, e});
      longest = std::max(longest, e - s0);
    }
    s0 = e;
  }
  // One worker per device (SURVEY section 8e: "LD prune = chromosomes -> GPUs, no collective"): each owns a pinned
  // buffer of the longest run, decodes a run straight into it and hands it to the function-face entry point on ITS
  // context; runs are taken largest first from a shared counter and write disjoint slices of `removed`.  With one
  // device this is the plain loop over the runs in file order.
  const uint32_t worker_ct = std::max(1u, std::min<uint32_t>({c.gpus, static_cast<uint32_t>(chr_runs.size()), static_cast<uint32_t>(std::max(1, pl2gpu_device_count() - c.device))}));
  if (c.gpus > 1 && worker_ct < c.gpus) logprintf("Note: --indep-pairwise on %u GPU%s (--gpus %u): one chromosome per device at a time.\n", worker_ct, worker_ct == 1 ? "" : "s", c.gpus);
  std::vector<Pl2GpuCtx*> ld_ctx(1, ctx);
  struct CtxGuard {
    std::vector<Pl2GpuCtx*>* v;
    ~CtxGuard() {
      for (size_t g = 1; g < v->size(); ++g) pl2gpu_ctx_destroy((*v)[g]);
    }
  } ctx_guard{&ld_ctx};
  for (uint32_t g = 1; g < worker_ct; ++g) {
    Pl2GpuCtx* cx = nullptr;
    if (pl2gpu_ctx_create(c.device + static_cast<int>(g), &cx)) return GpuFail("pl2gpu_ctx_create");
    ld_ctx.push_back(cx);
  }
  std::vector<uint32_t> order(chr_runs.size());
  for (uint32_t k = 0; k < order.size(); ++k) order[k] = k;
  if (worker_ct > 1) std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return chr_runs[a].v1 - chr_runs[a].v0 > chr_runs[b].v1 - chr_runs[b].v0; });
  std::atomic<uint32_t> next_run{0};
  std::vector<double> t_decode_w(worker_ct, 0.0), t_device_w(worker_ct, 0.0);
  std::vector<int> worker_rc(worker_ct, 0);
  std::vector<std::string> worker_msg(worker_ct);
  auto worker = [&](uint32_t g) {
    std::vector<uint32_t> vsub;
    BlockStreamer bs(ds, &vsub, founder_ct, std::max(longest, 1u));
    bs.threads = std::max(1u, g_decode_threads / worker_ct);
    if (founder_ct != n) bs.sample_include = inc.data();
    if (longest && !bs.Init()) {
      worker_rc[g] = kRetGpuFail;
      worker_msg[g] = std::string("pl2gpu_host_alloc: ") + pl2gpu_last_error();
      return;
    }
    for (;;) {
      const uint32_t slot = next_run.fetch_add(1);
      if (slot >= order.size()) return;
      for (uint32_t w = 0; w < worker_ct; ++w)
        if (worker_rc[w]) return;  // another worker failed: stop taking work
      const ChrRun& run = chr_runs[order[slot]];
      vsub.resize(run.v1 - run.v0);
      for (uint32_t v = run.v0; v < run.v1; ++v) vsub[v - run.v0] = v;
      bs.Rewind();
      std::string err;
      auto tp = std::chrono::steady_clock::now();
      const int got = bs.Next(&err);
      if (got != static_cast<int>(run.v1 - run.v0)) {
        worker_rc[g] = kRetMalformedInput;
        worker_msg[g] = got < 0 ? err : "short read";
        return;
      }
      t_decode_w[g] += g_clock.Since(tp);
      tp = std::chrono::steady_clock::now();
      const int rc = pl2_indep_pairwise_ex(ld_ctx[g], bs.buf, static_cast<uint64_t>(words) * 8, founder_ct, run.v1 - run.v0, V.chr_code.data() + run.v0, V.bp.data() + run.v0, c.indep_window, c.indep_step, c.indep_r2, c.indep_kb ? 1 : 0,
                                           ds->read_ref_freq.empty() ? nullptr : ds->read_ref_freq.data() + run.v0, preferred.empty() ? nullptr : preferred.data() + run.v0, 0, founder_sex.data(),
                                           c.indep_order1 ? kPl2LdPlink1Order : 0, removed.data() + run.v0);
      if (rc) {
        worker_rc[g] = kRetGpuFail;
        worker_msg[g] = std::string("pl2_indep_pairwise: ") + pl2gpu_last_error();  // thread-local in the library
        return;
      }
      t_device_w[g] += g_clock.Since(tp);
    }
  };
  {
    std::vector<std::thread> th;
    for (uint32_t g = 1; g < worker_ct; ++g) th.emplace_back(worker, g);
    worker(0);
    for (auto& t : th) t.join();
  }
  for (uint32_t g = 0; g < worker_ct; ++g) {
    if (worker_rc[g]) {
      logprintf("Error: %s\n", worker_msg[g].c_str());
      return worker_rc[g];
    }
  }
  double t_decode = 0, t_device = 0;
  for (uint32_t g = 0; g < worker_ct; ++g) {
    t_decode = std::max(t_decode, t_decode_w[g]);
    t_device = std::max(t_device, t_device_w[g]);
  }
  if (g_clock.on) fprintf(stderr, "[timing]   ld: decode %.3f s, counts + pair decisions + greedy walk %.3f s over %zu chromosome run%s\n", t_decode, t_device, chr_runs.size(), chr_runs.size() == 1 ? "" : "s");
  // LdPruneWrite (plink2_ld.cc:2464-2528)
  const std::string in_name = c.out + ".prune.in", out_name = c.out + ".prune.out";
  OutFile fin, fout;
  if (!fin.Open(in_name) || !fout.Open(out_name)) return kRetOpenFail;
  uint32_t removed_ct = 0, considered = 0;
  for (uint32_t v = 0; v < m; ++v) {
    if (removed[v] == 2) continue;
    ++considered;
    OutFile& f = removed[v] ? fout : fin;
    removed_ct += removed[v];
    f.Write(V.id[v].data(), V.id[v].size());
    f.Puts("\n");
  }
  if (!fin.Close() || !fout.Close()) return kRetWriteFail;
  logprintf("--indep-pairwise: %u/%u variant%s removed.\n", removed_ct, considered, considered == 1 ? "" : "s");
  logprintf("Variant lists written to %s and %s .\n", in_name.c_str(), out_name.c_str());
  return 0;
}

}  // namespace

// Host-only debug hooks used by the CPU test-suite (no GPU involved):
//   --debug-dtoa <in: raw doubles> <out: one dtoa_g line each>
//   --debug-dump-geno <pgen> <psam/fam> <pvar/bim> <out: one byte per genotype, variant-major>
int DebugHooks(int argc, char** argv) {
  if (argc == 4 && (!strcmp(argv[1], "--debug-dtoa") || !strcmp(argv[1], "--debug-dtoa-p8"))) {
    const bool p8 = argv[1][12] != 0;
    FILE* in = fopen(argv[2], "rb");
    OutFile out;
    if (!in || !out.Open(argv[3])) return kRetOpenFail;
    double x;
    while (fread(&x, 8, 1, in) == 1) {
      char* w = out.Reserve(64);
      w = p8 ? dtoa_g_p8(x, w) : dtoa_g(x, w);
      *w++ = '\n';
      out.Advance(w);
    }
    fclose(in);
    return out.Close() ? 0 : kRetWriteFail;
  }
  if (argc == 4 && !strcmp(argv[1], "--debug-rel-check-pairs")) {  // <.fam/.psam> <out: FID1 IID1 FID2 IID2 per pair, table order>
    SampleInfo S;
    std::string err;
    OutFile out;
    if (!LoadSamples(argv[2], &S, &err) || !out.Open(argv[3])) return kRetOpenFail;
    std::vector<uint32_t> pairs;
    RelCheckPairs(S, &pairs);
    for (size_t k = 0; k < pairs.size(); k += 2) {
      const std::string ln = S.fid[pairs[k]] + "\t" + S.iid[pairs[k]] + "\t" + S.fid[pairs[k + 1]] + "\t" + S.iid[pairs[k + 1]] + "\n";
      out.Write(ln.data(), ln.size());
    }
    return out.Close() ? 0 : kRetWriteFail;
  }
  if (argc == 4 && !strcmp(argv[1], "--debug-natural-sort")) {  // <in: one key per line> <out: the keys in natural order>
    std::vector<std::string> keys;
    std::string err;
    OutFile out;
    if (!ReadLines(argv[2], &keys, &err) || !out.Open(argv[3])) return kRetOpenFail;
    std::stable_sort(keys.begin(), keys.end(), [](const std::string& a, const std::string& b) { return NaturalCompare(a, b) < 0; });
    for (const std::string& k : keys) {
      out.Write(k.data(), k.size());
      out.Puts("\n");
    }
    return out.Close() ? 0 : kRetWriteFail;
  }
  if (argc == 4 && !strcmp(argv[1], "--debug-zst")) {  // <in> <out.zst>: the 'zs' writer on its own (mixed small and large writes)
    FILE* in = fopen(argv[2], "rb");
    OutFile out;
    if (!in || !out.Open(argv[3], true)) return kRetOpenFail;
    std::vector<char> chunk(3 << 20);
    size_t want = 7, got;
    while ((got = fread(chunk.data(), 1, std::min(want, chunk.size()), in)) > 0) {
      out.Write(chunk.data(), got);
      want = want * 5 + 3;
    }
    fclose(in);
    return out.Close() ? 0 : kRetWriteFail;
  }
  if (argc == 5 && !strcmp(argv[1], "--debug-sfmt")) {  // <seed> <count> <out: raw uint32>
    Sfmt19937 rng;
    rng.InitGenRand(static_cast<uint32_t>(strtoul(argv[2], nullptr, 10)));
    OutFile out;
    if (!out.Open(argv[4])) return kRetOpenFail;
    const unsigned long cnt = strtoul(argv[3], nullptr, 10);
    for (unsigned long k = 0; k < cnt; ++k) {
      const uint32_t v = rng.GenRandU32();
      out.Write(&v, 4);
    }
    return out.Close() ? 0 : kRetWriteFail;
  }
  if (argc == 6 && !strcmp(argv[1], "--debug-gauss")) {  // <seed> <pairs> <threads> <out: raw doubles>
    Sfmt19937 rng;
    rng.InitGenRand(static_cast<uint32_t>(strtoul(argv[2], nullptr, 10)));
    const uint64_t pairs = strtoull(argv[3], nullptr, 10);
    std::vector<double> g(2 * pairs);
    FillGaussian(pairs, static_cast<uint32_t>(strtoul(argv[4], nullptr, 10)), &rng, g.data());
    OutFile out;
    if (!out.Open(argv[5])) return kRetOpenFail;
    out.Write(g.data(), g.size() * 8);
    return out.Close() ? 0 : kRetWriteFail;
  }
  if (argc == 6 && !strcmp(argv[1], "--debug-dump-geno")) {
    Dataset ds;
    std::string err;
    if (!LoadSamples(argv[3], &ds.samples, &err) || !LoadVariants(argv[4], &ds.variants, &err) || !ds.reader.Open(argv[2], ds.samples.size(), ds.variants.size(), &err)) {
      fprintf(stderr, "Error: %s\n", err.c_str());
      return kRetMalformedInput;
    }
    OutFile out;
    if (!out.Open(argv[5])) return kRetOpenFail;
    const uint32_t n = ds.samples.size();
    std::vector<uint64_t> gv(PgenReader::WordsFor(n));
    std::vector<uint8_t> row(n);
    for (uint32_t v = 0; v < ds.variants.size(); ++v) {
      if (!ds.reader.Get(v, gv.data(), &err)) {
        fprintf(stderr, "Error: %s\n", err.c_str());
        return kRetMalformedInput;
      }
      for (uint32_t k = 0; k < n; ++k) row[k] = (gv[k / 32] >> (2 * (k % 32))) & 3;
      out.Write(row.data(), n);
    }
    return out.Close() ? 0 : kRetWriteFail;
  }
  return -1;
}

// `--r2-unphased` table (VcorTable, 2.0/plink2_ld.cc:11025; per-pair statistic ComputeR2 :6654-6682, report filter
// :10814-10818): squared correlation of the founders' hard-call dosages for every variant pair on one chromosome within
// --ld-window-kb (default 1000) / --ld-window, reported when r^2 >= --ld-window-r2 (default 0.2).
// Division of labour: the DEVICE screens every pair of the band with the pair-decision kernel the LD prune uses
// (pl2gpu_ld_band_flags: cov^2 > t var1 var2 on the exact integer sextuple, t a hair below the report threshold, so
// the flagged set is a superset); the HOST recomputes the sextuple of the few flagged pairs from bit planes of the
// block it already holds and applies the reference's own arithmetic (int64 -> double, cov^2 / (var0 var1), >= threshold).
// chrX pairs use the reference's sex-aware statistic (ComputeXR2) and are evaluated on the host without a device screen.
int RunR2Unphased(const Cmd& c, Dataset* ds, Pl2GpuCtx* ctx) {
  const SampleInfo& S = ds->samples;
  const VariantInfo& V = ds->variants;
  const uint32_t n = S.size(), m = V.size();
  const uint32_t bp_radius = c.ld_bp_radius == 0xFFFFFFFFu ? 1000000u : c.ld_bp_radius;
  const double min_r2 = c.ld_min_r2 == 2.0 ? 0.2 * (1 - 1.0 / 17592186044416.0) : c.ld_min_r2;
  if (c.parallel_tot != 1) {
    logprintf("Error: --r2-unphased cannot be used with --parallel in plink2_b200.\n");
    return kRetNotYetSupported;
  }
  if (!(min_r2 > 0.0)) {
    logprintf("Error: --r2-unphased needs a positive --ld-window-r2 in plink2_b200 (the device screens pairs against it).\n");
    return kRetNotYetSupported;
  }
  // founders; on chrY the reference sets female founders to missing (InterleavedSetMissing, plink2_ld.cc:11845), which
  // for a statistic over samples non-missing in both variants is the same as leaving them out
  uint32_t all_founder_ct = 0, y_founder_ct = 0;
  std::vector<uint64_t> inc_all((n + 63) / 64, 0), inc_y((n + 63) / 64, 0);
  std::vector<uint64_t> male_plane;  // one bit per founder (founder order): male
  for (uint32_t k = 0; k < n; ++k) {
    if (S.is_founder[k]) {
      if ((all_founder_ct & 63) == 0) male_plane.push_back(0);
      if (S.sex[k] == 1) male_plane.back() |= 1ull << (all_founder_ct & 63);
      inc_all[k / 64] |= 1ull << (k % 64);
      ++all_founder_ct;
      if (S.sex[k] != 2) {
        inc_y[k / 64] |= 1ull << (k % 64);
        ++y_founder_ct;
      }
    }
  }
  if (!all_founder_ct) {
    logprintf("Error: No founders for --r2-unphased.\n");
    return kRetDegenerateData;
  }
  logprintf("Running --r2-unphased with the following filters:\n");
  if (c.ld_var_radius < 0x7fffffff) logprintf("  --ld-window: %u\n", c.ld_var_radius + 1);
  logprintf("  --ld-window-kb: %g\n", 0.001 * bp_radius);
  logprintf("  --ld-window-r2: %g\n", min_r2);
  const std::string name = c.out + (c.r2_zs ? ".vcor.zst" : ".vcor");
  OutFile f;
  if (!f.Open(name, c.r2_zs)) return kRetOpenFail;
  f.Puts("#CHROM_A\tPOS_A\tID_A\tCHROM_B\tPOS_B\tID_B\tUNPHASED_R2\n");
  uint64_t reported = 0, flagged_total = 0;
  for (uint32_t s0 = 0; s0 < m;) {
    uint32_t e = s0 + 1;
    while (e < m && V.chr_code[e] == V.chr_code[s0]) ++e;
    const uint32_t len = e - s0;
    const bool is_y = V.chr_code[s0] == 24;
    // chrX: the reference's sex-aware statistic (ComputeXR2, plink2_ld.cc:7122-7187: every sum taken over all founders
    // minus half of the same sum over the male founders, genotypes counted as NON-MAJOR alleles).  The unweighted device
    // screen is not a superset for it, so every pair of the window is evaluated on the host for this chromosome.
    const bool is_x = V.chr_code[s0] == 23;
    const uint32_t founder_ct = is_y ? y_founder_ct : all_founder_ct;
    const std::vector<uint64_t>& inc = is_y ? inc_y : inc_all;
    const uint32_t words = PgenReader::WordsFor(founder_ct);
    const uint32_t pw = (founder_ct + 63) / 64;  // plane words per variant
    if (len >= 2 && founder_ct) {
      // window end per first variant a: [a + 1, win_end[a]) holds the partners within both radii; band = widest window
      std::vector<uint32_t> win_end(len);
      uint32_t band = 0, hi = 0;
      for (uint32_t a = 0; a < len; ++a) {
        if (hi < a + 1) hi = a + 1;
        while (hi < len && V.bp[s0 + hi] - V.bp[s0 + a] <= bp_radius) ++hi;
        win_end[a] = std::min<uint64_t>(hi, static_cast<uint64_t>(a) + 1 + c.ld_var_radius);
        band = std::max(band, win_end[a] - a - 1);
      }
      if (band) {
        if (static_cast<uint64_t>(len) * band > (1ull << 33)) {
          logprintf("Error: --r2-unphased window too wide for plink2_b200 on this chromosome (%u variants x %u partners); narrow --ld-window-kb / --ld-window.\n", len, band);
          return kRetNotYetSupported;
        }
        std::vector<uint32_t> vsub(len);
        for (uint32_t k = 0; k < len; ++k) vsub[k] = s0 + k;
        BlockStreamer bs(ds, &vsub, founder_ct, len);
        if (founder_ct != n) bs.sample_include = inc.data();
        if (!bs.Init()) return GpuFail("pl2gpu_host_alloc");
        std::string err;
        if (bs.Next(&err) != static_cast<int>(len)) {
          logprintf("Error: %s\n", err.empty() ? "short read" : err.c_str());
          return kRetMalformedInput;
        }
        std::vector<uint8_t> flags(is_x ? 0 : static_cast<uint64_t>(len) * band);
        if (!is_x && pl2gpu_ld_band_flags(ctx, bs.buf, static_cast<uint64_t>(words) * 8, founder_ct, len, 0, band, min_r2 * (1 - 1e-9), flags.data())) return GpuFail("pl2gpu_ld_band_flags");
        // bit planes of the block: het / hom-ALT / non-missing, one bit per founder
        std::vector<uint64_t> p_one(static_cast<uint64_t>(len) * pw, 0), p_two(static_cast<uint64_t>(len) * pw, 0), p_nm(static_cast<uint64_t>(len) * pw, 0);
        for (uint32_t k = 0; k < len; ++k) {
          const uint64_t* row = bs.buf + static_cast<uint64_t>(k) * words;
          for (uint32_t w = 0; w < words; ++w) {
            const uint64_t g = row[w];
            const uint64_t lo = _pext_u64(g, 0x5555555555555555ull), hi2 = _pext_u64(g, 0xAAAAAAAAAAAAAAAAull);
            uint64_t valid = 0xFFFFFFFFull;
            if (w == words - 1 && (founder_ct & 31)) valid = (1ull << (founder_ct & 31)) - 1;
            const uint64_t one = lo & ~hi2 & valid, two = hi2 & ~lo & valid, nm = ~(lo & hi2) & valid;
            const uint32_t sh = 32 * (w & 1);
            p_one[static_cast<uint64_t>(k) * pw + (w >> 1)] |= one << sh;
            p_two[static_cast<uint64_t>(k) * pw + (w >> 1)] |= two << sh;
            p_nm[static_cast<uint64_t>(k) * pw + (w >> 1)] |= nm << sh;
          }
          if (is_x) {
            // count NON-MAJOR alleles: when ALT is the major allele (founder REF frequency below 1/2, chrX accounting of
            // --freq, or the loaded / frozen value) hom-REF becomes the "two" class
            uint64_t n1 = 0, n2 = 0, m1 = 0, m2 = 0, nmc = 0, mnm = 0;
            for (uint32_t w = 0; w < pw; ++w) {
              const uint64_t o = p_one[static_cast<uint64_t>(k) * pw + w], t2 = p_two[static_cast<uint64_t>(k) * pw + w], nm = p_nm[static_cast<uint64_t>(k) * pw + w], ml = male_plane[w];
              n1 += __builtin_popcountll(o);
              n2 += __builtin_popcountll(t2);
              nmc += __builtin_popcountll(nm);
              m1 += __builtin_popcountll(o & ml);
              m2 += __builtin_popcountll(t2 & ml);
              mnm += __builtin_popcountll(nm & ml);
            }
            const uint64_t alt1 = 4 * n2 + 2 * n1 - 2 * m2 - m1, wobs = (2 * nmc - mnm) * 2;  // = (2 (F - n3) - males + m3) * 2
            double ref_freq = wobs ? static_cast<double>(wobs - alt1) * (1.0 / static_cast<double>(wobs)) : 0.5;
            if (!ds->read_ref_freq.empty() && ds->read_ref_freq[s0 + k] == ds->read_ref_freq[s0 + k]) ref_freq = ds->read_ref_freq[s0 + k];
            if (ref_freq < 0.5) {
              for (uint32_t w = 0; w < pw; ++w) {
                uint64_t& t2 = p_two[static_cast<uint64_t>(k) * pw + w];
                t2 = p_nm[static_cast<uint64_t>(k) * pw + w] & ~p_one[static_cast<uint64_t>(k) * pw + w] & ~t2;
              }
            }
          }
        }
        // rows are independent: host threads each take rows a = t, t + T, ... of a block of rows and write their lines to
        // per-row strings, which are emitted in row order (the table order of the reference)
        auto process_row = [&](uint32_t a, std::string* out_text, uint64_t* flagged_ct, uint64_t* reported_ct) {
          char line[64];
          for (uint32_t b = a + 1; b < win_end[a]; ++b) {
            if (!is_x && !flags[static_cast<uint64_t>(b) * band + (b - a - 1)]) continue;
            ++*flagged_ct;
            const uint64_t *o0 = &p_one[static_cast<uint64_t>(a) * pw], *t0 = &p_two[static_cast<uint64_t>(a) * pw], *n0 = &p_nm[static_cast<uint64_t>(a) * pw];
            const uint64_t *o1 = &p_one[static_cast<uint64_t>(b) * pw], *t1 = &p_two[static_cast<uint64_t>(b) * pw], *n1 = &p_nm[static_cast<uint64_t>(b) * pw];
            int64_t obs = 0, sum0 = 0, sum1 = 0, ssq0 = 0, ssq1 = 0, dot = 0;
            for (uint32_t w = 0; w < pw; ++w) {
              const uint64_t valid = n0[w] & n1[w];
              const int64_t a1 = __builtin_popcountll(o0[w] & valid), a2 = __builtin_popcountll(t0[w] & valid), b1 = __builtin_popcountll(o1[w] & valid), b2 = __builtin_popcountll(t1[w] & valid);
              obs += __builtin_popcountll(valid);
              sum0 += a1 + 2 * a2;
              ssq0 += a1 + 4 * a2;
              sum1 += b1 + 2 * b2;
              ssq1 += b1 + 4 * b2;
              dot += __builtin_popcountll(o0[w] & o1[w]) + 2 * (__builtin_popcountll(o0[w] & t1[w]) + __builtin_popcountll(t0[w] & o1[w])) + 4 * __builtin_popcountll(t0[w] & t1[w]);
            }
            if (!obs) continue;
            double r2;
            if (is_x) {
              int64_t mobs = 0, msum0 = 0, msum1 = 0, mssq0 = 0, mssq1 = 0, mdot = 0;
              for (uint32_t w = 0; w < pw; ++w) {
                const uint64_t ml = male_plane[w], valid = n0[w] & n1[w] & ml;
                const int64_t a1 = __builtin_popcountll(o0[w] & valid), a2 = __builtin_popcountll(t0[w] & valid), b1 = __builtin_popcountll(o1[w] & valid), b2 = __builtin_popcountll(t1[w] & valid);
                mobs += __builtin_popcountll(valid);
                msum0 += a1 + 2 * a2;
                mssq0 += a1 + 4 * a2;
                msum1 += b1 + 2 * b2;
                mssq1 += b1 + 4 * b2;
                mdot += __builtin_popcountll(o0[w] & o1[w] & ml) + 2 * (__builtin_popcountll(o0[w] & t1[w] & ml) + __builtin_popcountll(t0[w] & o1[w] & ml)) + 4 * __builtin_popcountll(t0[w] & t1[w] & ml);
              }
              const double dw = 0.5;  // male_downwt for two chrX variants
              const double wobs = std::fma(-dw, static_cast<double>(mobs), static_cast<double>(obs)), wn0 = std::fma(-dw, static_cast<double>(msum0), static_cast<double>(sum0)), wn1 = std::fma(-dw, static_cast<double>(msum1), static_cast<double>(sum1));
              const double ws0 = std::fma(-dw, static_cast<double>(mssq0), static_cast<double>(ssq0)), ws1 = std::fma(-dw, static_cast<double>(mssq1), static_cast<double>(ssq1)), wd = std::fma(-dw, static_cast<double>(mdot), static_cast<double>(dot));
              const double variance0 = std::fma(ws0, wobs, -wn0 * wn0), variance1 = std::fma(ws1, wobs, -wn1 * wn1);
              if (variance0 <= 0.0 || variance1 <= 0.0) continue;
              const double cov01 = std::fma(wd, wobs, -wn0 * wn1);
              r2 = std::min(1.0, cov01 * cov01 / (variance0 * variance1));
            } else {
              const int64_t var0 = ssq0 * obs - sum0 * sum0, var1 = ssq1 * obs - sum1 * sum1;
              const double variance_prod = static_cast<double>(var0) * static_cast<double>(var1);
              if (variance_prod == 0.0) continue;
              const double cov01 = static_cast<double>(dot * obs - sum0 * sum1);
              r2 = cov01 * cov01 / variance_prod;
            }
            if (!(r2 >= min_r2)) continue;
            const uint32_t va = s0 + a, vb = s0 + b;
            const std::string chr = ChrNameOut(V.chr_code[va], V.chr_name[va]);
            *out_text += chr;
            *out_text += '\t';
            *u32toa(V.bp[va], line) = '\0';
            *out_text += line;
            *out_text += '\t';
            *out_text += V.id[va];
            *out_text += '\t';
            *out_text += chr;
            *out_text += '\t';
            *u32toa(V.bp[vb], line) = '\0';
            *out_text += line;
            *out_text += '\t';
            *out_text += V.id[vb];
            *out_text += '\t';
            *dtoa_g(r2, line) = '\0';
            *out_text += line;
            *out_text += '\n';
            ++*reported_ct;
          }
        };
        const uint32_t worker_ct = std::max(1u, std::min(EffectiveHostThreads(c.threads), 64u));
        const uint32_t row_block = 8192;
        std::vector<std::string> row_text(std::min(row_block, len));
        std::vector<uint64_t> flagged_w(worker_ct, 0), reported_w(worker_ct, 0);
        for (uint32_t a0 = 0; a0 < len; a0 += row_block) {
          const uint32_t a1 = std::min(len, a0 + row_block);
          auto work = [&](uint32_t t) {
            for (uint32_t a = a0 + t; a < a1; a += worker_ct) {
              row_text[a - a0].clear();
              process_row(a, &row_text[a - a0], &flagged_w[t], &reported_w[t]);
            }
          };
          std::vector<std::thread> th;
          for (uint32_t t = 1; t < worker_ct; ++t) th.emplace_back(work, t);
          work(0);
          for (auto& x : th) x.join();
          for (uint32_t a = a0; a < a1; ++a) f.Write(row_text[a - a0].data(), row_text[a - a0].size());
        }
        for (uint32_t t = 0; t < worker_ct; ++t) {
          flagged_total += flagged_w[t];
          reported += reported_w[t];
        }
      }
    }
    s0 = e;
  }
  if (!f.Close()) return kRetWriteFail;
  if (g_clock.on) fprintf(stderr, "[timing]   r2: %llu pairs flagged by the device screen, %llu reported\n", static_cast<unsigned long long>(flagged_total), static_cast<unsigned long long>(reported));
  logprintf("--r2-unphased: Results written to %s .\n", name.c_str());
  return 0;
}

// --missing (WriteMissingnessReports, 2.0/plink2_misc.cc): .smiss / .vmiss from one host counting pass.  Written where the
// reference writes them: after the sample filters (incl. --mind), BEFORE the variant thresholds (--geno, --maf, ...).
int WriteMissingReports(const Cmd& c, Dataset* ds) {
  int rc;
  std::string err;
  // --missing (WriteMissingnessReports, 2.0/plink2_misc.cc): .smiss / .vmiss from one host counting pass over what the
  // filters left.  chrY calls are counted for males only (OBS_CT of a chrY variant = male count; a non-male's OBS_CT
  // excludes the chrY variants).  PHENOx columns say whether that phenotype is missing (Y) or not (N).
  VariantGenoCounts vc;
  std::vector<uint32_t> smiss;
  uint32_t y_ct = 0;
  rc = CountGenotypes(ds, EffectiveHostThreads(c.threads), &vc, &smiss, &y_ct, &err);
  if (rc) {
    logprintf("Error: %s\n", err.c_str());
    return rc;
  }
  const SampleInfo& S = ds->samples;
  const VariantInfo& V = ds->variants;
  const uint32_t n = S.size(), m = V.size();
  uint32_t male_ct = 0;
  for (uint8_t sx : S.sex) male_ct += sx == 1;
  char num[40];
  if (c.missing_sample) {
    std::vector<PhenoOut> phenos;
    for (size_t p = 0; p < S.pheno_names.size(); ++p) {
      PhenoOut po;
      if (TypePheno(S.pheno_names[p], S.pheno_tokens[p], &po)) phenos.push_back(std::move(po));
    }
    const std::string name = c.out + (c.missing_zs ? ".smiss.zst" : ".smiss");
    OutFile f;
    if (!f.Open(name, c.missing_zs)) return kRetOpenFail;
    std::string h = std::string("#") + (S.fid_present ? "FID\t" : "") + "IID" + (S.sid_present ? "\tSID" : "");
    for (const PhenoOut& po : phenos) h += "\t" + po.name;
    h += "\tMISSING_CT\tOBS_CT\tF_MISS\n";
    f.Puts(h.c_str());
    for (uint32_t k = 0; k < n; ++k) {
      std::string ln = (S.fid_present ? S.fid[k] + "\t" : std::string()) + S.iid[k] + (S.sid_present ? "\t" + S.sid[k] : std::string());
      for (const PhenoOut& po : phenos) ln += (po.text[k] == "NA" || po.text[k] == "NONE") ? "\tY" : "\tN";
      const uint32_t obs = m - (S.sex[k] == 1 ? 0 : y_ct);
      *dtoa_g(obs ? static_cast<double>(smiss[k]) / static_cast<double>(obs) : std::numeric_limits<double>::quiet_NaN(), num) = '\0';
      ln += "\t" + std::to_string(smiss[k]) + "\t" + std::to_string(obs) + "\t" + num + "\n";
      f.Puts(ln.c_str());
    }
    if (!f.Close()) return kRetWriteFail;
    logprintf("--missing: Sample missing data report written to %s .\n", name.c_str());
  }
  if (c.missing_variant) {
    const std::string name = c.out + (c.missing_zs ? ".vmiss.zst" : ".vmiss");
    OutFile f;
    if (!f.Open(name, c.missing_zs)) return kRetOpenFail;
    f.Puts("#CHROM\tID\tMISSING_CT\tOBS_CT\tF_MISS\n");
    for (uint32_t v = 0; v < m; ++v) {
      const bool is_y = V.chr_code[v] == 24;
      const uint32_t miss = is_y ? vc.male[4ull * v + 3] : vc.all[4ull * v + 3], obs = is_y ? male_ct : n;
      *dtoa_g(obs ? static_cast<double>(miss) / static_cast<double>(obs) : std::numeric_limits<double>::quiet_NaN(), num) = '\0';
      const std::string ln = ChrNameOut(V.chr_code[v], V.chr_name[v]) + "\t" + V.id[v] + "\t" + std::to_string(miss) + "\t" + std::to_string(obs) + "\t" + num + "\n";
      f.Puts(ln.c_str());
    }
    if (!f.Close()) return kRetWriteFail;
    logprintf("--missing: Variant missing data report written to %s .\n", name.c_str());
  }
  return 0;
}

// --mind, --geno, --maf / --max-maf / --mac / --max-mac on hard calls: one host counting pass each for the sample and
// the variant thresholds (MindFilter plink2_filter.cc:3329, EnforceGenoThresh :3498, EnforceFreqConstraints :3791).
// chrY: missingness over males only; frequencies are the founder frequencies --freq reports (or --read-freq's).
int ApplyCountFilters(const Cmd& c, Dataset* ds) {
  const FilterSpec& f = c.filters;
  const double eps = 1.0 / 17592186044416.0;  // kSmallEpsilon = 2^-44
  const uint32_t threads = EffectiveHostThreads(c.threads);
  std::string err;
  if (f.mind < 1.0) {
    std::vector<uint32_t> miss;
    uint32_t y_ct = 0;
    const int rc = CountGenotypes(ds, threads, nullptr, &miss, &y_ct, &err);
    if (rc) {
      logprintf("Error: %s\n", err.c_str());
      return rc;
    }
    const SampleInfo& S = ds->samples;
    const uint32_t n = S.size(), m = ds->variants.size();
    const double thr = f.mind * (1 + eps);
    const uint32_t max_nonmale = static_cast<uint32_t>(static_cast<int32_t>(static_cast<double>(m - y_ct) * thr)), max_male = static_cast<uint32_t>(static_cast<int32_t>(static_cast<double>(m) * thr));
    std::vector<uint8_t> keep(n, 1);
    std::vector<uint32_t> gone;
    for (uint32_t k = 0; k < n; ++k) {
      if (miss[k] > (S.sex[k] == 1 ? max_male : max_nonmale)) {
        keep[k] = 0;
        gone.push_back(k);
      }
    }
    logprintf("%zu sample%s removed due to missing genotype data (--mind).\n", gone.size(), gone.size() == 1 ? "" : "s");
    if (!gone.empty()) {
      const std::string name = c.out + ".mindrem.id";
      if (!WriteIdFile(name, S, gone, true)) return kRetWriteFail;
      logprintf("ID%s written to %s .\n", gone.size() == 1 ? "" : "s", name.c_str());
      if (gone.size() == n) {
        logprintf("Error: No samples remaining after main filters.\n");
        return kRetInconsistentInput;
      }
      KeepSamples(ds, keep);
    }
  }
  if (c.missing_report) {
    const int mrc = WriteMissingReports(c, ds);
    if (mrc) return mrc;
  }
  if (f.geno < 1.0 || f.min_maf != 0.0 || f.max_maf != 1.0 || f.min_mac || f.max_mac != ~0ull) {
    VariantGenoCounts vc;
    const int rc = CountGenotypes(ds, threads, &vc, nullptr, nullptr, &err, c.nonfounders);
    if (rc) {
      logprintf("Error: %s\n", err.c_str());
      return rc;
    }
    const SampleInfo& S = ds->samples;
    const VariantInfo& V = ds->variants;
    const uint32_t n = S.size(), m = V.size();
    uint32_t male_ct = 0, founder_ct = 0, founder_male_ct = 0;
    for (uint32_t k = 0; k < n; ++k) {
      male_ct += S.sex[k] == 1;
      founder_ct += S.is_founder[k] != 0 || c.nonfounders;
      founder_male_ct += (S.is_founder[k] || c.nonfounders) && S.sex[k] == 1;
    }
    if ((f.min_mac || f.max_mac != ~0ull) && founder_ct != n) {  // plink2.cc:2102
      logprintf("Error: --mac/--max-mac specified, but with neither --ac-founders nor --nonfounders; and nonfounders are present.\n");
      return kRetInconsistentInput;
    }
    std::vector<uint8_t> keep(m, 1);
    uint32_t left = m;
    if (f.geno < 1.0) {
      const double thr = f.geno * (1 + eps);
      const uint32_t max_nony = static_cast<uint32_t>(static_cast<int32_t>(thr * static_cast<double>(n))), max_y = static_cast<uint32_t>(static_cast<int32_t>(thr * static_cast<double>(male_ct)));
      uint32_t removed = 0;
      for (uint32_t v = 0; v < m; ++v) {
        const bool is_y = V.chr_code[v] == 24;
        if ((is_y ? vc.male[4ull * v + 3] : vc.all[4ull * v + 3]) > (is_y ? max_y : max_nony)) {
          keep[v] = 0;
          ++removed;
        }
      }
      left -= removed;
      logprintf("--geno: %u variant%s removed due to missing genotype data.\n", removed, removed == 1 ? "" : "s");
    }
    if (f.min_maf != 0.0 || f.max_maf != 1.0 || f.min_mac || f.max_mac != ~0ull) {
      const bool freq_filter = f.min_maf != 0.0 || f.max_maf != 1.0;
      const double lo = f.min_maf * (1.0 - eps), hi = f.max_maf * (1.0 + eps);
      uint32_t removed = 0;
      for (uint32_t v = 0; v < m; ++v) {
        if (!keep[v]) continue;
        uint64_t alt_dd, tot_dd;
        FounderAlleleDd(vc, v, V.chr_code[v], founder_ct, founder_male_ct, &alt_dd, &tot_dd);
        bool drop = false;
        if (freq_filter) {
          double ref_freq = tot_dd ? static_cast<double>(tot_dd - alt_dd) * (1.0 / static_cast<double>(tot_dd)) : 0.5;
          if (!ds->read_ref_freq.empty() && ds->read_ref_freq[v] == ds->read_ref_freq[v]) ref_freq = ds->read_ref_freq[v];
          const double nonref = 1.0 - ref_freq, maf = nonref < ref_freq ? nonref : ref_freq;
          drop = (f.min_maf != 0.0 && maf < lo) || (f.max_maf < 1.0 && maf > hi);
        }
        if (!drop && (f.min_mac || f.max_mac != ~0ull)) {
          const uint64_t nonmajor = std::min(alt_dd, tot_dd - alt_dd);
          drop = (f.min_mac && nonmajor < f.min_mac) || (f.max_mac != ~0ull && nonmajor > f.max_mac);
        }
        if (drop) {
          keep[v] = 0;
          ++removed;
        }
      }
      left -= removed;
      logprintf("%u variant%s removed due to allele frequency threshold(s) (--maf/--max-maf/--mac/--max-mac).\n", removed, removed == 1 ? "" : "s");
    }
    if (!left) {
      logprintf("Error: No variants remaining after main filters.\n");
      return kRetInconsistentInput;
    }
    if (left != m) KeepVariants(ds, keep);
  }
  if (f.min_bp_space) {
    // within a chromosome a variant closer than the given distance to the last KEPT variant is removed
    const VariantInfo& V = ds->variants;
    const uint32_t m = V.size();
    std::vector<uint8_t> keep(m, 1);
    uint32_t removed = 0, last_bp = 0;
    for (uint32_t v = 0; v < m; ++v) {
      if (!v || V.chr_code[v] != V.chr_code[v - 1]) {
        last_bp = V.bp[v];
      } else if (V.bp[v] < last_bp + f.min_bp_space) {
        keep[v] = 0;
        ++removed;
      } else {
        last_bp = V.bp[v];
      }
    }
    logprintf("--bp-space: %u variant%s removed (%u remaining).\n", removed, removed == 1 ? "" : "s", m - removed);
    if (removed) KeepVariants(ds, keep);
  }
  return 0;
}

int main(int argc, char** argv) {
  {
    const int dbg = DebugHooks(argc, argv);
    if (dbg >= 0) return dbg;
  }
  Cmd c;
  // the log file name depends on --out, so scan for it first
  for (int i = 1; i + 1 < argc; ++i)
    if (!strcmp(argv[i], "--out")) c.out = argv[i + 1];
  g_log = fopen((c.out + ".log").c_str(), "w");
  logprintf("plink2_b200: H100-native KING / GRM / PCA / --indep-pairwise (plink2 command-line face)\n");
  {
    std::string opts = "Options in effect:\n";
    for (int i = 1; i < argc; ++i) {
      if (argv[i][0] == '-' && argv[i][1] == '-') opts += std::string(i > 1 ? "\n" : "") + "  " + argv[i];
      else opts += std::string(" ") + argv[i];
    }
    logprintf("%s\n\n", opts.c_str());
  }
  int rc = ParseArgs(argc, argv, &c);
  if (rc) return rc;
  // CUDA initialisation (0.5 - 3 s on a cold box) runs beside the loading of the sample / variant files; runs that need
  // no device (file-driven --king-cutoff[-table], --make-bed, --write-snplist / --write-samples on their own) never start it
  const bool gpu_command = c.freq || c.r2_unphased || c.make_king || c.make_king_table || c.king_cutoff >= 0 || c.make_grm_bin || c.make_grm_list || c.make_grm_sparse || c.make_rel || c.pca || c.indep_pairwise || !c.score_file.empty() || !c.vscore_file.empty();
  const bool needs_gpu = gpu_command;
  Pl2GpuCtx* ctx = nullptr;
  int ctx_rc = 0;
  std::string ctx_err;
  std::thread ctx_thread;
  struct CtxJoin {
    std::thread* t;
    ~CtxJoin() {
      if (t->joinable()) t->join();
    }
  } ctx_join{&ctx_thread};
  if (needs_gpu) {
    ctx_thread = std::thread([&]() {
      ctx_rc = pl2gpu_ctx_create(c.device, &ctx);
      if (ctx_rc) ctx_err = pl2gpu_last_error();  // thread-local in the library: capture it here
    });
  }
  Dataset ds;
  std::string err;
  // --ped/--map: convert first (PedmapToPgen's role); the temporary fileset is removed when the run ends
  struct TempFileset {
    std::vector<std::string> paths;
    void Remove() {
      for (const std::string& p : paths) unlink(p.c_str());
      paths.clear();
    }
    ~TempFileset() { Remove(); }
  } temp_files;
  if (!c.ped.empty()) {
    const std::string prefix = c.pgen.substr(0, c.pgen.size() - 4);
    uint32_t pn = 0, pm = 0;
    rc = PedmapToBed(c.ped, c.map, prefix, &pn, &pm, &err);
    if (!c.keep_autoconv) temp_files.paths = {c.pgen, c.pvar, c.psam};
    if (rc) {
      logprintf("Error: %s\n", err.c_str());
      return rc;
    }
    logprintf("--pedmap: %u sample%s, %u variant%s; %s.bed + %s.bim + %s.fam written%s.\n", pn, pn == 1 ? "" : "s", pm, pm == 1 ? "" : "s", prefix.c_str(), prefix.c_str(), prefix.c_str(), c.keep_autoconv ? "" : " (temporary)");
  }
  if (!LoadSamples(c.psam, &ds.samples, &err) || !LoadVariants(c.pvar, &ds.variants, &err, c.allow_extra_chr)) {
    logprintf("Error: %s\n", err.c_str());
    return kRetOpenFail;
  }
  if (!ds.reader.Open(c.pgen, ds.samples.size(), ds.variants.size(), &err)) {
    logprintf("Error: %s\n", err.c_str());
    return kRetMalformedInput;
  }
  ds.variants.provisional_ref = ds.reader.nonref_flags_storage() == 2;
  uint32_t founder_ct = 0;
  for (uint8_t f : ds.samples.is_founder) founder_ct += f;
  logprintf("%u sample%s (%u founder%s) loaded from %s.\n", ds.samples.size(), ds.samples.size() == 1 ? "" : "s", founder_ct, founder_ct == 1 ? "" : "s", c.psam.c_str());
  logprintf("%u variant%s loaded from %s.\n", ds.variants.size(), ds.variants.size() == 1 ? "" : "s", c.pvar.c_str());
  if (!c.var_id_template.empty()) {
    // variant IDs from a template, assigned while the .pvar is loaded in the reference (plink2_pvar.cc VaridTemplate*):
    // before any ID-based filter.  Alleles longer than 23 characters are refused (--new-id-max-allele-len default).
    VariantInfo& V = ds.variants;
    uint32_t changed = 0;
    for (uint32_t v = 0; v < V.size(); ++v) {
      if (!c.var_id_all && V.id[v] != ".") continue;
      // the template sees the allele codes as written in the file: a '0' missing code stays '0' in the ID
      const std::string ref = (V.zero_allele[v] & 1) ? std::string("0") : V.ref[v];
      const std::string alt1 = (V.zero_allele[v] & 2) ? std::string("0") : V.alt[v].substr(0, V.alt[v].find(','));
      if (ref.size() > 23 || alt1.size() > 23) {
        logprintf("Error: Allele code of variant %u is longer than 23 characters; plink2_b200 does not implement --new-id-max-allele-len.\n", v + 1);
        return kRetInconsistentInput;
      }
      const bool ref_first = strcmp(ref.c_str(), alt1.c_str()) <= 0;
      std::string id;
      const std::string& t = c.var_id_template;
      for (size_t k = 0; k < t.size(); ++k) {
        if (t[k] == '@') id += ChrNameOut(V.chr_code[v], V.chr_name[v]);
        else if (t[k] == '#') id += std::to_string(V.bp[v]);
        else if (t[k] == '$' && k + 1 < t.size() && strchr("ra12", t[k + 1])) {
          const char sel = t[++k];
          id += sel == 'r' ? ref : sel == 'a' ? alt1 : ((sel == '1') == ref_first) ? ref : alt1;
        } else id += t[k];
      }
      V.id[v] = id;
      ++changed;
    }
    logprintf("--set-%s-var-ids: %u variant ID%s assigned.\n", c.var_id_all ? "all" : "missing", changed, changed == 1 ? "" : "s");
  }
  {  // .fam phenotype column of --make-bed: the first case/control or quantitative phenotype, typed over all loaded samples
    for (size_t p = 0; p < ds.samples.pheno_names.size() && ds.samples.fam_pheno.empty(); ++p) {
      PhenoOut po;
      if (!TypePheno(ds.samples.pheno_names[p], ds.samples.pheno_tokens[p], &po)) continue;
      if (po.categorical) continue;  // .fam files don't support categorical phenotypes (WriteFam, plink2_data.cc:1219)
      for (std::string& t : po.text)
        if (t == "NA") t = "-9";
      ds.samples.fam_pheno = std::move(po.text);
    }
  }
  if (c.filters.any()) {
    std::vector<std::string> flog;
    const int frc = ApplyFilters(c.filters, &ds, &flog, &err);
    for (const std::string& l : flog) logprintf("%s\n", l.c_str());
    if (frc) {
      logprintf("Error: %s\n", err.c_str());
      return frc;
    }
  }
  if (c.indep_pairwise && !c.bad_ld) {
    // plink2.cc:2065: checked once the main filters ran and BEFORE any relatedness prune - a --king-cutoff that
    // leaves fewer than 50 founders does not stop the LD prune chained behind it
    uint32_t fct = 0;
    for (uint8_t f : ds.samples.is_founder) fct += f;
    if (fct < 50) {
      logprintf("Error: This run estimates linkage disequilibrium between variants, but there are less than 50 %s to estimate from.  (Strictly speaking, you can also override this error with --bad-ld, but this is almost always a bad idea.)\n", ds.samples.size() < 50 ? "samples" : "founders");
      return kRetDegenerateData;
    }
  }
  if (!c.read_freq.empty()) {
    rc = LoadReadFreq(c, &ds);
    if (rc) return rc;
  }
  if (c.filters.any_count_filter() || c.missing_report) {
    rc = ApplyCountFilters(c, &ds);
    if (rc) return rc;
  }
  if (c.nonfounders && (c.r2_unphased || c.make_grm_bin || c.make_grm_list || c.make_grm_sparse || c.make_rel || c.pca || c.indep_pairwise || !c.score_file.empty() || !c.vscore_file.empty())) {
    // --nonfounders: allele frequencies from every sample (plink2.cc:2301).  One host counting pass, frozen as per-variant
    // overrides (the --read-freq mechanism) so that every later command - whose own founder-only estimate would differ -
    // uses them; entries loaded with --read-freq keep precedence.
    VariantGenoCounts vc;
    rc = CountGenotypes(&ds, EffectiveHostThreads(c.threads), &vc, nullptr, nullptr, &err, true);
    if (rc) {
      logprintf("Error: %s\n", err.c_str());
      return rc;
    }
    uint32_t male_ct = 0;
    for (uint8_t sx : ds.samples.sex) male_ct += sx == 1;
    if (ds.read_ref_freq.empty()) ds.read_ref_freq.assign(ds.variants.size(), std::numeric_limits<double>::quiet_NaN());
    for (uint32_t v = 0; v < ds.variants.size(); ++v) {
      if (ds.read_ref_freq[v] == ds.read_ref_freq[v]) continue;
      uint64_t alt_dd, tot_dd;
      FounderAlleleDd(vc, v, ds.variants.chr_code[v], ds.samples.size(), male_ct, &alt_dd, &tot_dd);
      ds.read_ref_freq[v] = tot_dd ? static_cast<double>(tot_dd - alt_dd) * (1.0 / static_cast<double>(tot_dd)) : 0.5;
    }
  }
  if (c.write_snplist) {  // WriteSnplist / --write-samples (plink2.cc:2030-2062): what the main filters left
    OutFile f;
    const std::string name = c.out + ".snplist";
    if (!f.Open(name)) return kRetOpenFail;
    for (const std::string& id : ds.variants.id) {
      f.Write(id.data(), id.size());
      f.Write("\n", 1);
    }
    if (!f.Close()) return kRetWriteFail;
    logprintf("--write-snplist: Variant IDs written to %s .\n", name.c_str());
  }
  if (c.write_samples) {
    const std::string name = c.out + ".id";
    if (!WriteAllIds(name, ds.samples, true)) return kRetWriteFail;
    logprintf("--write-samples: Sample IDs written to %s .\n", name.c_str());
  }
  g_clock.Mark("load .psam/.pvar, open .pgen");
  // ---- relatedness prune from a file, then the commands that see its survivors (Plink2Core order, plink2.cc:2523-2581)
  std::vector<uint8_t> cutoff_removed;
  const bool later_gpu_command = c.r2_unphased || c.make_grm_bin || c.make_grm_list || c.make_grm_sparse || c.make_rel || c.pca || c.indep_pairwise || !c.score_file.empty() || !c.vscore_file.empty();
  if (!c.king_cutoff_table.empty() || !c.king_cutoff_prefix.empty()) {
    if (!c.king_cutoff_table.empty() && (c.king_cutoff >= 0 || !c.king_cutoff_prefix.empty())) {
      logprintf("Error: --king-cutoff cannot be used with --king-cutoff-table.\n");
      return kRetInvalidCmdline;
    }
    if (c.make_king || c.make_king_table || c.king_cutoff >= 0) {
      logprintf("Error: file-driven --king-cutoff[-table] cannot be combined with --make-king[-table] in plink2_b200.\n");
      return kRetInvalidCmdline;
    }
    rc = c.king_cutoff_table.empty() ? RunKingCutoffBinary(c, &ds, &cutoff_removed) : RunKingCutoffTable(c, &ds, &cutoff_removed);
    if (rc) return rc;
  }
  auto write_bed = [&]() -> int {
    std::vector<uint64_t> finc;
    uint32_t fct = 0;
    if (c.debug_founders_bed) {
      finc.assign((ds.samples.size() + 63) / 64, 0);
      for (uint32_t k = 0; k < ds.samples.size(); ++k) {
        if (ds.samples.is_founder[k]) {
          finc[k / 64] |= 1ull << (k % 64);
          ++fct;
        }
      }
    }
    const int wrc = WriteBedFileset(&ds, c.out, EffectiveHostThreads(c.threads), &err, c.debug_founders_bed ? finc.data() : nullptr, fct);
    if (wrc) {
      logprintf("Error: %s\n", err.c_str());
      return wrc;
    }
    logprintf("--make-bed: %s.bed + %s.bim + %s.fam written.\n", c.out.c_str(), c.out.c_str(), c.out.c_str());
    return 0;
  };
  auto write_pgen = [&]() -> int {
    if (ds.reader.nonref_flags_storage() == 3) {
      logprintf("Error: --make-pgen from a .pgen with per-variant provisional-REF flags is not supported by plink2_b200.\n");
      return kRetNotYetSupported;
    }
    const int wrc = WritePgenFileset(&ds, c.out, EffectiveHostThreads(c.threads), ds.reader.nonref_flags_storage() != 1, &err);
    if (wrc) {
      logprintf("Error: %s\n", err.c_str());
      return wrc;
    }
    logprintf("--make-pgen: %s.pgen + %s.pvar + %s.psam written.\n", c.out.c_str(), c.out.c_str(), c.out.c_str());
    return 0;
  };
  auto any_removed = [&]() { return std::find(cutoff_removed.begin(), cutoff_removed.end(), 1) != cutoff_removed.end(); };
  auto drop_removed = [&]() {
    std::vector<uint8_t> keep(cutoff_removed.size());
    for (size_t k = 0; k < keep.size(); ++k) keep[k] = !cutoff_removed[k];
    KeepSamples(&ds, keep);
    cutoff_removed.clear();
  };
  if (!needs_gpu) {
    if (c.make_bed || c.make_pgen) {
      if (any_removed()) drop_removed();
      rc = c.make_bed ? write_bed() : 0;
      if (!rc && c.make_pgen) rc = write_pgen();
      if (rc) return rc;
    }
    return 0;  // host-only run (the ID lists were written above); these steps need no device in the reference either
  }
  g_decode_threads = EffectiveHostThreads(c.threads);
  if (ctx_thread.joinable()) ctx_thread.join();
  if (ctx_rc || !ctx) {
    logprintf("Error: GPU initialisation failed: %s\n", ctx_err.c_str());
    return kRetGpuFail;
  }
  g_clock.Mark("pl2gpu_ctx_create (overlapped with the file loading above)");
  if (c.freq) {
    rc = RunFreq(c, &ds, ctx);  // before any relatedness prune, like the reference's LoadAlleleAndGenoCounts stage
    if (rc) return rc;
  }
  bool rel_check_pairs = false;
  if (c.king_rel_check && c.king_table_subset.empty()) {
    // with a single FID in the dataset the modifier has no effect (the reference warns and computes the full table)
    for (uint32_t k = 1; k < ds.samples.size() && !rel_check_pairs; ++k) rel_check_pairs = ds.samples.fid[k] != ds.samples.fid[0];
    if (!rel_check_pairs) logprintf("Warning: --make-king-table 'rel-check' modifier has no effect since only one FID is present.\n");
  }
  if (!c.king_table_subset.empty() || rel_check_pairs || (!c.king_table_require.empty() && c.make_king_table)) {
    if (!c.make_king_table || c.make_king || c.king_cutoff >= 0) {
      logprintf("Error: --king-table-subset must be used with --make-king-table (and without --make-king / --king-cutoff).\n");
      return kRetInvalidCmdline;
    }
    rc = RunKingSubset(c, &ds, ctx, rel_check_pairs);
    if (rc) return rc;
  } else if (c.make_king || c.make_king_table || c.king_cutoff >= 0) {
    rc = RunKing(c, &ds, ctx, &cutoff_removed);
    if (rc) return rc;
  }
  if (any_removed() && (later_gpu_command || c.make_bed || c.make_pgen)) {
    // The commands after a relatedness prune see the surviving samples, but keep the allele frequencies estimated
    // BEFORE it: the reference computes allele_freqs once (plink2.cc:2280-2304) and only narrows sample_include /
    // founder_info afterwards (UpdateSampleSubsets, :2580).  Freeze those frequencies as per-variant overrides
    // (the --read-freq mechanism), then drop the samples from the view.
    if (later_gpu_command) {
      std::vector<uint64_t> alt_dd, tot_dd;
      rc = FounderAlleleDosages(&ds, ctx, AllVariants(ds), &alt_dd, &tot_dd);
      if (rc) return rc;
      if (ds.read_ref_freq.empty()) ds.read_ref_freq.assign(ds.variants.size(), std::numeric_limits<double>::quiet_NaN());
      for (uint32_t v = 0; v < ds.variants.size(); ++v) {
        if (ds.read_ref_freq[v] == ds.read_ref_freq[v]) continue;
        ds.read_ref_freq[v] = tot_dd[v] ? static_cast<double>(tot_dd[v] - alt_dd[v]) * (1.0 / static_cast<double>(tot_dd[v])) : 0.5;
      }
    }
    drop_removed();
    logprintf("%u sample%s remaining after the relatedness prune.\n", ds.samples.size(), ds.samples.size() == 1 ? "" : "s");
  }
  if (c.make_bed) {
    rc = write_bed();
    if (rc) return rc;
  }
  if (c.make_pgen) {
    rc = write_pgen();
    if (rc) return rc;
  }
  if (!c.score_file.empty()) {
    rc = RunScore(c, &ds, ctx);
    if (rc) return rc;
  }
  if (!c.vscore_file.empty()) {
    rc = RunVscore(c, &ds, ctx);
    if (rc) return rc;
  }
  {
    GrmJob grm_job;  // exact --pca's matrix, ended before the commands below
    const bool exact_pca = c.pca && !c.pca_approx;
    if (c.make_grm_bin || c.make_grm_list || c.make_grm_sparse || c.make_rel || exact_pca) {
      if (exact_pca && c.parallel_tot != 1) {
        logprintf("Error: --pca cannot be used with --parallel.\n");
        return kRetInvalidCmdline;
      }
      rc = RunGrm(c, &ds, ctx, exact_pca, &grm_job);
      if (rc) return rc;
    }
    if (c.pca) {
      rc = RunPca(c, &ds, ctx, grm_job.get());
      if (rc) return rc;
    }
  }
  if (c.indep_pairwise) {
    rc = RunLdPrune(c, &ds, ctx);
    if (rc) return rc;
  }
  if (c.r2_unphased) {
    rc = RunR2Unphased(c, &ds, ctx);
    if (rc) return rc;
  }
  pl2gpu_ctx_synchronize(ctx);
  g_clock.Mark("commands done");
  time_t now = time(nullptr);
  logprintf("End time: %s", ctime(&now));
  if (g_log) fclose(g_log);
  fflush(stdout);
  fflush(stderr);
  // All output files are closed.  Skip the explicit CUDA teardown (context destroy + pinned-memory
  // unmapping cost ~1.4 s here); the driver reclaims the device when the process exits.
  temp_files.Remove();
  _exit(0);
}
