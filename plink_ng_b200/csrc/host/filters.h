// filters.h - the sample / variant filters in front of the pairwise-genotype commands, and the .bed fileset writer
// that pins them.  In the reference every command receives sample_include / variant_include bitsets prepared by
// Plink2Core (2.0/plink2.cc:1423-1665: --chr / --not-chr / --autosome[-xy] at load, --extract / --exclude by ID,
// then --keep-fam, --keep, --remove-fam, --remove); here the same filters compact the Dataset tables and install the
// matching view in the PgenReader, so every command driver simply sees a smaller dataset.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "dataset.h"

namespace pl2host {

struct FilterSpec {
  std::vector<std::string> keep, remove, keep_fam, remove_fam;  // ID files (LoadSampleIds, plink2_common.cc:1707)
  std::vector<std::string> extract, exclude;                    // variant-ID token files (TokenExtractExclude)
  std::vector<uint8_t> chr_mask, not_chr_mask;                  // 27 flags each when the flag was given
  bool autosome = false, autosome_xy = false;
  uint32_t min_alleles = 0, max_alleles = 0xFFFFFFFFu;  // --min-alleles / --max-alleles (LoadPvar, plink2_pvar.cc:1939-1952)
  int snps_only = 0;                      // 1 --snps-only, 2 --snps-only just-acgt (LoadPvar, plink2_pvar.cc:1917-1931)
  int64_t from_bp = -1, to_bp = -1;       // --from-bp/-kb/-mb, --to-bp/-kb/-mb: with --chr naming one chromosome (plink2.cc:764-787)
  bool excl_males = false, excl_females = false, excl_nosex = false;  // --keep-males / --remove-females / ... (plink2.cc:1688)
  int founders_only = 0;                                               // 1 --keep-founders, 2 --keep-nonfounders (:1705)
  // thresholds on genotype counts (applied after --read-freq was loaded; plink2.cc:1748, :2338, :2460)
  double mind = 1.0, geno = 1.0, min_maf = 0.0, max_maf = 1.0;
  uint64_t min_mac = 0, max_mac = ~0ull;  // allele counts (the reference's ddosage bounds / 32768)
  uint32_t min_bp_space = 0;              // --bp-space: applied last (EnforceMinBpSpace, plink2_filter.cc:3904; plink2.cc:2479)
  bool any_count_filter() const { return mind < 1.0 || geno < 1.0 || min_maf != 0.0 || max_maf != 1.0 || min_mac || max_mac != ~0ull || min_bp_space; }
  bool any() const {
    if (excl_males || excl_females || excl_nosex || founders_only) return true;
    return any_id_filter();
  }
  bool any_id_filter() const { return !(keep.empty() && remove.empty() && keep_fam.empty() && remove_fam.empty() && extract.empty() && exclude.empty() && chr_mask.empty() && not_chr_mask.empty()) || autosome || autosome_xy || min_alleles || max_alleles != 0xFFFFFFFFu || snps_only || from_bp != -1 || to_bp != -1; }
};

// "1-4,22,X" style arguments (ParseChrRanges, plink2_common.cc:3695) -> 27 flags.  False + *err on a bad token.
bool ParseChrList(const std::vector<std::string>& args, const char* flag, std::vector<uint8_t>* mask, std::string* err);

// Applies the filters in the reference's order.  Log lines ("--keep: 61 samples remaining.") are appended to *log.
// Returns 0, or a PglErr-valued code with *err set (3 open failure, 6 malformed file, 7 nothing left).
int ApplyFilters(const FilterSpec& spec, Dataset* ds, std::vector<std::string>* log, std::string* err);

// Genotype counts of the current view, one host pass (the roles of LoadSampleMissingCts and LoadAlleleAndGenoCounts,
// 2.0/plink2_data.cc, for hard calls).  Per variant [4]: code counts 0 / 1 / 2 / 3 over the named sample set.
struct VariantGenoCounts {
  std::vector<uint32_t> all, male;                            // every sample; males (chrY missingness)
  std::vector<uint32_t> founder, founder_male, founder_nonfemale;  // allele-frequency sets (autosomes / chrX / chrY)
};
// sample_missing[k]: missing calls of sample k over all variants, chrY variants counted for males only (then
// *variant_ct_y = number of chrY variants).  Either output may be null.
// all_as_founders (--nonfounders): the three "founder" sets are taken over every sample.
int CountGenotypes(Dataset* ds, uint32_t thread_ct, VariantGenoCounts* vc, std::vector<uint32_t>* sample_missing, uint32_t* variant_ct_y, std::string* err, bool all_as_founders = false);
// REF allele "ddosage" pair of a variant from those counts (the numbers behind --freq; see RunFreq)
void FounderAlleleDd(const VariantGenoCounts& vc, uint32_t v, uint32_t chr_code, uint32_t founder_ct, uint32_t founder_male_ct, uint64_t* alt_dd, uint64_t* tot_dd);

// Marks the samples named in one or more ID files read like --keep files (LoadSampleIds with kfLoadSampleIdsMultifile,
// plink2_common.cc:1707: the lists are merged): (*marked)[k] = 1.  `flag` names the option in messages.  Returns 0, or 3
// (open failure) / 6 (malformed file) with *err set.  *dup_ct counts IDs named more than once.
int MarkSampleIds(const std::vector<std::string>& files, const char* flag, const SampleInfo& S, std::vector<uint8_t>* marked, uint64_t* dup_ct, std::string* err);

// keep[k] != 0: sample / variant k (current numbering) stays.  Compacts the tables and updates the reader view.
void KeepSamples(Dataset* ds, const std::vector<uint8_t>& keep);
void KeepVariants(Dataset* ds, const std::vector<uint8_t>& keep);

// --make-bed (MakePlink2NoVsort -> .bed/.bim/.fam writers, 2.0/plink2_data.cc): the current view as a PLINK 1 binary
// fileset.  Host-only.  Returns 0 or a code with *err set.  With `sample_include` (bitset over the view's samples,
// include_ct set bits) only the .bed of that subset is written: the test hook for the subset-of-a-view decode that
// the founder-only commands (LD prune, allele frequencies) use.
int WriteBedFileset(Dataset* ds, const std::string& out_prefix, uint32_t thread_ct, std::string* err, const uint64_t* sample_include = nullptr, uint32_t include_ct = 0);

// --make-pgen (host-only): the current view as <prefix>.pgen in the fixed-width storage mode 0x02 (pgen_spec.tex:137-139:
// 12-byte header, then ceil(n / 4) bytes of 2-bit hard calls per variant - no compression, every reader accepts it) with
// <prefix>.pvar (#CHROM POS ID REF ALT [CM], CM only when a nonzero value exists) and <prefix>.psam ([#FID] IID [PAT MAT]
// SEX [PHENO1], FID / parents only when some value is not 0; the column rules of the reference's writers).
// provisional_ref: header bits 6-7 (2 = every REF allele provisional, 1 = all trusted).
int WritePgenFileset(Dataset* ds, const std::string& out_prefix, uint32_t thread_ct, bool provisional_ref, std::string* err);

}  // namespace pl2host
