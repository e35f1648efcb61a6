#include "filters.h"

#include <algorithm>
#include <cstring>
#include <thread>
#include <unordered_map>
#include <unordered_set>

#include "text_util.h"

namespace pl2host {

namespace {

template <class T>
void Compact(std::vector<T>* v, const std::vector<uint8_t>& keep) {
  if (v->empty()) return;
  size_t w = 0;
  for (size_t k = 0; k < keep.size(); ++k) {
    if (keep[k]) {
      if (w != k) (*v)[w] = std::move((*v)[k]);
      ++w;
    }
  }
  v->resize(w);
}

void InstallView(Dataset* ds) {
  std::vector<uint64_t> sample_keep;
  if (!ds->sample_raw.empty()) {
    sample_keep.assign((static_cast<size_t>(ds->reader.raw_sample_ct()) + 63) / 64, 0);
    for (uint32_t r : ds->sample_raw) sample_keep[r >> 6] |= 1ull << (r & 63);
  }
  ds->reader.SetView(ds->variant_raw, std::move(sample_keep), static_cast<uint32_t>(ds->sample_raw.size()));
}

std::string Plural(uint32_t n, const char* noun) { return std::to_string(n) + " " + noun + (n == 1 ? "" : "s"); }

// One --keep / --remove style file (LoadSampleIds, plink2_common.cc:1770-1846): optional "#FID IID [SID]" / "#IID
// [SID]" header (other '#' lines before it are skipped); without one, "FID IID" lines, or a lone IID that is read with
// FID 0.  IDs without a FID column carry FID 0 (XidRead, :1280), so they only name samples whose own FID is 0.  A SID
// column is compared only when the dataset has SIDs; otherwise every sample with that FID + IID is marked.
int MarkSampleFile(const std::string& path, const char* flag, const SampleInfo& S, const std::unordered_multimap<std::string, uint32_t>& by_id, std::vector<uint8_t>* seen, uint64_t* dup_ct, std::string* err) {
  std::vector<std::string> lines;
  if (!ReadLines(path, &lines, err)) return 3;
  size_t li = 0;
  auto is_id_header = [](const std::string& l) {
    if (l.size() < 4 || l[0] != '#') return false;
    const std::string t = l.substr(1, 3);
    return (t == "FID" || t == "IID") && (l.size() == 4 || l[4] == ' ' || l[4] == '\t');
  };
  while (li < lines.size() && (lines[li].empty() || (lines[li][0] == '#' && !is_id_header(lines[li])))) ++li;
  if (li == lines.size()) return 0;  // empty file: nothing named
  bool fid_col = true, sid_col = false, headerless = true;
  if (lines[li][0] == '#') {
    headerless = false;
    const std::vector<std::string> h = SplitWs(lines[li].substr(1));
    size_t t = 0;
    fid_col = h[0] == "FID";
    if (fid_col) ++t;
    if (t >= h.size() || h[t] != "IID") {
      *err = "No IID column on line " + std::to_string(li + 1) + " of --" + flag + " file.";
      return 6;
    }
    ++t;
    sid_col = t < h.size() && h[t] == "SID";
    ++li;
  }
  const bool use_sid = sid_col && S.sid_present;
  for (; li < lines.size(); ++li) {
    if (lines[li].empty()) continue;
    const std::vector<std::string> t = SplitWs(lines[li]);
    if (t.empty()) continue;
    std::string fid = "0", iid, sid;
    if (headerless) {
      if (t.size() >= 2) {
        fid = t[0];
        iid = t[1];
      } else {
        iid = t[0];
      }
    } else {
      size_t q = 0;
      if (t.size() < static_cast<size_t>(fid_col ? 2 : 1) + (sid_col ? 1 : 0)) {
        *err = std::string("--") + flag + ": Line " + std::to_string(li + 1) + " of " + path + " has fewer tokens than expected.";
        return 6;
      }
      if (fid_col) fid = t[q++];
      iid = t[q++];
      if (sid_col) sid = t[q++];
    }
    const auto range = by_id.equal_range(fid + "\t" + iid);
    bool first = true;
    for (auto it = range.first; it != range.second; ++it) {
      const uint32_t k = it->second;
      if (use_sid && S.sid[k] != sid) continue;
      if (first && (*seen)[k]) {
        ++*dup_ct;
        break;
      }
      first = false;
      (*seen)[k] = 1;
    }
  }
  return 0;
}

// --keep-fam / --remove-fam files: the first token of every line is a family ID (LoadSampleIds kfLoadSampleIdsFamOnly,
// :1821-1845); no header handling.
int MarkFamilyFile(const std::string& path, const SampleInfo& S, const std::unordered_multimap<std::string, uint32_t>& by_fid, std::vector<uint8_t>* seen, uint64_t* dup_ct, std::string* err) {
  std::vector<std::string> lines;
  if (!ReadLines(path, &lines, err)) return 3;
  for (size_t li = 0; li < lines.size(); ++li) {
    const std::vector<std::string> t = SplitWs(lines[li]);
    if (t.empty()) continue;
    const auto range = by_fid.equal_range(t[0]);
    bool first = true;
    for (auto it = range.first; it != range.second; ++it) {
      if (first && (*seen)[it->second]) {
        ++*dup_ct;
        break;
      }
      first = false;
      (*seen)[it->second] = 1;
    }
  }
  return 0;
}

}  // namespace

int MarkSampleIds(const std::vector<std::string>& files, const char* flag, const SampleInfo& S, std::vector<uint8_t>* marked, uint64_t* dup_ct, std::string* err) {
  const uint32_t n = S.size();
  std::unordered_multimap<std::string, uint32_t> index;
  index.reserve(static_cast<size_t>(n) * 2);
  for (uint32_t k = n; k--;) index.emplace(S.fid[k] + "\t" + S.iid[k], k);
  marked->assign(n, 0);
  *dup_ct = 0;
  for (const std::string& path : files) {
    const int rc = MarkSampleFile(path, flag, S, index, marked, dup_ct, err);
    if (rc) return rc;
  }
  return 0;
}

bool ParseChrList(const std::vector<std::string>& args, const char* flag, std::vector<uint8_t>* mask, std::string* err) {
  mask->assign(27, 0);
  std::string joined;
  for (const std::string& a : args) joined += (joined.empty() ? "" : ",") + a;
  size_t pos = 0;
  while (pos <= joined.size()) {
    size_t end = joined.find(',', pos);
    if (end == std::string::npos) end = joined.size();
    const std::string tok = joined.substr(pos, end - pos);
    pos = end + 1;
    if (tok.empty()) continue;
    const size_t dash = tok.find('-');
    uint32_t c0, c1;
    if (dash == std::string::npos) {
      if (!ParseChr(tok, &c0)) {
        *err = std::string("Invalid --") + flag + " chromosome code '" + tok + "'.";
        return false;
      }
      (*mask)[c0] = 1;
      continue;
    }
    const std::string a = tok.substr(0, dash), b = tok.substr(dash + 1);
    if (!ParseChr(a, &c0) || !ParseChr(b, &c1)) {
      *err = std::string("Invalid --") + flag + " parameter '" + tok + "'.";
      return false;
    }
    if (c1 > 22) {
      *err = std::string("--") + flag + " chromosome code '" + b + "' cannot be the end of a range.";
      return false;
    }
    if (c1 <= c0) {
      *err = std::string("--") + flag + " chromosome code '" + b + "' is not greater than '" + a + "'.";
      return false;
    }
    for (uint32_t c = c0; c <= c1; ++c) (*mask)[c] = 1;
  }
  return true;
}

void KeepSamples(Dataset* ds, const std::vector<uint8_t>& keep) {
  SampleInfo& S = ds->samples;
  if (ds->sample_raw.empty()) {
    ds->sample_raw.resize(S.size());
    for (uint32_t k = 0; k < S.size(); ++k) ds->sample_raw[k] = k;
  }
  Compact(&ds->sample_raw, keep);
  Compact(&S.fid, keep);
  Compact(&S.iid, keep);
  Compact(&S.sid, keep);
  Compact(&S.pat, keep);
  Compact(&S.mat, keep);
  Compact(&S.is_founder, keep);
  Compact(&S.sex, keep);
  Compact(&S.fam_pheno, keep);
  for (auto& col : S.pheno_tokens) Compact(&col, keep);
  InstallView(ds);
}

void KeepVariants(Dataset* ds, const std::vector<uint8_t>& keep) {
  VariantInfo& V = ds->variants;
  if (ds->variant_raw.empty()) {
    ds->variant_raw.resize(V.size());
    for (uint32_t k = 0; k < V.size(); ++k) ds->variant_raw[k] = k;
  }
  Compact(&ds->variant_raw, keep);
  Compact(&V.chr_code, keep);
  Compact(&V.bp, keep);
  Compact(&V.id, keep);
  Compact(&V.chr_name, keep);
  Compact(&V.ref, keep);
  Compact(&V.alt, keep);
  Compact(&V.cm, keep);
  Compact(&V.zero_allele, keep);
  Compact(&ds->read_ref_freq, keep);
  InstallView(ds);
}

int ApplyFilters(const FilterSpec& spec, Dataset* ds, std::vector<std::string>* log, std::string* err) {
  // (count-based thresholds are applied by the caller after --read-freq: ApplyCountFilters in the host program)
  // ---- variants: chromosome flags (applied while the reference loads the .pvar), then --extract, then --exclude
  {
    const VariantInfo& V = ds->variants;
    const uint32_t m = V.size();
    std::vector<uint8_t> keep(m, 1);
    bool changed = false;
    if (!spec.chr_mask.empty() || !spec.not_chr_mask.empty() || spec.autosome || spec.autosome_xy) {
      uint32_t left = 0;
      for (uint32_t v = 0; v < m; ++v) {
        const uint32_t c = V.chr_code[v];
        bool ok = true;
        if (!spec.chr_mask.empty()) ok = c < 27 && spec.chr_mask[c];
        if (spec.autosome || spec.autosome_xy) ok = ok && ((c >= 1 && c <= 22) || (spec.autosome_xy && c == 25));
        if (!spec.not_chr_mask.empty() && c < 27 && spec.not_chr_mask[c]) ok = false;
        keep[v] = ok;
        left += ok;
      }
      log->push_back(std::to_string(m - left) + " variant" + (m - left == 1 ? "" : "s") + " excluded by chromosome filter, " + std::to_string(left) + " remaining.");
      changed = true;
    }
    if (spec.min_alleles || spec.max_alleles != 0xFFFFFFFFu) {
      // allele count = REF + comma-separated ALTs; a lone missing ALT code counts as no ALT allele (:1944-1948).  This is
      // what lets a file with some multiallelic records through: "--max-alleles 2" drops them before anything is decoded.
      uint32_t left = 0;
      for (uint32_t v = 0; v < m; ++v) {
        if (keep[v]) {
          const std::string& alt = V.alt[v];
          uint32_t ct = 2 + static_cast<uint32_t>(std::count(alt.begin(), alt.end(), ','));
          if (alt == ".") ct = 1;
          keep[v] = ct >= spec.min_alleles && ct <= spec.max_alleles;
          left += keep[v];
        }
      }
      log->push_back(std::to_string(m - left) + " variant" + (m - left == 1 ? "" : "s") + " excluded by --min-alleles / --max-alleles, " + std::to_string(left) + " remaining.");
      changed = true;
    }
    if (spec.snps_only) {
      auto acgt_or_missing = [](char ch) { return ch == '.' || ch == '0' || strchr("ACGTacgt", ch) != nullptr; };
      uint32_t left = 0;
      for (uint32_t v = 0; v < m; ++v) {
        if (keep[v]) {
          bool ok = V.ref[v].size() == 1 && V.alt[v].size() == 1;
          if (ok && spec.snps_only == 2) ok = acgt_or_missing(V.ref[v][0]) && acgt_or_missing(V.alt[v][0]);
          keep[v] = ok;
          left += ok;
        }
      }
      log->push_back("--snps-only: " + Plural(left, "variant") + " remaining.");
      changed = true;
    }
    if (spec.from_bp != -1 || spec.to_bp != -1) {
      uint32_t left = 0;
      for (uint32_t v = 0; v < m; ++v) {
        if (keep[v]) {
          const int64_t bp = V.bp[v];
          keep[v] = (spec.from_bp == -1 || bp >= spec.from_bp) && (spec.to_bp == -1 || bp <= spec.to_bp);
          left += keep[v];
        }
      }
      log->push_back("--from-bp/--to-bp: " + Plural(left, "variant") + " remaining.");
      changed = true;
    }
    for (int pass = 0; pass < 2; ++pass) {
      const std::vector<std::string>& files = pass ? spec.exclude : spec.extract;
      if (files.empty()) continue;
      std::unordered_set<std::string> ids;
      for (const std::string& path : files) {
        std::vector<std::string> lines;
        if (!ReadLines(path, &lines, err)) return 3;
        for (const std::string& l : lines)
          for (std::string& t : SplitWs(l)) ids.insert(std::move(t));
      }
      uint32_t left = 0;
      for (uint32_t v = 0; v < m; ++v) {
        if (keep[v]) {
          const bool named = ids.count(V.id[v]) != 0;
          keep[v] = pass ? !named : named;
          left += keep[v];
        }
      }
      log->push_back(std::string(pass ? "--exclude: " : "--extract: ") + Plural(left, "variant") + " remaining.");
      changed = true;
    }
    if (changed) {
      if (std::find(keep.begin(), keep.end(), 1) == keep.end()) {
        *err = "No variants remaining after main filters.";
        return 7;
      }
      KeepVariants(ds, keep);
    }
  }
  // ---- samples: --keep-fam, --keep, --remove-fam, --remove (plink2.cc:1645-1668); each sees the survivors of the last
  struct Step {
    const std::vector<std::string>* files;
    const char* flag;
    bool fam, remove;
  };
  const Step steps[4] = {{&spec.keep_fam, "keep-fam", true, false}, {&spec.keep, "keep", false, false}, {&spec.remove_fam, "remove-fam", true, true}, {&spec.remove, "remove", false, true}};
  for (const Step& st : steps) {
    if (st.files->empty()) continue;
    const SampleInfo& S = ds->samples;
    const uint32_t n = S.size();
    std::unordered_multimap<std::string, uint32_t> index;
    index.reserve(static_cast<size_t>(n) * 2);
    // inserted in reverse so equal_range walks the samples of one key in file order (insertion puts later ones first)
    for (uint32_t k = n; k--;) index.emplace(st.fam ? S.fid[k] : (S.fid[k] + "\t" + S.iid[k]), k);
    std::vector<uint8_t> seen(n, 0);
    uint64_t dup_ct = 0;
    for (const std::string& path : *st.files) {
      const int rc = st.fam ? MarkFamilyFile(path, S, index, &seen, &dup_ct, err) : MarkSampleFile(path, st.flag, S, index, &seen, &dup_ct, err);
      if (rc) return rc;
    }
    if (st.remove)
      for (auto& f : seen) f = !f;
    uint32_t left = 0;
    for (uint8_t f : seen) left += f;
    log->push_back(std::string("--") + st.flag + ": " + Plural(left, "sample") + " remaining.");
    if (dup_ct) log->push_back("Warning: At least " + std::to_string(dup_ct) + " duplicate ID" + (dup_ct == 1 ? "" : "s") + " in --" + st.flag + " file(s).");
    if (!left) {
      *err = "No samples remaining after main filters.";
      return 7;
    }
    KeepSamples(ds, seen);
  }
  if (spec.excl_males || spec.excl_females || spec.excl_nosex) {
    const SampleInfo& S = ds->samples;
    std::vector<uint8_t> keep(S.size());
    uint32_t removed = 0;
    for (uint32_t k = 0; k < S.size(); ++k) {
      keep[k] = !((S.sex[k] == 1 && spec.excl_males) || (S.sex[k] == 2 && spec.excl_females) || (S.sex[k] == 0 && spec.excl_nosex));
      removed += !keep[k];
    }
    log->push_back(Plural(removed, "sample") + " removed due to sex filter(s).");
    if (removed == S.size()) {
      *err = "No samples remaining after main filters.";
      return 7;
    }
    if (removed) KeepSamples(ds, keep);
  }
  if (spec.founders_only) {
    const SampleInfo& S = ds->samples;
    std::vector<uint8_t> keep(S.size());
    uint32_t removed = 0;
    for (uint32_t k = 0; k < S.size(); ++k) {
      keep[k] = (S.is_founder[k] != 0) == (spec.founders_only == 1);
      removed += !keep[k];
    }
    log->push_back(std::string("--keep-") + (spec.founders_only == 1 ? "" : "non") + "founders: " + Plural(removed, "sample") + " removed.");
    if (removed == S.size()) {
      *err = "No samples remaining after main filters.";
      return 7;
    }
    if (removed) KeepSamples(ds, keep);
  }
  return 0;
}

int CountGenotypes(Dataset* ds, uint32_t thread_ct, VariantGenoCounts* vc, std::vector<uint32_t>* sample_missing, uint32_t* variant_ct_y, std::string* err, bool all_as_founders) {
  const SampleInfo& S = ds->samples;
  const VariantInfo& V = ds->variants;
  const uint32_t n = S.size(), m = V.size();
  const uint32_t words = PgenReader::WordsFor(n);
  // one 0b01 lane per member sample, in genovec layout (32 samples per word)
  enum { kAll, kMale, kFounder, kFounderMale, kFounderNonfemale, kSets };
  std::vector<uint64_t> lane[kSets];
  for (auto& l : lane) l.assign(words, 0);
  for (uint32_t k = 0; k < n; ++k) {
    const uint64_t bit = 1ull << (2 * (k & 31));
    const bool f = all_as_founders || S.is_founder[k] != 0;
    lane[kAll][k >> 5] |= bit;
    if (S.sex[k] == 1) lane[kMale][k >> 5] |= bit;
    if (f) lane[kFounder][k >> 5] |= bit;
    if (f && S.sex[k] == 1) lane[kFounderMale][k >> 5] |= bit;
    if (f && S.sex[k] != 2) lane[kFounderNonfemale][k >> 5] |= bit;
  }
  std::vector<uint32_t>* out[kSets] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  if (vc) {
    out[kAll] = &vc->all;
    out[kMale] = &vc->male;
    out[kFounder] = &vc->founder;
    out[kFounderMale] = &vc->founder_male;
    out[kFounderNonfemale] = &vc->founder_nonfemale;
    for (auto* o : out) o->assign(4ull * m, 0);
  }
  uint32_t set_size[kSets];
  for (int s = 0; s < kSets; ++s) {
    uint64_t c = 0;
    for (uint64_t w : lane[s]) c += static_cast<uint64_t>(__builtin_popcountll(w));
    set_size[s] = static_cast<uint32_t>(c);
  }
  if (sample_missing) sample_missing->assign(n, 0);
  uint32_t y_ct = 0;
  const uint32_t batch = 8192;
  std::vector<uint64_t> buf(static_cast<size_t>(batch) * words);
  std::vector<uint32_t> vidx(batch);
  thread_ct = std::max(1u, thread_ct);
  std::vector<std::vector<uint32_t>> miss_part(sample_missing ? thread_ct : 0, std::vector<uint32_t>(sample_missing ? n : 0, 0));
  const uint64_t kLo = 0x5555555555555555ull;
  for (uint32_t v0 = 0; v0 < m; v0 += batch) {
    const uint32_t cnt = std::min(batch, m - v0);
    for (uint32_t k = 0; k < cnt; ++k) vidx[k] = v0 + k;
    if (!ds->reader.GetBlock(vidx.data(), cnt, nullptr, n, buf.data(), words, thread_ct, err)) return 6;
    auto work = [&](uint32_t t) {
      const uint32_t k0 = static_cast<uint32_t>(static_cast<uint64_t>(cnt) * t / thread_ct), k1 = static_cast<uint32_t>(static_cast<uint64_t>(cnt) * (t + 1) / thread_ct);
      for (uint32_t k = k0; k < k1; ++k) {
        const uint64_t* row = buf.data() + static_cast<size_t>(k) * words;
        const uint32_t v = v0 + k;
        const bool is_y = V.chr_code[v] == 24;
        uint32_t c[kSets][3] = {};
        for (uint32_t w = 0; w < words; ++w) {
          const uint64_t g = row[w], lo = g & kLo, hi = (g >> 1) & kLo;
          const uint64_t het = lo & ~hi, alt = hi & ~lo, mis = lo & hi;
          if (vc) {
            for (int s = 0; s < kSets; ++s) {
              const uint64_t l = lane[s][w];
              c[s][0] += static_cast<uint32_t>(__builtin_popcountll(het & l));
              c[s][1] += static_cast<uint32_t>(__builtin_popcountll(alt & l));
              c[s][2] += static_cast<uint32_t>(__builtin_popcountll(mis & l));
            }
          }
          if (sample_missing) {
            uint64_t mm = mis & (is_y ? lane[kMale][w] : lane[kAll][w]);
            while (mm) {
              const uint32_t b = static_cast<uint32_t>(__builtin_ctzll(mm));
              ++miss_part[t][w * 32 + (b >> 1)];
              mm &= mm - 1;
            }
          }
        }
        if (vc) {
          for (int s = 0; s < kSets; ++s) {
            uint32_t* dst = out[s]->data() + 4ull * v;
            dst[1] = c[s][0];
            dst[2] = c[s][1];
            dst[3] = c[s][2];
            dst[0] = set_size[s] - c[s][0] - c[s][1] - c[s][2];
          }
        }
      }
    };
    std::vector<std::thread> th;
    for (uint32_t t = 1; t < thread_ct; ++t) th.emplace_back(work, t);
    work(0);
    for (auto& x : th) x.join();
    for (uint32_t k = 0; k < cnt; ++k) y_ct += V.chr_code[v0 + k] == 24;
  }
  if (sample_missing)
    for (const auto& part : miss_part)
      for (uint32_t k = 0; k < n; ++k) (*sample_missing)[k] += part[k];
  if (variant_ct_y) *variant_ct_y = y_ct;
  return 0;
}

void FounderAlleleDd(const VariantGenoCounts& vc, uint32_t v, uint32_t chr_code, uint32_t founder_ct, uint32_t founder_male_ct, uint64_t* alt_dd, uint64_t* tot_dd) {
  const uint32_t* f = &vc.founder[4ull * v];
  const uint64_t n0 = f[0], n1 = f[1], n2 = f[2], n3 = f[3];
  if (chr_code == 23) {  // nonmales twice, males once (a male het counts half of each allele)
    const uint32_t* mc = &vc.founder_male[4ull * v];
    *alt_dd = (4 * n2 + 2 * n1 - 2ull * mc[2] - mc[1]) * 16384ull;
    *tot_dd = (2 * (founder_ct - n3) - founder_male_ct + mc[3]) * 2 * 16384ull;
  } else if (chr_code == 24) {  // nonfemale founders, haploid
    const uint32_t* y = &vc.founder_nonfemale[4ull * v];
    *alt_dd = (y[1] + 2ull * y[2]) * 16384ull;
    *tot_dd = 2ull * (static_cast<uint64_t>(y[0]) + y[1] + y[2]) * 16384ull;
  } else if (chr_code == 26) {
    *alt_dd = (n1 + 2 * n2) * 16384ull;
    *tot_dd = 2 * (n0 + n1 + n2) * 16384ull;
  } else {
    *alt_dd = (n1 + 2 * n2) * 32768ull;
    *tot_dd = 2 * (n0 + n1 + n2) * 32768ull;
  }
}

int WriteBedFileset(Dataset* ds, const std::string& out_prefix, uint32_t thread_ct, std::string* err, const uint64_t* sample_include, uint32_t include_ct) {
  const SampleInfo& S = ds->samples;
  const VariantInfo& V = ds->variants;
  const uint32_t m = V.size();
  const uint32_t n = sample_include ? include_ct : S.size();
  char num[40];
  if (!sample_include) {  // .fam: FID IID PAT MAT SEX PHENO (WriteFam, plink2_data.cc:1209); a missing FID column is written as 0
    OutFile f;
    if (!f.Open(out_prefix + ".fam")) {
      *err = "Failed to open " + out_prefix + ".fam for writing.";
      return 3;
    }
    for (uint32_t k = 0; k < n; ++k) {
      std::string line = S.fid[k] + "\t" + S.iid[k] + "\t" + S.pat[k] + "\t" + S.mat[k] + "\t";
      line += static_cast<char>('0' + S.sex[k]);
      line += "\t" + (S.fam_pheno.empty() ? std::string("-9") : S.fam_pheno[k]) + "\n";
      f.Write(line.data(), line.size());
    }
    if (!f.Close()) {
      *err = "File write failure.";
      return 5;
    }
  }
  if (!sample_include) {  // .bim: CHROM ID CM POS ALT REF
    OutFile f;
    if (!f.Open(out_prefix + ".bim")) {
      *err = "Failed to open " + out_prefix + ".bim for writing.";
      return 3;
    }
    for (uint32_t v = 0; v < m; ++v) {
      std::string cm = "0";
      if (!V.cm.empty()) {
        char* endp = nullptr;
        const double d = strtod(V.cm[v].c_str(), &endp);
        if (endp != V.cm[v].c_str()) {
          *dtoa_g(d, num) = '\0';
          cm = num;
        }
      }
      const std::string line = ChrNameOut(V.chr_code[v], V.chr_name[v]) + "\t" + V.id[v] + "\t" + cm + "\t" + std::to_string(V.bp[v]) + "\t" + V.alt[v] + "\t" + V.ref[v] + "\n";
      f.Write(line.data(), line.size());
    }
    if (!f.Close()) {
      *err = "File write failure.";
      return 5;
    }
  }
  // .bed: magic 6c 1b 01, then ceil(n / 4) bytes per variant.  PLINK 2 codes (0 hom-REF, 1 het, 2 hom-ALT, 3 missing)
  // -> .bed codes (3, 2, 0, 1) (PgrPlink2ToPlink1InplaceUnsafe, pgenlib_misc); padding entries of the last byte are 0.
  uint8_t lut[256];
  for (uint32_t b = 0; b < 256; ++b) {
    static const uint8_t map[4] = {3, 2, 0, 1};
    lut[b] = static_cast<uint8_t>(map[b & 3] | (map[(b >> 2) & 3] << 2) | (map[(b >> 4) & 3] << 4) | (map[(b >> 6) & 3] << 6));
  }
  OutFile f;
  if (!f.Open(out_prefix + ".bed")) {
    *err = "Failed to open " + out_prefix + ".bed for writing.";
    return 3;
  }
  const uint8_t magic[3] = {0x6c, 0x1b, 0x01};
  f.Write(magic, 3);
  const uint32_t words = PgenReader::WordsFor(n), bytes = (n + 3) / 4;
  const uint8_t last_mask = (n & 3) ? static_cast<uint8_t>((1u << (2 * (n & 3))) - 1) : 0xFF;
  const uint32_t batch = 4096;
  std::vector<uint64_t> buf(static_cast<size_t>(batch) * words);
  std::vector<uint32_t> vidx(batch);
  std::vector<uint8_t> row(bytes);
  for (uint32_t v0 = 0; v0 < m; v0 += batch) {
    const uint32_t cnt = std::min(batch, m - v0);
    for (uint32_t k = 0; k < cnt; ++k) vidx[k] = v0 + k;
    if (!ds->reader.GetBlock(vidx.data(), cnt, sample_include, n, buf.data(), words, thread_ct, err)) return 6;
    for (uint32_t k = 0; k < cnt; ++k) {
      const uint8_t* src = reinterpret_cast<const uint8_t*>(buf.data() + static_cast<size_t>(k) * words);
      for (uint32_t b = 0; b < bytes; ++b) row[b] = lut[src[b]];
      row[bytes - 1] &= last_mask;
      f.Write(row.data(), bytes);
    }
  }
  if (!f.Close()) {
    *err = "File write failure.";
    return 5;
  }
  return 0;
}

int WritePgenFileset(Dataset* ds, const std::string& out_prefix, uint32_t thread_ct, bool provisional_ref, std::string* err) {
  const SampleInfo& S = ds->samples;
  const VariantInfo& V = ds->variants;
  const uint32_t n = S.size(), m = V.size();
  char num[40];
  {  // .psam
    bool any_fid = false, any_parent = false;
    for (uint32_t k = 0; k < n; ++k) {
      any_fid = any_fid || S.fid[k] != "0";
      any_parent = any_parent || S.pat[k] != "0" || S.mat[k] != "0";
    }
    OutFile f;
    if (!f.Open(out_prefix + ".psam")) {
      *err = "Failed to open " + out_prefix + ".psam for writing.";
      return 3;
    }
    std::string h = any_fid ? "#FID\tIID" : "#IID";
    if (S.sid_present) h += "\tSID";
    if (any_parent) h += "\tPAT\tMAT";
    h += "\tSEX";
    if (!S.fam_pheno.empty()) h += "\tPHENO1";
    h += "\n";
    f.Write(h.data(), h.size());
    for (uint32_t k = 0; k < n; ++k) {
      std::string line = any_fid ? (S.fid[k] + "\t" + S.iid[k]) : S.iid[k];
      if (S.sid_present) line += "\t" + S.sid[k];
      if (any_parent) line += "\t" + S.pat[k] + "\t" + S.mat[k];
      line += S.sex[k] == 1 ? "\t1" : S.sex[k] == 2 ? "\t2" : "\tNA";
      if (!S.fam_pheno.empty()) line += "\t" + (S.fam_pheno[k] == "-9" ? std::string("NA") : S.fam_pheno[k]);
      line += "\n";
      f.Write(line.data(), line.size());
    }
    if (!f.Close()) return 5;
  }
  {  // .pvar
    bool any_cm = false;
    for (const std::string& cm : V.cm) any_cm = any_cm || strtod(cm.c_str(), nullptr) != 0.0;
    OutFile f;
    if (!f.Open(out_prefix + ".pvar")) {
      *err = "Failed to open " + out_prefix + ".pvar for writing.";
      return 3;
    }
    f.Puts(any_cm ? "#CHROM\tPOS\tID\tREF\tALT\tCM\n" : "#CHROM\tPOS\tID\tREF\tALT\n");
    for (uint32_t v = 0; v < m; ++v) {
      std::string line = ChrNameOut(V.chr_code[v], V.chr_name[v]) + "\t" + std::to_string(V.bp[v]) + "\t" + V.id[v] + "\t" + V.ref[v] + "\t" + V.alt[v];
      if (any_cm) {
        *dtoa_g(strtod(V.cm[v].c_str(), nullptr), num) = '\0';
        line += std::string("\t") + num;
      }
      line += "\n";
      f.Write(line.data(), line.size());
    }
    if (!f.Close()) return 5;
  }
  OutFile f;
  if (!f.Open(out_prefix + ".pgen")) {
    *err = "Failed to open " + out_prefix + ".pgen for writing.";
    return 3;
  }
  uint8_t hdr[12] = {0x6c, 0x1b, 0x02, 0, 0, 0, 0, 0, 0, 0, 0, static_cast<uint8_t>(provisional_ref ? 0x80 : 0x40)};
  for (int b = 0; b < 4; ++b) {
    hdr[3 + b] = static_cast<uint8_t>(m >> (8 * b));
    hdr[7 + b] = static_cast<uint8_t>(n >> (8 * b));
  }
  f.Write(hdr, 12);
  const uint32_t words = PgenReader::WordsFor(n), bytes = (n + 3) / 4;
  const uint32_t batch = 4096;
  std::vector<uint64_t> buf(static_cast<size_t>(batch) * words);
  std::vector<uint32_t> vidx(batch);
  for (uint32_t v0 = 0; v0 < m; v0 += batch) {
    const uint32_t cnt = std::min(batch, m - v0);
    for (uint32_t k = 0; k < cnt; ++k) vidx[k] = v0 + k;
    if (!ds->reader.GetBlock(vidx.data(), cnt, nullptr, n, buf.data(), words, thread_ct, err)) return 6;
    for (uint32_t k = 0; k < cnt; ++k) f.Write(buf.data() + static_cast<size_t>(k) * words, bytes);  // trailing entries are already 0
  }
  if (!f.Close()) {
    *err = "File write failure.";
    return 5;
  }
  return 0;
}

}  // namespace pl2host
