// score.cu - `--score` accumulation: replaces the dosage expansion + dgemm / difflist updates of ScoreReport's worker
// (CalcScoreThread, 2.0/plink2_matrix_calc.cc:6467-6890, driven by ScoreReport :6892) for diploid hard calls: per
// sample the weighted sum  sum_v w_v[g_vs]  over the scored (variant, allele) entries, the sum of named-allele dosages
// and the number of missing calls.  The caller supplies, per entry, the four weights of the genotype codes
// (coefficient x named-allele dosage for codes 0/1/2, coefficient x 2 x allele frequency for a missing call - or 0
// with 'no-mean-imputation', :6605-6607) and the integer named-allele dosages, so centring / dominant / recessive
// variants are a matter of the table the caller builds.  A job carries score_ct coefficient columns
// (--score-col-nums): the weight table is [entry][score_ct][4], the columns are scored in groups of kScoreGroup per
// launch over the batch already staged, and every column's adds are those of a one-column job in the same order.
// chrX (--xchr-model 1), chrY and MT entries (pl2gpu_score_add_variants_ploidy) run through score_ploidy_kernel, which
// picks per sample a diploid or haploid table (or none: chrY females) from the sex masks and counts dosages in half
// allele units with diploid and haploid missing calls apart; runs of diploid entries keep score_kernel and its plan.
// A job may keep several accumulator sets, one per class (--q-score-range: the entries whose p-values lie in the same
// set of ranges): each staged batch is gathered into class-major order on the device (score_row_gather_kernel), and
// each (class, ploidy class) run goes through the same kernels and launch plan into its class's accumulators.  With
// pl2gpu_score_add_entries several entries (--score-list: one per file that scores the variant) read one staged row,
// which the gather copies once per entry.
//
// Streaming: every 32-bit word of a variant row (16 samples) is read once.  A CTA covers 128 words x a chunk of
// variants and writes per-chunk partial sums; a second kernel adds the partials in chunk order, so results do not
// depend on scheduling.  The fp64 adds go through a two-variant lookup table, the integer sums are bit-parallel.
#include <algorithm>
#include <memory>
#include <utility>
#include <vector>

#include "../../include/plink2_b200.h"
#include "common.cuh"

using namespace pl2;

namespace {

constexpr uint32_t kScoreThreads = 128;
constexpr uint32_t kScoreTile = 64;  // variants whose tables are staged in shared memory at a time (even)

// One thread owns one 32-bit word column (16 samples) of a chunk of variants, for NC score columns of the entries.
//  * fp64 sums: variants are taken in PAIRS; s_t2[c][pair][ca + 4 cb] = w_a[c][ca] + w_b[c][cb] (16 doubles = 128
//    bytes, one bank group: conflict-free for any index pattern), and the two words are merged into per-sample nibbles
//    (x: even samples, y: odd samples), so a sample costs one bit-field extract, one LDS.64 and one DADD per TWO
//    variants and column.  Each column's adds are the same, in the same order, whatever NC is: column j of a
//    several-column job is bit-identical to a one-column job of column j.
//  * integer sums (kInts; they do not depend on the column, so one launch per batch computes them): the named-allele
//    dosage (0..2) and the missing flag are added bit-parallel for all 16 samples at once in 4-bit fields (8 samples
//    per register), spilled to 8-bit fields every 7 variants and to the 32-bit per-sample counters every 127 variants.
//    A REF-named entry flips hom-REF <-> hom-ALT first (w ^= (~w & 0x5555...) << 1), after which the dosage is the code
//    itself with "missing" cleared.
// raw: [variant][pitch] bytes (pitch multiple of 4, padding samples coded missing); w4: [variant][score_ct][4] weights,
// of which columns col0 .. col0 + NC - 1 are scored here; d4: [variant] packed named-allele dosages of codes 0..2 (2 bits
// each): 0x24 = ALT named, 0x06 = REF named; the 'dominant' / 'recessive' forms 0x14 / 0x05 and 0x10 / 0x01 count
// min(copies, 1) / max(copies - 1, 0).  part_sum: [chunk][NC][samples_padded].
template <int NC, bool kInts>
__global__ void __launch_bounds__(kScoreThreads, NC == 1 ? 8 : 3) score_kernel(const uint8_t* __restrict__ raw, uint32_t pitch, uint32_t words, uint32_t variant_ct, uint32_t chunk_variants, const double* __restrict__ w4, uint32_t score_ct,
                                                           uint32_t col0, const uint8_t* __restrict__ d4, double* __restrict__ part_sum, uint32_t* __restrict__ part_dos, uint32_t* __restrict__ part_miss,
                                                           uint32_t samples_padded) {
  __shared__ double s_t2[NC][(kScoreTile / 2) * 16];
  __shared__ uint32_t s_flip[kScoreTile];
  __shared__ uint8_t s_mode[kScoreTile];  // 0 additive, 1 dominant (dosage min(count, 1)), 2 recessive (max(count - 1, 0))
  const uint32_t widx = blockIdx.x * kScoreThreads + threadIdx.x;
  const uint32_t v_begin = blockIdx.y * chunk_variants, v_end = min(variant_ct, v_begin + chunk_variants);
  double sum[NC][16];
#pragma unroll
  for (int c = 0; c < NC; ++c)
#pragma unroll
    for (int s = 0; s < 16; ++s) sum[c][s] = 0.0;
  // the integer partial sums live in this thread's own 16 slots of the per-chunk partial arrays (zeroed here, added to
  // at every 8-bit spill): 32 registers fewer than keeping them in the thread
  const uint64_t base = static_cast<uint64_t>(blockIdx.y) * samples_padded + 16ull * widx;
  if (kInts && widx < words) {
#pragma unroll
    for (int s = 0; s < 16; ++s) {
      part_dos[base + s] = 0;
      part_miss[base + s] = 0;
    }
  }
  // 4-bit fields (even / odd samples) and 8-bit fields (sample s -> register s % 4 ... see spill lambdas)
  uint32_t d4e = 0, d4o = 0, m4e = 0, m4o = 0;
  uint32_t d8[4] = {0, 0, 0, 0}, m8[4] = {0, 0, 0, 0};
  uint32_t n4 = 0, n8 = 0;
  auto spill4 = [&]() {  // 4-bit -> 8-bit: nibble j of the even register is sample 2j, of the odd register sample 2j+1
    d8[0] += d4e & 0x0F0F0F0Fu;         // samples 0, 4, 8, 12
    d8[1] += (d4e >> 4) & 0x0F0F0F0Fu;  // samples 2, 6, 10, 14
    d8[2] += d4o & 0x0F0F0F0Fu;         // samples 1, 5, 9, 13
    d8[3] += (d4o >> 4) & 0x0F0F0F0Fu;  // samples 3, 7, 11, 15
    m8[0] += m4e & 0x0F0F0F0Fu;
    m8[1] += (m4e >> 4) & 0x0F0F0F0Fu;
    m8[2] += m4o & 0x0F0F0F0Fu;
    m8[3] += (m4o >> 4) & 0x0F0F0F0Fu;
    d4e = d4o = m4e = m4o = 0;
    n4 = 0;
  };
  auto spill8 = [&]() {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int s0 = (r == 0) ? 0 : (r == 1) ? 2 : (r == 2) ? 1 : 3;
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        part_dos[base + s0 + 4 * b] += (d8[r] >> (8 * b)) & 0xFFu;
        part_miss[base + s0 + 4 * b] += (m8[r] >> (8 * b)) & 0xFFu;
      }
      d8[r] = 0;
      m8[r] = 0;
    }
    n8 = 0;
  };
  for (uint32_t v0 = v_begin; v0 < v_end; v0 += kScoreTile) {
    const uint32_t tile = min(kScoreTile, v_end - v0);
    const uint32_t pairs = (tile + 1) / 2;
    __syncthreads();
    for (uint32_t e = threadIdx.x; e < pairs * 16; e += kScoreThreads) {
      const uint32_t pr = e >> 4, ca = e & 3, cb = (e >> 2) & 3;
      const uint32_t va = v0 + 2 * pr, vb = va + 1;
      const double* wa = w4 + 4ull * (static_cast<uint64_t>(va) * score_ct + col0) + ca;
      const double* wb = w4 + 4ull * (static_cast<uint64_t>(vb) * score_ct + col0) + cb;
#pragma unroll
      for (int c = 0; c < NC; ++c) s_t2[c][e] = wa[4 * c] + ((vb < v_end) ? wb[4 * c] : 0.0);
    }
    if (kInts) {
      for (uint32_t e = threadIdx.x; e < tile; e += kScoreThreads) {
        const uint32_t dd = d4[v0 + e], da = dd & 3, db = (dd >> 2) & 3, dc = (dd >> 4) & 3;
        s_flip[e] = da ? 0xFFFFFFFFu : 0u;  // dosage of code 0 nonzero: REF named
        s_mode[e] = (da == 2 || dc == 2) ? 0 : (db ? 1 : 2);
      }
    }
    __syncthreads();
    if (widx >= words) continue;
    for (uint32_t pr = 0; pr < pairs; ++pr) {
      const uint32_t va = v0 + 2 * pr;
      const bool has_b = 2 * pr + 1 < tile;
      const uint32_t wa = *reinterpret_cast<const uint32_t*>(raw + static_cast<uint64_t>(va) * pitch + 4ull * widx);
      const uint32_t wb = has_b ? *reinterpret_cast<const uint32_t*>(raw + static_cast<uint64_t>(va + 1) * pitch + 4ull * widx) : 0u;
      // fp64: combined nibbles (code_a | code_b << 2); a missing second word indexes cb = 0, whose table part is 0
      const uint32_t x = (wa & 0x33333333u) | ((wb & 0x33333333u) << 2);
      const uint32_t y = ((wa >> 2) & 0x33333333u) | (wb & 0xCCCCCCCCu);
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        const double* t2 = &s_t2[c][16 * pr];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          sum[c][2 * j] += t2[(x >> (4 * j)) & 15u];
          sum[c][2 * j + 1] += t2[(y >> (4 * j)) & 15u];
        }
      }
      if constexpr (kInts) {  // integers, bit-parallel
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (h && !has_b) break;
          uint32_t w = h ? wb : wa;
          const uint32_t ms = w & (w >> 1) & 0x55555555u;  // missing flag at the even bit of each 2-bit field
          w ^= ((~w & 0x55555555u) << 1) & s_flip[2 * pr + h];  // REF named: 0 <-> 2 (1 and 3 keep their value)
          uint32_t d = w ^ (ms * 3u);                         // missing -> 0
          const uint32_t mode = s_mode[2 * pr + h];
          if (mode == 1) d = (d | (d >> 1)) & 0x55555555u;    // dominant: 1 for one or two copies
          else if (mode == 2) d = (d >> 1) & 0x55555555u;     // recessive: 1 for two copies
          d4e += d & 0x33333333u;
          d4o += (d >> 2) & 0x33333333u;
          m4e += ms & 0x11111111u;
          m4o += (ms >> 2) & 0x11111111u;
          if (++n4 == 7) {
            spill4();
            if (++n8 == 18) spill8();  // 18 x 7 x 2 = 252 <= 255
          }
        }
      }
    }
  }
  if (widx >= words) return;
  if constexpr (kInts) {
    spill4();
    spill8();
  }
#pragma unroll
  for (int c = 0; c < NC; ++c)
#pragma unroll
    for (int s = 0; s < 16; ++s) part_sum[(static_cast<uint64_t>(blockIdx.y) * NC + c) * samples_padded + 16ull * widx + s] = sum[c][s];
}

// Entries whose samples do not all share one weight table (chrY; chrX under --xchr-model 1) and haploid entries (MT).
// Every entry of a launch has the same ploidy class (kPl2ScoreHaploidAll / ChrY / ChrXMaleHaploid); per 16-sample word
// the class and the sex masks select, per sample, the first (w_dip) or the second (w_hap) 4-entry table of the entry,
// or nothing (chrY females).  One variant at a time: s_t[c][entry][skip * 8 + hap * 4 + code] with the skip half zero,
// 128 bytes per entry and column (one bank line, conflict-free), one LDS.64 and one DADD per sample, variant and
// column.  The integer sums are bit-parallel as in score_kernel, in half allele units (a diploid sample's named-allele
// dosage counts twice, a haploid one's once) in 4-bit fields spilled every 3 entries, with the missing calls split
// into a diploid and a haploid count.  Per class (the reference's chrY worker zeroes the dosage of every nonmale, :6683-
// 6691, and counts the missing calls of every nonfemale as haploid, :7914-7956):
//   class            table hap / dip / none       dosage x2 / x1     missing diploid / haploid
//   HaploidAll       all / - / -                  - / all            - / all
//   ChrY             male / unknown sex / female  - / male           - / nonfemale
//   ChrXMaleHaploid  male / nonmale / -           nonmale / male     nonmale / male
// male2 / female2: [word] 2-bit-field masks (both bits of a sample's field set when the sample is male / female).
// w_dip / w_hap: [entry][score_ct][4]; part_sum as score_kernel's; part_dos half units, part_miss diploid, part_miss_hap
// haploid missing calls.  Only ALT- or REF-named additive entries (named dosages 0x24 / 0x06) reach this kernel.
template <int NC, bool kInts>
__global__ void __launch_bounds__(kScoreThreads, NC == 1 ? 6 : 2) score_ploidy_kernel(const uint8_t* __restrict__ raw, uint32_t pitch, uint32_t words, uint32_t variant_ct, uint32_t chunk_variants, uint32_t ploidy_class,
                                                                    const uint32_t* __restrict__ male2, const uint32_t* __restrict__ female2, const double* __restrict__ w_dip, const double* __restrict__ w_hap, uint32_t score_ct,
                                                                    uint32_t col0, const uint8_t* __restrict__ d4, double* __restrict__ part_sum, uint32_t* __restrict__ part_dos, uint32_t* __restrict__ part_miss,
                                                                    uint32_t* __restrict__ part_miss_hap, uint32_t samples_padded) {
  __shared__ double s_t[NC][kScoreTile * 16];
  __shared__ uint32_t s_flip[kScoreTile];
  const uint32_t widx = blockIdx.x * kScoreThreads + threadIdx.x;
  const uint32_t v_begin = blockIdx.y * chunk_variants, v_end = min(variant_ct, v_begin + chunk_variants);
  // per sample (2-bit-field masks, see the table above): second table, no table, dosage counted twice / once, missing
  // call counted diploid / haploid
  uint32_t hap = 0, skip = 0, dos2 = 0, dos1 = 0, mdip = 0, mhap = 0;
  if (widx < words) {
    const uint32_t male = male2[widx], female = female2[widx];
    if (ploidy_class == kPl2ScoreHaploidAll) {
      hap = dos1 = mhap = 0xFFFFFFFFu;
    } else if (ploidy_class == kPl2ScoreChrY) {
      hap = dos1 = male;
      skip = female;
      mhap = ~female;
    } else {
      hap = dos1 = mhap = male;
      dos2 = mdip = ~male;
    }
  }
  double sum[NC][16];
#pragma unroll
  for (int c = 0; c < NC; ++c)
#pragma unroll
    for (int s = 0; s < 16; ++s) sum[c][s] = 0.0;
  const uint64_t base = static_cast<uint64_t>(blockIdx.y) * samples_padded + 16ull * widx;
  if (kInts && widx < words) {
#pragma unroll
    for (int s = 0; s < 16; ++s) {
      part_dos[base + s] = 0;
      part_miss[base + s] = 0;
      part_miss_hap[base + s] = 0;
    }
  }
  uint32_t d4e = 0, d4o = 0, md4e = 0, md4o = 0, mh4e = 0, mh4o = 0;
  uint32_t d8[4] = {0, 0, 0, 0}, md8[4] = {0, 0, 0, 0}, mh8[4] = {0, 0, 0, 0};
  uint32_t n4 = 0, n8 = 0;
  auto spill4 = [&]() {  // nibble j of an even register is sample 2j, of an odd register sample 2j+1 (as score_kernel)
    d8[0] += d4e & 0x0F0F0F0Fu;
    d8[1] += (d4e >> 4) & 0x0F0F0F0Fu;
    d8[2] += d4o & 0x0F0F0F0Fu;
    d8[3] += (d4o >> 4) & 0x0F0F0F0Fu;
    md8[0] += md4e & 0x0F0F0F0Fu;
    md8[1] += (md4e >> 4) & 0x0F0F0F0Fu;
    md8[2] += md4o & 0x0F0F0F0Fu;
    md8[3] += (md4o >> 4) & 0x0F0F0F0Fu;
    mh8[0] += mh4e & 0x0F0F0F0Fu;
    mh8[1] += (mh4e >> 4) & 0x0F0F0F0Fu;
    mh8[2] += mh4o & 0x0F0F0F0Fu;
    mh8[3] += (mh4o >> 4) & 0x0F0F0F0Fu;
    d4e = d4o = md4e = md4o = mh4e = mh4o = 0;
    n4 = 0;
  };
  auto spill8 = [&]() {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int s0 = (r == 0) ? 0 : (r == 1) ? 2 : (r == 2) ? 1 : 3;
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        part_dos[base + s0 + 4 * b] += (d8[r] >> (8 * b)) & 0xFFu;
        part_miss[base + s0 + 4 * b] += (md8[r] >> (8 * b)) & 0xFFu;
        part_miss_hap[base + s0 + 4 * b] += (mh8[r] >> (8 * b)) & 0xFFu;
      }
      d8[r] = md8[r] = mh8[r] = 0;
    }
    n8 = 0;
  };
  for (uint32_t v0 = v_begin; v0 < v_end; v0 += kScoreTile) {
    const uint32_t tile = min(kScoreTile, v_end - v0);
    __syncthreads();
    for (uint32_t e = threadIdx.x; e < tile * 16; e += kScoreThreads) {
      const uint32_t t = e >> 4, h = (e >> 2) & 3, code = e & 3;
      const uint64_t off = 4ull * (static_cast<uint64_t>(v0 + t) * score_ct + col0) + code;
#pragma unroll
      for (int c = 0; c < NC; ++c) s_t[c][e] = h == 1 ? w_hap[off + 4 * c] : h == 0 ? w_dip[off + 4 * c] : 0.0;
    }
    if (kInts)
      for (uint32_t e = threadIdx.x; e < tile; e += kScoreThreads) s_flip[e] = (d4[v0 + e] & 3) ? 0xFFFFFFFFu : 0u;
    __syncthreads();
    if (widx >= words) continue;
    for (uint32_t t = 0; t < tile; ++t) {
      const uint32_t w = *reinterpret_cast<const uint32_t*>(raw + static_cast<uint64_t>(v0 + t) * pitch + 4ull * widx);
      // nibbles: bits 0-1 the code, bit 2 the second table, bit 3 the zero half
      const uint32_t x = (w & 0x33333333u) | ((hap & 0x11111111u) << 2) | ((skip & 0x11111111u) << 3);
      const uint32_t y = ((w >> 2) & 0x33333333u) | (hap & 0x44444444u) | ((skip & 0x44444444u) << 1);
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        const double* tt = &s_t[c][16 * t];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          sum[c][2 * j] += tt[(x >> (4 * j)) & 15u];
          sum[c][2 * j + 1] += tt[(y >> (4 * j)) & 15u];
        }
      }
      if constexpr (kInts) {
        uint32_t g = w;
        const uint32_t ms = g & (g >> 1) & 0x55555555u;
        g ^= ((~g & 0x55555555u) << 1) & s_flip[t];  // REF named: 0 <-> 2
        const uint32_t d = (g ^ (ms * 3u)) & (dos1 | dos2);  // missing and uncounted -> 0
        // half units: dos2 samples count twice, once the fields are nibbles (values up to 4 need three bits)
        const uint32_t de = d & 0x33333333u, dd = (d >> 2) & 0x33333333u;
        d4e += de + (de & dos2);
        d4o += dd + (dd & (dos2 >> 2));
        const uint32_t md = ms & mdip, mh = ms & mhap;
        md4e += md & 0x11111111u;
        md4o += (md >> 2) & 0x11111111u;
        mh4e += mh & 0x11111111u;
        mh4o += (mh >> 2) & 0x11111111u;
        if (++n4 == 3) {
          spill4();
          if (++n8 == 21) spill8();  // 21 x 3 x 4 = 252 <= 255
        }
      }
    }
  }
  if (widx >= words) return;
  if constexpr (kInts) {
    spill4();
    spill8();
  }
#pragma unroll
  for (int c = 0; c < NC; ++c)
#pragma unroll
    for (int s = 0; s < 16; ++s) part_sum[(static_cast<uint64_t>(blockIdx.y) * NC + c) * samples_padded + 16ull * widx + s] = sum[c][s];
}

// The integer partials of score_ploidy_kernel, added in chunk order: half-unit dosages and haploid missing calls to
// their own accumulators, diploid missing calls to the job's missing counts.
__global__ void __launch_bounds__(256, 1) score_ploidy_reduce_ints_kernel(const uint32_t* __restrict__ part_dos, const uint32_t* __restrict__ part_miss, const uint32_t* __restrict__ part_miss_hap, uint32_t chunks,
                                                                       uint32_t samples_padded, uint32_t sample_ct, unsigned long long* __restrict__ acc_hdos, uint32_t* __restrict__ acc_miss,
                                                                       uint32_t* __restrict__ acc_miss_hap) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= sample_ct) return;
  unsigned long long d = acc_hdos[s];
  uint32_t md = acc_miss[s], mh = acc_miss_hap[s];
  for (uint32_t k = 0; k < chunks; ++k) {
    const uint64_t i = static_cast<uint64_t>(k) * samples_padded + s;
    d += part_dos[i];
    md += part_miss[i];
    mh += part_miss_hap[i];
  }
  acc_hdos[s] = d;
  acc_miss[s] = md;
  acc_miss_hap[s] = mh;
}

// acc_sum: [sample][score_ct]; columns col0 .. col0 + NC - 1 get the partials of this launch, added in chunk order.
template <int NC, bool kInts>
__global__ void __launch_bounds__(256, 1) score_reduce_kernel(const double* __restrict__ part_sum, const uint32_t* __restrict__ part_dos, const uint32_t* __restrict__ part_miss, uint32_t chunks, uint32_t samples_padded, uint32_t sample_ct,
                                                          uint32_t score_ct, uint32_t col0, double* __restrict__ acc_sum, unsigned long long* __restrict__ acc_dos, uint32_t* __restrict__ acc_miss) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= sample_ct) return;
#pragma unroll
  for (int c = 0; c < NC; ++c) {
    double* acc = acc_sum + static_cast<uint64_t>(s) * score_ct + col0 + c;
    double a = *acc;
    for (uint32_t k = 0; k < chunks; ++k) a += part_sum[(static_cast<uint64_t>(k) * NC + c) * samples_padded + s];
    *acc = a;
  }
  if (!kInts) return;
  unsigned long long d = acc_dos[s];
  uint32_t m = acc_miss[s];
  for (uint32_t k = 0; k < chunks; ++k) {
    d += part_dos[static_cast<uint64_t>(k) * samples_padded + s];
    m += part_miss[static_cast<uint64_t>(k) * samples_padded + s];
  }
  acc_dos[s] = d;
  acc_miss[s] = m;
}

constexpr uint32_t kScoreStageVariants = 16384;
constexpr uint32_t kScoreMaxChunks = 64;
// Score columns per launch: 16 fp64 sums per column and thread live in registers, so 4 columns (128 of them) is the most
// that compiles without spills (ptxas -v: 168 registers, three CTAs per SM) with the integer sums alongside.  The
// one-column kernel keeps the 64 registers (eight CTAs per SM) of the one-column-only kernel it replaced.
constexpr uint32_t kScoreGroup = 4;

struct ScoreLaunch {
  const uint8_t* raw;
  uint32_t pitch, words, variant_ct, chunk_variants, chunks, col_ctas, score_ct, col0, samples_padded, sample_ct;
  const double* w4;
  const uint8_t* d4;
  double* part_sum;
  uint32_t *part_dos, *part_miss;
  double* acc_sum;
  unsigned long long* acc_dos;
  uint32_t* acc_miss;
};

template <int NC, bool kInts>
void LaunchScoreGroup(const ScoreLaunch& a, cudaStream_t st) {
  score_kernel<NC, kInts><<<dim3(a.col_ctas, a.chunks), kScoreThreads, 0, st>>>(a.raw, a.pitch, a.words, a.variant_ct, a.chunk_variants, a.w4, a.score_ct, a.col0, a.d4, a.part_sum, a.part_dos, a.part_miss, a.samples_padded);
  score_reduce_kernel<NC, kInts><<<DivUpU32(a.sample_ct, 256), 256, 0, st>>>(a.part_sum, a.part_dos, a.part_miss, a.chunks, a.samples_padded, a.sample_ct, a.score_ct, a.col0, a.acc_sum, a.acc_dos, a.acc_miss);
}

template <bool kInts>
void LaunchScoreGroup(uint32_t nc, const ScoreLaunch& a, cudaStream_t st) {
  static_assert(kScoreGroup == 4, "one case per group width");
  switch (nc) {
    case 1: LaunchScoreGroup<1, kInts>(a, st); break;
    case 2: LaunchScoreGroup<2, kInts>(a, st); break;
    case 3: LaunchScoreGroup<3, kInts>(a, st); break;
    default: LaunchScoreGroup<4, kInts>(a, st); break;
  }
}

// score_ploidy_kernel's extra operands; the fp64 partials reduce through score_reduce_kernel<NC, false> into acc_sum
struct PloidyLaunch {
  uint32_t ploidy_class;
  const uint32_t *male2, *female2;
  const double* w_hap;
  uint32_t* part_miss_hap;
  unsigned long long* acc_hdos;
  uint32_t* acc_miss_hap;
};

template <int NC, bool kInts>
void LaunchPloidyGroup(const ScoreLaunch& a, const PloidyLaunch& p, cudaStream_t st) {
  score_ploidy_kernel<NC, kInts><<<dim3(a.col_ctas, a.chunks), kScoreThreads, 0, st>>>(a.raw, a.pitch, a.words, a.variant_ct, a.chunk_variants, p.ploidy_class, p.male2, p.female2, a.w4, p.w_hap, a.score_ct, a.col0, a.d4, a.part_sum,
                                                                                   a.part_dos, a.part_miss, p.part_miss_hap, a.samples_padded);
  score_reduce_kernel<NC, false><<<DivUpU32(a.sample_ct, 256), 256, 0, st>>>(a.part_sum, nullptr, nullptr, a.chunks, a.samples_padded, a.sample_ct, a.score_ct, a.col0, a.acc_sum, nullptr, nullptr);
  if (kInts)
    score_ploidy_reduce_ints_kernel<<<DivUpU32(a.sample_ct, 256), 256, 0, st>>>(a.part_dos, a.part_miss, p.part_miss_hap, a.chunks, a.samples_padded, a.sample_ct, p.acc_hdos, a.acc_miss, p.acc_miss_hap);
}

template <bool kInts>
void LaunchPloidyGroup(uint32_t nc, const ScoreLaunch& a, const PloidyLaunch& p, cudaStream_t st) {
  switch (nc) {
    case 1: LaunchPloidyGroup<1, kInts>(a, p, st); break;
    case 2: LaunchPloidyGroup<2, kInts>(a, p, st); break;
    case 3: LaunchPloidyGroup<3, kInts>(a, p, st); break;
    default: LaunchPloidyGroup<4, kInts>(a, p, st); break;
  }
}

// Class jobs (pl2gpu_score_add_variants_classes): row r of out is row perm[r] of in, so each class's entries of a
// staged batch lie next to each other and run through the kernels above as one block.  pitch16: 16-byte words per row.
__global__ void __launch_bounds__(256) score_row_gather_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, uint32_t pitch16, const uint32_t* __restrict__ perm) {
  const uint4* src = in + static_cast<uint64_t>(perm[blockIdx.y]) * pitch16;
  uint4* dst = out + static_cast<uint64_t>(blockIdx.y) * pitch16;
  for (uint32_t i = blockIdx.x * 256 + threadIdx.x; i < pitch16; i += gridDim.x * 256) dst[i] = src[i];
}

}  // namespace

struct Pl2ScoreJob {
  explicit Pl2ScoreJob(Pl2GpuCtx* x) : ctx(x) {}
  ~Pl2ScoreJob() {  // the kernels and copies that use the buffers finish before they are freed
    cudaSetDevice(ctx->c.device);
    cudaStreamSynchronize(ctx->c.stream);
  }
  Pl2GpuCtx* ctx;
  uint32_t sample_ct = 0, score_ct = 1;
  uint32_t class_ct = 1;  // accumulator sets (pl2gpu_score_begin_classes): class k's start k x samples_padded (x score_ct) in
                          // d_acc_sum, d_acc_dos, d_acc_miss, d_acc_hdos and d_acc_miss_hap
  uint32_t stage_variants = kScoreStageVariants;  // entries per staged batch
  GenoStage stage;
  DevArray<double> d_w4, d_part_sum, d_acc_sum;
  DevArray<uint8_t> d_d4;
  DevArray<uint32_t> d_part_dos, d_part_miss, d_acc_miss;
  DevArray<unsigned long long> d_acc_dos;
  uint64_t entries = 0;
  // entries of the haploid / sex-dependent classes (pl2gpu_score_add_variants_ploidy), allocated on first use
  DevArray<uint32_t> d_male2, d_female2;  // [word] 2-bit-field sex masks (pl2gpu_score_set_sex)
  DevArray<double> d_w4h;
  DevArray<uint32_t> d_part_miss_hap, d_acc_miss_hap;
  DevArray<unsigned long long> d_acc_hdos;
  // batches whose entries span several classes: the class-major copy of the stage and its row order, on first use
  DevArray<uint8_t> d_raw_grouped;
  DevArray<uint32_t> d_perm;
};

extern "C" {

int pl2gpu_score_end(Pl2ScoreJob* job) {
  if (!job) return 0;
  delete job;
  cudaGetLastError();
  return 0;
}

}  // extern "C"

namespace {

// class_ct accumulator sets; a job of several classes (fn = pl2gpu_score_begin_classes) also gets the haploid
// accumulators from the start, so that every per-class buffer is sized before the first entry
int ScoreBegin(Pl2GpuCtx* ctx, uint32_t sample_ct, uint32_t score_ct, uint32_t class_ct, const char* fn, Pl2ScoreJob** job_ptr) {
  if (job_ptr) *job_ptr = nullptr;
  if (!ctx || !job_ptr || !sample_ct || !score_ct || !class_ct) {
    set_error("%s: bad arguments", fn);
    return 1;
  }
  PL2_CUDA_OK(cudaSetDevice(ctx->c.device));
  std::unique_ptr<Pl2ScoreJob, int (*)(Pl2ScoreJob*)> job(new Pl2ScoreJob(ctx), pl2gpu_score_end);
  job->sample_ct = sample_ct;
  job->score_ct = score_ct;
  job->class_ct = class_ct;
  PL2_TRY(StageAlloc(sample_ct, kScoreStageVariants, &job->stage, 64));
  const uint64_t np = job->stage.sample_ct_padded;
  const uint64_t group = std::min(score_ct, kScoreGroup);
  const char* oom = "%s: insufficient device memory for %u samples x %u score columns";
  if (job->d_d4.alloc(kScoreStageVariants, oom, fn, sample_ct, score_ct) || job->d_part_sum.alloc(np * kScoreMaxChunks * group, oom, fn, sample_ct, score_ct) || job->d_part_dos.alloc(np * kScoreMaxChunks, oom, fn, sample_ct, score_ct) ||
      job->d_part_miss.alloc(np * kScoreMaxChunks, oom, fn, sample_ct, score_ct))
    return 1;
  // the accumulators: class_ct x (8 score_ct + 24) bytes per padded sample
  const char* oom_acc = "%s: insufficient device memory for the accumulators of %u classes x %u score columns x %u samples (%llu bytes)";
  const unsigned long long acc_bytes = class_ct * np * (8ull * score_ct + (class_ct > 1 ? 24 : 12));
  if (job->d_acc_sum.alloc(np * score_ct * class_ct, oom_acc, fn, class_ct, score_ct, sample_ct, acc_bytes) || job->d_acc_dos.alloc(np * class_ct, oom_acc, fn, class_ct, score_ct, sample_ct, acc_bytes) ||
      job->d_acc_miss.alloc(np * class_ct, oom_acc, fn, class_ct, score_ct, sample_ct, acc_bytes))
    return 1;
  if (class_ct > 1 && (job->d_acc_hdos.alloc(np * class_ct, oom_acc, fn, class_ct, score_ct, sample_ct, acc_bytes) || job->d_acc_miss_hap.alloc(np * class_ct, oom_acc, fn, class_ct, score_ct, sample_ct, acc_bytes))) return 1;
  // the staged weights ([entry][score_ct][4]) are the one buffer that grows with the column count and the batch: when
  // they do not fit, batches get fewer entries (then the chunk plan, and so the last bits of a sum, can differ from a
  // job with fewer columns)
  while (job->d_w4.alloc(4ull * score_ct * job->stage_variants, "%s: insufficient device memory for the weights of %u score columns", fn, score_ct)) {
    if (job->stage_variants <= kScoreTile) return 1;
    job->stage_variants /= 2;
  }
  if (cudaMemsetAsync(job->d_acc_sum, 0, 8 * np * score_ct * class_ct, ctx->c.stream) != cudaSuccess || cudaMemsetAsync(job->d_acc_dos, 0, 8 * np * class_ct, ctx->c.stream) != cudaSuccess ||
      cudaMemsetAsync(job->d_acc_miss, 0, 4 * np * class_ct, ctx->c.stream) != cudaSuccess ||
      (job->d_acc_hdos && (cudaMemsetAsync(job->d_acc_hdos, 0, 8 * np * class_ct, ctx->c.stream) != cudaSuccess || cudaMemsetAsync(job->d_acc_miss_hap, 0, 4 * np * class_ct, ctx->c.stream) != cudaSuccess))) {
    set_error("%s: %s", fn, cudaGetErrorString(cudaGetLastError()));
    return 1;
  }
  *job_ptr = job.release();
  return 0;
}

}  // namespace

extern "C" {

int pl2gpu_score_begin_cols(Pl2GpuCtx* ctx, uint32_t sample_ct, uint32_t score_ct, Pl2ScoreJob** job_ptr) { return ScoreBegin(ctx, sample_ct, score_ct, 1, "pl2gpu_score_begin_cols", job_ptr); }

int pl2gpu_score_begin_classes(Pl2GpuCtx* ctx, uint32_t sample_ct, uint32_t score_ct, uint32_t class_ct, Pl2ScoreJob** job_ptr) { return ScoreBegin(ctx, sample_ct, score_ct, class_ct, "pl2gpu_score_begin_classes", job_ptr); }

int pl2gpu_score_begin(Pl2GpuCtx* ctx, uint32_t sample_ct, Pl2ScoreJob** job_ptr) { return pl2gpu_score_begin_cols(ctx, sample_ct, 1, job_ptr); }

}  // extern "C"

namespace {

// Scores variant_ct staged rows (raw, the stage's pitch) of one ploidy class into the accumulators of class cls: class
// kPl2ScoreDiploid through score_kernel, the others through score_ploidy_kernel.  w4 / w4h / d4: the rows' device tables.
int ScoreLaunchRun(Pl2ScoreJob* job, const uint8_t* raw, uint32_t variant_ct, const double* w4, const double* w4h, const uint8_t* d4, uint32_t ploidy_class, uint32_t cls) {
  Ctx* c = &job->ctx->c;
  const uint32_t np = job->stage.sample_ct_padded, words = np / 16;
  const uint64_t acc = static_cast<uint64_t>(cls) * np;
  // enough chunks to fill the GPU, each a multiple of the shared-memory tile; the plan does not depend on the column
  // count, so every column is added in the order of a one-column job
  const uint32_t col_ctas = DivUpU32(words, kScoreThreads);
  uint32_t chunks = std::max(1u, std::min({kScoreMaxChunks, DivUpU32(7 * static_cast<uint32_t>(c->sm_count), col_ctas), DivUpU32(variant_ct, kScoreTile)}));
  const uint32_t chunk_variants = RoundUpU32(DivUpU32(variant_ct, chunks), kScoreTile);
  chunks = DivUpU32(variant_ct, chunk_variants);
  ScoreLaunch a{raw, job->stage.pitch, words, variant_ct, chunk_variants, chunks, col_ctas, job->score_ct, 0, np, job->sample_ct, w4, d4, job->d_part_sum, job->d_part_dos, job->d_part_miss,
                job->d_acc_sum + acc * job->score_ct, job->d_acc_dos + acc, job->d_acc_miss + acc};
  const PloidyLaunch p{ploidy_class, job->d_male2, job->d_female2, w4h, job->d_part_miss_hap, job->d_acc_hdos + (job->d_acc_hdos ? acc : 0), job->d_acc_miss_hap + (job->d_acc_miss_hap ? acc : 0)};
  // column groups over the resident batch; the first also adds the integer sums
  for (uint32_t col0 = 0; col0 < job->score_ct; col0 += kScoreGroup) {
    a.col0 = col0;
    const uint32_t nc = std::min(kScoreGroup, job->score_ct - col0);
    if (ploidy_class == kPl2ScoreDiploid) {
      if (col0 == 0) LaunchScoreGroup<true>(nc, a, c->stream);
      else LaunchScoreGroup<false>(nc, a, c->stream);
      c->launches += 2;
    } else {
      if (col0 == 0) LaunchPloidyGroup<true>(nc, a, p, c->stream);
      else LaunchPloidyGroup<false>(nc, a, p, c->stream);
      c->launches += col0 == 0 ? 3 : 2;
    }
  }
  PL2_CUDA_OK(cudaGetLastError());
  return 0;
}

// Stages and scores variant_ct entries of one ploidy class into class cls: class kPl2ScoreDiploid exactly as
// pl2gpu_score_add_variants always has, the others with their haploid tables w_hap.
int ScoreAddRun(Pl2ScoreJob* job, const uint8_t* src, uint64_t variant_stride_bytes, uint32_t variant_ct, int src_is_device, const double* weights4, const double* w_hap, const uint8_t* named_dosages, uint32_t ploidy_class,
                uint32_t cls = 0) {
  Ctx* c = &job->ctx->c;
  const uint64_t w_row = 4ull * job->score_ct;  // doubles of weights per entry
  for (uint32_t done = 0; done < variant_ct;) {
    const uint32_t cur = std::min(job->stage_variants, variant_ct - done);
    uint32_t padded = 0;
    PL2_TRY(StageUpload(c, &job->stage, src + static_cast<uint64_t>(done) * variant_stride_bytes, variant_stride_bytes, cur, src_is_device, &padded));
    PL2_CUDA_OK(cudaMemcpyAsync(job->d_w4, weights4 + w_row * done, 8 * w_row * cur, cudaMemcpyHostToDevice, c->stream));
    if (ploidy_class != kPl2ScoreDiploid) PL2_CUDA_OK(cudaMemcpyAsync(job->d_w4h, w_hap + w_row * done, 8 * w_row * cur, cudaMemcpyHostToDevice, c->stream));
    PL2_CUDA_OK(cudaMemcpyAsync(job->d_d4, named_dosages + done, cur, cudaMemcpyHostToDevice, c->stream));
    PL2_TRY(ScoreLaunchRun(job, job->stage.d_raw, cur, job->d_w4, job->d_w4h, job->d_d4, ploidy_class, cls));
    PL2_CUDA_OK(cudaStreamSynchronize(c->stream));  // host tables and a host source may be reused by the caller
    job->entries += cur;
    done += cur;
  }
  return 0;
}

bool ValidNamedDosages(const uint8_t* named_dosages, uint32_t variant_ct, const char* fn) {
  for (uint32_t v = 0; v < variant_ct; ++v) {
    const uint8_t dd = named_dosages[v];
    if (dd != 0x24 && dd != 0x06 && dd != 0x14 && dd != 0x05 && dd != 0x10 && dd != 0x01) {
      set_error("%s: entry %u has named-allele dosages 0x%02x (ALT / REF named: additive 0x24 / 0x06, dominant 0x14 / 0x05, recessive 0x10 / 0x01)", fn, v, dd);
      return false;
    }
  }
  return true;
}

// the buffers only entries of the haploid / sex-dependent classes use: all of them or none
// (a job of several classes has its haploid accumulators from the start)
int ScoreAllocPloidy(Pl2ScoreJob* job) {
  if (job->d_w4h) return 0;
  Ctx* c = &job->ctx->c;
  const uint64_t np = job->stage.sample_ct_padded;
  const char* oom = "pl2gpu_score_add_variants_ploidy: insufficient device memory for the haploid tables of %u samples x %u score columns";
  DevArray<double> w4h;
  DevArray<uint32_t> part_miss_hap;
  if (w4h.alloc(4ull * job->score_ct * job->stage_variants, oom, job->sample_ct, job->score_ct) || part_miss_hap.alloc(np * kScoreMaxChunks, oom, job->sample_ct, job->score_ct)) return 1;
  if (!job->d_acc_hdos) {
    DevArray<uint32_t> acc_miss_hap;
    DevArray<unsigned long long> acc_hdos;
    if (acc_miss_hap.alloc(np, oom, job->sample_ct, job->score_ct) || acc_hdos.alloc(np, oom, job->sample_ct, job->score_ct)) return 1;
    PL2_CUDA_OK(cudaMemsetAsync(acc_miss_hap, 0, 4 * np, c->stream));
    PL2_CUDA_OK(cudaMemsetAsync(acc_hdos, 0, 8 * np, c->stream));
    job->d_acc_miss_hap = std::move(acc_miss_hap);
    job->d_acc_hdos = std::move(acc_hdos);
  }
  job->d_w4h = std::move(w4h);
  job->d_part_miss_hap = std::move(part_miss_hap);
  return 0;
}

// the checks of pl2gpu_score_add_variants_ploidy on its ploidy classes (fn names the entry point in the messages)
bool ValidPloidyClasses(const Pl2ScoreJob* job, const uint8_t* ploidy_classes, uint32_t variant_ct, const double* weights4_haploid, const uint8_t* named_dosages, const char* fn) {
  for (uint32_t v = 0; v < variant_ct; ++v) {
    const uint8_t pc = ploidy_classes[v];
    if (pc > kPl2ScoreChrXMaleHaploid) {
      set_error("%s: entry %u has ploidy class %u", fn, v, pc);
      return false;
    }
    if (pc == kPl2ScoreDiploid) continue;
    if (!weights4_haploid) {
      set_error("%s: entry %u is haploid for some samples but weights4_haploid is NULL", fn, v);
      return false;
    }
    if (named_dosages[v] != 0x24 && named_dosages[v] != 0x06) {
      set_error("%s: entry %u of ploidy class %u is not additive (named-allele dosages 0x%02x)", fn, v, pc, named_dosages[v]);
      return false;
    }
    if (pc != kPl2ScoreHaploidAll && !job->d_male2) {
      set_error("%s: entry %u of ploidy class %u needs the sample sexes (pl2gpu_score_set_sex)", fn, v, pc);
      return false;
    }
  }
  return true;
}

// runs of consecutive entries of one ploidy class into class cls; a diploid-only call is one run of the plain score path
int ScoreAddPloidyRuns(Pl2ScoreJob* job, const uint8_t* src, uint64_t variant_stride_bytes, uint32_t variant_ct, int src_is_device, const uint8_t* ploidy_classes, const double* weights4_diploid, const double* weights4_haploid,
                       const uint8_t* named_dosages, uint32_t cls) {
  const uint64_t w_row = 4ull * job->score_ct;
  for (uint32_t r0 = 0; r0 < variant_ct;) {
    const uint32_t pc = ploidy_classes ? ploidy_classes[r0] : kPl2ScoreDiploid;
    uint32_t r1 = r0 + 1;
    while (r1 < variant_ct && (ploidy_classes ? ploidy_classes[r1] : kPl2ScoreDiploid) == pc) ++r1;
    if (pc != kPl2ScoreDiploid && ScoreAllocPloidy(job)) return 1;
    PL2_TRY(ScoreAddRun(job, src + static_cast<uint64_t>(r0) * variant_stride_bytes, variant_stride_bytes, r1 - r0, src_is_device, weights4_diploid + w_row * r0, pc == kPl2ScoreDiploid ? nullptr : weights4_haploid + w_row * r0,
                        named_dosages + r0, pc, cls));
    r0 = r1;
  }
  return 0;
}

// Entries of several classes, each reading one staged row (entry_rows NULL: entry e reads row e).  Each batch is as many
// whole rows as fit the stage whose entries also fit the entry buffers (stage_variants each), so no row's entries are
// split between batches.  A batch's rows are uploaded once; its entries are gathered on the device into class-major
// order (a row is copied once per entry that reads it), stably, with their tables in the same order, and each class's
// block runs, in runs of one ploidy class, through the kernels and launch plan of the plain path.  One class for every
// entry with one entry per row: the ploidy runs of the plain path, into that class, with no gather.
int ScoreAddEntries(Pl2ScoreJob* job, const void* genovecs, uint64_t variant_stride_bytes, uint32_t row_ct, int src_is_device, uint32_t entry_ct, const uint32_t* entry_rows, const uint32_t* entry_classes, const uint8_t* ploidy_classes,
                    const double* weights4_diploid, const double* weights4_haploid, const uint8_t* named_dosages, const char* fn) {
  if (!job || (entry_ct && (!genovecs || !entry_classes || !weights4_diploid || !named_dosages))) {
    set_error("%s: bad arguments", fn);
    return 1;
  }
  if (!ValidNamedDosages(named_dosages, entry_ct, fn)) return 1;
  if (ploidy_classes && !ValidPloidyClasses(job, ploidy_classes, entry_ct, weights4_haploid, named_dosages, fn)) return 1;
  for (uint32_t e = 0; e < entry_ct; ++e) {
    if (entry_classes[e] >= job->class_ct) {
      set_error("%s: entry %u has class %u of a job of %u classes", fn, e, entry_classes[e], job->class_ct);
      return 1;
    }
  }
  auto row_of = [&](uint32_t e) { return entry_rows ? entry_rows[e] : e; };
  for (uint32_t e0 = 0; e0 < entry_ct;) {
    uint32_t e1 = e0 + 1;
    while (e1 < entry_ct && row_of(e1) == row_of(e0)) ++e1;
    if (e1 - e0 > job->stage_variants) {
      set_error("%s: row %u has %u entries, more than the %u of a staged batch", fn, row_of(e0), e1 - e0, job->stage_variants);
      return 1;
    }
    e0 = e1;
  }
  PL2_CUDA_OK(cudaSetDevice(job->ctx->c.device));
  const uint8_t* src = static_cast<const uint8_t*>(genovecs);
  if (!entry_rows && std::all_of(entry_classes, entry_classes + entry_ct, [&](uint32_t k) { return k == entry_classes[0]; }))
    return ScoreAddPloidyRuns(job, src, variant_stride_bytes, entry_ct, src_is_device, ploidy_classes, weights4_diploid, weights4_haploid, named_dosages, entry_ct ? entry_classes[0] : 0);
  Ctx* c = &job->ctx->c;
  if (ploidy_classes && std::any_of(ploidy_classes, ploidy_classes + entry_ct, [](uint8_t pc) { return pc != kPl2ScoreDiploid; }) && ScoreAllocPloidy(job)) return 1;
  if (!job->d_raw_grouped) {  // the class-major copy holds a batch's entries (stage_variants rows of the stage's pitch)
    DevArray<uint8_t> raw;
    DevArray<uint32_t> perm;
    if (raw.alloc(static_cast<uint64_t>(job->stage_variants) * job->stage.pitch, "%s: insufficient device memory for a class-major copy of the %u-sample genotype stage", fn, job->sample_ct) ||
        perm.alloc(job->stage_variants, "%s: insufficient device memory", fn))
      return 1;
    job->d_raw_grouped = std::move(raw);
    job->d_perm = std::move(perm);
  }
  const uint64_t w_row = 4ull * job->score_ct;
  const uint32_t pitch16 = job->stage.pitch / 16;
  std::vector<uint32_t> perm, first(job->class_ct + 1);
  std::vector<double> w4, w4h;
  std::vector<uint8_t> d4, pcs;
  for (uint32_t done = 0; done < entry_ct;) {
    // whole rows from the batch's first row while the rows fit the stage and their entries the entry buffers
    const uint32_t r0 = row_of(done);
    uint32_t end = done;
    while (end < entry_ct && row_of(end) - r0 < job->stage_variants) {
      uint32_t next = end + 1;
      while (next < entry_ct && row_of(next) == row_of(end)) ++next;
      if (next - done > job->stage_variants) break;
      end = next;
    }
    const uint32_t cur = end - done, rows = row_of(end - 1) - r0 + 1;
    const uint32_t* cls = entry_classes + done;
    std::fill(first.begin(), first.end(), 0u);
    for (uint32_t e = 0; e < cur; ++e) ++first[cls[e] + 1];
    for (uint32_t k = 0; k < job->class_ct; ++k) first[k + 1] += first[k];
    perm.resize(cur);
    {
      std::vector<uint32_t> next(first.begin(), first.end() - 1);
      for (uint32_t e = 0; e < cur; ++e) perm[next[cls[e]]++] = done + e;
    }
    w4.resize(w_row * cur);
    d4.resize(cur);
    pcs.assign(cur, kPl2ScoreDiploid);
    const bool any_hap = ploidy_classes && std::any_of(ploidy_classes + done, ploidy_classes + done + cur, [](uint8_t pc) { return pc != kPl2ScoreDiploid; });
    if (any_hap) w4h.assign(w_row * cur, 0.0);
    for (uint32_t r = 0; r < cur; ++r) {
      const uint32_t e = perm[r];
      std::copy_n(weights4_diploid + w_row * e, w_row, w4.data() + w_row * r);
      d4[r] = named_dosages[e];
      if (ploidy_classes) pcs[r] = ploidy_classes[e];
      if (any_hap && pcs[r] != kPl2ScoreDiploid) std::copy_n(weights4_haploid + w_row * e, w_row, w4h.data() + w_row * r);
      perm[r] = row_of(e) - r0;  // the entry's row in the staged batch
    }
    uint32_t padded = 0;
    PL2_TRY(StageUpload(c, &job->stage, src + static_cast<uint64_t>(r0) * variant_stride_bytes, variant_stride_bytes, rows, src_is_device, &padded));
    PL2_CUDA_OK(cudaMemcpyAsync(job->d_perm, perm.data(), 4ull * cur, cudaMemcpyHostToDevice, c->stream));
    PL2_CUDA_OK(cudaMemcpyAsync(job->d_w4, w4.data(), 8 * w_row * cur, cudaMemcpyHostToDevice, c->stream));
    if (any_hap) PL2_CUDA_OK(cudaMemcpyAsync(job->d_w4h, w4h.data(), 8 * w_row * cur, cudaMemcpyHostToDevice, c->stream));
    PL2_CUDA_OK(cudaMemcpyAsync(job->d_d4, d4.data(), cur, cudaMemcpyHostToDevice, c->stream));
    score_row_gather_kernel<<<dim3(std::min(DivUpU32(pitch16, 256), 64u), cur), 256, 0, c->stream>>>(reinterpret_cast<const uint4*>(job->stage.d_raw.get()), reinterpret_cast<uint4*>(job->d_raw_grouped.get()), pitch16, job->d_perm);
    ++c->launches;
    PL2_CUDA_OK(cudaGetLastError());
    for (uint32_t k = 0; k < job->class_ct; ++k) {
      for (uint32_t r0k = first[k]; r0k < first[k + 1];) {
        uint32_t r1k = r0k + 1;
        while (r1k < first[k + 1] && pcs[r1k] == pcs[r0k]) ++r1k;
        PL2_TRY(ScoreLaunchRun(job, job->d_raw_grouped.get() + static_cast<uint64_t>(r0k) * job->stage.pitch, r1k - r0k, job->d_w4 + w_row * r0k, job->d_w4h ? job->d_w4h + w_row * r0k : nullptr, job->d_d4 + r0k, pcs[r0k], k));
        r0k = r1k;
      }
    }
    PL2_CUDA_OK(cudaStreamSynchronize(c->stream));  // host tables and a host source may be reused by the caller
    job->entries += cur;
    done = end;
  }
  return 0;
}

}  // namespace

extern "C" {

int pl2gpu_score_add_variants(Pl2ScoreJob* job, const void* genovecs, uint64_t variant_stride_bytes, uint32_t variant_ct, int src_is_device, const double* weights4, const uint8_t* named_dosages) {
  if (!job || (variant_ct && (!genovecs || !weights4 || !named_dosages))) {
    set_error("pl2gpu_score_add_variants: bad arguments");
    return 1;
  }
  if (!ValidNamedDosages(named_dosages, variant_ct, "pl2gpu_score_add_variants")) return 1;
  PL2_CUDA_OK(cudaSetDevice(job->ctx->c.device));
  return ScoreAddRun(job, static_cast<const uint8_t*>(genovecs), variant_stride_bytes, variant_ct, src_is_device, weights4, nullptr, named_dosages, kPl2ScoreDiploid);
}

int pl2gpu_score_set_sex(Pl2ScoreJob* job, const uint8_t* sample_sex) {
  if (!job || !sample_sex) {
    set_error("pl2gpu_score_set_sex: bad arguments");
    return 1;
  }
  const uint32_t words = job->stage.sample_ct_padded / 16;
  std::vector<uint32_t> male2(words, 0), female2(words, 0);
  for (uint32_t s = 0; s < job->sample_ct; ++s) {
    if (sample_sex[s] > 2) {
      set_error("pl2gpu_score_set_sex: sample %u has sex code %u (0 unknown, 1 male, 2 female)", s, sample_sex[s]);
      return 1;
    }
    if (sample_sex[s] == 1) male2[s / 16] |= 3u << (2 * (s % 16));
    if (sample_sex[s] == 2) female2[s / 16] |= 3u << (2 * (s % 16));
  }
  Ctx* c = &job->ctx->c;
  PL2_CUDA_OK(cudaSetDevice(c->device));
  if (!job->d_male2) {  // both masks or neither
    DevArray<uint32_t> d_male2, d_female2;
    if (d_male2.alloc(words, "pl2gpu_score_set_sex: insufficient device memory") || d_female2.alloc(words, "pl2gpu_score_set_sex: insufficient device memory")) return 1;
    job->d_male2 = std::move(d_male2);
    job->d_female2 = std::move(d_female2);
  }
  PL2_CUDA_OK(cudaMemcpyAsync(job->d_male2, male2.data(), 4ull * words, cudaMemcpyHostToDevice, c->stream));
  PL2_CUDA_OK(cudaMemcpyAsync(job->d_female2, female2.data(), 4ull * words, cudaMemcpyHostToDevice, c->stream));
  PL2_CUDA_OK(cudaStreamSynchronize(c->stream));
  return 0;
}

int pl2gpu_score_add_variants_ploidy(Pl2ScoreJob* job, const void* genovecs, uint64_t variant_stride_bytes, uint32_t variant_ct, int src_is_device, const uint8_t* ploidy_classes, const double* weights4_diploid,
                                     const double* weights4_haploid, const uint8_t* named_dosages) {
  if (!job || (variant_ct && (!genovecs || !ploidy_classes || !weights4_diploid || !named_dosages))) {
    set_error("pl2gpu_score_add_variants_ploidy: bad arguments");
    return 1;
  }
  if (!ValidNamedDosages(named_dosages, variant_ct, "pl2gpu_score_add_variants_ploidy")) return 1;
  if (!ValidPloidyClasses(job, ploidy_classes, variant_ct, weights4_haploid, named_dosages, "pl2gpu_score_add_variants_ploidy")) return 1;
  PL2_CUDA_OK(cudaSetDevice(job->ctx->c.device));
  return ScoreAddPloidyRuns(job, static_cast<const uint8_t*>(genovecs), variant_stride_bytes, variant_ct, src_is_device, ploidy_classes, weights4_diploid, weights4_haploid, named_dosages, 0);
}

int pl2gpu_score_add_variants_classes(Pl2ScoreJob* job, const void* genovecs, uint64_t variant_stride_bytes, uint32_t variant_ct, int src_is_device, const uint32_t* entry_classes, const uint8_t* ploidy_classes,
                                      const double* weights4_diploid, const double* weights4_haploid, const uint8_t* named_dosages) {
  return ScoreAddEntries(job, genovecs, variant_stride_bytes, variant_ct, src_is_device, variant_ct, nullptr, entry_classes, ploidy_classes, weights4_diploid, weights4_haploid, named_dosages, "pl2gpu_score_add_variants_classes");
}

int pl2gpu_score_add_entries(Pl2ScoreJob* job, const void* genovecs, uint64_t variant_stride_bytes, uint32_t row_ct, int src_is_device, uint32_t entry_ct, const uint32_t* entry_rows, const uint32_t* entry_classes,
                             const uint8_t* ploidy_classes, const double* weights4_diploid, const double* weights4_haploid, const uint8_t* named_dosages) {
  const char* fn = "pl2gpu_score_add_entries";
  if (!job || (entry_ct && !entry_rows)) {
    set_error("%s: bad arguments", fn);
    return 1;
  }
  for (uint32_t e = 0; e < entry_ct; ++e) {
    if (entry_rows[e] >= row_ct || (e && entry_rows[e] < entry_rows[e - 1])) {
      set_error("%s: entry %u has row %u (rows must be < %u and non-decreasing)", fn, e, entry_rows[e], row_ct);
      return 1;
    }
  }
  // one entry per row, in row order: the rows are the entries
  bool identity = entry_ct == row_ct;
  for (uint32_t e = 0; identity && e < entry_ct; ++e) identity = entry_rows[e] == e;
  return ScoreAddEntries(job, genovecs, variant_stride_bytes, row_ct, src_is_device, entry_ct, identity ? nullptr : entry_rows, entry_classes, ploidy_classes, weights4_diploid, weights4_haploid, named_dosages, fn);
}

int pl2gpu_score_get_class(Pl2ScoreJob* job, uint32_t class_idx, double* score_sums, uint64_t* named_half_dosage_sums, uint32_t* missing_diploid_cts, uint32_t* missing_haploid_cts) {
  if (!job || !score_sums || class_idx >= job->class_ct) {
    set_error("pl2gpu_score_get_class: bad arguments");
    return 1;
  }
  const uint32_t n = job->sample_ct;
  const uint64_t acc = static_cast<uint64_t>(class_idx) * job->stage.sample_ct_padded;
  std::vector<uint64_t> dos(n), hdos(n, 0);
  Ctx* c = &job->ctx->c;
  PL2_CUDA_OK(cudaSetDevice(c->device));
  PL2_CUDA_OK(cudaMemcpyAsync(score_sums, job->d_acc_sum + acc * job->score_ct, 8ull * n * job->score_ct, cudaMemcpyDeviceToHost, c->stream));
  PL2_CUDA_OK(cudaMemcpyAsync(dos.data(), job->d_acc_dos + acc, 8ull * n, cudaMemcpyDeviceToHost, c->stream));
  if (missing_diploid_cts) PL2_CUDA_OK(cudaMemcpyAsync(missing_diploid_cts, job->d_acc_miss + acc, 4ull * n, cudaMemcpyDeviceToHost, c->stream));
  if (job->d_acc_hdos) {
    PL2_CUDA_OK(cudaMemcpyAsync(hdos.data(), job->d_acc_hdos + acc, 8ull * n, cudaMemcpyDeviceToHost, c->stream));
    if (missing_haploid_cts) PL2_CUDA_OK(cudaMemcpyAsync(missing_haploid_cts, job->d_acc_miss_hap + acc, 4ull * n, cudaMemcpyDeviceToHost, c->stream));
  } else if (missing_haploid_cts) {
    std::fill(missing_haploid_cts, missing_haploid_cts + n, 0u);
  }
  PL2_CUDA_OK(cudaStreamSynchronize(c->stream));
  if (named_half_dosage_sums)
    for (uint32_t s = 0; s < n; ++s) named_half_dosage_sums[s] = 2 * dos[s] + hdos[s];
  return 0;
}

int pl2gpu_score_get_ploidy(Pl2ScoreJob* job, double* score_sums, uint64_t* named_half_dosage_sums, uint32_t* missing_diploid_cts, uint32_t* missing_haploid_cts) {
  if (!job || !score_sums) {
    set_error("pl2gpu_score_get_ploidy: bad arguments");
    return 1;
  }
  return pl2gpu_score_get_class(job, 0, score_sums, named_half_dosage_sums, missing_diploid_cts, missing_haploid_cts);
}

int pl2gpu_score_get(Pl2ScoreJob* job, double* score_sums, uint64_t* named_dosage_sums, uint32_t* missing_cts) {
  if (!job || !score_sums) {
    set_error("pl2gpu_score_get: bad arguments");
    return 1;
  }
  Ctx* c = &job->ctx->c;
  PL2_CUDA_OK(cudaSetDevice(c->device));
  PL2_CUDA_OK(cudaMemcpyAsync(score_sums, job->d_acc_sum, 8ull * job->sample_ct * job->score_ct, cudaMemcpyDeviceToHost, c->stream));
  if (named_dosage_sums) PL2_CUDA_OK(cudaMemcpyAsync(named_dosage_sums, job->d_acc_dos, 8ull * job->sample_ct, cudaMemcpyDeviceToHost, c->stream));
  if (missing_cts) PL2_CUDA_OK(cudaMemcpyAsync(missing_cts, job->d_acc_miss, 4ull * job->sample_ct, cudaMemcpyDeviceToHost, c->stream));
  PL2_CUDA_OK(cudaStreamSynchronize(c->stream));
  return 0;
}

}  // extern "C"
