// mock_king_mapped.cc - TEST INFRASTRUCTURE, never shipped and never linked into the product: the CPU stand-in library
// (mock_pl2gpu.cc, included unchanged) plus the mapped KING job of pl2gpu_king_begin_mapped, so that the
// `--king-table-require[-xor]` driver replays on the CPU like every other device-backed driver.  A mapped job keeps
// its codes in device-position order (the rows are permuted as they arrive) and returns only the pairs of positions
// (j, i), row_start <= j < row_end, i < min(j, col_end), in the library's order; "1" = the smaller position.
// Build: g++ -O2 -std=c++17 -ffp-contract=off -shared -fPIC -o mock_king_mapped.so mock_king_mapped.cc
#include <unordered_map>

// the stand-in's own KING entry points stay reachable under these names; the exported ones below route to them
#define pl2gpu_king_add_variants mock_base_king_add_variants
#define pl2gpu_king_get_counts mock_base_king_get_counts
#define pl2gpu_king_get_kinship mock_base_king_get_kinship
#define pl2gpu_king_get_filtered mock_base_king_get_filtered
#define pl2gpu_king_end mock_base_king_end
#include "mock_pl2gpu.cc"
#undef pl2gpu_king_add_variants
#undef pl2gpu_king_get_counts
#undef pl2gpu_king_get_kinship
#undef pl2gpu_king_get_filtered
#undef pl2gpu_king_end

namespace {
struct Mapped {
  std::vector<uint32_t> order;  // position -> sample index (empty: identity)
  uint32_t col_end;
};
std::mutex g_mapped_mu;
std::unordered_map<const Pl2KingJob*, Mapped> g_mapped;

const Mapped* FindMapped(const Pl2KingJob* job) {
  std::lock_guard<std::mutex> lock(g_mapped_mu);
  const auto it = g_mapped.find(job);
  return it == g_mapped.end() ? nullptr : &it->second;
}
uint64_t PairsBelow(uint64_t r, uint64_t col_end) { return r <= col_end ? (r ? r * (r - 1) / 2 : 0) : col_end * (col_end - 1) / 2 + (r - col_end) * col_end; }
}  // namespace

extern "C" {

uint64_t pl2gpu_king_mapped_mem_required(uint32_t sample_ct, uint32_t row_start, uint32_t row_end, uint32_t col_end, uint32_t) {
  return 2048ull * (PairsBelow(row_end, col_end) - PairsBelow(row_start, col_end)) + 4096ull * sample_ct;
}

int pl2gpu_king_begin_mapped(Pl2GpuCtx* ctx, uint32_t sample_ct, const uint32_t* order, uint32_t row_start, uint32_t row_end, uint32_t col_end, uint32_t, Pl2KingJob** job_ptr) {
  Log("king_begin_mapped device=%d rows=%u\n", ctx->device, row_end - row_start);
  *job_ptr = new Pl2KingJob{sample_ct, row_start, row_end, {}, 0};
  std::lock_guard<std::mutex> lock(g_mapped_mu);
  g_mapped[*job_ptr] = Mapped{order ? std::vector<uint32_t>(order, order + sample_ct) : std::vector<uint32_t>(), col_end};
  return 0;
}

int pl2gpu_king_add_variants(Pl2KingJob* job, const void* genovecs, uint64_t stride, uint32_t variant_ct, int src) {
  const uint64_t first = job->variants;
  const int rc = mock_base_king_add_variants(job, genovecs, stride, variant_ct, src);
  const Mapped* m = FindMapped(job);
  if (rc || !m || m->order.empty()) return rc;
  std::vector<uint8_t> row(job->n);
  for (uint64_t v = first; v < job->variants; ++v) {
    uint8_t* codes = &job->codes[v * job->n];
    for (uint32_t p = 0; p < job->n; ++p) row[p] = codes[m->order[p]];
    memcpy(codes, row.data(), job->n);
  }
  return 0;
}

int pl2gpu_king_get_counts(Pl2KingJob* job, uint32_t r0, uint32_t r1, uint32_t* dst, int dst_is_device) {
  const Mapped* m = FindMapped(job);
  if (!m) return mock_base_king_get_counts(job, r0, r1, dst, dst_is_device);
  for (uint32_t j = r0; j < r1; ++j)
    for (uint32_t i = 0; i < j && i < m->col_end; ++i, dst += 5) PairCounts(job, j, i, dst);
  return 0;
}

int pl2gpu_king_get_kinship(Pl2KingJob* job, uint32_t r0, uint32_t r1, double* dst, int dst_is_device) {
  const Mapped* m = FindMapped(job);
  if (!m) return mock_base_king_get_kinship(job, r0, r1, dst, dst_is_device);
  for (uint32_t j = r0; j < r1; ++j) {
    for (uint32_t i = 0; i < j && i < m->col_end; ++i) {
      uint32_t c[5];
      PairCounts(job, j, i, c);
      *dst++ = Kinship(c);
    }
  }
  return 0;
}

int pl2gpu_king_get_filtered(Pl2KingJob* job, uint32_t r0, uint32_t r1, double min_kinship, uint64_t max_out, uint32_t* pairs_out, uint32_t* counts_out, double* kinship_out, uint64_t* n_found) {
  const Mapped* m = FindMapped(job);
  if (!m) return mock_base_king_get_filtered(job, r0, r1, min_kinship, max_out, pairs_out, counts_out, kinship_out, n_found);
  uint64_t k = 0;
  for (uint32_t j = r0; j < r1; ++j) {
    for (uint32_t i = 0; i < j && i < m->col_end; ++i) {
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

int pl2gpu_king_end(Pl2KingJob* job) {
  {
    std::lock_guard<std::mutex> lock(g_mapped_mu);
    g_mapped.erase(job);
  }
  return mock_base_king_end(job);
}

}  // extern "C"
