// common.cuh - shared declarations of the pl2gpu library (internal; the public face is
// include/plink2_b200.h).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

namespace pl2 {

// ---- error plumbing: every CUDA call is checked; failures become `return 1` + message ----
void set_error(const char* fmt, ...);
const char* get_error();

#define PL2_CUDA_OK(expr)                                                                                  \
  do {                                                                                                     \
    cudaError_t err__ = (expr);                                                                            \
    if (err__ != cudaSuccess) {                                                                            \
      pl2::set_error("%s failed at %s:%d: %s", #expr, __FILE__, __LINE__, cudaGetErrorString(err__));      \
      return 1;                                                                                            \
    }                                                                                                      \
  } while (0)

#define PL2_TRY(expr)  \
  do {                 \
    if ((expr)) {      \
      return 1;        \
    }                  \
  } while (0)

// ---- pair-tile geometry shared by every N x N kernel ----
// Output tiles are kTileRows (larger-index samples, "sample 2") x kTileCols (smaller-index
// samples, "sample 1").  A tensor kernel runs a tile as two CTAs of 64 rows (the wgmma M dimension), each
// keeping its five 32-bit accumulator blocks (5 x 64 x 96 int32) in the registers of two warpgroups.
constexpr uint32_t kTileRows = 128;
constexpr uint32_t kTileCols = 96;
constexpr uint32_t kKingAccs = 5;                                   // TT, TH, HT, HH, SS
constexpr uint32_t kKingTileAccCols = kKingAccs * kTileCols;        // 480
constexpr uint32_t kKingTileAccWords = kKingTileAccCols * kTileRows;  // int32 per tile
// Samples are padded to a multiple of lcm(128, 96) with "missing" so every tile read is in-bounds.
constexpr uint32_t kSamplePad = 384;

// Position p of a 16-byte expanded vector holds sample kPosToSample(p) of the 16-sample group
// (a by-product of the PRMT expansion, which handles even and odd samples separately).
__host__ __device__ constexpr uint32_t PosToSample(uint32_t p) { return (p < 8) ? (2 * p) : (2 * (p - 8) + 1); }
__host__ __device__ constexpr uint32_t SampleToPos(uint32_t s) { return (s & 1) ? (8 + (s >> 1)) : (s >> 1); }

struct Ctx {
  int device = -1;
  cudaStream_t stream = nullptr;       // compute stream: every tensor / popcount / finalize kernel
  cudaStream_t copy_stream = nullptr;  // high-priority prep stream: H2D / D2D copies, all-gathers, padding, re-tiling
  int sm_count = 0;
  uint64_t launches = 0;
  cudaEvent_t events[16] = {};
  // optional NCCL communicator (one rank per context; pl2gpu_comm_init), loaded lazily with dlopen
  void* comm = nullptr;
  int comm_rank = 0, comm_world = 1;
};

// NCCL plumbing (pl2gpu.cu): in-place all-gather of `bytes_per_rank` bytes per rank over buf (rank r's part
// already sits at buf + r * bytes_per_rank), and an in-place fp64 sum all-reduce, both enqueued on `stream`.
int CommAllGatherInPlace(Ctx* ctx, void* buf, uint64_t bytes_per_rank, cudaStream_t stream);
int CommAllReduceSumF64(Ctx* ctx, double* buf, uint64_t count, cudaStream_t stream);

struct TileList {
  // tiles of the strict lower triangle restricted to rows [row_start, row_end)
  uint32_t row_tile_first = 0;  // row_start / kTileRows
  uint32_t row_tile_ct = 0;
  uint32_t tile_ct = 0;
  uint32_t* d_tile_rt = nullptr;       // [tile_ct] row-tile index (absolute)
  uint32_t* d_tile_tc = nullptr;       // [tile_ct] col-tile index
  uint32_t* d_rowtile_offset = nullptr;  // [row_tile_ct + 1] first tile of each row tile
  uint32_t* d_tile_order = nullptr;      // [tile_ct] launch order: 12 x 12 tile blocks so co-resident CTAs share L2 lines
  std::vector<uint32_t> h_rowtile_offset;  // host copy of the same
};

// col_end: tiles that lie entirely at or past this column are left out (a KING job cut at a column bound)
uint64_t CountTiles(uint32_t row_start, uint32_t row_end, bool include_diag, uint32_t tile_cols = kTileCols, uint32_t col_end = 0xFFFFFFFFu);
int BuildTileList(uint32_t row_start, uint32_t row_end, bool include_diag, TileList* tl, uint32_t tile_cols = kTileCols, uint32_t col_end = 0xFFFFFFFFu);
void FreeTileList(TileList* tl);

// ---- staged genotype block on the device (implemented in pl2gpu.cu) ----
struct GenoStage {
  uint8_t* d_raw = nullptr;  // [variant_cap][pitch]
  uint32_t pitch = 0;        // bytes per variant row = sample_ct_padded / 4
  uint32_t sample_ct = 0;
  uint32_t sample_ct_padded = 0;
  uint32_t variant_cap = 0;  // multiple of kVariantPad
};
constexpr uint32_t kVariantPad = 256;      // lcm(popcount chunk 8*32, tensor stage 64)
constexpr uint32_t kMaxStageVariants = 65536;        // default capacity of a staged block
constexpr uint32_t kMaxStageVariantsEx = 1u << 20;   // largest capacity pl2gpu_king_begin_ex accepts
// pad_genotypes_kernel launcher (kernel lives in pl2gpu.cu's translation unit); stream = nullptr: the compute stream
int LaunchPadGenotypes(Ctx* ctx, uint8_t* dst, uint32_t pitch, uint32_t sample_ct, uint32_t variant_ct, uint32_t variant_ct_padded, cudaStream_t stream = nullptr);
int StageAlloc(uint32_t sample_ct, uint32_t variant_cap, GenoStage* gs, uint32_t sample_pad = kSamplePad);
void StageFree(GenoStage* gs);
// Copies variant_ct (<= variant_cap) rows starting at destination row dst_row and forces padding
// samples / rows [dst_row + variant_ct, dst_row + padded) to "missing".
int StageUpload(Ctx* ctx, GenoStage* gs, const void* src, uint64_t src_stride, uint32_t variant_ct, int src_is_device, uint32_t* padded_ct_ptr, uint32_t dst_row = 0, uint32_t pad_to = kVariantPad);

static inline uint32_t DivUpU32(uint32_t a, uint32_t b) { return (a + b - 1) / b; }
static inline uint64_t DivUpU64(uint64_t a, uint64_t b) { return (a + b - 1) / b; }
static inline uint32_t RoundUpU32(uint32_t a, uint32_t b) { return DivUpU32(a, b) * b; }

}  // namespace pl2

struct Pl2GpuCtx {
  pl2::Ctx c;
};
