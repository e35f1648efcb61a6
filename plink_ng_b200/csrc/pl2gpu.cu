// pl2gpu.cu - C-ABI entry points (include/plink2_b200.h): context, staging, KING job driver.
#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <cstdarg>
#include <cstring>
#include <mutex>
#include <vector>

#include "../../include/plink2_b200.h"
#include "common.cuh"
#include "king_kernels.cuh"
#include "king_ts_kernel.cuh"
#include "king_pairs_kernel.cuh"
#include "ld_kernels.cuh"
#include "wgmma_probe.cuh"

namespace pl2 {

static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* get_error() { return g_err; }

// ---- tile list over the strict lower triangle restricted to rows [row_start,row_end) ----
static uint32_t ColTilesForRowTile(uint32_t rt, uint32_t row_end, bool include_diag, uint32_t tile_cols, uint32_t col_end) {
  uint32_t tile_row_end = (rt + 1) * kTileRows;
  if (tile_row_end > row_end) tile_row_end = row_end;
  // columns 0 .. tile_row_end-2 are needed (.. tile_row_end-1 with the diagonal), none at or past col_end
  uint32_t cols = include_diag ? tile_row_end : (tile_row_end ? tile_row_end - 1 : 0);
  if (cols > col_end) cols = col_end;
  if (!cols) return 0;
  return DivUpU32(cols, tile_cols);
}

uint64_t CountTiles(uint32_t row_start, uint32_t row_end, bool include_diag, uint32_t tile_cols, uint32_t col_end) {
  if (row_end <= row_start) return 0;
  uint64_t n = 0;
  for (uint32_t rt = row_start / kTileRows; rt * kTileRows < row_end; ++rt) n += ColTilesForRowTile(rt, row_end, include_diag, tile_cols, col_end);
  return n;
}

int BuildTileList(uint32_t row_start, uint32_t row_end, bool include_diag, TileList* tl, uint32_t tile_cols, uint32_t col_end) {
  std::vector<uint32_t> rt_v, tc_v, off_v;
  tl->row_tile_first = row_start / kTileRows;
  uint32_t rt = tl->row_tile_first;
  // an empty row range (a rank of a multi-GPU team that owns no rows) has no tiles at all
  for (; row_end > row_start && rt * kTileRows < row_end; ++rt) {
    off_v.push_back(static_cast<uint32_t>(rt_v.size()));
    const uint32_t nct = ColTilesForRowTile(rt, row_end, include_diag, tile_cols, col_end);
    for (uint32_t tc = 0; tc < nct; ++tc) {
      rt_v.push_back(rt);
      tc_v.push_back(tc);
    }
  }
  off_v.push_back(static_cast<uint32_t>(rt_v.size()));
  tl->row_tile_ct = rt - tl->row_tile_first;
  tl->tile_ct = static_cast<uint32_t>(rt_v.size());
  const size_t nb = (rt_v.size() + 1) * sizeof(uint32_t);
  PL2_CUDA_OK(cudaMalloc(&tl->d_tile_rt, nb));
  PL2_CUDA_OK(cudaMalloc(&tl->d_tile_tc, nb));
  PL2_CUDA_OK(cudaMalloc(&tl->d_rowtile_offset, off_v.size() * sizeof(uint32_t)));
  if (!rt_v.empty()) {
    PL2_CUDA_OK(cudaMemcpy(tl->d_tile_rt, rt_v.data(), rt_v.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    PL2_CUDA_OK(cudaMemcpy(tl->d_tile_tc, tc_v.data(), tc_v.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
  }
  PL2_CUDA_OK(cudaMemcpy(tl->d_rowtile_offset, off_v.data(), off_v.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
  tl->h_rowtile_offset = off_v;
  // launch order: blocks of kBand x kBand tiles (144, about one wave on the 132 SMs of an H100 SXM) so that the
  // CTAs resident at the same time stream the same few row/column sample ranges and hit in L2
  constexpr uint32_t kBand = 12;
  std::vector<uint32_t> order;
  order.reserve(rt_v.size());
  const uint32_t n_rt = tl->row_tile_ct;
  for (uint32_t rb = 0; rb < n_rt; rb += kBand) {
    const uint32_t rb_end = std::min(n_rt, rb + kBand);
    uint32_t max_cols = 0;
    for (uint32_t r = rb; r < rb_end; ++r) max_cols = std::max(max_cols, off_v[r + 1] - off_v[r]);
    for (uint32_t cb = 0; cb < max_cols; cb += kBand) {
      for (uint32_t r = rb; r < rb_end; ++r) {
        const uint32_t ncols = off_v[r + 1] - off_v[r];
        for (uint32_t c = cb; c < std::min(ncols, cb + kBand); ++c) order.push_back(off_v[r] + c);
      }
    }
  }
  PL2_CUDA_OK(cudaMalloc(&tl->d_tile_order, nb));
  if (!order.empty()) PL2_CUDA_OK(cudaMemcpy(tl->d_tile_order, order.data(), order.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
  return 0;
}

void FreeTileList(TileList* tl) {
  cudaFree(tl->d_tile_rt);
  cudaFree(tl->d_tile_tc);
  cudaFree(tl->d_rowtile_offset);
  cudaFree(tl->d_tile_order);
  tl->d_tile_order = nullptr;
  tl->d_tile_rt = tl->d_tile_tc = tl->d_rowtile_offset = nullptr;
}

// ---- NCCL, loaded on first use: the library has no link-time dependency on it, and inside a process that
// already carries an NCCL (torch.distributed) the same copy is shared ----
namespace {
struct NcclApi {
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool ok = false;
};
NcclApi g_nccl;
std::once_flag g_nccl_once;

void LoadNccl() {
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) return;
  g_nccl.GetUniqueId = reinterpret_cast<decltype(g_nccl.GetUniqueId)>(dlsym(h, "ncclGetUniqueId"));
  g_nccl.CommInitRank = reinterpret_cast<decltype(g_nccl.CommInitRank)>(dlsym(h, "ncclCommInitRank"));
  g_nccl.CommDestroy = reinterpret_cast<decltype(g_nccl.CommDestroy)>(dlsym(h, "ncclCommDestroy"));
  g_nccl.AllGather = reinterpret_cast<decltype(g_nccl.AllGather)>(dlsym(h, "ncclAllGather"));
  g_nccl.AllReduce = reinterpret_cast<decltype(g_nccl.AllReduce)>(dlsym(h, "ncclAllReduce"));
  g_nccl.GetErrorString = reinterpret_cast<decltype(g_nccl.GetErrorString)>(dlsym(h, "ncclGetErrorString"));
  g_nccl.ok = g_nccl.GetUniqueId && g_nccl.CommInitRank && g_nccl.CommDestroy && g_nccl.AllGather && g_nccl.AllReduce && g_nccl.GetErrorString;
}
bool HaveNccl() {
  std::call_once(g_nccl_once, LoadNccl);
  if (!g_nccl.ok) set_error("NCCL (libnccl.so.2) could not be loaded: %s", dlerror() ? dlerror() : "symbols missing");
  return g_nccl.ok;
}
}  // namespace

#define PL2_NCCL_OK(expr)                                                                              \
  do {                                                                                                 \
    ncclResult_t r__ = (expr);                                                                         \
    if (r__ != ncclSuccess) {                                                                          \
      pl2::set_error("%s failed at %s:%d: %s", #expr, __FILE__, __LINE__, g_nccl.GetErrorString(r__)); \
      return 1;                                                                                        \
    }                                                                                                  \
  } while (0)

int CommAllGatherInPlace(Ctx* ctx, void* buf, uint64_t bytes_per_rank, cudaStream_t stream) {
  if (!ctx->comm) {
    set_error("no communicator attached to the context");
    return 1;
  }
  const uint8_t* mine = static_cast<const uint8_t*>(buf) + static_cast<uint64_t>(ctx->comm_rank) * bytes_per_rank;
  PL2_NCCL_OK(g_nccl.AllGather(mine, buf, bytes_per_rank, ncclUint8, static_cast<ncclComm_t>(ctx->comm), stream));
  return 0;
}

int CommAllReduceSumF64(Ctx* ctx, double* buf, uint64_t count, cudaStream_t stream) {
  if (!ctx->comm) {
    set_error("no communicator attached to the context");
    return 1;
  }
  PL2_NCCL_OK(g_nccl.AllReduce(buf, buf, count, ncclDouble, ncclSum, static_cast<ncclComm_t>(ctx->comm), stream));
  return 0;
}

// ---- staged genotype block on the device ----
int StageAlloc(uint32_t sample_ct, uint32_t variant_cap, GenoStage* gs, uint32_t sample_pad) {
  gs->sample_ct = sample_ct;
  gs->sample_ct_padded = RoundUpU32(sample_ct, sample_pad);
  gs->pitch = gs->sample_ct_padded / 4;
  gs->variant_cap = RoundUpU32(variant_cap, kVariantPad);
  if (cudaMalloc(&gs->d_raw, static_cast<uint64_t>(gs->variant_cap) * gs->pitch) != cudaSuccess) {
    cudaGetLastError();
    gs->d_raw = nullptr;
    set_error("insufficient device memory for a %u-variant x %u-sample genotype stage", gs->variant_cap, sample_ct);
    return 1;
  }
  return 0;
}

int LaunchPadGenotypes(Ctx* ctx, uint8_t* dst, uint32_t pitch, uint32_t sample_ct, uint32_t variant_ct, uint32_t variant_ct_padded, cudaStream_t stream) {
  if (!variant_ct_padded) return 0;
  pad_genotypes_kernel<<<variant_ct_padded, 128, 0, stream ? stream : ctx->stream>>>(dst, pitch, sample_ct, variant_ct, variant_ct_padded);
  ctx->launches++;
  PL2_CUDA_OK(cudaGetLastError());
  return 0;
}

void StageFree(GenoStage* gs) {
  cudaFree(gs->d_raw);
  gs->d_raw = nullptr;
}

int StageUpload(Ctx* ctx, GenoStage* gs, const void* src, uint64_t src_stride, uint32_t variant_ct, int src_is_device, uint32_t* padded_ct_ptr, uint32_t dst_row, uint32_t pad_to) {
  const uint32_t padded = RoundUpU32(variant_ct, pad_to);
  if (dst_row + padded > gs->variant_cap) {
    set_error("StageUpload: %u + %u rows exceed the stage capacity %u", dst_row, padded, gs->variant_cap);
    return 1;
  }
  const uint32_t width = DivUpU32(gs->sample_ct, 4);
  uint8_t* dst = gs->d_raw + static_cast<uint64_t>(dst_row) * gs->pitch;
  if (variant_ct) {
    PL2_CUDA_OK(cudaMemcpy2DAsync(dst, gs->pitch, src, src_stride, width, variant_ct, src_is_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, ctx->stream));
  }
  if (padded) {
    pad_genotypes_kernel<<<padded, 128, 0, ctx->stream>>>(dst, gs->pitch, gs->sample_ct, variant_ct, padded);
    ctx->launches++;
    PL2_CUDA_OK(cudaGetLastError());
  }
  *padded_ct_ptr = padded;
  return 0;
}

}  // namespace pl2

using namespace pl2;

struct Pl2KingJob {
  Pl2GpuCtx* ctx = nullptr;
  uint32_t sample_ct = 0, row_start = 0, row_end = 0;
  uint32_t col_end = 0;              // pairs with a column at or past this are never returned (sample_ct: none cut)
  uint32_t* d_order = nullptr;       // mapped job: device position -> sample index; null = identity
  uint8_t* d_unmapped = nullptr;     // mapped job: the block as the caller gave it, before the gather into position order
  int algo = kPl2KingAlgoTensor;
  TileList tiles;
  // TS path: two staged blocks + two row-side re-tiled copies, so that the copy / all-gather, padding and
  // row re-tiling of batch k+1 (prep stream) overlap the tensor kernel of batch k (compute stream).
  // The other algorithms use buffer 0 on the compute stream only.
  GenoStage stage[2];
  uint8_t* d_raw_t[2] = {nullptr, nullptr};  // tensor paths: sample-major copy of the staged block (geno_tile.cuh; split form on the TS path)
  cudaEvent_t ev_prep_done[2] = {nullptr, nullptr};
  cudaEvent_t ev_kernel_start[2] = {nullptr, nullptr};  // timing-enabled pair around the tensor kernel (pl2gpu_king_last_kernel_ms)
  cudaEvent_t ev_kernel_done[2] = {nullptr, nullptr};
  int last_buf = -1;
  bool kernel_pending[2] = {false, false};
  uint32_t buf_idx = 0;
  uint32_t* d_planes = nullptr;  // popcount path only
  uint32_t tile_cols = kTileCols;
  int32_t* d_raw_acc = nullptr;
  void* d_out_stage = nullptr;   // bounded staging for host downloads
  uint64_t out_stage_bytes = 0;
  uint64_t variants_added = 0;
  cudaEvent_t ev_copied = nullptr;     // the caller's buffer has been consumed (prep stream)
  cudaEvent_t ev_src_ready = nullptr;  // device sources ordered on the compute stream
};

extern "C" {

int pl2gpu_abi_version(void) { return 2; }

const char* pl2gpu_last_error(void) { return get_error(); }

int pl2gpu_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

int pl2gpu_ctx_create(int device_idx, Pl2GpuCtx** ctx_ptr) {
  *ctx_ptr = nullptr;
  int n = 0;
  PL2_CUDA_OK(cudaGetDeviceCount(&n));
  if (device_idx < 0 || device_idx >= n) {
    set_error("pl2gpu_ctx_create: device %d out of range (%d CUDA devices visible); there is no CPU fallback", device_idx, n);
    return 1;
  }
  cudaDeviceProp prop;
  PL2_CUDA_OK(cudaGetDeviceProperties(&prop, device_idx));
  if (prop.major != 9 || prop.minor != 0) {
    set_error("pl2gpu_ctx_create: device %d is sm_%d%d; this library contains sm_90a code only", device_idx, prop.major, prop.minor);
    return 1;
  }
  PL2_CUDA_OK(cudaSetDevice(device_idx));
  Pl2GpuCtx* ctx = new Pl2GpuCtx();
  ctx->c.device = device_idx;
  ctx->c.sm_count = prop.multiProcessorCount;
  PL2_CUDA_OK(cudaStreamCreateWithFlags(&ctx->c.stream, cudaStreamNonBlocking));
  {
    // the prep stream outranks the compute stream: its short copy / pad / re-tile / all-gather kernels must get
    // SM slots while a long tensor kernel keeps every SM busy
    int prio_lo = 0, prio_hi = 0;
    PL2_CUDA_OK(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
    PL2_CUDA_OK(cudaStreamCreateWithPriority(&ctx->c.copy_stream, cudaStreamNonBlocking, prio_hi));
  }
  PL2_CUDA_OK(cudaFuncSetAttribute(king_wg_kernel<kTileCols>, cudaFuncAttributeMaxDynamicSharedMemorySize, KingWgShape<kTileCols>::kSmemBytes));
  PL2_CUDA_OK(cudaFuncSetAttribute(king_b1_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kKb1SmemBytes));
  *ctx_ptr = ctx;
  return 0;
}

int pl2gpu_ctx_destroy(Pl2GpuCtx* ctx) {
  if (!ctx) return 0;
  cudaSetDevice(ctx->c.device);
  pl2gpu_comm_destroy(ctx);
  if (ctx->c.stream) cudaStreamDestroy(ctx->c.stream);
  if (ctx->c.copy_stream) cudaStreamDestroy(ctx->c.copy_stream);
  for (auto& e : ctx->c.events)
    if (e) cudaEventDestroy(e);
  delete ctx;
  return 0;
}

int pl2gpu_ctx_synchronize(Pl2GpuCtx* ctx) {
  PL2_CUDA_OK(cudaSetDevice(ctx->c.device));
  PL2_CUDA_OK(cudaStreamSynchronize(ctx->c.stream));
  return 0;
}

void* pl2gpu_ctx_stream(Pl2GpuCtx* ctx) { return ctx ? static_cast<void*>(ctx->c.stream) : nullptr; }

uint64_t pl2gpu_ctx_launch_count(Pl2GpuCtx* ctx) { return ctx ? ctx->c.launches : 0; }

int pl2gpu_ctx_mem_info(Pl2GpuCtx* ctx, uint64_t* free_bytes, uint64_t* total_bytes) {
  if (!ctx) {
    set_error("pl2gpu_ctx_mem_info: null context");
    return 1;
  }
  PL2_CUDA_OK(cudaSetDevice(ctx->c.device));
  size_t f = 0, t = 0;
  PL2_CUDA_OK(cudaMemGetInfo(&f, &t));
  if (free_bytes) *free_bytes = f;
  if (total_bytes) *total_bytes = t;
  return 0;
}

int pl2gpu_host_alloc(uint64_t bytes, void** ptr) {
  *ptr = nullptr;
  PL2_CUDA_OK(cudaHostAlloc(ptr, bytes ? bytes : 1, cudaHostAllocDefault));
  return 0;
}

int pl2gpu_host_free(void* ptr) {
  if (ptr) PL2_CUDA_OK(cudaFreeHost(ptr));
  return 0;
}

int pl2gpu_ctx_event_record(Pl2GpuCtx* ctx, int slot) {
  if (!ctx || slot < 0 || slot >= 16) {
    set_error("pl2gpu_ctx_event_record: bad arguments");
    return 1;
  }
  PL2_CUDA_OK(cudaSetDevice(ctx->c.device));
  if (!ctx->c.events[slot]) PL2_CUDA_OK(cudaEventCreate(&ctx->c.events[slot]));
  PL2_CUDA_OK(cudaEventRecord(ctx->c.events[slot], ctx->c.stream));
  return 0;
}

int pl2gpu_ctx_event_elapsed_ms(Pl2GpuCtx* ctx, int slot_from, int slot_to, float* ms) {
  if (!ctx || slot_from < 0 || slot_from >= 16 || slot_to < 0 || slot_to >= 16 || !ctx->c.events[slot_from] || !ctx->c.events[slot_to]) {
    set_error("pl2gpu_ctx_event_elapsed_ms: bad arguments");
    return 1;
  }
  PL2_CUDA_OK(cudaSetDevice(ctx->c.device));
  PL2_CUDA_OK(cudaEventSynchronize(ctx->c.events[slot_to]));
  PL2_CUDA_OK(cudaEventElapsedTime(ms, ctx->c.events[slot_from], ctx->c.events[slot_to]));
  return 0;
}

// ------------------------------------------------------------------------------------------ communicator

int pl2gpu_comm_unique_id(uint8_t* id_out) {
  if (!id_out || !HaveNccl()) {
    if (!id_out) set_error("pl2gpu_comm_unique_id: null output");
    return 1;
  }
  static_assert(sizeof(ncclUniqueId) == PL2GPU_COMM_ID_BYTES, "ncclUniqueId size");
  ncclUniqueId id;
  PL2_NCCL_OK(g_nccl.GetUniqueId(&id));
  memcpy(id_out, &id, sizeof(id));
  return 0;
}

int pl2gpu_comm_init(Pl2GpuCtx* ctx, int rank, int world, const uint8_t* id) {
  if (!ctx || !id || world < 1 || rank < 0 || rank >= world) {
    set_error("pl2gpu_comm_init: bad arguments");
    return 1;
  }
  if (ctx->c.comm) {
    set_error("pl2gpu_comm_init: the context already has a communicator");
    return 1;
  }
  if (!HaveNccl()) return 1;
  PL2_CUDA_OK(cudaSetDevice(ctx->c.device));
  ncclUniqueId uid;
  memcpy(&uid, id, sizeof(uid));
  ncclComm_t comm = nullptr;
  PL2_NCCL_OK(g_nccl.CommInitRank(&comm, world, uid, rank));
  ctx->c.comm = comm;
  ctx->c.comm_rank = rank;
  ctx->c.comm_world = world;
  return 0;
}

int pl2gpu_comm_destroy(Pl2GpuCtx* ctx) {
  if (!ctx || !ctx->c.comm) return 0;
  cudaSetDevice(ctx->c.device);
  cudaStreamSynchronize(ctx->c.stream);
  cudaStreamSynchronize(ctx->c.copy_stream);
  g_nccl.CommDestroy(static_cast<ncclComm_t>(ctx->c.comm));
  ctx->c.comm = nullptr;
  ctx->c.comm_rank = 0;
  ctx->c.comm_world = 1;
  return 0;
}

int pl2gpu_comm_allreduce_sum_f64(Pl2GpuCtx* ctx, double* device_buf, uint64_t count) {
  if (!ctx || !device_buf) {
    set_error("pl2gpu_comm_allreduce_sum_f64: bad arguments");
    return 1;
  }
  PL2_CUDA_OK(cudaSetDevice(ctx->c.device));
  return CommAllReduceSumF64(&ctx->c, device_buf, count, ctx->c.stream);
}

// ------------------------------------------------------------------------------------------ KING

static uint32_t ClampStageCap(uint32_t max_variants_per_add) {
  uint32_t cap = max_variants_per_add ? max_variants_per_add : kMaxStageVariants;
  if (cap > kMaxStageVariantsEx) cap = kMaxStageVariantsEx;
  return RoundUpU32(cap, kVariantPad);
}
constexpr uint64_t kKingOutStageBytes = 256ull << 20;

uint64_t pl2gpu_king_mem_required(uint32_t sample_ct, uint32_t row_start, uint32_t row_end, uint32_t max_variants_per_add) {
  // Upper bound over the algorithms (the caller does not pass one) of exactly what pl2gpu_king_begin_ex
  // allocates for the same max_variants_per_add: accumulators + staged block(s) and their per-algorithm
  // re-layouts + tile lists + the output staging buffer, plus slack for allocator granularity.
  const uint64_t cap = ClampStageCap(max_variants_per_add);
  const uint64_t slack = 128ull << 20;
  // 128 x 96 tiles (tensor / popcount): raw block + its sample-major copy (tensor) or 3 bit planes (popcount)
  const uint64_t tiles = CountTiles(row_start, row_end, false);
  const uint64_t npad = RoundUpU32(sample_ct, kSamplePad);
  const uint64_t need_ss = tiles * kKingTileAccWords * 4 + cap * (npad / 4) + 3ull * (cap / 32) * npad * 4 + tiles * 16;
  // 128 x 64 tiles (the default): two raw blocks + two sample-major copies
  const uint64_t tiles_ts = CountTiles(row_start, row_end, false, kKingTsCols);
  const uint64_t npad_ts = RoundUpU32(sample_ct, kTsSamplePad);
  const uint64_t need_ts = tiles_ts * kKingTsTileAccWords * 4 + 4 * cap * (npad_ts / 4) + tiles_ts * 16;
  return (need_ss > need_ts ? need_ss : need_ts) + kKingOutStageBytes + slack;
}

int pl2gpu_king_begin(Pl2GpuCtx* ctx, uint32_t sample_ct, uint32_t row_start, uint32_t row_end, int algo, Pl2KingJob** job_ptr) {
  return pl2gpu_king_begin_ex(ctx, sample_ct, row_start, row_end, algo, 0, job_ptr);
}

uint64_t pl2gpu_king_mapped_mem_required(uint32_t sample_ct, uint32_t row_start, uint32_t row_end, uint32_t col_end, uint32_t max_variants_per_add) {
  // what pl2gpu_king_begin_mapped allocates: the TS accumulators of the cut tile list, two raw blocks + two sample-major
  // copies, the unmapped block, the position map, the output staging buffer, plus slack for allocator granularity
  const uint64_t cap = ClampStageCap(max_variants_per_add);
  const uint64_t tiles_ts = CountTiles(row_start, row_end, false, kKingTsCols, col_end);
  const uint64_t npad_ts = RoundUpU32(sample_ct, kTsSamplePad);
  return tiles_ts * kKingTsTileAccWords * 4 + 5 * cap * (npad_ts / 4) + tiles_ts * 16 + 4ull * sample_ct + kKingOutStageBytes + (128ull << 20);
}

static int KingBegin(Pl2GpuCtx* ctx, uint32_t sample_ct, const uint32_t* order, uint32_t row_start, uint32_t row_end, uint32_t col_end, int algo, uint32_t max_variants_per_add, Pl2KingJob** job_ptr) {
  *job_ptr = nullptr;
  if (!ctx) {
    set_error("pl2gpu_king_begin: null context");
    return 1;
  }
  if (sample_ct < 2 || row_end > sample_ct || row_start > row_end) {  // row_start == row_end: a rank that only takes part in the all-gathers
    set_error("pl2gpu_king_begin: bad row range [%u,%u) for %u samples", row_start, row_end, sample_ct);
    return 1;
  }
  if (!col_end || col_end > sample_ct) {
    set_error("pl2gpu_king_begin: bad column bound %u for %u samples", col_end, sample_ct);
    return 1;
  }
  if (algo == kPl2KingAlgoAuto) algo = kPl2KingAlgoTensorTS;
  if (algo != kPl2KingAlgoPopcount && algo != kPl2KingAlgoTensor && algo != kPl2KingAlgoTensorTS) {
    set_error("pl2gpu_king_begin: unknown algo %d", algo);
    return 1;
  }
  PL2_CUDA_OK(cudaSetDevice(ctx->c.device));
  Pl2KingJob* job = new Pl2KingJob();
  job->ctx = ctx;
  job->sample_ct = sample_ct;
  job->row_start = row_start;
  job->row_end = row_end;
  job->col_end = col_end;
  job->algo = algo;
  auto fail = [&]() {
    pl2gpu_king_end(job);
    return 1;
  };
  const bool ts = algo == kPl2KingAlgoTensorTS;
  const uint32_t cap = ClampStageCap(max_variants_per_add);
  bool ev_ok = cudaEventCreateWithFlags(&job->ev_copied, cudaEventDisableTiming) == cudaSuccess && cudaEventCreateWithFlags(&job->ev_src_ready, cudaEventDisableTiming) == cudaSuccess;
  for (int b = 0; b < 2 && ev_ok; ++b) {
    ev_ok = cudaEventCreateWithFlags(&job->ev_prep_done[b], cudaEventDisableTiming) == cudaSuccess && cudaEventCreate(&job->ev_kernel_start[b]) == cudaSuccess && cudaEventCreate(&job->ev_kernel_done[b]) == cudaSuccess;
  }
  if (!ev_ok) {
    set_error("pl2gpu_king_begin: cudaEventCreate failed");
    return fail();
  }
  job->tile_cols = ts ? kKingTsCols : kTileCols;
  if (BuildTileList(row_start, row_end, false, &job->tiles, job->tile_cols, col_end)) return fail();
  if (order && (cudaMalloc(&job->d_order, 4ull * sample_ct) != cudaSuccess || cudaMemcpy(job->d_order, order, 4ull * sample_ct, cudaMemcpyHostToDevice) != cudaSuccess)) {
    set_error("pl2gpu_king_begin_mapped: position map upload failed: %s", cudaGetErrorString(cudaGetLastError()));
    return fail();
  }
  for (int b = 0; b < (ts ? 2 : 1); ++b) {
    if (StageAlloc(sample_ct, cap, &job->stage[b], ts ? kTsSamplePad : kSamplePad)) return fail();
    if (order && b == 0 && cudaMalloc(&job->d_unmapped, static_cast<uint64_t>(job->stage[0].variant_cap) * job->stage[0].pitch) != cudaSuccess) {
      cudaGetLastError();
      set_error("pl2gpu_king_begin_mapped: insufficient device memory for the unmapped genotype block");
      return fail();
    }
    if (algo != kPl2KingAlgoPopcount) {
      const uint64_t raw_t_bytes = static_cast<uint64_t>(job->stage[b].sample_ct_padded) * (job->stage[b].variant_cap / 4);
      if (cudaMalloc(&job->d_raw_t[b], raw_t_bytes) != cudaSuccess) {
        cudaGetLastError();
        set_error("pl2gpu_king_begin: insufficient device memory for the sample-major genotype copy");
        return fail();
      }
    }
  }
  const uint64_t acc_bytes = static_cast<uint64_t>(job->tiles.tile_ct) * (5ull * job->tile_cols * kTileRows) * sizeof(int32_t);
  if (cudaMalloc(&job->d_raw_acc, acc_bytes ? acc_bytes : 4) != cudaSuccess) {
    cudaGetLastError();
    set_error("pl2gpu_king_begin: insufficient device memory for %u pair tiles (%.1f GB of accumulators); narrow the row range", job->tiles.tile_ct, acc_bytes / 1e9);
    return fail();
  }
  if (cudaMemsetAsync(job->d_raw_acc, 0, acc_bytes, ctx->c.stream) != cudaSuccess) {
    set_error("pl2gpu_king_begin: cudaMemsetAsync failed: %s", cudaGetErrorString(cudaGetLastError()));
    return fail();
  }
  if (algo == kPl2KingAlgoPopcount) {
    const uint64_t plane_bytes = 3ull * (job->stage[0].variant_cap / 32) * job->stage[0].sample_ct_padded * sizeof(uint32_t);
    if (cudaMalloc(&job->d_planes, plane_bytes) != cudaSuccess) {
      cudaGetLastError();
      set_error("pl2gpu_king_begin: insufficient device memory for bit planes");
      return fail();
    }
  }
  job->out_stage_bytes = kKingOutStageBytes;
  if (cudaMalloc(&job->d_out_stage, job->out_stage_bytes) != cudaSuccess) {
    cudaGetLastError();
    set_error("pl2gpu_king_begin: insufficient device memory for output staging");
    return fail();
  }
  *job_ptr = job;
  return 0;
}

int pl2gpu_king_begin_ex(Pl2GpuCtx* ctx, uint32_t sample_ct, uint32_t row_start, uint32_t row_end, int algo, uint32_t max_variants_per_add, Pl2KingJob** job_ptr) {
  return KingBegin(ctx, sample_ct, nullptr, row_start, row_end, sample_ct, algo, max_variants_per_add, job_ptr);
}

int pl2gpu_king_begin_mapped(Pl2GpuCtx* ctx, uint32_t sample_ct, const uint32_t* order, uint32_t row_start, uint32_t row_end, uint32_t col_end, uint32_t max_variants_per_add, Pl2KingJob** job_ptr) {
  if (order) {
    // a permutation of the samples: every index once
    std::vector<uint8_t> seen(sample_ct, 0);
    for (uint32_t p = 0; p < sample_ct; ++p) {
      if (order[p] >= sample_ct || seen[order[p]]++) {
        *job_ptr = nullptr;
        set_error("pl2gpu_king_begin_mapped: order[] is not a permutation of the %u samples (position %u)", sample_ct, p);
        return 1;
      }
    }
  }
  return KingBegin(ctx, sample_ct, order, row_start, row_end, col_end, kPl2KingAlgoTensorTS, max_variants_per_add, job_ptr);
}

// TS path: the staged block stage[b] holds `cur` variants (rows [0, cur)); pad it, write its sample-major copy
// and queue the tensor kernel.  Everything up to the kernel runs on the prep stream.
static int KingTsPrepAndLaunch(Pl2KingJob* job, uint32_t b, uint32_t cur, bool pad_valid_rows) {
  Ctx* c = &job->ctx->c;
  cudaStream_t prep = c->copy_stream;
  GenoStage& st = job->stage[b];
  const uint32_t padded = RoundUpU32(cur, kVariantPad);
  // pad_valid_rows == false: the valid rows were already padded slice by slice (sharded add); only the tail rows remain
  if (pad_valid_rows) {
    PL2_TRY(LaunchPadGenotypes(c, st.d_raw, st.pitch, st.sample_ct, cur, padded, prep));
  } else if (padded > cur) {
    PL2_TRY(LaunchPadGenotypes(c, st.d_raw + static_cast<uint64_t>(cur) * st.pitch, st.pitch, st.sample_ct, 0, padded - cur, prep));
  }
  if (!job->tiles.tile_ct) {  // nothing to count on this rank: only order later reuse of the buffer behind the gather
    PL2_CUDA_OK(cudaEventRecord(job->ev_kernel_done[b], prep));
    job->kernel_pending[b] = true;
    return 0;
  }
  geno_tile_rows_kernel<true><<<dim3(padded / 64, st.sample_ct_padded / 64), 256, 0, prep>>>(st.d_raw, st.pitch, padded / 32, 0, job->d_raw_t[b]);
  c->launches++;
  PL2_CUDA_OK(cudaGetLastError());
  PL2_CUDA_OK(cudaEventRecord(job->ev_prep_done[b], prep));
  PL2_CUDA_OK(cudaStreamWaitEvent(c->stream, job->ev_prep_done[b], 0));
  PL2_CUDA_OK(cudaEventRecord(job->ev_kernel_start[b], c->stream));
  king_b1_kernel<<<job->tiles.tile_ct, kKwThreads, kKb1SmemBytes, c->stream>>>(job->d_raw_t[b], padded, job->tiles.d_tile_order, job->tiles.d_tile_rt, job->tiles.d_tile_tc, job->d_raw_acc);
  c->launches++;
  PL2_CUDA_OK(cudaGetLastError());
  PL2_CUDA_OK(cudaEventRecord(job->ev_kernel_done[b], c->stream));
  job->kernel_pending[b] = true;
  job->last_buf = static_cast<int>(b);
  return 0;
}

int pl2gpu_king_add_variants(Pl2KingJob* job, const void* genovecs, uint64_t variant_stride_bytes, uint32_t variant_ct, int src_is_device) {
  if (!job) {
    set_error("pl2gpu_king_add_variants: null job");
    return 1;
  }
  Ctx* c = &job->ctx->c;
  PL2_CUDA_OK(cudaSetDevice(c->device));
  const uint64_t min_stride = 8ull * DivUpU32(job->sample_ct, 32);
  if (variant_stride_bytes < DivUpU32(job->sample_ct, 4)) {
    set_error("pl2gpu_king_add_variants: variant stride %llu < %u bytes of genotype data (PgrGet rows are %llu bytes)", static_cast<unsigned long long>(variant_stride_bytes), DivUpU32(job->sample_ct, 4), static_cast<unsigned long long>(min_stride));
    return 1;
  }
  const uint8_t* src = static_cast<const uint8_t*>(genovecs);
  const bool ts = job->algo == kPl2KingAlgoTensorTS;
  uint32_t done = 0;
  while (done < variant_ct) {
    uint32_t cur = variant_ct - done;
    if (cur > job->stage[0].variant_cap) cur = job->stage[0].variant_cap;
    const uint8_t* src_cur = src + static_cast<uint64_t>(done) * variant_stride_bytes;
    if (ts && job->tiles.tile_ct) {
      // Double-buffered: copy + pad + row re-tiling on the prep stream while the previous batch's tensor
      // kernel (which reads the OTHER staged block through its tensor map) is still running.
      const uint32_t b = job->buf_idx;
      job->buf_idx ^= 1;
      GenoStage& st = job->stage[b];
      cudaStream_t prep = c->copy_stream;
      if (job->kernel_pending[b]) PL2_CUDA_OK(cudaStreamWaitEvent(prep, job->ev_kernel_done[b], 0));
      if (src_is_device == 1) {
        // device source produced by work the caller ordered on the context's stream
        PL2_CUDA_OK(cudaEventRecord(job->ev_src_ready, c->stream));
        PL2_CUDA_OK(cudaStreamWaitEvent(prep, job->ev_src_ready, 0));
      }
      // a mapped job lands the caller's rows in d_unmapped and gathers them into position order (the prep stream runs
      // copy and gather in turn, so one unmapped block serves both staged buffers)
      uint8_t* const land = job->d_order ? job->d_unmapped : st.d_raw;
      PL2_CUDA_OK(cudaMemcpy2DAsync(land, st.pitch, src_cur, variant_stride_bytes, DivUpU32(st.sample_ct, 4), cur, src_is_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, prep));
      PL2_CUDA_OK(cudaEventRecord(job->ev_copied, prep));
      for (uint32_t v0 = 0; job->d_order && v0 < cur; v0 += 32768) {  // grid.y is at most 65,535 rows
        const uint32_t rows = std::min(cur - v0, 32768u);
        geno_gather_kernel<<<dim3(DivUpU32(st.pitch, 256), rows), 256, 0, prep>>>(land + static_cast<uint64_t>(v0) * st.pitch, st.pitch, st.d_raw + static_cast<uint64_t>(v0) * st.pitch, st.pitch, job->d_order, st.sample_ct);
        c->launches++;
        PL2_CUDA_OK(cudaGetLastError());
      }
      PL2_TRY(KingTsPrepAndLaunch(job, b, cur, true));
      if (!src_is_device) PL2_CUDA_OK(cudaEventSynchronize(job->ev_copied));  // the caller may reuse its buffer; the kernels keep running
    } else {
      uint32_t padded = 0;
      PL2_TRY(StageUpload(c, &job->stage[0], src_cur, variant_stride_bytes, cur, src_is_device, &padded));
      if (job->tiles.tile_ct) {
        if (job->algo == kPl2KingAlgoPopcount) {
          const uint32_t word_ct = padded / 32;
          const uint64_t warps = static_cast<uint64_t>(job->stage[0].sample_ct_padded / 32) * word_ct;
          split_transpose_kernel<<<static_cast<uint32_t>(DivUpU64(warps, 8)), 256, 0, c->stream>>>(job->stage[0].d_raw, job->stage[0].pitch, job->stage[0].sample_ct_padded, word_ct, job->d_planes);
          c->launches++;
          king_popc_kernel<<<job->tiles.tile_ct * 2, 256, 0, c->stream>>>(job->d_planes, job->stage[0].sample_ct_padded, word_ct, job->tiles.d_tile_rt, job->tiles.d_tile_tc, job->d_raw_acc);
          c->launches++;
        } else {
          const GenoStage& st = job->stage[0];
          geno_tile_rows_kernel<<<dim3(padded / 64, st.sample_ct_padded / 64), 256, 0, c->stream>>>(st.d_raw, st.pitch, padded / 32, 0, job->d_raw_t[0]);
          c->launches++;
          king_wg_kernel<kTileCols><<<2 * job->tiles.tile_ct, kKwThreads, KingWgShape<kTileCols>::kSmemBytes, c->stream>>>(job->d_raw_t[0], padded, job->tiles.d_tile_order, job->tiles.d_tile_rt, job->tiles.d_tile_tc, job->d_raw_acc);
          c->launches++;
        }
        PL2_CUDA_OK(cudaGetLastError());
      }
      // host source on the compute stream: it has been consumed once the stream reaches here
      if (!src_is_device) PL2_CUDA_OK(cudaStreamSynchronize(c->stream));
    }
    done += cur;
  }
  job->variants_added += variant_ct;
  return 0;
}

int pl2gpu_king_add_variants_sharded(Pl2KingJob* job, const void* slice, uint64_t variant_stride_bytes, uint32_t slice_variant_ct, int src_is_device) {
  if (!job || !job->ctx->c.comm) {
    set_error("pl2gpu_king_add_variants_sharded: %s", job ? "no communicator attached to the context (pl2gpu_comm_init)" : "null job");
    return 1;
  }
  Ctx* c = &job->ctx->c;
  PL2_CUDA_OK(cudaSetDevice(c->device));
  if (job->algo != kPl2KingAlgoTensorTS) {
    set_error("pl2gpu_king_add_variants_sharded: only the default (TS tensor) algorithm is sharded");
    return 1;
  }
  if (job->d_order || job->col_end != job->sample_ct) {
    set_error("pl2gpu_king_add_variants_sharded: a mapped job (pl2gpu_king_begin_mapped) runs on one device");
    return 1;
  }
  const uint64_t total64 = static_cast<uint64_t>(slice_variant_ct) * c->comm_world;
  if (!slice_variant_ct || total64 > job->stage[0].variant_cap) {
    set_error("pl2gpu_king_add_variants_sharded: %u variants x %d ranks exceed the stage capacity %u", slice_variant_ct, c->comm_world, job->stage[0].variant_cap);
    return 1;
  }
  if (variant_stride_bytes < DivUpU32(job->sample_ct, 4)) {
    set_error("pl2gpu_king_add_variants_sharded: variant stride too small");
    return 1;
  }
  const uint32_t total = static_cast<uint32_t>(total64);
  const uint32_t b = job->buf_idx;
  job->buf_idx ^= 1;
  GenoStage& st = job->stage[b];
  cudaStream_t prep = c->copy_stream;
  if (job->kernel_pending[b]) PL2_CUDA_OK(cudaStreamWaitEvent(prep, job->ev_kernel_done[b], 0));
  if (src_is_device == 1) {
    PL2_CUDA_OK(cudaEventRecord(job->ev_src_ready, c->stream));
    PL2_CUDA_OK(cudaStreamWaitEvent(prep, job->ev_src_ready, 0));
  }
  // this rank's variants land at rows [rank * slice, (rank + 1) * slice) of the staged block, are padded
  // there, and ONE in-place all-gather of the genotype column tile makes the block complete on every GPU
  uint8_t* mine = st.d_raw + static_cast<uint64_t>(c->comm_rank) * slice_variant_ct * st.pitch;
  PL2_CUDA_OK(cudaMemcpy2DAsync(mine, st.pitch, slice, variant_stride_bytes, DivUpU32(st.sample_ct, 4), slice_variant_ct, src_is_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, prep));
  PL2_CUDA_OK(cudaEventRecord(job->ev_copied, prep));
  PL2_TRY(LaunchPadGenotypes(c, mine, st.pitch, st.sample_ct, slice_variant_ct, slice_variant_ct, prep));
  PL2_TRY(CommAllGatherInPlace(c, st.d_raw, static_cast<uint64_t>(slice_variant_ct) * st.pitch, prep));
  PL2_TRY(KingTsPrepAndLaunch(job, b, total, false));
  if (!src_is_device) PL2_CUDA_OK(cudaEventSynchronize(job->ev_copied));
  job->variants_added += total;
  return 0;
}

static int KingGet(Pl2KingJob* job, uint32_t r0, uint32_t r1, void* dst, int dst_is_device, bool kinship) {
  if (!job) {
    set_error("pl2gpu_king_get: null job");
    return 1;
  }
  if (r0 < job->row_start || r1 > job->row_end || r0 > r1) {
    set_error("pl2gpu_king_get: rows [%u,%u) outside the job's [%u,%u)", r0, r1, job->row_start, job->row_end);
    return 1;
  }
  Ctx* c = &job->ctx->c;
  PL2_CUDA_OK(cudaSetDevice(c->device));
  const uint64_t bytes_per_pair = kinship ? 8 : 20;
  const uint32_t col_end = job->col_end;
  auto tri = [col_end](uint64_t r) { return KingPairsBelow(r, col_end); };
  uint8_t* out = static_cast<uint8_t*>(dst);
  uint32_t cur0 = r0;
  while (cur0 < r1) {
    uint32_t cur1;
    void* d_dst;
    if (dst_is_device) {
      cur1 = r1;
      d_dst = out;
    } else {
      // largest row block whose pairs fit the staging buffer (at least one row)
      cur1 = cur0 + 1;
      while (cur1 < r1 && (tri(cur1 + 1) - tri(cur0)) * bytes_per_pair <= job->out_stage_bytes) ++cur1;
      if ((tri(cur1) - tri(cur0)) * bytes_per_pair > job->out_stage_bytes) {
        set_error("pl2gpu_king_get: a single row exceeds the staging buffer");
        return 1;
      }
      d_dst = job->d_out_stage;
    }
    const uint64_t pairs = tri(cur1) - tri(cur0);
    if (pairs) {
      const uint32_t rt_a = cur0 / kTileRows - job->tiles.row_tile_first;
      const uint32_t rt_b = (cur1 - 1) / kTileRows - job->tiles.row_tile_first;
      const uint32_t tile_a = job->tiles.h_rowtile_offset[rt_a];
      const uint32_t tile_b = job->tiles.h_rowtile_offset[rt_b + 1];
      if (tile_b > tile_a) {
        const uint32_t grid = (tile_b - tile_a) * 8;
        const int32_t* acc0 = job->d_raw_acc + static_cast<uint64_t>(tile_a) * (5ull * job->tile_cols * kTileRows);
        const uint32_t* trt = job->tiles.d_tile_rt + tile_a;
        const uint32_t* ttc = job->tiles.d_tile_tc + tile_a;
        if (job->tile_cols == kKingTsCols) {
          if (kinship) king_finalize_kernel<true, kKingTsCols><<<grid, 256, 0, c->stream>>>(acc0, trt, ttc, job->sample_ct, col_end, cur0, cur1, nullptr, static_cast<double*>(d_dst));
          else king_finalize_kernel<false, kKingTsCols><<<grid, 256, 0, c->stream>>>(acc0, trt, ttc, job->sample_ct, col_end, cur0, cur1, static_cast<uint32_t*>(d_dst), nullptr);
        } else {
          if (kinship) king_finalize_kernel<true, kTileCols><<<grid, 256, 0, c->stream>>>(acc0, trt, ttc, job->sample_ct, col_end, cur0, cur1, nullptr, static_cast<double*>(d_dst));
          else king_finalize_kernel<false, kTileCols><<<grid, 256, 0, c->stream>>>(acc0, trt, ttc, job->sample_ct, col_end, cur0, cur1, static_cast<uint32_t*>(d_dst), nullptr);
        }
        c->launches++;
        PL2_CUDA_OK(cudaGetLastError());
      }
      if (!dst_is_device) {
        PL2_CUDA_OK(cudaMemcpyAsync(out, d_dst, pairs * bytes_per_pair, cudaMemcpyDeviceToHost, c->stream));
        PL2_CUDA_OK(cudaStreamSynchronize(c->stream));
        out += pairs * bytes_per_pair;
      }
    }
    cur0 = cur1;
  }
  if (dst_is_device) {
    // caller synchronises through pl2gpu_ctx_synchronize / its own stream ordering
  }
  return 0;
}

int pl2gpu_king_get_counts(Pl2KingJob* job, uint32_t out_row_start, uint32_t out_row_end, uint32_t* dst, int dst_is_device) {
  return KingGet(job, out_row_start, out_row_end, dst, dst_is_device, false);
}

int pl2gpu_king_get_kinship(Pl2KingJob* job, uint32_t out_row_start, uint32_t out_row_end, double* dst, int dst_is_device) {
  return KingGet(job, out_row_start, out_row_end, dst, dst_is_device, true);
}

int pl2gpu_king_get_filtered(Pl2KingJob* job, uint32_t r0, uint32_t r1, double min_kinship, uint64_t max_out, uint32_t* pairs_out, uint32_t* counts_out, double* kinship_out, uint64_t* n_found) {
  if (!job || !n_found || (max_out && (!pairs_out || !counts_out || !kinship_out))) {
    set_error("pl2gpu_king_get_filtered: bad arguments");
    return 1;
  }
  if (r0 < job->row_start || r1 > job->row_end || r0 > r1) {
    set_error("pl2gpu_king_get_filtered: rows [%u,%u) outside the job's [%u,%u)", r0, r1, job->row_start, job->row_end);
    return 1;
  }
  *n_found = 0;
  Ctx* c = &job->ctx->c;
  PL2_CUDA_OK(cudaSetDevice(c->device));
  if (!job->tiles.tile_ct || r0 == r1) return 0;
  unsigned long long* d_found = nullptr;
  uint32_t *d_pairs = nullptr, *d_counts = nullptr;
  double* d_kin = nullptr;
  const uint64_t cap = max_out ? max_out : 1;
  int rc = 1;
  do {
    if (cudaMalloc(&d_found, 8) != cudaSuccess || cudaMalloc(&d_pairs, cap * 8) != cudaSuccess || cudaMalloc(&d_counts, cap * 20) != cudaSuccess || cudaMalloc(&d_kin, cap * 8) != cudaSuccess) {
      cudaGetLastError();
      set_error("pl2gpu_king_get_filtered: insufficient device memory for %llu result slots", static_cast<unsigned long long>(max_out));
      break;
    }
    if (cudaMemsetAsync(d_found, 0, 8, c->stream) != cudaSuccess) break;
    if (job->tile_cols == kKingTsCols) {
      king_filter_kernel<kKingTsCols><<<job->tiles.tile_ct, kTileRows, 0, c->stream>>>(job->d_raw_acc, job->tiles.d_tile_rt, job->tiles.d_tile_tc, job->sample_ct, job->col_end, r0, r1, min_kinship, max_out, d_found, d_pairs, d_counts, d_kin);
    } else {
      king_filter_kernel<kTileCols><<<job->tiles.tile_ct, kTileRows, 0, c->stream>>>(job->d_raw_acc, job->tiles.d_tile_rt, job->tiles.d_tile_tc, job->sample_ct, job->col_end, r0, r1, min_kinship, max_out, d_found, d_pairs, d_counts, d_kin);
    }
    c->launches++;
    unsigned long long found = 0;
    if (cudaGetLastError() != cudaSuccess || cudaMemcpyAsync(&found, d_found, 8, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess || cudaStreamSynchronize(c->stream) != cudaSuccess) {
      set_error("pl2gpu_king_get_filtered: %s", cudaGetErrorString(cudaGetLastError()));
      break;
    }
    *n_found = found;
    const uint64_t k = found < max_out ? found : max_out;
    if (k) {
      std::vector<uint32_t> hp(2 * k), hc(5 * k);
      std::vector<double> hk(k);
      if (cudaMemcpy(hp.data(), d_pairs, k * 8, cudaMemcpyDeviceToHost) != cudaSuccess || cudaMemcpy(hc.data(), d_counts, k * 20, cudaMemcpyDeviceToHost) != cudaSuccess || cudaMemcpy(hk.data(), d_kin, k * 8, cudaMemcpyDeviceToHost) != cudaSuccess) {
        set_error("pl2gpu_king_get_filtered: %s", cudaGetErrorString(cudaGetLastError()));
        break;
      }
      std::vector<uint64_t> order(k);
      for (uint64_t q = 0; q < k; ++q) order[q] = q;
      std::sort(order.begin(), order.end(), [&](uint64_t a, uint64_t b) { return hp[2 * a] != hp[2 * b] ? hp[2 * a] < hp[2 * b] : hp[2 * a + 1] < hp[2 * b + 1]; });
      for (uint64_t q = 0; q < k; ++q) {
        const uint64_t src = order[q];
        pairs_out[2 * q] = hp[2 * src];
        pairs_out[2 * q + 1] = hp[2 * src + 1];
        memcpy(counts_out + 5 * q, &hc[5 * src], 20);
        kinship_out[q] = hk[src];
      }
    }
    rc = 0;
  } while (0);
  cudaFree(d_found);
  cudaFree(d_pairs);
  cudaFree(d_counts);
  cudaFree(d_kin);
  return rc;
}

uint64_t pl2gpu_king_variants_added(Pl2KingJob* job) { return job ? job->variants_added : 0; }

int pl2gpu_king_last_kernel_ms(Pl2KingJob* job, float* ms) {
  if (!job || !ms || job->last_buf < 0) {
    set_error("pl2gpu_king_last_kernel_ms: no tensor-kernel launch has been recorded (TS algorithm only)");
    return 1;
  }
  PL2_CUDA_OK(cudaSetDevice(job->ctx->c.device));
  PL2_CUDA_OK(cudaEventSynchronize(job->ev_kernel_done[job->last_buf]));
  PL2_CUDA_OK(cudaEventElapsedTime(ms, job->ev_kernel_start[job->last_buf], job->ev_kernel_done[job->last_buf]));
  return 0;
}

int pl2gpu_king_end(Pl2KingJob* job) {
  if (!job) return 0;
  if (job->ctx) {
    cudaSetDevice(job->ctx->c.device);
    cudaStreamSynchronize(job->ctx->c.stream);
    if (job->ctx->c.copy_stream) cudaStreamSynchronize(job->ctx->c.copy_stream);
  }
  if (job->ev_copied) cudaEventDestroy(job->ev_copied);
  if (job->ev_src_ready) cudaEventDestroy(job->ev_src_ready);
  FreeTileList(&job->tiles);
  for (int b = 0; b < 2; ++b) {
    if (job->ev_prep_done[b]) cudaEventDestroy(job->ev_prep_done[b]);
    if (job->ev_kernel_start[b]) cudaEventDestroy(job->ev_kernel_start[b]);
    if (job->ev_kernel_done[b]) cudaEventDestroy(job->ev_kernel_done[b]);
    StageFree(&job->stage[b]);
    cudaFree(job->d_raw_t[b]);
  }
  cudaFree(job->d_order);
  cudaFree(job->d_unmapped);
  cudaFree(job->d_planes);
  cudaFree(job->d_raw_acc);
  cudaFree(job->d_out_stage);
  cudaGetLastError();
  delete job;
  return 0;
}

// ------------------------------------------------------------------------------------------ pair list

struct Pl2KingPairJob {
  Pl2GpuCtx* ctx = nullptr;
  uint32_t sample_ct = 0;
  uint64_t pair_ct = 0;
  GenoStage stage;
  uint8_t* d_raw_t = nullptr;   // sample-major 2-bit copy of the staged block
  uint32_t* d_pairs = nullptr;  // [pair][2]
  uint32_t* d_counts = nullptr; // [pair][5]
};

int pl2gpu_king_pairs_begin(Pl2GpuCtx* ctx, uint32_t sample_ct, const uint32_t* pairs_host, uint64_t pair_ct, Pl2KingPairJob** job_ptr) {
  if (job_ptr) *job_ptr = nullptr;
  if (!ctx || !job_ptr || !sample_ct || (pair_ct && !pairs_host)) {
    set_error("pl2gpu_king_pairs_begin: bad arguments");
    return 1;
  }
  for (uint64_t p = 0; p < 2 * pair_ct; ++p) {
    if (pairs_host[p] >= sample_ct) {
      set_error("pl2gpu_king_pairs_begin: pair %llu names sample %u of %u", static_cast<unsigned long long>(p / 2), pairs_host[p], sample_ct);
      return 1;
    }
  }
  PL2_CUDA_OK(cudaSetDevice(ctx->c.device));
  Pl2KingPairJob* job = new Pl2KingPairJob();
  job->ctx = ctx;
  job->sample_ct = sample_ct;
  job->pair_ct = pair_ct;
  auto fail = [&]() {
    pl2gpu_king_pairs_end(job);
    return 1;
  };
  if (StageAlloc(sample_ct, kMaxStageVariants, &job->stage, 64)) return fail();
  const uint64_t n_alloc = pair_ct ? pair_ct : 1;
  if (cudaMalloc(&job->d_raw_t, static_cast<uint64_t>(job->stage.sample_ct_padded) * (job->stage.variant_cap / 4)) != cudaSuccess || cudaMalloc(&job->d_pairs, n_alloc * 8) != cudaSuccess ||
      cudaMalloc(&job->d_counts, n_alloc * 20) != cudaSuccess) {
    cudaGetLastError();
    set_error("pl2gpu_king_pairs_begin: insufficient device memory for %llu pairs", static_cast<unsigned long long>(pair_ct));
    return fail();
  }
  if (cudaMemcpyAsync(job->d_pairs, pairs_host, pair_ct * 8, cudaMemcpyHostToDevice, ctx->c.stream) != cudaSuccess || cudaMemsetAsync(job->d_counts, 0, n_alloc * 20, ctx->c.stream) != cudaSuccess ||
      cudaStreamSynchronize(ctx->c.stream) != cudaSuccess) {
    set_error("pl2gpu_king_pairs_begin: %s", cudaGetErrorString(cudaGetLastError()));
    return fail();
  }
  *job_ptr = job;
  return 0;
}

int pl2gpu_king_pairs_add_variants(Pl2KingPairJob* job, const void* genovecs, uint64_t variant_stride_bytes, uint32_t variant_ct, int src_is_device) {
  if (!job || (!genovecs && variant_ct)) {
    set_error("pl2gpu_king_pairs_add_variants: bad arguments");
    return 1;
  }
  Ctx* c = &job->ctx->c;
  PL2_CUDA_OK(cudaSetDevice(c->device));
  const uint64_t min_stride = static_cast<uint64_t>(DivUpU32(job->sample_ct, 4));
  if (variant_stride_bytes < min_stride) {
    set_error("pl2gpu_king_pairs_add_variants: variant stride %llu < %llu bytes of genotype data", static_cast<unsigned long long>(variant_stride_bytes), static_cast<unsigned long long>(min_stride));
    return 1;
  }
  const uint8_t* src = static_cast<const uint8_t*>(genovecs);
  uint32_t done = 0;
  while (done < variant_ct) {
    uint32_t cur = variant_ct - done;
    if (cur > job->stage.variant_cap) cur = job->stage.variant_cap;
    uint32_t padded = 0;
    PL2_TRY(StageUpload(c, &job->stage, src + static_cast<uint64_t>(done) * variant_stride_bytes, variant_stride_bytes, cur, src_is_device, &padded));
    if (job->pair_ct) {
      const uint32_t pitch_t = padded / 4;
      geno_transpose_kernel<<<dim3(padded / 64, job->stage.sample_ct_padded / 64), 256, 0, c->stream>>>(job->stage.d_raw, job->stage.pitch, job->d_raw_t, pitch_t);
      king_pairs_kernel<<<static_cast<uint32_t>(DivUpU64(job->pair_ct, 8)), 256, 0, c->stream>>>(job->d_raw_t, pitch_t, padded / 32, job->d_pairs, job->pair_ct, job->d_counts);
      c->launches += 2;
      PL2_CUDA_OK(cudaGetLastError());
    }
    if (!src_is_device) PL2_CUDA_OK(cudaStreamSynchronize(c->stream));
    done += cur;
  }
  return 0;
}

int pl2gpu_king_pairs_get_counts(Pl2KingPairJob* job, uint64_t pair_start, uint64_t pair_end, uint32_t* dst, int dst_is_device) {
  if (!job || pair_start > pair_end || pair_end > job->pair_ct || (!dst && pair_end > pair_start)) {
    set_error("pl2gpu_king_pairs_get_counts: bad arguments");
    return 1;
  }
  Ctx* c = &job->ctx->c;
  PL2_CUDA_OK(cudaSetDevice(c->device));
  if (pair_end > pair_start) {
    PL2_CUDA_OK(cudaMemcpyAsync(dst, job->d_counts + 5 * pair_start, (pair_end - pair_start) * 20, dst_is_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, c->stream));
  }
  PL2_CUDA_OK(cudaStreamSynchronize(c->stream));
  return 0;
}

int pl2gpu_king_pairs_end(Pl2KingPairJob* job) {
  if (!job) return 0;
  if (job->ctx) {
    cudaSetDevice(job->ctx->c.device);
    cudaStreamSynchronize(job->ctx->c.stream);
  }
  StageFree(&job->stage);
  cudaFree(job->d_raw_t);
  cudaFree(job->d_pairs);
  cudaFree(job->d_counts);
  cudaGetLastError();
  delete job;
  return 0;
}

// ------------------------------------------------------------------------------------------ probe

int pl2gpu_int8_peak(Pl2GpuCtx* ctx, uint32_t n_cols, int form, double min_seconds, double* tops_out, double* seconds_out) {
  if (!ctx || !tops_out || (form != 1 && form != 2) || (n_cols != 64 && n_cols != 128 && (form == 2 || (n_cols != 80 && n_cols != 96)))) {
    set_error("pl2gpu_int8_peak: bad arguments (form 1 = int8, n_cols 64, 80, 96 or 128; form 2 = b1 AND-POPC, n_cols 64 or 128)");
    return 1;
  }
  Ctx* c = &ctx->c;
  PL2_CUDA_OK(cudaSetDevice(c->device));
  int32_t* d_sink = nullptr;
  PL2_CUDA_OK(cudaMalloc(&d_sink, 256 * sizeof(int32_t)));
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  PL2_CUDA_OK(cudaEventCreate(&e0));
  PL2_CUDA_OK(cudaEventCreate(&e1));
  const uint32_t blocks = 4096;  // x 32 wgmmas x 2 warpgroups per SM
  const double k_per_wgmma = form == 2 ? 256 : 32;
  const double ops_per_launch = 2.0 * 64 * n_cols * k_per_wgmma * 32.0 * 2 * blocks * c->sm_count;
  auto launch = [&]() {
    if (form == 2 && n_cols == 64) wgmma_b1_peak_kernel<64><<<c->sm_count, 256, 0, c->stream>>>(blocks, d_sink);
    else if (form == 2) wgmma_b1_peak_kernel<128><<<c->sm_count, 256, 0, c->stream>>>(blocks, d_sink);
    else if (n_cols == 64) wgmma_peak_kernel<64><<<c->sm_count, 256, 0, c->stream>>>(blocks, d_sink);
    else if (n_cols == 80) wgmma_peak_kernel<80><<<c->sm_count, 256, 0, c->stream>>>(blocks, d_sink);
    else if (n_cols == 96) wgmma_peak_kernel<96><<<c->sm_count, 256, 0, c->stream>>>(blocks, d_sink);
    else wgmma_peak_kernel<128><<<c->sm_count, 256, 0, c->stream>>>(blocks, d_sink);
    c->launches++;
  };
  launch();  // warm-up
  PL2_CUDA_OK(cudaStreamSynchronize(c->stream));
  PL2_CUDA_OK(cudaGetLastError());
  double total_s = 0, total_ops = 0;
  const uint32_t per_batch = 8;
  while (total_s < min_seconds) {
    PL2_CUDA_OK(cudaEventRecord(e0, c->stream));
    for (uint32_t k = 0; k < per_batch; ++k) launch();
    PL2_CUDA_OK(cudaEventRecord(e1, c->stream));
    PL2_CUDA_OK(cudaEventSynchronize(e1));
    PL2_CUDA_OK(cudaGetLastError());
    float ms = 0;
    PL2_CUDA_OK(cudaEventElapsedTime(&ms, e0, e1));
    total_s += ms * 1e-3;
    total_ops += ops_per_launch * per_batch;
    if (min_seconds <= 0) break;
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  cudaFree(d_sink);
  *tops_out = total_ops / total_s / 1e12;
  if (seconds_out) *seconds_out = total_s;
  return 0;
}

int pl2gpu_bulk_read_rate(Pl2GpuCtx* ctx, uint64_t working_set_bytes, uint32_t inflight_bytes, double min_seconds, double* tbps_out, double* seconds_out) {
  const uint64_t max_inflight = (kKwSmemLimit - 128) / (kFeedChunk + 8) * kFeedChunk;
  if (!ctx || !tbps_out || inflight_bytes == 0 || inflight_bytes % kFeedChunk || inflight_bytes > max_inflight || working_set_bytes < kFeedChunk || working_set_bytes / kFeedChunk > 0xFFFFFFFFull) {
    set_error("pl2gpu_bulk_read_rate: bad arguments (inflight_bytes: a multiple of %u up to %llu; working_set_bytes: at least %u)", kFeedChunk, static_cast<unsigned long long>(max_inflight), kFeedChunk);
    return 1;
  }
  Ctx* c = &ctx->c;
  PL2_CUDA_OK(cudaSetDevice(c->device));
  const uint32_t ws_chunks = static_cast<uint32_t>(working_set_bytes / kFeedChunk);
  const uint32_t chunks = inflight_bytes / kFeedChunk;
  const uint32_t smem = chunks * (kFeedChunk + 8) + 128;
  // about 64 MB per SM and launch
  const uint32_t rounds = std::max<uint32_t>(2, (64u << 20) / inflight_bytes);
  const double bytes_per_launch = static_cast<double>(kFeedChunk) * chunks * rounds * c->sm_count;
  uint8_t* d_src = nullptr;
  PL2_CUDA_OK(cudaMalloc(&d_src, static_cast<uint64_t>(ws_chunks) * kFeedChunk));
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  auto release = [&]() {
    cudaFree(d_src);
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
  };
  auto fail = [&]() {
    release();
    return 1;
  };
  if (cudaMemsetAsync(d_src, 0x5A, static_cast<uint64_t>(ws_chunks) * kFeedChunk, c->stream) != cudaSuccess || cudaEventCreate(&e0) != cudaSuccess || cudaEventCreate(&e1) != cudaSuccess ||
      cudaFuncSetAttribute(bulk_read_probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) {
    set_error("pl2gpu_bulk_read_rate: set-up failed: %s", cudaGetErrorString(cudaGetLastError()));
    return fail();
  }
  auto launch = [&]() {
    bulk_read_probe_kernel<<<c->sm_count, 32, smem, c->stream>>>(d_src, ws_chunks, chunks, rounds);
    c->launches++;
  };
  launch();  // warm-up: also brings an L2-sized working set into L2
  double total_s = 0, total_bytes = 0;
  const uint32_t per_batch = 4;
  while (true) {
    if (cudaEventRecord(e0, c->stream) != cudaSuccess) return fail();
    for (uint32_t k = 0; k < per_batch; ++k) launch();
    float ms = 0;
    if (cudaEventRecord(e1, c->stream) != cudaSuccess || cudaEventSynchronize(e1) != cudaSuccess || cudaGetLastError() != cudaSuccess || cudaEventElapsedTime(&ms, e0, e1) != cudaSuccess) {
      set_error("pl2gpu_bulk_read_rate: probe run failed: %s", cudaGetErrorString(cudaGetLastError()));
      return fail();
    }
    total_s += ms * 1e-3;
    total_bytes += bytes_per_launch * per_batch;
    if (total_s >= min_seconds) break;
  }
  release();
  *tbps_out = total_bytes / total_s / 1e12;
  if (seconds_out) *seconds_out = total_s;
  return 0;
}

// The int8 wgmma form of every tensor kernel (A fragments in registers, B K-major in shared memory) against a
// scalar product on the host: M = 64, N = 80, K = 64 (two k-steps); then the binary AND-POPC form against a host
// popcount: M = 64, N = 64, K = 512 bits (two k256 steps), which fixes how the 32 K-bits of an A fragment register
// line up with the bits of a B row in shared memory.
int pl2gpu_selftest_umma(Pl2GpuCtx* ctx, int verbose) {
  if (!ctx) {
    set_error("pl2gpu_selftest_umma: null context");
    return 1;
  }
  Ctx* c = &ctx->c;
  PL2_CUDA_OK(cudaSetDevice(c->device));
  const uint32_t M = 64, N = kProbeN, K = kProbeK;
  std::vector<int8_t> a(M * K), b(N * K);
  uint32_t seed = 12345;
  auto rnd = [&]() {
    seed = seed * 1664525u + 1013904223u;
    return static_cast<int8_t>(static_cast<int>((seed >> 24) % 255) - 127);
  };
  for (auto& v : a) v = rnd();
  for (auto& v : b) v = rnd();
  int8_t *d_a = nullptr, *d_b = nullptr;
  int32_t* d_d = nullptr;
  std::vector<int32_t> d(M * N);
  PL2_CUDA_OK(cudaMalloc(&d_a, M * K));
  PL2_CUDA_OK(cudaMalloc(&d_b, N * K));
  PL2_CUDA_OK(cudaMalloc(&d_d, 4ull * M * N));
  PL2_CUDA_OK(cudaMemcpyAsync(d_a, a.data(), M * K, cudaMemcpyHostToDevice, c->stream));
  PL2_CUDA_OK(cudaMemcpyAsync(d_b, b.data(), N * K, cudaMemcpyHostToDevice, c->stream));
  wgmma_probe_kernel<<<1, 128, 0, c->stream>>>(d_a, d_b, d_d);
  c->launches++;
  PL2_CUDA_OK(cudaGetLastError());
  PL2_CUDA_OK(cudaMemcpyAsync(d.data(), d_d, 4ull * M * N, cudaMemcpyDeviceToHost, c->stream));
  PL2_CUDA_OK(cudaStreamSynchronize(c->stream));
  cudaFree(d_a);
  cudaFree(d_b);
  cudaFree(d_d);
  uint32_t bad = 0;
  for (uint32_t m = 0; m < M; ++m)
    for (uint32_t n = 0; n < N; ++n) {
      int32_t ref = 0;
      for (uint32_t k = 0; k < K; ++k) ref += static_cast<int32_t>(a[m * K + k]) * b[n * K + k];
      if (ref != d[m * N + n]) {
        if (verbose && bad < 8) fprintf(stderr, "selftest_umma mismatch m=%u n=%u got=%d want=%d\n", m, n, d[m * N + n], ref);
        ++bad;
      }
    }
  if (bad) {
    set_error("pl2gpu_selftest_umma: %u of %u accumulator entries differ from the scalar reference", bad, M * N);
    return 1;
  }

  constexpr uint32_t kB1Words = kProbeB1K / 32, kB1N = kProbeB1N;
  std::vector<uint32_t> ab(M * kB1Words), bb(kB1N * kB1Words);
  for (auto& v : ab) v = (seed = seed * 1664525u + 1013904223u);
  for (auto& v : bb) v = (seed = seed * 1664525u + 1013904223u) ^ (seed >> 13);
  std::vector<int32_t> db(M * kB1N);
  uint32_t *d_ab = nullptr, *d_bb = nullptr;
  PL2_CUDA_OK(cudaMalloc(&d_ab, 4ull * ab.size()));
  PL2_CUDA_OK(cudaMalloc(&d_bb, 4ull * bb.size()));
  PL2_CUDA_OK(cudaMalloc(&d_d, 4ull * db.size()));
  PL2_CUDA_OK(cudaMemcpyAsync(d_ab, ab.data(), 4ull * ab.size(), cudaMemcpyHostToDevice, c->stream));
  PL2_CUDA_OK(cudaMemcpyAsync(d_bb, bb.data(), 4ull * bb.size(), cudaMemcpyHostToDevice, c->stream));
  wgmma_b1_probe_kernel<<<1, 128, 0, c->stream>>>(d_ab, d_bb, d_d);
  c->launches++;
  PL2_CUDA_OK(cudaGetLastError());
  PL2_CUDA_OK(cudaMemcpyAsync(db.data(), d_d, 4ull * db.size(), cudaMemcpyDeviceToHost, c->stream));
  PL2_CUDA_OK(cudaStreamSynchronize(c->stream));
  cudaFree(d_ab);
  cudaFree(d_bb);
  cudaFree(d_d);
  for (uint32_t m = 0; m < M; ++m)
    for (uint32_t n = 0; n < kB1N; ++n) {
      int32_t ref = 0;
      for (uint32_t w = 0; w < kB1Words; ++w) ref += __builtin_popcount(ab[m * kB1Words + w] & bb[n * kB1Words + w]);
      if (ref != db[m * kB1N + n]) {
        if (verbose && bad < 8) fprintf(stderr, "selftest_umma b1 mismatch m=%u n=%u got=%d want=%d\n", m, n, db[m * kB1N + n], ref);
        ++bad;
      }
    }
  if (bad) {
    set_error("pl2gpu_selftest_umma: %u of %u binary AND-POPC accumulator entries differ from the host popcount", bad, M * kB1N);
    return 1;
  }
  return 0;
}

}  // extern "C"
