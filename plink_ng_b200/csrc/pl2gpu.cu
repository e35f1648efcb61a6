// pl2gpu.cu - C-ABI entry points (include/plink2_b200.h): context, staging, KING job driver.
#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <cstdarg>
#include <cstring>
#include <memory>
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

int BuildTileList(uint32_t row_start, uint32_t row_end, bool include_diag, TileList* tl, uint32_t tile_cols, uint32_t col_end, bool row_pairs) {
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
  const char* oom = "BuildTileList: insufficient device memory for the tile list of %u tiles: %s";
  PL2_TRY(tl->d_tile_rt.alloc(rt_v.size() + 1, oom, tl->tile_ct));
  PL2_TRY(tl->d_tile_tc.alloc(rt_v.size() + 1, oom, tl->tile_ct));
  PL2_TRY(tl->d_rowtile_offset.alloc(off_v.size(), oom, tl->tile_ct));
  if (!rt_v.empty()) {
    PL2_CUDA_OK(cudaMemcpy(tl->d_tile_rt, rt_v.data(), rt_v.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    PL2_CUDA_OK(cudaMemcpy(tl->d_tile_tc, tc_v.data(), tc_v.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
  }
  PL2_CUDA_OK(cudaMemcpy(tl->d_rowtile_offset, off_v.data(), off_v.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
  tl->h_rowtile_offset = off_v;
  // launch order: blocks of kBand x kBand tiles (144, about one wave on the 132 SMs of an H100 SXM) so that the
  // CTAs resident at the same time stream the same few row/column sample ranges and hit in L2.  With row_pairs the
  // row tiles of a block go two at a time (kBand is even, so a pair never straddles two blocks): a column tile both
  // rows have becomes a pair, next to each other in the order; the rest, the second row's last column tiles at the
  // triangle edge and a last unpaired row, go to the end in the same blocked order.
  constexpr uint32_t kBand = 12;
  std::vector<uint32_t> order, lone;
  order.reserve(rt_v.size());
  const uint32_t n_rt = tl->row_tile_ct;
  const uint32_t r_step = row_pairs ? 2 : 1;
  for (uint32_t rb = 0; rb < n_rt; rb += kBand) {
    const uint32_t rb_end = std::min(n_rt, rb + kBand);
    uint32_t max_cols = 0;
    for (uint32_t r = rb; r < rb_end; ++r) max_cols = std::max(max_cols, off_v[r + 1] - off_v[r]);
    for (uint32_t cb = 0; cb < max_cols; cb += kBand) {
      for (uint32_t r = rb; r < rb_end; r += r_step) {
        const uint32_t n0 = off_v[r + 1] - off_v[r];
        const uint32_t n1 = row_pairs && r + 1 < rb_end ? off_v[r + 2] - off_v[r + 1] : 0;
        for (uint32_t c = cb; c < std::min(std::max(n0, n1), cb + kBand); ++c) {
          if (c < n0 && c < n1) {
            order.push_back(off_v[r] + c);
            order.push_back(off_v[r + 1] + c);
          } else {
            (row_pairs ? lone : order).push_back(c < n0 ? off_v[r] + c : off_v[r + 1] + c);
          }
        }
      }
    }
  }
  tl->pair_tile_ct = row_pairs ? static_cast<uint32_t>(order.size()) : 0;
  order.insert(order.end(), lone.begin(), lone.end());
  PL2_TRY(tl->d_tile_order.alloc(rt_v.size() + 1, oom, tl->tile_ct));
  if (!order.empty()) PL2_CUDA_OK(cudaMemcpy(tl->d_tile_order, order.data(), order.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
  return 0;
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
  return gs->d_raw.alloc(static_cast<uint64_t>(gs->variant_cap) * gs->pitch, "insufficient device memory for a %u-variant x %u-sample genotype stage", gs->variant_cap, sample_ct);
}

int LaunchPadGenotypes(Ctx* ctx, uint8_t* dst, uint32_t pitch, uint32_t sample_ct, uint32_t variant_ct, uint32_t variant_ct_padded, cudaStream_t stream) {
  if (!variant_ct_padded) return 0;
  pad_genotypes_kernel<<<variant_ct_padded, 128, 0, stream ? stream : ctx->stream>>>(dst, pitch, sample_ct, variant_ct, variant_ct_padded);
  ctx->launches++;
  PL2_CUDA_OK(cudaGetLastError());
  return 0;
}

int StageUpload(Ctx* ctx, GenoStage* gs, const void* src, uint64_t src_stride, uint32_t variant_ct, int src_is_device, uint32_t* padded_ct_ptr, uint32_t dst_row, uint32_t pad_to) {
  const uint32_t padded = RoundUpU32(variant_ct, pad_to);
  if (dst_row + padded > gs->variant_cap) {
    set_error("StageUpload: %u + %u rows exceed the stage capacity %u", dst_row, padded, gs->variant_cap);
    return 1;
  }
  const uint32_t width = DivUpU32(gs->sample_ct, 4);
  uint8_t* dst = gs->d_raw.get() + static_cast<uint64_t>(dst_row) * gs->pitch;
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

int StageRing::alloc(Ctx* c, uint32_t sample_ct, uint32_t variant_cap, uint32_t sample_pad) {
  ctx = c;
  const char* fail = "StageRing: cudaEventCreate failed: %s";
  for (int s = 0; s < 2; ++s) {
    PL2_TRY(StageAlloc(sample_ct, variant_cap, &stage[s], sample_pad));
    PL2_TRY(ev_prep_done[s].create(cudaEventDisableTiming, fail));
    PL2_TRY(ev_free[s].create(cudaEventDefault, fail));
  }
  PL2_TRY(ev_src_ready.create(cudaEventDisableTiming, fail));
  return ev_copied.create(cudaEventDisableTiming, fail);
}

int StageRing::acquire(int src_is_device, uint32_t* slot) {
  const uint32_t s = next;
  next ^= 1;
  if (free_pending[s]) PL2_CUDA_OK(cudaStreamWaitEvent(ctx->copy_stream, ev_free[s], 0));
  if (src_is_device == 1) {
    PL2_CUDA_OK(cudaEventRecord(ev_src_ready, ctx->stream));
    PL2_CUDA_OK(cudaStreamWaitEvent(ctx->copy_stream, ev_src_ready, 0));
  }
  *slot = s;
  return 0;
}

int StageRing::land(uint32_t slot, uint8_t* dst, const void* src, uint64_t src_stride, uint32_t rows, int src_is_device) {
  const GenoStage& st = stage[slot];
  PL2_CUDA_OK(cudaMemcpy2DAsync(dst ? dst : st.d_raw.get(), st.pitch, src, src_stride, DivUpU32(st.sample_ct, 4), rows, src_is_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, ctx->copy_stream));
  PL2_CUDA_OK(cudaEventRecord(ev_copied, ctx->copy_stream));
  return 0;
}

int StageRing::land_slice(uint32_t slot, const void* src, uint64_t src_stride, uint32_t slice_rows, int src_is_device) {
  const GenoStage& st = stage[slot];
  uint8_t* mine = st.d_raw.get() + static_cast<uint64_t>(ctx->comm_rank) * slice_rows * st.pitch;
  PL2_TRY(land(slot, mine, src, src_stride, slice_rows, src_is_device));
  PL2_TRY(LaunchPadGenotypes(ctx, mine, st.pitch, st.sample_ct, slice_rows, slice_rows, ctx->copy_stream));
  return CommAllGatherInPlace(ctx, st.d_raw, static_cast<uint64_t>(slice_rows) * st.pitch, ctx->copy_stream);
}

int StageRing::pad(uint32_t slot, uint32_t cur, bool pad_valid_rows, uint32_t pad_to, uint32_t* padded) {
  const GenoStage& st = stage[slot];
  *padded = RoundUpU32(cur, pad_to);
  if (pad_valid_rows) return LaunchPadGenotypes(ctx, st.d_raw, st.pitch, st.sample_ct, cur, *padded, ctx->copy_stream);
  if (*padded > cur) return LaunchPadGenotypes(ctx, st.d_raw.get() + static_cast<uint64_t>(cur) * st.pitch, st.pitch, st.sample_ct, 0, *padded - cur, ctx->copy_stream);
  return 0;
}

int StageRing::fence(uint32_t slot) {
  PL2_CUDA_OK(cudaEventRecord(ev_prep_done[slot], ctx->copy_stream));
  PL2_CUDA_OK(cudaStreamWaitEvent(ctx->stream, ev_prep_done[slot], 0));
  return 0;
}

int StageRing::mark_busy(uint32_t slot, cudaStream_t stream) {
  PL2_CUDA_OK(cudaEventRecord(ev_free[slot], stream));
  free_pending[slot] = true;
  return 0;
}

int StageRing::release_host_source(int src_is_device) {
  if (!src_is_device) PL2_CUDA_OK(cudaEventSynchronize(ev_copied));  // the kernels keep running
  return 0;
}

}  // namespace pl2

using namespace pl2;

struct Pl2KingJob {
  explicit Pl2KingJob(Pl2GpuCtx* x) : ctx(x) {}
  ~Pl2KingJob() {  // the kernels and copies that use the buffers finish before they are freed
    cudaSetDevice(ctx->c.device);
    cudaStreamSynchronize(ctx->c.stream);
    cudaStreamSynchronize(ctx->c.copy_stream);
  }
  Pl2GpuCtx* ctx;
  uint32_t sample_ct = 0, row_start = 0, row_end = 0;
  uint32_t col_end = 0;              // pairs with a column at or past this are never returned (sample_ct: none cut)
  DevArray<uint32_t> d_order;        // mapped job: device position -> sample index; null = identity
  DevArray<uint8_t> d_unmapped;      // mapped job: the block as the caller gave it, before the gather into position order
  int algo = kPl2KingAlgoTensor;
  TileList tiles;
  StageRing ring;   // TS path: the row re-tiling of each slot also runs on the prep stream
  GenoStage stage;  // the other algorithms: one block on the compute stream
  DevArray<uint8_t> d_raw_t[2];       // tensor paths: sample-major copy of the staged block (geno_tile.cuh; split form on the TS path)
  DevArray<uint8_t> d_col_planes[2];  // TS path: the column plane images of the staged block (geno_tile.cuh)
  Event ev_kernel_start[2];           // with the ring's ev_free, the timed pair around the tensor kernel (pl2gpu_king_last_kernel_ms)
  int last_buf = -1;
  DevArray<uint32_t> d_planes;  // popcount path only
  uint32_t tile_cols = kTileCols;
  DevArray<int32_t> d_raw_acc;
  DevArray<uint8_t> d_out_stage;  // bounded staging for host downloads
  uint64_t out_stage_bytes = 0;
  uint64_t variants_added = 0;
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
  std::unique_ptr<Pl2GpuCtx> ctx(new Pl2GpuCtx());
  ctx->c.device = device_idx;
  ctx->c.sm_count = prop.multiProcessorCount;
  // the prep stream outranks the compute stream (default priority 0): its short copy / pad / re-tile / all-gather
  // kernels must get SM slots while a long tensor kernel keeps every SM busy
  int prio_lo = 0, prio_hi = 0;
  PL2_TRY(ctx->c.stream.create(0, "pl2gpu_ctx_create: cudaStreamCreate failed: %s"));
  PL2_CUDA_OK(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
  PL2_TRY(ctx->c.copy_stream.create(prio_hi, "pl2gpu_ctx_create: cudaStreamCreate failed: %s"));
  PL2_CUDA_OK(cudaFuncSetAttribute(king_wg_kernel<kTileCols>, cudaFuncAttributeMaxDynamicSharedMemorySize, KingWgShape<kTileCols>::kSmemBytes));
  PL2_CUDA_OK(cudaFuncSetAttribute(king_b1_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, kKb1SmemBytes));
  PL2_CUDA_OK(cudaFuncSetAttribute(king_b1_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, kKb1SmemBytes));
  *ctx_ptr = ctx.release();
  return 0;
}

int pl2gpu_ctx_destroy(Pl2GpuCtx* ctx) {
  if (!ctx) return 0;
  cudaSetDevice(ctx->c.device);
  pl2gpu_comm_destroy(ctx);
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
  if (!ctx->c.events[slot]) PL2_TRY(ctx->c.events[slot].create(cudaEventDefault, "pl2gpu_ctx_event_record: cudaEventCreate failed: %s"));
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
  // 128 x 64 tiles (the default): two raw blocks + two sample-major copies (each the size of a raw block) + two copies
  // of the column planes (twice that size)
  const uint64_t tiles_ts = CountTiles(row_start, row_end, false, kKingTsCols);
  const uint64_t npad_ts = RoundUpU32(sample_ct, kTsSamplePad);
  const uint64_t need_ts = tiles_ts * kKingTsTileAccWords * 4 + 8 * cap * (npad_ts / 4) + tiles_ts * 16;
  return (need_ss > need_ts ? need_ss : need_ts) + kKingOutStageBytes + slack;
}

int pl2gpu_king_begin(Pl2GpuCtx* ctx, uint32_t sample_ct, uint32_t row_start, uint32_t row_end, int algo, Pl2KingJob** job_ptr) {
  return pl2gpu_king_begin_ex(ctx, sample_ct, row_start, row_end, algo, 0, job_ptr);
}

uint64_t pl2gpu_king_mapped_mem_required(uint32_t sample_ct, uint32_t row_start, uint32_t row_end, uint32_t col_end, uint32_t max_variants_per_add) {
  // what pl2gpu_king_begin_mapped allocates: the TS accumulators of the cut tile list, two raw blocks + two sample-major
  // copies + two copies of the column planes (twice their size), the unmapped block, the position map, the output
  // staging buffer, plus slack for allocator granularity
  const uint64_t cap = ClampStageCap(max_variants_per_add);
  const uint64_t tiles_ts = CountTiles(row_start, row_end, false, kKingTsCols, col_end);
  const uint64_t npad_ts = RoundUpU32(sample_ct, kTsSamplePad);
  return tiles_ts * kKingTsTileAccWords * 4 + 9 * cap * (npad_ts / 4) + tiles_ts * 16 + 4ull * sample_ct + kKingOutStageBytes + (128ull << 20);
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
  std::unique_ptr<Pl2KingJob, int (*)(Pl2KingJob*)> job(new Pl2KingJob(ctx), pl2gpu_king_end);
  job->sample_ct = sample_ct;
  job->row_start = row_start;
  job->row_end = row_end;
  job->col_end = col_end;
  job->algo = algo;
  const bool ts = algo == kPl2KingAlgoTensorTS;
  const uint32_t cap = ClampStageCap(max_variants_per_add);
  for (Event& ev : job->ev_kernel_start) PL2_TRY(ev.create(cudaEventDefault, "pl2gpu_king_begin: cudaEventCreate failed"));
  job->tile_cols = ts ? kKingTsCols : kTileCols;
  PL2_TRY(BuildTileList(row_start, row_end, false, &job->tiles, job->tile_cols, col_end, ts));
  if (order) {
    const char* fail = "pl2gpu_king_begin_mapped: position map upload failed: %s";
    PL2_TRY(job->d_order.alloc(sample_ct, fail));
    if (cudaMemcpy(job->d_order, order, 4ull * sample_ct, cudaMemcpyHostToDevice) != cudaSuccess) {
      set_error(fail, cudaGetErrorString(cudaGetLastError()));
      return 1;
    }
  }
  PL2_TRY(ts ? job->ring.alloc(&ctx->c, sample_ct, cap, kTsSamplePad) : StageAlloc(sample_ct, cap, &job->stage, kSamplePad));
  const GenoStage& st0 = ts ? job->ring.stage[0] : job->stage;
  if (order) PL2_TRY(job->d_unmapped.alloc(static_cast<uint64_t>(st0.variant_cap) * st0.pitch, "pl2gpu_king_begin_mapped: insufficient device memory for the unmapped genotype block"));
  for (int b = 0; b < (ts ? 2 : 1) && algo != kPl2KingAlgoPopcount; ++b) {
    PL2_TRY(job->d_raw_t[b].alloc(static_cast<uint64_t>(st0.sample_ct_padded) * (st0.variant_cap / 4), "pl2gpu_king_begin: insufficient device memory for the sample-major genotype copy"));
    const uint64_t plane_bytes = static_cast<uint64_t>(st0.sample_ct_padded) * (st0.variant_cap / 2);
    if (ts) PL2_TRY(job->d_col_planes[b].alloc(plane_bytes, "pl2gpu_king_begin: insufficient device memory for the column plane copy (%.1f GB per staged block); lower the variants per batch", plane_bytes / 1e9));
  }
  const uint64_t acc_words = static_cast<uint64_t>(job->tiles.tile_ct) * (5ull * job->tile_cols * kTileRows);
  PL2_TRY(job->d_raw_acc.alloc(acc_words ? acc_words : 1, "pl2gpu_king_begin: insufficient device memory for %u pair tiles (%.1f GB of accumulators); narrow the row range", job->tiles.tile_ct, acc_words * 4 / 1e9));
  if (cudaMemsetAsync(job->d_raw_acc, 0, acc_words * 4, ctx->c.stream) != cudaSuccess) {
    set_error("pl2gpu_king_begin: cudaMemsetAsync failed: %s", cudaGetErrorString(cudaGetLastError()));
    return 1;
  }
  if (algo == kPl2KingAlgoPopcount) PL2_TRY(job->d_planes.alloc(3ull * (job->stage.variant_cap / 32) * job->stage.sample_ct_padded, "pl2gpu_king_begin: insufficient device memory for bit planes"));
  job->out_stage_bytes = kKingOutStageBytes;
  PL2_TRY(job->d_out_stage.alloc(job->out_stage_bytes, "pl2gpu_king_begin: insufficient device memory for output staging"));
  *job_ptr = job.release();
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

// TS path: ring slot b holds `cur` variants (rows [0, cur)); pad it, write its sample-major copy and queue the
// tensor kernel.  Everything up to the kernel runs on the prep stream.
static int KingTsPrepAndLaunch(Pl2KingJob* job, uint32_t b, uint32_t cur, bool pad_valid_rows) {
  Ctx* c = &job->ctx->c;
  const GenoStage& st = job->ring.stage[b];
  uint32_t padded;
  PL2_TRY(job->ring.pad(b, cur, pad_valid_rows, kVariantPad, &padded));
  if (!job->tiles.tile_ct) return job->ring.mark_busy(b, c->copy_stream);  // nothing to count on this rank
  geno_tile_rows_kernel<true><<<dim3(padded / 256, st.sample_ct_padded / 64), 256, 0, c->copy_stream>>>(st.d_raw, st.pitch, padded / 32, 0, job->d_raw_t[b], job->d_col_planes[b]);
  c->launches++;
  PL2_CUDA_OK(cudaGetLastError());
  PL2_TRY(job->ring.fence(b));
  PL2_CUDA_OK(cudaEventRecord(job->ev_kernel_start[b], c->stream));
  // tile pairs as 2-CTA clusters that share their plane copies, then the tiles without a partner
  const uint8_t* raw_t = job->d_raw_t[b];
  const uint8_t* planes = job->d_col_planes[b];
  const uint32_t pair_tiles = job->tiles.pair_tile_ct, lone_tiles = job->tiles.tile_ct - pair_tiles;
  if (pair_tiles) {
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute cluster = {};
    cluster.id = cudaLaunchAttributeClusterDimension;
    cluster.val.clusterDim.x = 2;
    cluster.val.clusterDim.y = cluster.val.clusterDim.z = 1;
    cfg.gridDim = dim3(pair_tiles);
    cfg.blockDim = dim3(kKwThreads);
    cfg.dynamicSmemBytes = kKb1SmemBytes;
    cfg.stream = c->stream;
    cfg.attrs = &cluster;
    cfg.numAttrs = 1;
    const uint32_t* order = job->tiles.d_tile_order;
    PL2_CUDA_OK(cudaLaunchKernelEx(&cfg, king_b1_kernel<2>, raw_t, planes, padded, order, static_cast<const uint32_t*>(job->tiles.d_tile_rt), static_cast<const uint32_t*>(job->tiles.d_tile_tc), job->d_raw_acc));
    c->launches++;
  }
  if (lone_tiles) {
    king_b1_kernel<1><<<lone_tiles, kKwThreads, kKb1SmemBytes, c->stream>>>(raw_t, planes, padded, job->tiles.d_tile_order + pair_tiles, job->tiles.d_tile_rt, job->tiles.d_tile_tc, job->d_raw_acc);
    c->launches++;
  }
  PL2_CUDA_OK(cudaGetLastError());
  PL2_TRY(job->ring.mark_busy(b, c->stream));
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
  const uint32_t cap = (ts ? job->ring.stage[0] : job->stage).variant_cap;
  for (uint32_t done = 0; done < variant_ct;) {
    const uint32_t cur = std::min(cap, variant_ct - done);
    const uint8_t* src_cur = src + static_cast<uint64_t>(done) * variant_stride_bytes;
    if (ts) {
      uint32_t b;
      PL2_TRY(job->ring.acquire(src_is_device, &b));
      const GenoStage& st = job->ring.stage[b];
      // a mapped job lands the caller's rows in d_unmapped and gathers them into position order (the prep stream runs
      // copy and gather in turn, so one unmapped block serves both slots); without tiles nothing reads the slot
      PL2_TRY(job->ring.land(b, job->d_unmapped, src_cur, variant_stride_bytes, cur, src_is_device));
      for (uint32_t v0 = 0; job->d_order && job->tiles.tile_ct && v0 < cur; v0 += 32768) {  // grid.y is at most 65,535 rows
        const uint32_t rows = std::min(cur - v0, 32768u);
        geno_gather_kernel<<<dim3(DivUpU32(st.pitch, 256), rows), 256, 0, c->copy_stream>>>(job->d_unmapped + static_cast<uint64_t>(v0) * st.pitch, st.pitch, st.d_raw + static_cast<uint64_t>(v0) * st.pitch, st.pitch, job->d_order, st.sample_ct);
        c->launches++;
        PL2_CUDA_OK(cudaGetLastError());
      }
      PL2_TRY(KingTsPrepAndLaunch(job, b, cur, true));
      PL2_TRY(job->ring.release_host_source(src_is_device));
    } else {
      uint32_t padded = 0;
      PL2_TRY(StageUpload(c, &job->stage, src_cur, variant_stride_bytes, cur, src_is_device, &padded));
      if (job->tiles.tile_ct) {
        if (job->algo == kPl2KingAlgoPopcount) {
          const uint32_t word_ct = padded / 32;
          const uint64_t warps = static_cast<uint64_t>(job->stage.sample_ct_padded / 32) * word_ct;
          split_transpose_kernel<<<static_cast<uint32_t>(DivUpU64(warps, 8)), 256, 0, c->stream>>>(job->stage.d_raw, job->stage.pitch, job->stage.sample_ct_padded, word_ct, job->d_planes);
          c->launches++;
          king_popc_kernel<<<job->tiles.tile_ct * 2, 256, 0, c->stream>>>(job->d_planes, job->stage.sample_ct_padded, word_ct, job->tiles.d_tile_rt, job->tiles.d_tile_tc, job->d_raw_acc);
          c->launches++;
        } else {
          const GenoStage& st = job->stage;
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
  if (!slice_variant_ct || total64 > job->ring.stage[0].variant_cap) {
    set_error("pl2gpu_king_add_variants_sharded: %u variants x %d ranks exceed the stage capacity %u", slice_variant_ct, c->comm_world, job->ring.stage[0].variant_cap);
    return 1;
  }
  if (variant_stride_bytes < DivUpU32(job->sample_ct, 4)) {
    set_error("pl2gpu_king_add_variants_sharded: variant stride too small");
    return 1;
  }
  const uint32_t total = static_cast<uint32_t>(total64);
  uint32_t b;
  PL2_TRY(job->ring.acquire(src_is_device, &b));
  PL2_TRY(job->ring.land_slice(b, slice, variant_stride_bytes, slice_variant_ct, src_is_device));
  PL2_TRY(KingTsPrepAndLaunch(job, b, total, false));
  PL2_TRY(job->ring.release_host_source(src_is_device));
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
  DevArray<unsigned long long> d_found;
  DevArray<uint32_t> d_pairs, d_counts;
  DevArray<double> d_kin;
  const uint64_t cap = max_out ? max_out : 1;
  const char* oom = "pl2gpu_king_get_filtered: insufficient device memory for %llu result slots";
  const unsigned long long max_out_ull = max_out;
  if (d_found.alloc(1, oom, max_out_ull) || d_pairs.alloc(cap * 2, oom, max_out_ull) || d_counts.alloc(cap * 5, oom, max_out_ull) || d_kin.alloc(cap, oom, max_out_ull)) return 1;
  if (cudaMemsetAsync(d_found, 0, 8, c->stream) != cudaSuccess) return 1;
  if (job->tile_cols == kKingTsCols) {
    king_filter_kernel<kKingTsCols><<<job->tiles.tile_ct, kTileRows, 0, c->stream>>>(job->d_raw_acc, job->tiles.d_tile_rt, job->tiles.d_tile_tc, job->sample_ct, job->col_end, r0, r1, min_kinship, max_out, d_found, d_pairs, d_counts, d_kin);
  } else {
    king_filter_kernel<kTileCols><<<job->tiles.tile_ct, kTileRows, 0, c->stream>>>(job->d_raw_acc, job->tiles.d_tile_rt, job->tiles.d_tile_tc, job->sample_ct, job->col_end, r0, r1, min_kinship, max_out, d_found, d_pairs, d_counts, d_kin);
  }
  c->launches++;
  unsigned long long found = 0;
  if (cudaGetLastError() != cudaSuccess || cudaMemcpyAsync(&found, d_found, 8, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess || cudaStreamSynchronize(c->stream) != cudaSuccess) {
    set_error("pl2gpu_king_get_filtered: %s", cudaGetErrorString(cudaGetLastError()));
    return 1;
  }
  *n_found = found;
  const uint64_t k = found < max_out ? found : max_out;
  if (k) {
    std::vector<uint32_t> hp(2 * k), hc(5 * k);
    std::vector<double> hk(k);
    if (cudaMemcpy(hp.data(), d_pairs, k * 8, cudaMemcpyDeviceToHost) != cudaSuccess || cudaMemcpy(hc.data(), d_counts, k * 20, cudaMemcpyDeviceToHost) != cudaSuccess || cudaMemcpy(hk.data(), d_kin, k * 8, cudaMemcpyDeviceToHost) != cudaSuccess) {
      set_error("pl2gpu_king_get_filtered: %s", cudaGetErrorString(cudaGetLastError()));
      return 1;
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
  return 0;
}

uint64_t pl2gpu_king_variants_added(Pl2KingJob* job) { return job ? job->variants_added : 0; }

int pl2gpu_king_last_kernel_ms(Pl2KingJob* job, float* ms) {
  if (!job || !ms || job->last_buf < 0) {
    set_error("pl2gpu_king_last_kernel_ms: no tensor-kernel launch has been recorded (TS algorithm only)");
    return 1;
  }
  PL2_CUDA_OK(cudaSetDevice(job->ctx->c.device));
  PL2_CUDA_OK(cudaEventSynchronize(job->ring.ev_free[job->last_buf]));
  PL2_CUDA_OK(cudaEventElapsedTime(ms, job->ev_kernel_start[job->last_buf], job->ring.ev_free[job->last_buf]));
  return 0;
}

int pl2gpu_king_last_planes(Pl2KingJob* job, void* dst, uint64_t bytes) {
  if (!job || !dst || job->last_buf < 0 || bytes > static_cast<uint64_t>(job->ring.stage[0].sample_ct_padded) * (job->ring.stage[0].variant_cap / 2)) {
    set_error("pl2gpu_king_last_planes: no default-algorithm launch recorded, or more bytes than the plane copy holds");
    return 1;
  }
  PL2_CUDA_OK(cudaSetDevice(job->ctx->c.device));
  PL2_CUDA_OK(cudaEventSynchronize(job->ring.ev_free[job->last_buf]));
  PL2_CUDA_OK(cudaMemcpy(dst, job->d_col_planes[job->last_buf], bytes, cudaMemcpyDeviceToHost));
  return 0;
}

int pl2gpu_king_end(Pl2KingJob* job) {
  if (!job) return 0;
  delete job;
  cudaGetLastError();
  return 0;
}

// ------------------------------------------------------------------------------------------ pair list

struct Pl2KingPairJob {
  explicit Pl2KingPairJob(Pl2GpuCtx* x) : ctx(x) {}
  ~Pl2KingPairJob() {
    cudaSetDevice(ctx->c.device);
    cudaStreamSynchronize(ctx->c.stream);
  }
  Pl2GpuCtx* ctx;
  uint32_t sample_ct = 0;
  uint64_t pair_ct = 0;
  GenoStage stage;
  DevArray<uint8_t> d_raw_t;    // sample-major 2-bit copy of the staged block
  DevArray<uint32_t> d_pairs;   // [pair][2]
  DevArray<uint32_t> d_counts;  // [pair][5]
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
  std::unique_ptr<Pl2KingPairJob, int (*)(Pl2KingPairJob*)> job(new Pl2KingPairJob(ctx), pl2gpu_king_pairs_end);
  job->sample_ct = sample_ct;
  job->pair_ct = pair_ct;
  PL2_TRY(StageAlloc(sample_ct, kMaxStageVariants, &job->stage, 64));
  const uint64_t n_alloc = pair_ct ? pair_ct : 1;
  const char* oom = "pl2gpu_king_pairs_begin: insufficient device memory for %llu pairs";
  const unsigned long long pair_ct_ull = pair_ct;
  if (job->d_raw_t.alloc(static_cast<uint64_t>(job->stage.sample_ct_padded) * (job->stage.variant_cap / 4), oom, pair_ct_ull) || job->d_pairs.alloc(n_alloc * 2, oom, pair_ct_ull) ||
      job->d_counts.alloc(n_alloc * 5, oom, pair_ct_ull))
    return 1;
  if (cudaMemcpyAsync(job->d_pairs, pairs_host, pair_ct * 8, cudaMemcpyHostToDevice, ctx->c.stream) != cudaSuccess || cudaMemsetAsync(job->d_counts, 0, n_alloc * 20, ctx->c.stream) != cudaSuccess ||
      cudaStreamSynchronize(ctx->c.stream) != cudaSuccess) {
    set_error("pl2gpu_king_pairs_begin: %s", cudaGetErrorString(cudaGetLastError()));
    return 1;
  }
  *job_ptr = job.release();
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
  delete job;
  cudaGetLastError();
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
  DevArray<int32_t> d_sink;
  Event e0, e1;
  PL2_TRY(d_sink.alloc(256, "pl2gpu_int8_peak: cudaMalloc failed: %s"));
  PL2_TRY(e0.create(cudaEventDefault, "pl2gpu_int8_peak: cudaEventCreate failed: %s"));
  PL2_TRY(e1.create(cudaEventDefault, "pl2gpu_int8_peak: cudaEventCreate failed: %s"));
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
  DevArray<uint8_t> d_src;
  Event e0, e1;
  const char* setup_failed = "pl2gpu_bulk_read_rate: set-up failed: %s";
  PL2_TRY(d_src.alloc(static_cast<uint64_t>(ws_chunks) * kFeedChunk, "pl2gpu_bulk_read_rate: cudaMalloc failed: %s"));
  if (cudaMemsetAsync(d_src, 0x5A, static_cast<uint64_t>(ws_chunks) * kFeedChunk, c->stream) != cudaSuccess) {
    set_error(setup_failed, cudaGetErrorString(cudaGetLastError()));
    return 1;
  }
  PL2_TRY(e0.create(cudaEventDefault, setup_failed));
  PL2_TRY(e1.create(cudaEventDefault, setup_failed));
  if (cudaFuncSetAttribute(bulk_read_probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) {
    set_error(setup_failed, cudaGetErrorString(cudaGetLastError()));
    return 1;
  }
  auto launch = [&]() {
    bulk_read_probe_kernel<<<c->sm_count, 32, smem, c->stream>>>(d_src, ws_chunks, chunks, rounds);
    c->launches++;
  };
  launch();  // warm-up: also brings an L2-sized working set into L2
  double total_s = 0, total_bytes = 0;
  const uint32_t per_batch = 4;
  while (true) {
    if (cudaEventRecord(e0, c->stream) != cudaSuccess) return 1;
    for (uint32_t k = 0; k < per_batch; ++k) launch();
    float ms = 0;
    if (cudaEventRecord(e1, c->stream) != cudaSuccess || cudaEventSynchronize(e1) != cudaSuccess || cudaGetLastError() != cudaSuccess || cudaEventElapsedTime(&ms, e0, e1) != cudaSuccess) {
      set_error("pl2gpu_bulk_read_rate: probe run failed: %s", cudaGetErrorString(cudaGetLastError()));
      return 1;
    }
    total_s += ms * 1e-3;
    total_bytes += bytes_per_launch * per_batch;
    if (total_s >= min_seconds) break;
  }
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
  const char* oom = "pl2gpu_selftest_umma: cudaMalloc failed: %s";
  std::vector<int32_t> d(M * N);
  {
    DevArray<int8_t> d_a, d_b;
    DevArray<int32_t> d_d;
    PL2_TRY(d_a.alloc(M * K, oom));
    PL2_TRY(d_b.alloc(N * K, oom));
    PL2_TRY(d_d.alloc(M * N, oom));
    PL2_CUDA_OK(cudaMemcpyAsync(d_a, a.data(), M * K, cudaMemcpyHostToDevice, c->stream));
    PL2_CUDA_OK(cudaMemcpyAsync(d_b, b.data(), N * K, cudaMemcpyHostToDevice, c->stream));
    wgmma_probe_kernel<<<1, 128, 0, c->stream>>>(d_a, d_b, d_d);
    c->launches++;
    PL2_CUDA_OK(cudaGetLastError());
    PL2_CUDA_OK(cudaMemcpyAsync(d.data(), d_d, 4ull * M * N, cudaMemcpyDeviceToHost, c->stream));
    PL2_CUDA_OK(cudaStreamSynchronize(c->stream));
  }
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
  {
    DevArray<uint32_t> d_ab, d_bb;
    DevArray<int32_t> d_d;
    PL2_TRY(d_ab.alloc(ab.size(), oom));
    PL2_TRY(d_bb.alloc(bb.size(), oom));
    PL2_TRY(d_d.alloc(db.size(), oom));
    PL2_CUDA_OK(cudaMemcpyAsync(d_ab, ab.data(), 4ull * ab.size(), cudaMemcpyHostToDevice, c->stream));
    PL2_CUDA_OK(cudaMemcpyAsync(d_bb, bb.data(), 4ull * bb.size(), cudaMemcpyHostToDevice, c->stream));
    wgmma_b1_probe_kernel<<<1, 128, 0, c->stream>>>(d_ab, d_bb, d_d);
    c->launches++;
    PL2_CUDA_OK(cudaGetLastError());
    PL2_CUDA_OK(cudaMemcpyAsync(db.data(), d_d, 4ull * db.size(), cudaMemcpyDeviceToHost, c->stream));
    PL2_CUDA_OK(cudaStreamSynchronize(c->stream));
  }
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
