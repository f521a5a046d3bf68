// Frame recorder (tfl_recorder_*): a scalar grid leaves the device in `.vbox` order behind the running step.
// capture packs the field into one device staging frame on the context's stream (k_pack_vbox) and a copy stream
// moves the staging frame into the next free slot of a ring of pinned host frames; take / release hand the frames
// to the host strictly first in, first out.  Nothing here synchronises except take(wait = 1), which waits for that
// one frame's copy, and destroy.
//
// A z-slab recorder (tfl_recorder_create_slab) gathers one frame from every rank of a z-slab run.  Rank 0 is the
// writer: its recorder is the one above with the global depth, and its staging frame carries a counter area behind
// it (arrived[rank], freed), exported as one CUDA IPC allocation.  Every other rank maps it and packs its owned planes
// straight into it (remote stores over NVLink), after a bounded device-side wait for `freed` to show that the copy
// of the previous frame out of the staging frame is done; the pack's last CTA publishes the frame's sequence number
// in arrived[rank].  Rank 0's copy stream waits (bounded) for every rank's arrival before its copy to the host and
// publishes `freed` after it, so rank 0's own stream never waits for the other ranks' packs.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "tfl_api_internal.h"
#include "../../include/tfl.h"

constexpr int kPackTile = 32;     // a 32 x 32 (z, x) tile per block
constexpr int kPackRows = 8;      // 32 x 8 threads, 4 rows each
constexpr int kMaxRanks = 64;
// Behind the staging frame of a z-slab recorder: arrived[kMaxRanks], then freed (unsigned words, sequence numbers).
constexpr int kCounterWords = kMaxRanks + 64;
constexpr long long kWaitCycles = 4000000000LL;     // ~2 s at the H100's clock, as the slab exchanges' waits
constexpr int32_t kHandleMagic = 0x52464c54;        // "TLFR"

// Global planes [z0, z1) of in ([nz_local][ny][nx], x fastest; local plane 0 is global plane z_offset) -> out, a
// frame of depth gnz: the value at global (x, y, z) goes to out[(x * ny + y) * gnz + z] (z fastest), `permute(3, 2, 1)`
// of the grid, the order the demo writes to a `.vbox` file.  Block (bx, bz, y) moves the (z, x) tile
// [z0 + bz * 32, +32) x [bx * 32, +32) of plane y through shared memory: the load walks x in 128-byte rows, the store
// walks z in runs of up to 32 words (128-byte rows for a whole grid, z0 = 0).  The row of 33 words keeps the
// transposed read free of bank conflicts.  A bit copy (32-bit words, no arithmetic): -0.0, denormals and NaN payloads
// arrive unchanged.  The whole grid is [0, nz), z_offset = 0, gnz = nz, with no gate and no arrival counter.
// A z-slab rank other than the writer passes `gate` (the pack runs only if the wait before it stored `seq` there) and
// `arrived`: after the last CTA's stores, fenced at system scope, `seq` is stored there with release semantics
// (the k_slab_push pattern; `done` counts the finished CTAs and is reset by the last one).
// Not in an anonymous namespace: the kernel keeps a stable name in traces and profiles.
__global__ void __launch_bounds__(kPackTile * kPackRows)
k_pack_vbox(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, int z0, int z1, int z_offset, int gnz, int ny,
            int nx, const unsigned int* gate, unsigned int seq, unsigned int* done, unsigned int* arrived) {
  if (gate && *gate != seq) return;                 // the wait before timed out: write nothing, publish nothing
  __shared__ uint32_t tile[kPackTile][kPackTile + 1];
  const int x0 = blockIdx.x * kPackTile, zt = z0 + blockIdx.y * kPackTile, y = blockIdx.z;
  const int tx = threadIdx.x, ty = threadIdx.y;
  const long long plane = (long long)ny * nx;
  const int x = x0 + tx;
#pragma unroll
  for (int r = ty; r < kPackTile; r += kPackRows) {
    const int z = zt + r;
    if (z < z1 && x < nx) tile[r][tx] = __ldg(in + (z - z_offset) * plane + (long long)y * nx + x);
  }
  __syncthreads();
  const int z = zt + tx;
#pragma unroll
  for (int r = ty; r < kPackTile; r += kPackRows) {
    const int xo = x0 + r;
    if (xo < nx && z < z1) out[((long long)xo * ny + y) * gnz + z] = tile[tx][r];
  }
  if (!arrived) return;
  __threadfence_system();
  __syncthreads();
  if (tx == 0 && ty == 0) {
    const unsigned int blocks = gridDim.x * gridDim.y * gridDim.z;
    if (atomicAdd(done, 1u) == blocks - 1) {        // every CTA's stores are fenced: publish
      *done = 0u;
      __threadfence_system();
      asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(arrived), "r"(seq) : "memory");
    }
  }
}

namespace {

// Bounded wait of a z-slab rank other than the writer: until the writer's `freed` reaches seq - 1 (the previous
// frame left the staging frame), then *gate = seq.  A wait that times out stores nothing and raises the fault counter.
__global__ void k_rec_wait_freed(const unsigned int* freed, unsigned int seq, unsigned int* gate,
                                 unsigned long long* faults) {
  const long long t0 = clock64();
  for (;;) {
    unsigned int v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(freed) : "memory");
    if ((int)(v - (seq - 1u)) >= 0) break;
    if (clock64() - t0 > kWaitCycles) { if (faults) atomicAdd(faults, 1ULL); return; }
    __nanosleep(200);
  }
  *gate = seq;
}

// The writer's copy stream, before the copy to the host: a bounded wait for every other rank's arrival of `seq`.
// *missing = the ranks whose planes did not land (bit r; 0: all did); a timeout also raises the fault counter.
__global__ void k_rec_wait_arrived(const unsigned int* arrived, int world, unsigned int seq,
                                   unsigned long long* missing, unsigned long long* faults) {
  __shared__ unsigned long long miss;
  const int t = threadIdx.x;
  if (t == 0) miss = 0ULL;
  __syncthreads();
  if (t >= 1 && t < world) {
    const long long t0 = clock64();
    for (;;) {
      unsigned int v;
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(arrived + t) : "memory");
      if ((int)(v - seq) >= 0) break;
      if (clock64() - t0 > kWaitCycles) { atomicOr(&miss, 1ULL << t); break; }
      __nanosleep(200);
    }
  }
  __syncthreads();
  if (t == 0) {
    *missing = miss;
    if (miss && faults) atomicAdd(faults, 1ULL);
  }
}

// ... and after it: freed = seq, so the other ranks may pack the next frame.
__global__ void k_rec_publish_freed(unsigned int* freed, unsigned int seq) {
  __threadfence_system();
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(freed), "r"(seq) : "memory");
}

}  // namespace

// Launches k_pack_vbox on `st` for global planes [z0, z1); returns the number of kernels launched (1).
static int launch_pack_vbox(const float* in, float* out, int z0, int z1, int z_offset, int gnz, int ny, int nx,
                            const unsigned int* gate, unsigned int seq, unsigned int* done, unsigned int* arrived,
                            cudaStream_t st) {
  const dim3 block(kPackTile, kPackRows);
  const dim3 grid((nx + kPackTile - 1) / kPackTile, (z1 - z0 + kPackTile - 1) / kPackTile, ny);
  k_pack_vbox<<<grid, block, 0, st>>>((const uint32_t*)in, (uint32_t*)out, z0, z1, z_offset, gnz, ny, nx, gate, seq,
                                      done, arrived);
  return 1;
}

// Slots in use form one run of the ring starting at `first`: `taken` frames handed to the host (oldest first), then
// `captured` frames whose copies are enqueued or done.  The next capture fills slot (first + taken + captured).
// A z-slab recorder has nz = the global depth; rank 0 holds the ring, the other ranks only `frame_dev` (mapped).
struct tfl_recorder {
  int nz = 0, ny = 0, nx = 0, slots = 0;
  int rank = 0, world = 1, z0 = 0, z1 = 0;   // this rank's planes (the whole grid for one rank)
  size_t bytes = 0;                          // one frame
  DevPtr<float> stage;                       // rank 0: the packed frame (then the counters), read by the copy stream
  IpcPtr<float> mapped;                      // other ranks: rank 0's staging frame and counters
  float* frame_dev = nullptr;                // the staging frame this rank packs into
  unsigned int* counters = nullptr;          // arrived[kMaxRanks], freed (world > 1)
  DevPtr<unsigned int> local;                // world > 1: [0] done (pack CTAs), [1] gate, [2..3] missing ranks (u64)
  bool connected = false;
  std::vector<PinnedPtr<float>> host;        // [slots] host frames
  PinnedPtr<unsigned long long> missing;     // [slots] ranks whose planes did not land in the slot's frame
  std::vector<EventPtr> copied;              // [slots] recorded on `copy` after the slot's copy
  std::vector<int64_t> frame;                // [slots] index of the frame the slot holds
  StreamPtr copy;
  EventPtr packed;                           // recorded on the context's stream after the pack
  int first = 0, taken = 0, captured = 0;
  int last_slot = -1;                        // slot of the latest copy out of `stage` (the next pack waits on it)
  int64_t next_frame = 0;
};

// Counter area offset (floats) behind a frame of `cells` floats: 256-byte aligned.
static size_t counter_offset(size_t cells) { return (cells + 63) / 64 * 64; }

// Everything but the argument checks of create / create_slab.
static int recorder_new(tfl_ctx* ctx, int gnz, int ny, int nx, int rank, int world, int slots, tfl_recorder** out) {
  std::unique_ptr<tfl_recorder> r(new tfl_recorder());
  r->nz = gnz; r->ny = ny; r->nx = nx; r->rank = rank; r->world = world;
  slab_planes(gnz, world, rank, &r->z0, &r->z1);
  r->connected = world == 1;
  const size_t cells = (size_t)gnz * ny * nx;
  r->bytes = cells * sizeof(float);
  if (world > 1 && !(r->local = dev_zeros<unsigned int>(4)))
    return fail(ctx, "recorder_create: cudaMalloc of the recorder's counters failed");
  if (rank > 0) {                             // packs into rank 0's staging frame once connected
    r->slots = 0;
    *out = r.release();
    return 0;
  }
  r->slots = slots;
  r->stage = world > 1 ? dev_zeros<float>(counter_offset(cells) + kCounterWords) : dev_alloc<float>(cells);
  if (!r->stage) return fail(ctx, "recorder_create: cudaMalloc of the staging frame failed");
  r->frame_dev = r->stage.get();
  if (world > 1) r->counters = reinterpret_cast<unsigned int*>(r->stage.get() + counter_offset(cells));
  if (!(r->copy = new_stream(cudaStreamNonBlocking)) || !(r->packed = new_event(cudaEventDisableTiming)))
    return fail(ctx, "recorder_create: creating the copy stream or its events failed");
  if (!(r->missing = pinned_alloc<unsigned long long>(slots)))
    return fail(ctx, "recorder_create: pinned status words failed");
  for (int i = 0; i < slots; ++i) {
    r->missing.get()[i] = 0ULL;
    PinnedPtr<float> h = pinned_alloc<float>(cells);
    EventPtr e = new_event(cudaEventDisableTiming);
    if (!h || !e) return fail(ctx, "recorder_create: pinned host frame %d of %d or its event failed", i, slots);
    r->host.push_back(std::move(h));
    r->copied.push_back(std::move(e));
  }
  r->frame.assign(slots, -1);
  *out = r.release();
  return 0;
}

// Capture of global planes [r->z0, r->z1) from `field`, whose local plane 0 is global plane z_offset (checked).
static int recorder_capture(tfl_ctx* ctx, tfl_recorder* r, const tfl_grid* field, int z_offset, int64_t* frame_out) {
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  TFL_CUDA(ctx, cudaStreamIsCapturing(ctx->stream, &cs));
  if (cs != cudaStreamCaptureStatusNone)
    return fail(ctx, "recorder_capture: the context's stream is being captured into a graph; record outside the capture");
  cudaStream_t st = ctx->stream;
  const unsigned int seq = (unsigned int)(r->next_frame + 1);     // sequence numbers start at 1 (counters start at 0)
  if (r->rank > 0) {
    unsigned int* l = r->local.get();
    k_rec_wait_freed<<<1, 1, 0, st>>>(r->counters + kMaxRanks, seq, l + 1, ctx->counters.get());
    ctx->launches += 1;
    ctx->launches += launch_pack_vbox(field->data, r->frame_dev, r->z0, r->z1, z_offset, r->nz, r->ny, r->nx, l + 1, seq,
                                      l, r->counters + r->rank, st);
    if (check_launch(ctx, "k_pack_vbox")) return 1;
    if (frame_out) *frame_out = r->next_frame;
    r->next_frame++;
    return 0;
  }
  const int slot = (r->first + r->taken + r->captured) % r->slots;
  // The staging frame is free once the previous copy out of it has run: a device-side wait, never a host one.
  if (r->last_slot >= 0) TFL_CUDA(ctx, cudaStreamWaitEvent(st, r->copied[r->last_slot].get(), 0));
  ctx->launches += launch_pack_vbox(field->data, r->frame_dev, r->z0, r->z1, z_offset, r->nz, r->ny, r->nx, nullptr, 0,
                                    nullptr, nullptr, st);
  if (check_launch(ctx, "k_pack_vbox")) return 1;
  TFL_CUDA(ctx, cudaEventRecord(r->packed.get(), st));
  cudaStream_t cp = r->copy.get();
  TFL_CUDA(ctx, cudaStreamWaitEvent(cp, r->packed.get(), 0));
  if (r->world > 1) {
    unsigned long long* miss = reinterpret_cast<unsigned long long*>(r->local.get() + 2);
    k_rec_wait_arrived<<<1, kMaxRanks, 0, cp>>>(r->counters, r->world, seq, miss, ctx->counters.get());
    ctx->launches += 1;
    TFL_CUDA(ctx, cudaMemcpyAsync(r->missing.get() + slot, miss, sizeof(*miss), cudaMemcpyDeviceToHost, cp));
  }
  TFL_CUDA(ctx, cudaMemcpyAsync(r->host[slot].get(), r->stage.get(), r->bytes, cudaMemcpyDeviceToHost, cp));
  if (r->world > 1) {
    k_rec_publish_freed<<<1, 1, 0, cp>>>(r->counters + kMaxRanks, seq);
    ctx->launches += 1;
    if (check_launch(ctx, "recorder_capture (copy stream)")) return 1;
  }
  TFL_CUDA(ctx, cudaEventRecord(r->copied[slot].get(), cp));
  r->last_slot = slot;
  r->frame[slot] = r->next_frame;
  if (frame_out) *frame_out = r->next_frame;
  r->next_frame++;
  r->captured++;
  return 0;
}

extern "C" {

int tfl_recorder_create(tfl_ctx* ctx, int32_t nz, int32_t ny, int32_t nx, int32_t slots, tfl_recorder** out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!ctx) return 1;
  if (!out) return fail(ctx, "recorder_create: out is nil");
  *out = nullptr;
  if (nz < 1 || ny < 1 || nx < 1) return fail(ctx, "recorder_create: every grid extent must be >= 1 (got %d x %d x %d)", nz, ny, nx);
  if (slots < 1) return fail(ctx, "recorder_create: slots must be >= 1 (got %d)", slots);
  if (grid_too_large((long long)nz * ny * nx, 1)) return fail(ctx, "recorder_create: grid too large");
  return recorder_new(ctx, nz, ny, nx, 0, 1, slots, out);
}

int tfl_recorder_create_slab(tfl_ctx* ctx, int32_t gnz, int32_t ny, int32_t nx, int32_t rank, int32_t world,
                             int32_t slots, tfl_recorder** out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!ctx) return 1;
  if (!out) return fail(ctx, "recorder_create_slab: out is nil");
  *out = nullptr;
  if (gnz < 1 || ny < 1 || nx < 1)
    return fail(ctx, "recorder_create_slab: every grid extent must be >= 1 (got %d x %d x %d)", gnz, ny, nx);
  if (world < 1 || world > kMaxRanks || rank < 0 || rank >= world)
    return fail(ctx, "recorder_create_slab: rank %d of world %d (1 <= world <= %d)", rank, world, kMaxRanks);
  if (gnz / world < 1)
    return fail(ctx, "recorder_create_slab: %d planes over %d ranks leave empty slabs", gnz, world);
  if (rank == 0 && slots < 1) return fail(ctx, "recorder_create_slab: slots must be >= 1 on rank 0 (got %d)", slots);
  if (grid_too_large((long long)gnz * ny * nx, 1)) return fail(ctx, "recorder_create_slab: grid too large");
  return recorder_new(ctx, gnz, ny, nx, rank, world, rank == 0 ? slots : 0, out);
}

void tfl_recorder_destroy(tfl_ctx* ctx, tfl_recorder* r) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (r && r->copy) cudaStreamSynchronize(r->copy.get());   // copies in flight write into the host frames
  if (r && r->rank > 0 && ctx) cudaStreamSynchronize(ctx->stream);   // packs in flight write into rank 0's frame
  delete r;
}

// Rank 0's staging frame and counters as TFL_RECORDER_HANDLE_BYTES: the CUDA IPC handle, then gnz, ny, nx, world.
int tfl_recorder_ipc_export(tfl_ctx* ctx, tfl_recorder* r, char* handle_out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!ctx) return 1;
  if (!r || !handle_out) return fail(ctx, "recorder_ipc_export: nil argument");
  if (r->world == 1) return fail(ctx, "recorder_ipc_export: a recorder of one rank has nothing to share");
  if (r->rank != 0) return fail(ctx, "recorder_ipc_export: rank %d does not export; rank 0 (the writer) does", r->rank);
  static_assert(sizeof(cudaIpcMemHandle_t) + 5 * sizeof(int32_t) <= TFL_RECORDER_HANDLE_BYTES, "handle fits the ABI buffer");
  cudaIpcMemHandle_t h;
  TFL_CUDA(ctx, cudaIpcGetMemHandle(&h, r->stage.get()));
  memset(handle_out, 0, TFL_RECORDER_HANDLE_BYTES);
  memcpy(handle_out, &h, sizeof(h));
  const int32_t meta[5] = {kHandleMagic, r->nz, r->ny, r->nx, r->world};
  memcpy(handle_out + sizeof(h), meta, sizeof(meta));
  r->connected = true;
  return 0;
}

int tfl_recorder_ipc_connect(tfl_ctx* ctx, tfl_recorder* r, const char* handle) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!ctx) return 1;
  if (!r || !handle) return fail(ctx, "recorder_ipc_connect: nil argument");
  if (r->rank == 0) return fail(ctx, "recorder_ipc_connect: rank 0 (the writer) exports its frame, it does not connect");
  if (r->connected) return fail(ctx, "recorder_ipc_connect: rank %d is already connected", r->rank);
  cudaIpcMemHandle_t h;
  int32_t meta[5];
  memcpy(&h, handle, sizeof(h));
  memcpy(meta, handle + sizeof(h), sizeof(meta));
  if (meta[0] != kHandleMagic) return fail(ctx, "recorder_ipc_connect: the bytes are not a recorder's handle");
  if (meta[1] != r->nz || meta[2] != r->ny || meta[3] != r->nx || meta[4] != r->world)
    return fail(ctx, "recorder_ipc_connect: the handle is of a %d x %d x %d recorder over %d ranks, this one is "
                     "%d x %d x %d over %d ranks", meta[1], meta[2], meta[3], meta[4], r->nz, r->ny, r->nx, r->world);
  void* q = nullptr;
  const cudaError_t e = cudaIpcOpenMemHandle(&q, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return fail(ctx, "recorder_ipc_connect: cudaIpcOpenMemHandle (rank 0's frame): %s", cudaGetErrorString(e));
  }
  r->mapped.reset((float*)q);
  r->frame_dev = (float*)q;
  r->counters = reinterpret_cast<unsigned int*>(r->frame_dev + counter_offset((size_t)r->nz * r->ny * r->nx));
  r->connected = true;
  return 0;
}

int tfl_recorder_capture(tfl_ctx* ctx, tfl_recorder* r, const tfl_grid* field, int64_t* frame_out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!ctx) return 1;
  if (frame_out) *frame_out = -1;
  if (!r) return fail(ctx, "recorder_capture: recorder is nil");
  if (r->world > 1)
    return fail(ctx, "recorder_capture: a z-slab recorder of %d ranks captures with tfl_recorder_capture_slab", r->world);
  if (r->taken + r->captured == r->slots)
    return fail(ctx, "recorder_capture: the %d x %d x %d recorder's %d slot(s) all hold frames not yet released "
                     "(take and release the oldest first)", r->nz, r->ny, r->nx, r->slots);
  if (!field || !field->data) return fail(ctx, "recorder_capture: field is nil");
  if (field->nb != 1) return fail(ctx, "recorder_capture: field has nb = %d; a recorder takes one batch entry (nb = 1)", field->nb);
  if (field->nc != 1) return fail(ctx, "recorder_capture: field has nc = %d; a recorder takes a scalar field (nc = 1)", field->nc);
  if (field->nz != r->nz || field->ny != r->ny || field->nx != r->nx)
    return fail(ctx, "recorder_capture: field is %d x %d x %d (z, y, x), the recorder's frames are %d x %d x %d",
                field->nz, field->ny, field->nx, r->nz, r->ny, r->nx);
  return recorder_capture(ctx, r, field, 0, frame_out);
}

int tfl_recorder_capture_slab(tfl_ctx* ctx, tfl_recorder* r, const tfl_grid* field, int32_t z_offset, int64_t* frame_out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!ctx) return 1;
  if (frame_out) *frame_out = -1;
  if (!r) return fail(ctx, "recorder_capture_slab: recorder is nil");
  if (!r->connected)
    return fail(ctx, "recorder_capture_slab: rank %d of %d is not connected (export on rank 0, connect on the others, "
                     "then a barrier)", r->rank, r->world);
  if (r->rank == 0 && r->taken + r->captured == r->slots)
    return fail(ctx, "recorder_capture_slab: the %d x %d x %d recorder's %d slot(s) all hold frames not yet released "
                     "(take and release the oldest first)", r->nz, r->ny, r->nx, r->slots);
  if (!field || !field->data) return fail(ctx, "recorder_capture_slab: field is nil");
  if (field->nb != 1) return fail(ctx, "recorder_capture_slab: field has nb = %d; a recorder takes one batch entry (nb = 1)", field->nb);
  if (field->nc != 1) return fail(ctx, "recorder_capture_slab: field has nc = %d; a recorder takes a scalar field (nc = 1)", field->nc);
  if (field->ny != r->ny || field->nx != r->nx)
    return fail(ctx, "recorder_capture_slab: field planes are %d x %d (y, x), the recorder's are %d x %d",
                field->ny, field->nx, r->ny, r->nx);
  if (z_offset < 0 || z_offset > r->z0 || r->z1 - z_offset > field->nz)
    return fail(ctx, "recorder_capture_slab: a field of %d planes from global plane %d does not hold rank %d's planes "
                     "[%d, %d)", field->nz, z_offset, r->rank, r->z0, r->z1);
  return recorder_capture(ctx, r, field, z_offset, frame_out);
}

int tfl_recorder_take(tfl_ctx* ctx, tfl_recorder* r, int wait, const float** host_out, int64_t* frame_out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!ctx) return 1;
  if (host_out) *host_out = nullptr;
  if (frame_out) *frame_out = -1;
  if (!r) return fail(ctx, "recorder_take: recorder is nil");
  if (r->rank > 0) return fail(ctx, "recorder_take: rank %d has no frames; rank 0 (the writer) takes them", r->rank);
  if (!host_out || !frame_out) return fail(ctx, "recorder_take: host_out and frame_out must not be nil");
  if (r->captured == 0) return fail(ctx, "recorder_take: no captured frame left to take");
  const int slot = (r->first + r->taken) % r->slots;
  cudaEvent_t e = r->copied[slot].get();
  if (wait) {
    TFL_CUDA(ctx, cudaEventSynchronize(e));
  } else {
    const cudaError_t q = cudaEventQuery(e);
    if (q == cudaErrorNotReady) {                         // not an error: *frame_out stays -1
      cudaGetLastError();                                 // and no later launch check may report it
      return 0;
    }
    if (q != cudaSuccess) return fail(ctx, "recorder_take: cudaEventQuery: %s", cudaGetErrorString(q));
  }
  r->taken++;
  r->captured--;
  const unsigned long long miss = r->missing ? r->missing.get()[slot] : 0ULL;
  if (miss) {                    // taken without its planes: *frame_out names it, the caller releases it as usual
    *frame_out = r->frame[slot];
    std::string ranks;
    for (int k = 1; k < r->world; k++)
      if (miss >> k & 1ULL) ranks += (ranks.empty() ? "" : ", ") + std::to_string(k);
    return fail(ctx, "recorder_take: frame %lld is incomplete: the planes of rank(s) %s did not arrive within the wait "
                     "bound (release it to go on)", (long long)r->frame[slot], ranks.c_str());
  }
  *host_out = r->host[slot].get();
  *frame_out = r->frame[slot];
  return 0;
}

int tfl_recorder_release(tfl_ctx* ctx, tfl_recorder* r) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!ctx) return 1;
  if (!r) return fail(ctx, "recorder_release: recorder is nil");
  if (r->rank > 0) return fail(ctx, "recorder_release: rank %d has no frames; rank 0 (the writer) releases them", r->rank);
  if (r->taken == 0) return fail(ctx, "recorder_release: no taken frame to release");
  r->frame[r->first] = -1;
  r->first = (r->first + 1) % r->slots;
  r->taken--;
  return 0;
}

}  // extern "C"
