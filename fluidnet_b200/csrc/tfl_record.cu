// Frame recorder (tfl_recorder_*): a scalar grid leaves the device in `.vbox` order behind the running step.
// capture packs the field into one device staging frame on the context's stream (k_pack_vbox) and a copy stream
// moves the staging frame into the next free slot of a ring of pinned host frames; take / release hand the frames
// to the host strictly first in, first out.  Nothing here synchronises except take(wait = 1), which waits for that
// one frame's copy, and destroy.
#include <cuda_runtime.h>
#include <stdint.h>

#include "tfl_api_internal.h"
#include "../../include/tfl.h"

constexpr int kPackTile = 32;     // a 32 x 32 (z, x) tile per block
constexpr int kPackRows = 8;      // 32 x 8 threads, 4 rows each

// in [nz][ny][nx] (x fastest) -> out[(x * ny + y) * nz + z] (z fastest): `permute(3, 2, 1)` of the grid, the
// order the demo writes to a `.vbox` file.  Block (bx, bz, y) moves the (z, x) tile [bz * 32, +32) x [bx * 32, +32)
// of plane y through shared memory: the load walks x and the store walks z, both coalesced (128 bytes per warp).
// The row of 33 words keeps the transposed read free of bank conflicts.  A bit copy (32-bit words, no arithmetic):
// -0.0, denormals and NaN payloads arrive unchanged.
// Not in an anonymous namespace: the kernel keeps a stable name in traces and profiles.
__global__ void __launch_bounds__(kPackTile * kPackRows)
k_pack_vbox(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, int nz, int ny, int nx) {
  __shared__ uint32_t tile[kPackTile][kPackTile + 1];
  const int x0 = blockIdx.x * kPackTile, z0 = blockIdx.y * kPackTile, y = blockIdx.z;
  const int tx = threadIdx.x, ty = threadIdx.y;
  const long long plane = (long long)ny * nx;
  const int x = x0 + tx;
#pragma unroll
  for (int r = ty; r < kPackTile; r += kPackRows) {
    const int z = z0 + r;
    if (z < nz && x < nx) tile[r][tx] = __ldg(in + z * plane + (long long)y * nx + x);
  }
  __syncthreads();
  const int z = z0 + tx;
#pragma unroll
  for (int r = ty; r < kPackTile; r += kPackRows) {
    const int xo = x0 + r;
    if (xo < nx && z < nz) out[((long long)xo * ny + y) * nz + z] = tile[tx][r];
  }
}

// Launches k_pack_vbox on `st`; returns the number of kernels launched (1).
static int launch_pack_vbox(const float* in, float* out, int nz, int ny, int nx, cudaStream_t st) {
  const dim3 block(kPackTile, kPackRows);
  const dim3 grid((nx + kPackTile - 1) / kPackTile, (nz + kPackTile - 1) / kPackTile, ny);
  k_pack_vbox<<<grid, block, 0, st>>>((const uint32_t*)in, (uint32_t*)out, nz, ny, nx);
  return 1;
}

// Slots in use form one run of the ring starting at `first`: `taken` frames handed to the host (oldest first), then
// `captured` frames whose copies are enqueued or done.  The next capture fills slot (first + taken + captured).
struct tfl_recorder {
  int nz = 0, ny = 0, nx = 0, slots = 0;
  size_t bytes = 0;                          // one frame
  DevPtr<float> stage;                       // the packed frame, read by the copy stream
  std::vector<PinnedPtr<float>> host;        // [slots] host frames
  std::vector<EventPtr> copied;              // [slots] recorded on `copy` after the slot's copy
  std::vector<int64_t> frame;                // [slots] index of the frame the slot holds
  StreamPtr copy;
  EventPtr packed;                           // recorded on the context's stream after the pack
  int first = 0, taken = 0, captured = 0;
  int last_slot = -1;                        // slot of the latest copy out of `stage` (the next pack waits on it)
  int64_t next_frame = 0;
};

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
  std::unique_ptr<tfl_recorder> r(new tfl_recorder());
  r->nz = nz; r->ny = ny; r->nx = nx; r->slots = slots;
  const size_t cells = (size_t)nz * ny * nx;
  r->bytes = cells * sizeof(float);
  if (!(r->stage = dev_alloc<float>(cells))) return fail(ctx, "recorder_create: cudaMalloc of the staging frame failed");
  if (!(r->copy = new_stream(cudaStreamNonBlocking)) || !(r->packed = new_event(cudaEventDisableTiming)))
    return fail(ctx, "recorder_create: creating the copy stream or its events failed");
  for (int i = 0; i < slots; ++i) {
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

void tfl_recorder_destroy(tfl_ctx* ctx, tfl_recorder* r) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (r && r->copy) cudaStreamSynchronize(r->copy.get());   // copies in flight write into the host frames
  delete r;
}

int tfl_recorder_capture(tfl_ctx* ctx, tfl_recorder* r, const tfl_grid* field, int64_t* frame_out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!ctx) return 1;
  if (frame_out) *frame_out = -1;
  if (!r) return fail(ctx, "recorder_capture: recorder is nil");
  if (r->taken + r->captured == r->slots)
    return fail(ctx, "recorder_capture: the %d x %d x %d recorder's %d slot(s) all hold frames not yet released "
                     "(take and release the oldest first)", r->nz, r->ny, r->nx, r->slots);
  if (!field || !field->data) return fail(ctx, "recorder_capture: field is nil");
  if (field->nb != 1) return fail(ctx, "recorder_capture: field has nb = %d; a recorder takes one batch entry (nb = 1)", field->nb);
  if (field->nc != 1) return fail(ctx, "recorder_capture: field has nc = %d; a recorder takes a scalar field (nc = 1)", field->nc);
  if (field->nz != r->nz || field->ny != r->ny || field->nx != r->nx)
    return fail(ctx, "recorder_capture: field is %d x %d x %d (z, y, x), the recorder's frames are %d x %d x %d",
                field->nz, field->ny, field->nx, r->nz, r->ny, r->nx);
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  TFL_CUDA(ctx, cudaStreamIsCapturing(ctx->stream, &cs));
  if (cs != cudaStreamCaptureStatusNone)
    return fail(ctx, "recorder_capture: the context's stream is being captured into a graph; record outside the capture");
  const int slot = (r->first + r->taken + r->captured) % r->slots;
  cudaStream_t st = ctx->stream;
  // The staging frame is free once the previous copy out of it has run: a device-side wait, never a host one.
  if (r->last_slot >= 0) TFL_CUDA(ctx, cudaStreamWaitEvent(st, r->copied[r->last_slot].get(), 0));
  ctx->launches += launch_pack_vbox(field->data, r->stage.get(), r->nz, r->ny, r->nx, st);
  if (check_launch(ctx, "k_pack_vbox")) return 1;
  TFL_CUDA(ctx, cudaEventRecord(r->packed.get(), st));
  TFL_CUDA(ctx, cudaStreamWaitEvent(r->copy.get(), r->packed.get(), 0));
  TFL_CUDA(ctx, cudaMemcpyAsync(r->host[slot].get(), r->stage.get(), r->bytes, cudaMemcpyDeviceToHost, r->copy.get()));
  TFL_CUDA(ctx, cudaEventRecord(r->copied[slot].get(), r->copy.get()));
  r->last_slot = slot;
  r->frame[slot] = r->next_frame;
  if (frame_out) *frame_out = r->next_frame;
  r->next_frame++;
  r->captured++;
  return 0;
}

int tfl_recorder_take(tfl_ctx* ctx, tfl_recorder* r, int wait, const float** host_out, int64_t* frame_out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!ctx) return 1;
  if (host_out) *host_out = nullptr;
  if (frame_out) *frame_out = -1;
  if (!r) return fail(ctx, "recorder_take: recorder is nil");
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
  *host_out = r->host[slot].get();
  *frame_out = r->frame[slot];
  r->taken++;
  r->captured--;
  return 0;
}

int tfl_recorder_release(tfl_ctx* ctx, tfl_recorder* r) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!ctx) return 1;
  if (!r) return fail(ctx, "recorder_release: recorder is nil");
  if (r->taken == 0) return fail(ctx, "recorder_release: no taken frame to release");
  r->frame[r->first] = -1;
  r->first = (r->first + 1) % r->slots;
  r->taken--;
  return 0;
}

}  // extern "C"
