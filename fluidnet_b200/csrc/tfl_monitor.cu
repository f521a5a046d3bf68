// Step monitor (tfl_monitor_*): after a step, one call enqueues a reduction over U and the flags as the stream leaves
// them and yields one record per batch entry -- div_norm = sqrt(sum d^2) and div_max = max |d| of the divergence d that
// tfl_velocity_divergence_forward writes, and u_max = max |U| over every face and component -- the quantities
// calc_stats.lua:81-123 of the reference takes after every tfluids.simulate.  Nothing here synchronises except
// take(wait = 1), which waits for that one record, and destroy.
//
// Reduction order (fp64, fixed by the field alone):
//   k_monitor_chunks  one CTA per (batch entry, plane, chunk): a plane of ny rows is cut into min(ny, 8) chunks of
//                     whole rows (chunk c: rows [c ny / C, (c + 1) ny / C)); each thread adds its cells in order, the
//                     CTA's warps reduce in a fixed tree and warp 0 adds the eight warp sums in order.
//   k_monitor_finish  one CTA: a plane's partial is its chunks summed in chunk order; the total is the planes' partials
//                     summed in ascending global z, starting from 0, then the square root.
// The partial of a plane depends on (ny, nx) and the plane's cells only, so a z-slab rank (a context with a slab
// placement) yields the very partials the whole grid would; it hands them out per plane with their global index, and a
// host adding them in ascending z repeats the device's last step bit for bit.
//
// Records go straight into a ring of pinned, mapped host slots: the finishing CTA stores the record's doubles, fences
// at system scope and stores the record's sequence number last with release semantics (tfl_peer.cuh).  The host polls
// that word; there is no copy stream and no event per record.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include <thread>

#include "tfl_device.cuh"
#include "tfl_api_internal.h"
#include "tfl_peer.cuh"
#include "../../include/tfl.h"

constexpr int kMonThreads = 256;
constexpr int kMonChunks = 8;         // chunks per plane at most: 2048 cells per CTA at 128^2, 8192 at 256^2

// max that propagates NaN (fmaxf / fmax drop it): a field that went NaN shows in div_max and u_max, not only in div_norm
template <typename T>
__device__ __forceinline__ T nan_max(T a, T b) { return (b > a || b != b) ? b : a; }

// Chunk partials (sum d^2, max |d|, max |U|) of planes [zlo, zlo + gridDim.y) (local) of batch entry blockIdx.z.
// d is k_divergence's expression, evaluated in the same order (compiled with -fmad=false as that kernel is).
// Not in an anonymous namespace: the kernel keeps a stable name in traces and profiles.
template <bool IS3D>
__global__ void __launch_bounds__(kMonThreads)
k_monitor_chunks(const float* __restrict__ U, const float* __restrict__ flags, Geo gin, int zlo, int nchunks,
                 double* __restrict__ part) {
  const Geo g = static_geo<IS3D>(gin);
  const int c = blockIdx.x, pl = blockIdx.y, b = blockIdx.z, k = zlo + pl;
  const int r0 = (int)((long long)c * g.ny / nchunks), r1 = (int)((long long)(c + 1) * g.ny / nchunks);
  const float* fl = flags + b * g.n;
  const float* ub = U + (long long)b * g.nc * g.n;
  const int base = k * g.ny * g.nx;
  double s = 0.0;
  float dm = 0.0f, um = 0.0f;
  for (int t = r0 * g.nx + threadIdx.x; t < r1 * g.nx; t += kMonThreads) {
    const int j = t / g.nx, i = t - j * g.nx, cc = base + t;
    float r = 0.0f;
    if (!on_border(g, k, j, i) && (flag_at(fl, cc) & kFluid)) {
      r = __ldg(ub + cc) - __ldg(ub + cc + 1) + __ldg(ub + g.n + cc) - __ldg(ub + g.n + cc + g.nx);
      if (g.is3d) r += (__ldg(ub + 2 * g.n + cc) - __ldg(ub + 2 * g.n + cc + (long long)g.nx * g.ny));
    }
    s += (double)r * (double)r;                     // a float's square is exact in double
    dm = nan_max(dm, fabsf(r));
#pragma unroll
    for (int a = 0; a < g.nc; a++) um = nan_max(um, fabsf(__ldg(ub + a * g.n + cc)));
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    s += __shfl_down_sync(0xffffffffu, s, off);
    dm = nan_max(dm, __shfl_down_sync(0xffffffffu, dm, off));
    um = nan_max(um, __shfl_down_sync(0xffffffffu, um, off));
  }
  __shared__ double ws[kMonThreads / 32];
  __shared__ float wd[kMonThreads / 32], wu[kMonThreads / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) { ws[w] = s; wd[w] = dm; wu[w] = um; }
  __syncthreads();
  if (threadIdx.x == 0) {
    s = 0.0;
    dm = 0.0f;
    um = 0.0f;
    for (int q = 0; q < kMonThreads / 32; q++) { s += ws[q]; dm = nan_max(dm, wd[q]); um = nan_max(um, wu[q]); }
    double* o = part + (((long long)b * gridDim.y + pl) * nchunks + c) * 3;
    o[0] = s;
    o[1] = dm;
    o[2] = um;
  }
}

// Plane partials from the chunk partials, then (whole grid) the totals; both land in the mapped host slot `rec`, whose
// sequence word `seq_word` is stored last.  planes_only: a z-slab record (nb x planes x {sum d^2, max |d|, max |U|});
// otherwise nb x {div_norm, div_max, u_max}.  The planes go through shared memory 256 at a time, where thread 0 adds
// them in order (a sequential walk over global memory would pay its latency once per plane).
__global__ void __launch_bounds__(kMonThreads)
k_monitor_finish(const double* __restrict__ part, int nb, int nplanes, int nchunks, int planes_only, double* rec,
                 unsigned long long* seq_word, unsigned long long seq) {
  __shared__ double sp[kMonThreads][3];
  for (int b = 0; b < nb; b++) {
    double s = 0.0, dm = 0.0, um = 0.0;                   // thread 0's running totals
    for (int z0 = 0; z0 < nplanes; z0 += kMonThreads) {
      const int z = z0 + threadIdx.x;
      if (z < nplanes) {
        const double* p = part + ((long long)b * nplanes + z) * nchunks * 3;
        double ps = 0.0, pd = 0.0, pu = 0.0;
        for (int c = 0; c < nchunks; c++) { ps += p[3 * c]; pd = nan_max(pd, p[3 * c + 1]); pu = nan_max(pu, p[3 * c + 2]); }
        if (planes_only) {
          double* o = rec + ((long long)b * nplanes + z) * 3;
          o[0] = ps; o[1] = pd; o[2] = pu;
        }
        sp[threadIdx.x][0] = ps; sp[threadIdx.x][1] = pd; sp[threadIdx.x][2] = pu;
      }
      __syncthreads();
      if (threadIdx.x == 0 && !planes_only) {
        const int n = nplanes - z0 < kMonThreads ? nplanes - z0 : kMonThreads;
        for (int q = 0; q < n; q++) { s += sp[q][0]; dm = nan_max(dm, sp[q][1]); um = nan_max(um, sp[q][2]); }
      }
      __syncthreads();
    }
    if (threadIdx.x == 0 && !planes_only) { rec[3 * b] = sqrt(s); rec[3 * b + 1] = dm; rec[3 * b + 2] = um; }
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) store_release_sys(seq_word, seq);
}

// A ring of `capacity` mapped host slots; slot = [sequence word][nb x gnz x 3 doubles].  Records in flight or
// finished and not yet taken are `count` slots from `head`.
struct tfl_monitor {
  int nb = 0, gnz = 0, capacity = 0;
  int nc = 0, ny = 0, nx = 0;                // fixed by the first record (0: none yet)
  size_t slot_doubles = 0;
  DevPtr<double> part;                       // chunk partials [nb][gnz][kMonChunks][3]
  PinnedPtr<double> ring;                    // [capacity][slot_doubles], mapped
  double* ring_dev = nullptr;
  EventPtr done;                             // after the latest record: a record on another stream waits on it
  bool any = false;
  struct Slot {
    int64_t index = -1;
    int z0 = 0, planes = 0;                  // planes > 0: a z-slab record of global planes [z0, z0 + planes)
    cudaStream_t stream = nullptr;
  };
  std::vector<Slot> slots;
  int head = 0, count = 0;
  int64_t next = 0;
  cudaStream_t last_stream = nullptr;
};

static volatile unsigned long long* seq_of(const tfl_monitor* m, int slot) {
  return reinterpret_cast<volatile unsigned long long*>(m->ring.get() + (size_t)slot * m->slot_doubles);
}

int monitor_precheck(tfl_ctx* ctx, const tfl_monitor* m, int nb, int gnz) {
  if (m->count == m->capacity)
    return fail(ctx, "monitor_record: the monitor's %d record slot(s) all hold records not yet taken (take the oldest "
                     "first)", m->capacity);
  if (nb != m->nb) return fail(ctx, "monitor_record: the grid has nb = %d, the monitor's nb is %d", nb, m->nb);
  if (gnz != m->gnz)
    return fail(ctx, "monitor_record: the grid has gnz = %d (global planes), the monitor's gnz is %d", gnz, m->gnz);
  return 0;
}

extern "C" {

int tfl_monitor_create(tfl_ctx* ctx, int32_t nb, int32_t gnz, int32_t capacity, tfl_monitor** out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!ctx) return 1;
  if (!out) return fail(ctx, "monitor_create: out is nil");
  *out = nullptr;
  if (nb < 1 || gnz < 1) return fail(ctx, "monitor_create: nb and gnz must be >= 1 (got nb = %d, gnz = %d)", nb, gnz);
  if (capacity < 1) return fail(ctx, "monitor_create: capacity must be >= 1 (got %d)", capacity);
  if ((long long)nb * gnz * kMonChunks * 3 >= (1LL << 31)) return fail(ctx, "monitor_create: nb x gnz too large");
  if (nb > kMaxGridYZ || gnz > kMaxGridYZ)      // k_monitor_chunks: one block per entry on z, per plane on y
    return fail(ctx, "monitor_create: nb = %d and gnz = %d must each be at most %lld (blocks along gridDim.z and y)",
                nb, gnz, kMaxGridYZ);
  std::unique_ptr<tfl_monitor> m(new tfl_monitor());
  m->nb = nb; m->gnz = gnz; m->capacity = capacity;
  m->slot_doubles = 1 + (size_t)nb * gnz * 3;
  if (!(m->part = dev_alloc<double>((size_t)nb * gnz * kMonChunks * 3)))
    return fail(ctx, "monitor_create: cudaMalloc of the partial sums failed");
  double* h = nullptr;
  TFL_CUDA(ctx, cudaHostAlloc((void**)&h, (size_t)capacity * m->slot_doubles * sizeof(double), cudaHostAllocMapped));
  m->ring.reset(h);
  memset(h, 0, (size_t)capacity * m->slot_doubles * sizeof(double));
  TFL_CUDA(ctx, cudaHostGetDevicePointer((void**)&m->ring_dev, h, 0));
  if (!(m->done = new_event(cudaEventDisableTiming))) return fail(ctx, "monitor_create: creating its event failed");
  m->slots.resize(capacity);
  *out = m.release();
  return 0;
}

void tfl_monitor_destroy(tfl_ctx* ctx, tfl_monitor* m) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!m) return;
  for (int q = 0; q < m->count; q++) {        // records in flight write into the host slots
    cudaStream_t st = m->slots[(m->head + q) % m->capacity].stream;
    cudaStreamSynchronize(st);
  }
  delete m;
}

int tfl_monitor_record(tfl_ctx* ctx, tfl_monitor* m, const tfl_grid* U, const tfl_grid* flags, int64_t* index_out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!ctx) return 1;
  if (index_out) *index_out = -1;
  if (!m) return fail(ctx, "monitor_record: monitor is nil");
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  TFL_CUDA(ctx, cudaStreamIsCapturing(ctx->stream, &cs));
  if (cs != cudaStreamCaptureStatusNone)
    return fail(ctx, "monitor_record: the context's stream is being captured into a graph; record after the graph's launch");
  if (m->count == m->capacity) return monitor_precheck(ctx, m, m->nb, m->gnz);   // the full ring first
  if (!flags || !flags->data) return fail(ctx, "monitor_record: flags is nil");
  if (!U || !U->data) return fail(ctx, "monitor_record: U is nil");
  if (flags->nc != 1) return fail(ctx, "monitor_record: flags has nc = %d, a scalar field has 1", flags->nc);
  if (U->nc != 2 && U->nc != 3) return fail(ctx, "monitor_record: U has nc = %d (3-D: 3, 2-D: 2)", U->nc);
  if (U->nc == 2 && U->nz != 1) return fail(ctx, "monitor_record: U has 2 channels but nz = %d (2-D grids have nz = 1)", U->nz);
  if (!same_spatial(U, flags))
    return fail(ctx, "monitor_record: U is %d x %d x %d x %d and flags %d x %d x %d x %d (nb, z, y, x): shape mismatch",
                U->nb, U->nz, U->ny, U->nx, flags->nb, flags->nz, flags->ny, flags->nx);
  if (monitor_precheck(ctx, m, flags->nb, ctx->slab ? ctx->gnz : flags->nz)) return 1;
  if (m->any && (U->nc != m->nc || flags->ny != m->ny || flags->nx != m->nx))
    return fail(ctx, "monitor_record: the grid's shape (nc %d, ny %d, nx %d) differs from the monitor's first record's "
                     "(nc %d, ny %d, nx %d)", U->nc, flags->ny, flags->nx, m->nc, m->ny, m->nx);
  Geo g;
  if (make_geo(ctx, flags, U->nc == 3, &g)) return fail(ctx, "monitor_record: %s", ctx->err.c_str());
  // d on plane k reads U on plane k + 1: the local grid must hold it unless k is the global grid's last plane
  if (g.zhi == g.nz && g.zoff + g.nz < g.gnz)
    return fail(ctx, "monitor_record: the slab placement's last plane (global %d) needs the plane above it in the local "
                     "grid", g.zoff + g.zhi - 1);
  const int nplanes = g.zhi - g.zlo, nchunks = g.ny < kMonChunks ? g.ny : kMonChunks;
  cudaStream_t st = ctx->stream;
  if (m->last_stream && m->last_stream != st) TFL_CUDA(ctx, cudaStreamWaitEvent(st, m->done.get(), 0));
  const int slot = (m->head + m->count) % m->capacity;
  const unsigned long long seq = (unsigned long long)m->next + 1;
  double* rec = m->ring_dev + (size_t)slot * m->slot_doubles;
  const dim3 grid(nchunks, nplanes, g.nb);
  if (g.is3d) k_monitor_chunks<true><<<grid, kMonThreads, 0, st>>>(U->data, flags->data, g, g.zlo, nchunks, m->part.get());
  else k_monitor_chunks<false><<<grid, kMonThreads, 0, st>>>(U->data, flags->data, g, g.zlo, nchunks, m->part.get());
  k_monitor_finish<<<1, kMonThreads, 0, st>>>(m->part.get(), g.nb, nplanes, nchunks, ctx->slab ? 1 : 0, rec + 1,
                                              reinterpret_cast<unsigned long long*>(rec), seq);
  ctx->launches += 2;
  if (check_launch(ctx, "monitor_record")) return 1;
  TFL_CUDA(ctx, cudaEventRecord(m->done.get(), st));
  m->last_stream = st;
  if (!m->any) { m->any = true; m->nc = U->nc; m->ny = flags->ny; m->nx = flags->nx; }
  tfl_monitor::Slot& s = m->slots[slot];
  s.index = m->next;
  s.z0 = ctx->slab ? g.zoff + g.zlo : 0;
  s.planes = ctx->slab ? nplanes : 0;
  s.stream = st;
  if (index_out) *index_out = m->next;
  m->next++;
  m->count++;
  return 0;
}

int tfl_monitor_take(tfl_ctx* ctx, tfl_monitor* m, int wait, int64_t* index_out, double* values_out, int32_t* z0_out,
                     int32_t* planes_out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!ctx) return 1;
  if (index_out) *index_out = -1;
  if (!m) return fail(ctx, "monitor_take: monitor is nil");
  if (!index_out || !values_out) return fail(ctx, "monitor_take: index_out and values_out must not be nil");
  if (m->count == 0) return fail(ctx, "monitor_take: the monitor holds no record (nothing recorded since the last take)");
  const tfl_monitor::Slot& s = m->slots[m->head];
  const unsigned long long want = (unsigned long long)s.index + 1;
  volatile unsigned long long* word = seq_of(m, m->head);
  while (*word != want) {
    if (!wait) return 0;                                  // not an error: *index_out stays -1
    const cudaError_t q = cudaStreamQuery(s.stream);
    if (q == cudaSuccess) {                               // the stream drained: the store must be visible now
      if (*word == want) break;
      return fail(ctx, "monitor_take: record %lld's stream finished without publishing it", (long long)s.index);
    }
    if (q != cudaErrorNotReady) return fail(ctx, "monitor_take: cudaStreamQuery: %s", cudaGetErrorString(q));
    cudaGetLastError();
    std::this_thread::yield();
  }
  __atomic_thread_fence(__ATOMIC_ACQUIRE);
  const double* rec = m->ring.get() + (size_t)m->head * m->slot_doubles + 1;
  const size_t n = (size_t)m->nb * (s.planes ? s.planes : 1) * 3;
  memcpy(values_out, rec, n * sizeof(double));
  *index_out = s.index;
  if (z0_out) *z0_out = s.z0;
  if (planes_out) *planes_out = s.planes;
  m->head = (m->head + 1) % m->capacity;
  m->count--;
  return 0;
}

}  // extern "C"
