// C ABI of the z-slab driver (include/tfl.h): the NCCL loader, the halo exchange and all-reduce kernels, and
// tfl_comm_* / tfl_slab_sim_* / tfl_slab_graph_*.
#include <dlfcn.h>
#include <string.h>
#include <algorithm>
#include <vector>

#include "tfl_api_internal.h"
#include "tfl_peer.cuh"

// ---------------------------------------------------------------------------------------
// One domain split into z-slabs over the GPUs of a node (SURVEY.md 8e).  The reference is
// single-GPU; this is the multi-GPU form of the same step: rank r owns the planes [z0, z1) of every
// field plus `halo` ghost planes per interior side, every kernel works in GLOBAL coordinates
// (tfl_set_slab), and ghost planes are refreshed by neighbour ncclSend / ncclRecv pairs one
// message per neighbour and direction (a gather kernel packs the planes of every channel, a scatter kernel
// unpacks them), grouped into one NCCL operation per phase:
//     exchange U, density (halo = 2 * margin + 2)  -> advectScalar, advectVel
//     exchange U, density (4)                      -> buoyancy / gravity on owned +- 3, vorticity confinement
//     exchange U, p (5)                            -> wall mask + (sum, sum^2) on owned planes
//     all-reduce of the two doubles                -> conv stack on the local slab, velocity update
// simMethod 'jacobi' replaces the last two phases (tfl_slab_jacobi_schedule):
//     exchange U (w <= halo)                       -> divergence and Jacobi mask on owned +- (w - 1)
//     blocks of up to `halo` sweeps, p exchanged   -> velocity update on owned planes
//     before each block but the first
// ---------------------------------------------------------------------------------------
namespace {

struct NcclApi {
  void* lib = nullptr;
  decltype(&ncclGetUniqueId) GetUniqueId = nullptr;
  decltype(&ncclCommInitRank) CommInitRank = nullptr;
  decltype(&ncclCommDestroy) CommDestroy = nullptr;
  decltype(&ncclGroupStart) GroupStart = nullptr;
  decltype(&ncclGroupEnd) GroupEnd = nullptr;
  decltype(&ncclSend) Send = nullptr;
  decltype(&ncclRecv) Recv = nullptr;
  decltype(&ncclAllReduce) AllReduce = nullptr;
  decltype(&ncclGetErrorString) GetErrorString = nullptr;
};
NcclApi* nccl_api() {
  static NcclApi api;
  static bool tried = false;
  if (!tried) {
    tried = true;
    // a host that already carries an NCCL (e.g. the one bundled with PyTorch) gets that copy back
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (h) {
      api.lib = h;
#define TFL_NCCL_SYM(name) api.name = (decltype(api.name))dlsym(h, "nccl" #name)
      TFL_NCCL_SYM(GetUniqueId); TFL_NCCL_SYM(CommInitRank); TFL_NCCL_SYM(CommDestroy); TFL_NCCL_SYM(GroupStart);
      TFL_NCCL_SYM(GroupEnd); TFL_NCCL_SYM(Send); TFL_NCCL_SYM(Recv); TFL_NCCL_SYM(AllReduce); TFL_NCCL_SYM(GetErrorString);
#undef TFL_NCCL_SYM
      if (!api.GetUniqueId || !api.CommInitRank || !api.CommDestroy || !api.GroupStart || !api.GroupEnd || !api.Send ||
          !api.Recv || !api.AllReduce || !api.GetErrorString)
        api.lib = nullptr;
    }
  }
  return api.lib ? &api : nullptr;
}
#define TFL_NCCL(ctx, call)                                                                       \
  do {                                                                                            \
    ncclResult_t r_ = (call);                                                                     \
    if (r_ != ncclSuccess) return fail(ctx, "%s: %s", #call, nccl_api()->GetErrorString(r_));     \
  } while (0)

}  // namespace

// A rank's inbox: the one allocation its peers store into over peer memory (exported as one CUDA IPC handle).  Every
// rank's has this layout, in floats, with the counters written and waited on as tfl_peer.cuh describes:
//   [3 phases][2 from][xbuf_side]        halo messages (from 0: the rank below, 1: the rank above)
//   [64]                                  their counters, [phase][from], carrying the step number
//   [2 parities][kMaxRanks][2] doubles    the all-reduce's pair from each rank, parity = step number & 1
//   [2 parities][kMaxRanks]               their counters, carrying the step number
//   [2 parities][2 from][p_side]          the Jacobi p exchange's messages, parity = p sequence & 1
//   [64]                                  their counters, [parity][from], carrying the p sequence
//   [2 parities][r_side] doubles          the Jacobi tolerance solve's per-plane residuals of one block, [sweep][global
//                                         plane]: every rank stores its owned planes, parity = r sequence & 1
//   [2 parities][kMaxRanks]               their counters, [parity][rank], carrying the r sequence
// Alternating parities let a rank push the next all-reduce or p exchange while its peer still reads the current one.
// The step number and the p and r sequences live on the device (tfl_slab_sim::seq, SlabSeq), so a replayed step
// (tfl_slab_graph_launch) advances them exactly as a direct one does.
struct SlabInbox {
  size_t xbuf_side, p_side;             // floats of one halo message / one p message
  size_t r_side;                        // doubles of one block's residuals: halo sweeps x gnz planes
  static constexpr int kCounterFloats = 64;
  static constexpr int kSumSlotFloats = 2 * kMaxRanks * 2 * 2;
  static constexpr int kSumFloats = kSumSlotFloats + 2 * kMaxRanks;
  __host__ __device__ float* halo(float* inbox, int phase, int from) const {
    return inbox + ((size_t)phase * 2 + from) * xbuf_side;
  }
  __host__ __device__ unsigned int* halo_flag(float* inbox, int phase, int from) const {
    return (unsigned int*)(inbox + 6 * xbuf_side) + phase * 2 + from;
  }
  __host__ __device__ double* sum_slot(float* inbox, int parity, int rank) const {
    return reinterpret_cast<double*>(inbox + 6 * xbuf_side + kCounterFloats) + ((size_t)parity * kMaxRanks + rank) * 2;
  }
  __host__ __device__ unsigned int* sum_flag(float* inbox, int parity, int rank) const {
    return reinterpret_cast<unsigned int*>(inbox + 6 * xbuf_side + kCounterFloats + kSumSlotFloats) + parity * kMaxRanks + rank;
  }
  __host__ __device__ float* p_area(float* inbox) const { return inbox + 6 * xbuf_side + kCounterFloats + kSumFloats; }
  __host__ __device__ float* p_buf(float* inbox, int parity, int from) const {
    return p_area(inbox) + ((size_t)parity * 2 + from) * p_side;
  }
  __host__ __device__ unsigned int* p_flag(float* inbox, int parity, int from) const {
    return (unsigned int*)(p_area(inbox) + 4 * p_side) + parity * 2 + from;
  }
  // behind the p area, at an even float offset (xbuf_side and p_side are multiples of the even halo)
  __host__ __device__ double* r_buf(float* inbox, int parity) const {
    return reinterpret_cast<double*>(p_area(inbox) + 4 * p_side + kCounterFloats) + (size_t)parity * r_side;
  }
  __host__ __device__ unsigned int* r_flag(float* inbox, int parity, int rank) const {
    return reinterpret_cast<unsigned int*>(r_buf(inbox, 2)) + parity * kMaxRanks + rank;
  }
  size_t floats() const {
    return 6 * xbuf_side + kCounterFloats + kSumFloats + 4 * p_side + kCounterFloats + 4 * r_side + 2 * kMaxRanks;
  }
};

// The z-slab Jacobi tolerance solve's device state (slab_jacobi_tol), zeroed at the start of every solve.
struct SlabTolState {
  int done;        // the solve has stopped: every gated kernel and p exchange of the loop returns at once
  int blk;         // blocks decided so far
  int iter;        // the iteration counter of the whole-grid loop
  float res;       // residual of the last sweep run
  int stop_blk;    // the block of the stopping sweep
  int rollback;    // the stop fell before the last sweep of its block: p is rebuilt from the block's start
  int odd;         // the final iterate lies in p2 (an odd count of kept sweeps in the stopping block)
  int fix;         // the stop fell on the last sweep of a block that leaves p stale below the owned planes
};

struct tfl_slab_sim {
  int gnz = 0, ny = 0, nx = 0, margin = 2, halo = 6;
  int rank = 0, world = 1;
  int z0 = 0, z1 = 0, lo_halo = 0, hi_halo = 0, zoff = 0, nz = 0, own_lo = 0, own_hi = 0;
  size_t cells = 0, plane = 0;      // local cells / cells per plane
  tfl_state st;                     // views of the field buffers below
  DevPtr<float> flags, p, U, density, U_bc, U_bc_inv, d_bc, d_bc_inv;
  DevPtr<float> U1;
  DevPtr<double> sums;
  DevPtr<float> xbuf;               // [send down | send up | recv from below | recv from above], xbuf_side floats each
  size_t xbuf_side = 0;
  // Peer-memory exchanges (CUDA IPC over NVLink, tfl_slab_sim_ipc_*): this rank's inbox, which the peers' push kernels
  // fill with remote stores, and the other ranks' inboxes mapped into this process.
  DevPtr<float> inbox;              // exported, laid out as SlabInbox
  std::vector<IpcPtr<float>> mapped;           // the other ranks' inboxes, empty at [rank]
  float* peer_inbox[2] = {nullptr, nullptr};   // lower / upper neighbour's inbox
  std::vector<float*> all_inbox;               // every rank's inbox (own pointer at [rank]): the all-reduce's targets
  DevPtr<float*> all_inbox_dev;                // the same table on the device
  DevPtr<unsigned int> push_done;              // CTAs of the running push kernel that finished their stores
  // The exchanges' sequence numbers, two words each (SlabSeq): [0, 2) the step number, which the halo and all-reduce
  // counters carry, [2, 4) the p sequence, which the Jacobi p exchanges and tfl_slab_sim_monitor_record advance, and
  // [4, 6) the r sequence of the tolerance solve's residual gathers.
  DevPtr<unsigned int> seq;
  bool peer_ok = false;
  unsigned long long peer_gen = 0;             // bumped by every tfl_slab_sim_ipc_connect (the mapped inboxes change)
  bool capturing = false;                      // tfl_slab_graph_create is capturing a step
  // The last direct step, which sized every buffer a capture of the same step uses (tfl_slab_graph_create)
  struct {
    bool done = false;
    const tfl_cnn* cnn = nullptr;
    int sim_method = -1;
    BufferGens gens;
  } last;
  EventPtr ev[4][2];
  size_t bytes_sent[3] = {0, 0, 0};
  // Jacobi projection (simMethod 'jacobi'): divergence, second p buffer and mask of the local slab; the p exchanges
  // land in their own inbox area and carry the p sequence instead of the step number.
  DevPtr<float> div;
  DevPtr<float> p2;
  DevPtr<unsigned char> mask;
  size_t p_side = 0;                // halo planes of one channel
  std::vector<int32_t> jsched;
  std::vector<EventPtr> jev;        // [2 * exchange] begin / end of the last step's p exchanges
  int jx = 0;                       // p exchanges of the last step
  size_t jbytes = 0;
  // Jacobi to a tolerance (tfl_slab_sim_set_jacobi_tolerance; slab_jacobi_tol): allocated when a tolerance is first set
  float p_tol = 0.0f;
  bool tol_stepped = false;         // a step has run with a tolerance (tfl_slab_sim_jacobi_status)
  bool tol_last = false;            // the last step ran with one: its p exchange count comes from tol_state
  std::vector<int> tol_widths;      // width of the p exchange before each block of the last step's solve (0: none)
  DevPtr<float> p_save;             // p at the start of the running block, ghost planes included
  DevPtr<double> tol_slots;         // [halo sweeps][owned planes][tiles] per-tile residuals of the running block
  DevPtr<double> tol_send, tol_recv;   // [halo sweeps][gnz] per-plane residuals: this rank's planes / every rank's
  DevPtr<SlabTolState> tol_state;
  DevPtr<int> tol_rerun;            // [halo]: 0 for each sweep of the stopping block that runs again
  SlabInbox layout() const { return {xbuf_side, p_side, (size_t)halo * gnz}; }
};

int ipc_export(tfl_ctx* ctx, void* dev, char* out, size_t bytes) {
  cudaIpcMemHandle_t h;
  TFL_CUDA(ctx, cudaIpcGetMemHandle(&h, dev));
  memset(out, 0, bytes);
  memcpy(out, &h, sizeof(h));
  return 0;
}

int ipc_map(tfl_ctx* ctx, const char* handle, IpcPtr<float>* out, const char* who, const char* which, const char* tail) {
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, sizeof(h));
  void* q = nullptr;
  const cudaError_t e = cudaIpcOpenMemHandle(&q, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return fail(ctx, "%s: cudaIpcOpenMemHandle%s: %s%s", who, which, cudaGetErrorString(e), tail);
  }
  out->reset((float*)q);
  return 0;
}

extern "C" {

int tfl_comm_unique_id(tfl_ctx* ctx, char* id_out) {
  NcclApi* nc = nccl_api();
  if (!nc) return fail(ctx, "comm: libnccl.so.2 not found");
  static_assert(sizeof(ncclUniqueId) <= TFL_COMM_ID_BYTES, "unique id fits the ABI buffer");
  ncclUniqueId id;
  TFL_NCCL(ctx, nc->GetUniqueId(&id));
  memset(id_out, 0, TFL_COMM_ID_BYTES);
  memcpy(id_out, &id, sizeof(id));
  return 0;
}

int tfl_comm_init(tfl_ctx* ctx, const char* id_bytes, int32_t rank, int32_t world) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!ctx || world < 1 || rank < 0 || rank >= world) return fail(ctx, "comm_init: bad rank / world");
  tfl_comm_destroy(ctx);
  ctx->comm_rank = rank;
  ctx->comm_world = world;
  if (world == 1 || !id_bytes) return 0;       // nil id: a rank's workload without its neighbours (profiling)
  NcclApi* nc = nccl_api();
  if (!nc) return fail(ctx, "comm_init: libnccl.so.2 not found");
  ncclUniqueId id;
  memcpy(&id, id_bytes, sizeof(id));
  TFL_NCCL(ctx, nc->CommInitRank(&ctx->comm, world, id, rank));
  return 0;
}

int tfl_comm_destroy(tfl_ctx* ctx) {
  if (ctx && ctx->comm) {
    DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
    cudaStreamSynchronize(ctx->stream);
    nccl_api()->CommDestroy(ctx->comm);
    ctx->comm = nullptr;
  }
  if (ctx) { ctx->comm_rank = 0; ctx->comm_world = 1; }
  return 0;
}

void tfl_slab_sim_destroy(tfl_ctx* ctx, tfl_slab_sim* s) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (s && ctx) cudaStreamSynchronize(ctx->stream);
  delete s;
}

// All host arrays are GLOBAL [c][gnz][ny][nx] fields, identical on every rank; each rank keeps its slab.
int tfl_slab_sim_create(tfl_ctx* ctx, int32_t gnz, int32_t ny, int32_t nx, int32_t margin, const float* flags,
                        const float* U_bc, const float* U_bc_inv, const float* d_bc, const float* d_bc_inv,
                        tfl_slab_sim** out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!out || !flags || gnz < 3 || ny < 3 || nx < 3 || margin < 2) return fail(ctx, "slab_sim: bad arguments (margin >= 2)");
  std::unique_ptr<tfl_slab_sim> s(new tfl_slab_sim());
  memset(&s->st, 0, sizeof(s->st));
  s->gnz = gnz; s->ny = ny; s->nx = nx; s->margin = margin; s->halo = 2 * margin + 2;
  s->rank = ctx->comm_rank; s->world = ctx->comm_world;
  const int base = gnz / s->world;
  if (s->world > 1 && base < s->halo) return fail(ctx, "slab_sim: slabs of %d planes are thinner than the halo (%d)", base, s->halo);
  slab_planes(gnz, s->world, s->rank, &s->z0, &s->z1);
  s->lo_halo = std::min(s->halo, s->z0);
  s->hi_halo = std::min(s->halo, gnz - s->z1);
  s->zoff = s->z0 - s->lo_halo;
  s->nz = (s->z1 - s->z0) + s->lo_halo + s->hi_halo;
  s->own_lo = s->lo_halo;
  s->own_hi = s->lo_halo + (s->z1 - s->z0);
  s->plane = (size_t)ny * nx;
  s->cells = s->plane * s->nz;
  const size_t gcells = s->plane * gnz;
  s->xbuf_side = (size_t)s->halo * s->plane * 4;          // the widest exchange: halo planes of 4 channels
  s->p_side = (size_t)s->halo * s->plane;
  // d <- this rank's planes of the GLOBAL host field (zeros without one) of nc channels; g views it
  auto mk = [&](DevPtr<float>& d, tfl_grid* g, int nc, const float* host) {
    d = host ? dev_alloc<float>(s->cells * nc) : dev_zeros<float>(s->cells * nc);
    for (int c = 0; host && d && c < nc; c++)
      if (cudaMemcpy(d.get() + c * s->cells, host + c * gcells + (size_t)s->zoff * s->plane, s->cells * 4,
                     cudaMemcpyHostToDevice) != cudaSuccess)
        d.reset();
    *g = {d.get(), 1, nc, s->nz, ny, nx};
    return d != nullptr;
  };
  tfl_state& st = s->st;
  constexpr char kFailed[] = "slab_sim: allocation failed";
  if (!mk(s->flags, &st.flags, 1, flags) || !mk(s->p, &st.p, 1, nullptr) || !mk(s->U, &st.U, 3, nullptr) ||
      !mk(s->density, &st.density, 1, nullptr) ||
      (U_bc && U_bc_inv && (!mk(s->U_bc, &st.U_bc, 3, U_bc) || !mk(s->U_bc_inv, &st.U_bc_inv_mask, 3, U_bc_inv))) ||
      (d_bc && d_bc_inv && (!mk(s->d_bc, &st.density_bc, 1, d_bc) || !mk(s->d_bc_inv, &st.density_bc_inv_mask, 1, d_bc_inv))))
    return fail(ctx, kFailed);
  if (!(s->U1 = dev_alloc<float>(s->cells * 3)) || !(s->sums = dev_alloc<double>(2)) ||
      !(s->xbuf = dev_alloc<float>(4 * s->xbuf_side)) || !(s->div = dev_alloc<float>(s->cells)) ||
      !(s->p2 = dev_alloc<float>(s->cells)) || !(s->mask = dev_alloc<unsigned char>(s->cells)))
    return fail(ctx, kFailed);
  if (s->world > 1 &&
      (!(s->inbox = dev_zeros<float>(s->layout().floats())) ||
       !(s->push_done = dev_zeros<unsigned int>(1)) || !(s->seq = dev_zeros<unsigned int>(6))))
    return fail(ctx, kFailed);
  for (auto& pr : s->ev)
    for (EventPtr& e : pr)
      if (!(e = new_event(cudaEventDefault))) return fail(ctx, kFailed);
  *out = s.release();
  return 0;
}

// info: zoff, nz, own_lo, own_hi, z0, z1 (local storage and owned planes of this rank)
int tfl_slab_sim_layout(const tfl_slab_sim* s, tfl_state* state_out, int32_t info[6]) {
  if (!s) return 1;
  if (state_out) *state_out = s->st;
  if (info) { info[0] = s->zoff; info[1] = s->nz; info[2] = s->own_lo; info[3] = s->own_hi; info[4] = s->z0; info[5] = s->z1; }
  return 0;
}

// GLOBAL host arrays -> this rank's slab (ghost planes included); any pointer may be NULL.
int tfl_slab_sim_upload(tfl_ctx* ctx, tfl_slab_sim* s, const float* p, const float* U, const float* density) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!s) return fail(ctx, "slab_sim is nil");
  const size_t gcells = s->plane * s->gnz, off = (size_t)s->zoff * s->plane;
  TFL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (p) TFL_CUDA(ctx, cudaMemcpy(s->st.p.data, p + off, s->cells * 4, cudaMemcpyHostToDevice));
  if (density) TFL_CUDA(ctx, cudaMemcpy(s->st.density.data, density + off, s->cells * 4, cudaMemcpyHostToDevice));
  if (U) for (int c = 0; c < 3; c++)
    TFL_CUDA(ctx, cudaMemcpy(s->st.U.data + c * s->cells, U + c * gcells + off, s->cells * 4, cudaMemcpyHostToDevice));
  return 0;
}

// This rank's OWNED planes -> the same planes of GLOBAL host arrays (the rest is left alone).
int tfl_slab_sim_download(tfl_ctx* ctx, tfl_slab_sim* s, float* p, float* U, float* density) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!s) return fail(ctx, "slab_sim is nil");
  const size_t gcells = s->plane * s->gnz, goff = (size_t)s->z0 * s->plane, loff = (size_t)s->own_lo * s->plane;
  const size_t cnt = (size_t)(s->z1 - s->z0) * s->plane * 4;
  TFL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (p) TFL_CUDA(ctx, cudaMemcpy(p + goff, s->st.p.data + loff, cnt, cudaMemcpyDeviceToHost));
  if (density) TFL_CUDA(ctx, cudaMemcpy(density + goff, s->st.density.data + loff, cnt, cudaMemcpyDeviceToHost));
  if (U) for (int c = 0; c < 3; c++)
    TFL_CUDA(ctx, cudaMemcpy(U + c * gcells + goff, s->st.U.data + c * s->cells + loff, cnt, cudaMemcpyDeviceToHost));
  return 0;
}

}  // extern "C"

namespace {

// Gather / scatter of the planes one halo exchange moves: every channel of the listed fields, `cnt` floats per
// channel and side, to / from one contiguous buffer per neighbour (one NCCL message per neighbour and direction
// instead of one per channel: 4 p2p operations in the group instead of 16).
struct SlabPack {
  float* chan[8];
  int nchan;
  long long cnt;                    // floats per channel and side = width * ny * nx
  long long src_lo, src_hi;         // float offset (within a channel) of the planes sent down / up
  long long dst_lo, dst_hi;         // ... of the ghost planes filled from below / above
  float* send_lo; float* send_hi; float* recv_lo; float* recv_hi;     // null: no neighbour on that side
  // Grid-stride walk over both sides' messages: float r of side `side`'s message is float e of channel c's planes.
  template <typename F> __device__ __forceinline__ void walk(F f) const {
    const long long per_side = cnt * nchan;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < 2 * per_side; t += (long long)gridDim.x * blockDim.x) {
      const int side = t >= per_side;
      const long long r = t - side * per_side;
      const int c = (int)(r / cnt);
      f(side, r, c, r - c * cnt);
    }
  }
  // The planes sent down / up -> the messages to the lower / upper neighbour (null: none).
  __device__ __forceinline__ void gather(float* lo, float* hi) const {
    walk([&](int side, long long r, int c, long long e) {
      float* buf = side ? hi : lo;
      if (buf) buf[r] = chan[c][(side ? src_hi : src_lo) + e];
    });
  }
  // The messages from below / above (null: none) -> the ghost planes; CG loads past L1 (a peer's remote stores).
  template <bool CG> __device__ __forceinline__ void scatter(const float* lo, const float* hi) const {
    walk([&](int side, long long r, int c, long long e) {
      const float* buf = side ? hi : lo;
      if (buf) chan[c][(side ? dst_hi : dst_lo) + e] = CG ? __ldcg(buf + r) : buf[r];
    });
  }
};
template <bool UNPACK>
__global__ void k_slab_pack(SlabPack d) {
  if (!UNPACK) d.gather(d.send_lo, d.send_hi);
  else d.scatter<false>(d.recv_lo, d.recv_hi);
}

// The sequence number of one peer-memory exchange, read on the device.  word[0] is the number of the sequence's last
// exchange.  The push takes word[0] + advance (advance 1: a new number -- the step's first halo exchange, every p
// exchange; 0: the step's later halos) and leaves it in word[1]; the pull takes word[1] and commits it to word[0].
// Every CTA reads the word the kernel does not write and writes the same value, so neither kernel races with itself,
// and stream order carries the number from push to pull and on to the next exchange.  The message and counter of
// parity 1 lie buf_stride floats / flag_stride words past parity 0's (both 0 for the halos' single slot).
// gate (the tolerance solve's p exchanges): unless null, the exchange runs only while *gate == run_if; otherwise both
// kernels return at once on every rank alike and leave the words as they are.
struct SlabSeq {
  unsigned int* word;
  unsigned int advance;
  long long buf_stride;
  int flag_stride;
  const int* gate = nullptr;
  int run_if = 0;
  template <typename T> __device__ __forceinline__ T* at(T* p0, unsigned int seq, long long stride) const {
    return p0 ? p0 + (seq & 1u) * stride : nullptr;
  }
  __device__ __forceinline__ bool skipped() const { return gate && __ldcg(gate) != run_if; }
};

// Peer-memory exchange, sending half: every channel's boundary planes are written straight into the neighbours'
// inboxes (remote stores over NVLink), then the last CTA publishes the sequence number in the neighbours' counters.
// The buffers and counters are given for parity 0.
__global__ void k_slab_push(SlabPack d, float* peer_lo_buf, float* peer_hi_buf, unsigned int* peer_lo_flag,
                            unsigned int* peer_hi_flag, SlabSeq q, unsigned int* done) {
  if (q.skipped()) return;
  const unsigned int seq = q.word[0] + q.advance;
  if (threadIdx.x == 0) q.word[1] = seq;
  d.gather(q.at(peer_lo_buf, seq, q.buf_stride), q.at(peer_hi_buf, seq, q.buf_stride));
  last_cta_publish(done, gridDim.x, threadIdx.x == 0, q.at(peer_lo_flag, seq, q.flag_stride),
                   q.at(peer_hi_flag, seq, q.flag_stride), seq);
}
// ... receiving half: wait until the neighbours' counters have reached the push's number, then scatter the inbox into
// the ghost planes.  A neighbour that never arrives raises the fault counter, and nothing is scattered.
__global__ void k_slab_pull(SlabPack d, const float* buf_lo, const float* buf_hi, const unsigned int* flag_lo,
                            const unsigned int* flag_hi, SlabSeq q, unsigned long long* faults) {
  __shared__ int ok;
  if (q.skipped()) return;
  const unsigned int seq = q.word[1];
  if (threadIdx.x == 0) {
    q.word[0] = seq;
    ok = 1;
    const long long t0 = clock64();
    for (int sde = 0; sde < 2; sde++) {
      const unsigned int* f = q.at(sde ? flag_hi : flag_lo, seq, q.flag_stride);
      if (f && !wait_seq(f, seq, t0, 200)) ok = 0;
    }
    if (!ok && blockIdx.x == 0 && faults) atomicAdd(faults, 1ULL);
  }
  __syncthreads();
  if (!ok) return;
  d.scatter<true>(q.at(buf_lo, seq, q.buf_stride), q.at(buf_hi, seq, q.buf_stride));
}

// All-reduce of the two partial sums over peer memory: every rank stores its pair into slot [parity][rank] of every
// rank's inbox and raises that rank's counter [parity][rank]; then waits for all counters of its own inbox and adds
// the pairs in rank order (the same order on every rank: identical results everywhere, independent of timing).
// `step_word` is the step number's word[0] (SlabSeq), which the step's halo exchanges have already advanced.
__global__ void k_sum_push(const double* __restrict__ mine, float* const* __restrict__ inboxes, SlabInbox box, int rank,
                           int world, const unsigned int* step_word) {
  const int t = threadIdx.x;
  if (t >= world) return;
  const unsigned int step = *step_word;
  const int parity = step & 1;
  double* slot = box.sum_slot(inboxes[t], parity, rank);
  slot[0] = mine[0];
  slot[1] = mine[1];
  publish_seq(box.sum_flag(inboxes[t], parity, rank), step);
}
__global__ void k_sum_pull(double* __restrict__ out, float* inbox, SlabInbox box, int world,
                           const unsigned int* step_word, unsigned long long* faults) {
  __shared__ int ok;
  const unsigned int step = *step_word;
  const int t = threadIdx.x, parity = step & 1;
  if (t == 0) ok = 1;
  __syncthreads();
  if (t < world) {
    const long long t0 = clock64();
    if (!wait_seq(box.sum_flag(inbox, parity, t), step, t0, 100)) ok = 0;
  }
  __syncthreads();
  if (t == 0) {
    if (!ok) { if (faults) atomicAdd(faults, 1ULL); return; }
    double s0 = 0.0, s1 = 0.0;
    for (int r = 0; r < world; r++) {
      const volatile double* slot = box.sum_slot(inbox, parity, r);
      s0 += slot[0];
      s1 += slot[1];
    }
    out[0] = s0;
    out[1] = s1;
  }
}

// ---- Jacobi to a tolerance on z-slabs (slab_jacobi_tol) ----
// dst <- src (n floats) while *gate == run_if.
__global__ void k_slab_gated_copy(float* __restrict__ dst, const float* __restrict__ src, long long n, const int* gate,
                                  int run_if) {
  if (__ldcg(gate) != run_if) return;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    dst[i] = src[i];
}

// Gather, sending half: the block's per-tile residuals (k sweeps x nown owned planes x `tiles`) added tile by tile into
// one double per sweep and plane, stored at [sweep][z0 + plane] of `local` (one rank, NCCL) or of the r area of every
// rank's inbox (peer memory: then every rank's counter [parity][rank] takes the r sequence's next number).
__global__ void k_tol_push(const double* __restrict__ slots, int k, int nown, int tiles, int z0, int gnz,
                           double* local, float* const* __restrict__ inboxes, SlabInbox box, int rank, int world,
                           unsigned int* rword, const int* done) {
  if (__ldcg(done)) return;
  const unsigned int seq = inboxes ? rword[0] + 1 : 0u;
  if (inboxes && threadIdx.x == 0) rword[1] = seq;
  for (int e = threadIdx.x; e < k * nown; e += blockDim.x) {
    const int sw = e / nown;
    const double* sl = slots + (size_t)e * tiles;
    double v = 0.0;
    for (int t = 0; t < tiles; t++) v += sl[t];
    const size_t at = (size_t)sw * gnz + z0 + (e - sw * nown);
    if (!inboxes) local[at] = v;
    else for (int r = 0; r < world; r++) box.r_buf(inboxes[r], seq & 1)[at] = v;
  }
  if (!inboxes) return;
  __threadfence_system();
  __syncthreads();
  if ((int)threadIdx.x < world) store_release_sys(box.r_flag(inboxes[threadIdx.x], seq & 1, rank), seq);
}

// Gather, receiving half, and the stop decision of one block of k sweeps: wait for every rank's residuals (peer
// memory), add the planes of each sweep in ascending global z from zero, then apply the whole-grid loop's test in
// sweep order to global sweep blk * kb + s.  Every rank adds the same doubles in the same order and so decides alike.
// A stop records where p is (SlabTolState) and arms the rerun of the kept sweeps when it fell inside the block.  In a
// graph the WHILE node over the middle blocks runs again while the solve goes on and a middle block is left.
__global__ void k_tol_decide(const double* local, float* inbox, SlabInbox box, int world, unsigned int* rword,
                             SlabTolState* st, int* rerun, float tol, int max_iter, int kb, int k, int nblk,
                             int fix_at_end, int gnz, cudaGraphConditionalHandle loop, int has_loop,
                             unsigned long long* faults) {
  extern __shared__ double res2[];
  __shared__ int ok;
  if (__ldcg(&st->done)) return;
  const int t = threadIdx.x;
  const volatile double* vec = local;
  if (inbox) {
    const unsigned int seq = rword[1];
    if (t == 0) ok = 1;
    __syncthreads();
    if (t == 0) rword[0] = seq;
    if (t < world && !wait_seq(box.r_flag(inbox, seq & 1, t), seq, clock64(), 100)) ok = 0;
    __syncthreads();
    if (!ok) {                       // a rank that never arrived: stop here, counted as a fault
      if (t == 0) {
        if (faults) atomicAdd(faults, 1ULL);
        st->done = 1;
        if (has_loop) cudaGraphSetConditional(loop, 0u);
      }
      return;
    }
    vec = box.r_buf(inbox, seq & 1);
  }
  for (int sw = t; sw < k; sw += blockDim.x) {
    double v = 0.0;
    for (int z = 0; z < gnz; z++) v += vec[(size_t)sw * gnz + z];
    res2[sw] = v;
  }
  __syncthreads();
  if (t != 0) return;
  const int b = st->blk;
  int stop = -1, iter = 0;
  float res = 0.0f;
  for (int sw = 0; sw < k && stop < 0; sw++) {
    res = (float)sqrt(res2[sw]);
    if (jacobi_stops(res, tol, b * kb + sw, max_iter, &iter)) stop = sw;
  }
  st->iter = iter;
  st->res = res;
  st->blk = b + 1;
  if (stop >= 0) {
    const int keep = stop + 1;
    st->stop_blk = b;
    st->rollback = keep < k;
    st->odd = keep & 1;
    st->fix = fix_at_end && keep == k;
    if (keep < k)
      for (int i = 0; i < keep; i++) rerun[i] = 0;
    st->done = 1;
  }
  if (has_loop) cudaGraphSetConditional(loop, stop < 0 && b + 1 < nblk - 1 ? 1u : 0u);
}

// The Jacobi p exchange: several per step, so its inbox slots alternate with the parity of a sequence number (a rank
// may push exchange e + 1 while its neighbour still scatters exchange e; it cannot push e + 2 before the neighbour
// has pushed e + 1, which that neighbour does after scattering e).
constexpr int kPhaseP = 4;

// Records one of the step's statistics events; while a step is captured (tfl_slab_graph_create) it becomes an
// event-record node, so that the statistics after a replay time the replayed exchanges.
int slab_event(tfl_ctx* ctx, const tfl_slab_sim* s, const EventPtr& e) {
  TFL_CUDA(ctx, cudaEventRecordWithFlags(e.get(), ctx->stream, s->capturing ? cudaEventRecordExternal : cudaEventRecordDefault));
  return 0;
}

// Refresh `width` ghost planes on both sides of the listed fields from the neighbours' owned planes.
// gate / run_if (p exchanges of the tolerance solve, SlabSeq): the peer-memory kernels run only while *gate == run_if;
// such an exchange records no events and is not counted here (tfl_slab_sim_jacobi_stats counts it from the device).
// NCCL exchanges cannot be gated: the caller enqueues them only when they run.
int slab_exchange(tfl_ctx* ctx, tfl_slab_sim* s, std::initializer_list<const tfl_grid*> fields, int width, int phase,
                  const int* gate = nullptr, int run_if = 0) {
  const bool pph = phase == kPhaseP, counted = !gate;
  if (!pph) {
    if (slab_event(ctx, s, s->ev[phase][0])) return 1;
    s->bytes_sent[phase] = 0;
  }
  if (s->world > 1 && width > 0 && (ctx->comm || s->peer_ok)) {
    if (width > s->halo) return fail(ctx, "slab exchange of %d planes exceeds the halo (%d)", width, s->halo);
    if (pph && counted) {
      while ((int)s->jev.size() < 2 * (s->jx + 1)) {
        cudaEvent_t e = nullptr;
        TFL_CUDA(ctx, cudaEventCreate(&e));
        s->jev.emplace_back(e);
      }
      if (slab_event(ctx, s, s->jev[2 * s->jx])) return 1;
    }
    SlabPack d;
    d.nchan = 0;
    for (const tfl_grid* f : fields)
      for (int c = 0; c < f->nc && d.nchan < 8; c++) d.chan[d.nchan++] = f->data + (size_t)c * s->cells;
    d.cnt = (long long)width * s->plane;
    d.src_lo = (long long)s->own_lo * s->plane;
    d.src_hi = (long long)(s->own_hi - width) * s->plane;
    d.dst_lo = (long long)(s->own_lo - width) * s->plane;
    d.dst_hi = (long long)s->own_hi * s->plane;
    const size_t side = (size_t)d.cnt * d.nchan;                  // floats per message
    if (side > s->xbuf_side || (pph && side > s->p_side)) return fail(ctx, "slab exchange buffer too small");
    size_t sent = 0;
    const bool lo = s->rank > 0, hi = s->rank < s->world - 1;
    const int blocks = (int)std::min<size_t>((2 * side + 255) / 256, 132 * 4);
    if (s->peer_ok) {
      const SlabInbox box = s->layout();
      // the step's first halo exchange takes the next step number, every p exchange the next p sequence number
      const SlabSeq q = pph ? SlabSeq{s->seq.get() + 2, 1u, 2 * (long long)s->p_side, 2, gate, run_if}
                            : SlabSeq{s->seq.get(), phase == 0 ? 1u : 0u, 0, 0};
      auto buf = [&](float* base, int from) { return pph ? box.p_buf(base, 0, from) : box.halo(base, phase, from); };
      auto flag = [&](float* base, int from) { return pph ? box.p_flag(base, 0, from) : box.halo_flag(base, phase, from); };
      d.send_lo = d.send_hi = d.recv_lo = d.recv_hi = nullptr;
      // my first owned planes land in the lower neighbour's "from above" slot, my last ones in the upper neighbour's "from below"
      k_slab_push<<<blocks, 256, 0, ctx->stream>>>(d, lo ? buf(s->peer_inbox[0], 1) : nullptr, hi ? buf(s->peer_inbox[1], 0) : nullptr,
                                                   lo ? flag(s->peer_inbox[0], 1) : nullptr, hi ? flag(s->peer_inbox[1], 0) : nullptr,
                                                   q, s->push_done.get());
      float* inbox = s->inbox.get();
      k_slab_pull<<<blocks, 256, 0, ctx->stream>>>(d, lo ? buf(inbox, 0) : nullptr, hi ? buf(inbox, 1) : nullptr,
                                                   lo ? flag(inbox, 0) : nullptr, hi ? flag(inbox, 1) : nullptr,
                                                   q, ctx->counters.get());
      sent = (size_t)(lo + hi) * side * 4;
      ctx->launches += 2;
    } else {
      NcclApi* nc = nccl_api();
      float* xbuf = s->xbuf.get();
      d.send_lo = lo ? xbuf : nullptr;
      d.send_hi = hi ? xbuf + s->xbuf_side : nullptr;
      d.recv_lo = lo ? xbuf + 2 * s->xbuf_side : nullptr;
      d.recv_hi = hi ? xbuf + 3 * s->xbuf_side : nullptr;
      k_slab_pack<false><<<blocks, 256, 0, ctx->stream>>>(d);
      TFL_NCCL(ctx, nc->GroupStart());
      if (lo) {                                       // lower neighbour: my first owned planes go down
        TFL_NCCL(ctx, nc->Send(d.send_lo, side, ncclFloat, s->rank - 1, ctx->comm, ctx->stream));
        TFL_NCCL(ctx, nc->Recv(d.recv_lo, side, ncclFloat, s->rank - 1, ctx->comm, ctx->stream));
        sent += side * 4;
      }
      if (hi) {                                       // upper neighbour
        TFL_NCCL(ctx, nc->Send(d.send_hi, side, ncclFloat, s->rank + 1, ctx->comm, ctx->stream));
        TFL_NCCL(ctx, nc->Recv(d.recv_hi, side, ncclFloat, s->rank + 1, ctx->comm, ctx->stream));
        sent += side * 4;
      }
      TFL_NCCL(ctx, nc->GroupEnd());
      k_slab_pack<true><<<blocks, 256, 0, ctx->stream>>>(d);
      ctx->launches += 2;
    }
    if (pph) {
      if (!counted) return 0;
      if (slab_event(ctx, s, s->jev[2 * s->jx + 1])) return 1;
      s->jx += 1;
      s->jbytes += sent;
      return 0;
    }
    s->bytes_sent[phase] = sent;
  }
  return pph ? 0 : slab_event(ctx, s, s->ev[phase][1]);
}

struct SlabScope {       // slab placement of the context for the enclosed calls
  tfl_ctx* ctx;
  SlabScope(tfl_ctx* c, const tfl_slab_sim* s, int zlo, int zhi) : ctx(c) {
    c->slab = true; c->zoff = s->zoff; c->gnz = s->gnz; c->zlo = zlo; c->zhi = zhi; c->slab_margin = s->margin;
  }
  ~SlabScope() { ctx->slab = false; ctx->slab_margin = 2; }
};

// The Jacobi solve to s->p_tol on this rank's slab, from p = p2 = 0 on a prepared divergence and mask (`planes` and `g`
// of slab_jacobi_projection); leaves the whole-grid loop's final iterate in p on the owned planes and the plane below.
// Blocks of `halo` sweeps (the schedule's at world > 1, without its closing 1-plane exchange; at one rank the same
// lengths over the whole slab), each one:
//   p exchange (gated on done)  ->  p_save <- p  ->  per sweep: the gated sweep and its per-plane residual
//   ->  k_tol_push (+ the NCCL all-reduce)  ->  k_tol_decide
// Every block starts on p (halo is even).  A direct step enqueues 1, 2, 4 .. 32 blocks at a time and reads done after
// each chunk (one block at a time over NCCL, whose exchanges cannot be gated); a captured one is block 0, one WHILE
// node over the middle blocks and the last block.  Then, gated by the decision: p <- p_save and the stopping block's
// kept sweeps again (on the widest block range, which keeps the owned planes and the plane below right for every
// block), p <- p2 when the result lies there, and the 1-plane p exchange when the stop left p stale below the owned
// planes.
int slab_jacobi_tol(tfl_ctx* ctx, tfl_slab_sim* s, int iters, const int32_t planes[3], const Geo& g) {
  struct Blk { int k, w, z_lo, z_hi, shr_lo, shr_hi, fix_at_end; };
  std::vector<Blk> blocks;
  const int kb = s->halo;
  if (s->world == 1) {
    for (int b0 = 0; b0 < iters; b0 += kb) blocks.push_back({std::min(kb, iters - b0), 0, 0, s->nz, 0, 0, 0});
  } else {
    const int nsched = (int)(s->jsched.size() / TFL_JACOBI_BLOCK_INTS);
    for (int b = 0; b < nsched; b++) {
      const int32_t* o = s->jsched.data() + (size_t)b * TFL_JACOBI_BLOCK_INTS;
      if (o[0] > 0) blocks.push_back({o[0], o[1], o[2], o[3], o[4], o[5], b + 1 < nsched ? 1 : 0});
    }
  }
  const int nblk = (int)blocks.size();
  s->tol_widths.clear();
  int kmax = 0;
  for (const Blk& o : blocks) {
    s->tol_widths.push_back(o.w);
    kmax = std::max(kmax, o.k);
  }
  const tfl_state& st = s->st;
  float* p = st.p.data;
  float* p2 = s->p2.get();
  const unsigned char* mask = s->mask.get();
  const float* div = s->div.get();
  SlabTolState* S = s->tol_state.get();
  const int* done = &S->done;
  const int nown = s->z1 - s->z0, tiles = jacobi_plane_tiles(s->nx, s->ny);
  const bool peer = s->world > 1 && s->peer_ok && s->all_inbox_dev, nccl = s->world > 1 && !peer && ctx->comm;
  const unsigned copy_blocks = (unsigned)std::min<size_t>((s->cells + 1023) / 1024, 1184);
  const SlabInbox box = s->layout();
  TFL_CUDA(ctx, cudaMemsetAsync(S, 0, sizeof(SlabTolState), ctx->stream));
  TFL_CUDA(ctx, cudaMemsetAsync(s->tol_rerun.get(), 1, sizeof(int) * kb, ctx->stream));     // nonzero: skipped
  auto block = [&](const Blk& o, cudaGraphConditionalHandle loop, int has_loop) -> int {
    cudaStream_t q = ctx->stream;
    if (o.w > 0 && slab_exchange(ctx, s, {&st.p}, o.w, kPhaseP, done, 0)) return 1;
    // where the fixed count takes the cooperative block kernel, so does the tolerance: one launch that also saves the
    // block's start and leaves the per-plane residuals; elsewhere the copy, then a sweep and a residual pass per sweep
    JacobiTolArgs t;
    t.slots = s->tol_slots.get();
    t.gate = done;
    t.save = s->p_save.get();
    t.own_lo = s->own_lo;
    t.own_hi = s->own_hi;
    if (launch_jacobi_block_planes(mask, div, p, p2, g, o.z_lo, o.z_hi, o.shr_lo, o.shr_hi, o.k, t, q)) {
      ctx->launches += 1;
    } else {
      k_slab_gated_copy<<<copy_blocks, 256, 0, q>>>(s->p_save.get(), p, (long long)s->cells, done, 0);
      for (int sw = 0; sw < o.k; sw++) {
        Geo gs = g;
        gs.zlo = o.z_lo + sw * o.shr_lo;
        gs.zhi = o.z_hi - sw * o.shr_hi;
        float* prev = (sw & 1) ? p2 : p;
        float* cur = (sw & 1) ? p : p2;
        launch_jacobi_iter(mask, div, prev, cur, gs, q, done);
        launch_jacobi_plane_residual(cur, prev, s->nx, s->ny, s->own_lo, nown,
                                     s->tol_slots.get() + (size_t)sw * nown * tiles, done, q);
      }
      ctx->launches += 2 * o.k + 1;
    }
    k_tol_push<<<1, 256, 0, q>>>(s->tol_slots.get(), o.k, nown, tiles, s->z0, s->gnz, s->tol_send.get(),
                                 peer ? s->all_inbox_dev.get() : nullptr, box, s->rank, s->world, s->seq.get() + 4, done);
    if (nccl)
      TFL_NCCL(ctx, nccl_api()->AllReduce(s->tol_send.get(), s->tol_recv.get(), (size_t)kb * s->gnz, ncclDouble,
                                          ncclSum, ctx->comm, q));
    k_tol_decide<<<1, 256, sizeof(double) * kb, q>>>(nccl ? s->tol_recv.get() : s->tol_send.get(),
                                                      peer ? s->inbox.get() : nullptr, box, s->world, s->seq.get() + 4,
                                                      S, s->tol_rerun.get(), s->p_tol, iters, kb, o.k, nblk,
                                                      o.fix_at_end, s->gnz, loop, has_loop, ctx->counters.get());
    ctx->launches += 2;
    return 0;
  };
  if (s->capturing) {
    const int has_loop = nblk >= 3;             // the middle blocks are alike: the WHILE node's body is one of them
    cudaGraphConditionalHandle loop = 0;
    if (has_loop) TFL_CUDA(ctx, capture_while_handle(ctx->stream, 0, &loop));
    if (block(blocks[0], loop, has_loop)) return 1;
    if (has_loop) {
      // the body block enqueues on ctx->stream, slab_exchange included
      cudaStream_t main = ctx->stream;
      int rc = 0;
      const cudaError_t loop_capture = capture_while(main, loop, ctx->loop_body.get(), [&](cudaStream_t bs) {
        ctx->stream = bs;
        rc = block(blocks[1], loop, 1);
        ctx->stream = main;
        return rc ? cudaErrorUnknown : cudaSuccess;     // ctx->err names a failed block
      });
      if (rc) return 1;
      TFL_CUDA(ctx, loop_capture);
    }
    if (nblk >= 2 && block(blocks[nblk - 1], loop, has_loop)) return 1;
  } else {
    if (run_until_done(ctx, "slab_sim_step", done, nblk, 1, nccl ? 1 : 32, [&](int b0, int n) {
          for (int b = b0; b < b0 + n; b++)
            if (block(blocks[b], 0, 0)) return 1;
          return 0;
        }))
      return 1;
  }
  // the stopping block again from its start, up to its stopping sweep
  k_slab_gated_copy<<<copy_blocks, 256, 0, ctx->stream>>>(p, s->p_save.get(), (long long)s->cells, &S->rollback, 1);
  const int lo = s->rank > 0, hi = s->rank < s->world - 1;
  for (int sw = 0; sw + 1 < kmax; sw++) {
    Geo gs = g;
    gs.zlo = planes[0] + sw * lo;
    gs.zhi = planes[1] - sw * hi;
    launch_jacobi_iter(mask, div, (sw & 1) ? p2 : p, (sw & 1) ? p : p2, gs, ctx->stream, s->tol_rerun.get() + sw);
  }
  k_slab_gated_copy<<<copy_blocks, 256, 0, ctx->stream>>>(p, p2, (long long)s->cells, &S->odd, 1);
  ctx->launches += kmax + 1;
  if (peer) return slab_exchange(ctx, s, {&st.p}, 1, kPhaseP, &S->fix, 1);
  if (nccl) {                                   // direct only (NCCL is not captured): the host learns the stop
    SlabTolState h;
    TFL_CUDA(ctx, cudaMemcpyAsync(&h, S, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
    TFL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (h.fix) return slab_exchange(ctx, s, {&st.p}, 1, kPhaseP, &S->fix, 1);
  }
  return 0;
}

// lib/simulate.lua:275-303 on this rank's slab: divergence, `iters` Jacobi sweeps from p = 0 in the blocks of
// tfl_slab_jacobi_schedule, velocity update on the owned planes.  Every cell sees the single-GPU sweep's operands, so
// with pTol = 0 p and U are bit-identical to tfl_simulate_step's; with a tolerance (slab_jacobi_tol) they are those of
// the whole-grid operators with tfl_solve_linear_system_jacobi_dev as the solve.
int slab_jacobi_projection(tfl_ctx* ctx, tfl_slab_sim* s, int iters) {
  const tfl_state& st = s->st;
  int32_t planes[3];
  const int nblk = tfl_slab_jacobi_schedule(s->gnz, s->world, s->rank, s->margin, iters, planes, nullptr, 0);
  if (nblk < 1) return fail(ctx, "slab_sim_step: no Jacobi schedule for this slab");
  s->jsched.resize((size_t)nblk * TFL_JACOBI_BLOCK_INTS);
  tfl_slab_jacobi_schedule(s->gnz, s->world, s->rank, s->margin, iters, planes, s->jsched.data(), nblk);
  if (slab_exchange(ctx, s, {&st.U}, planes[2], 2)) return 1;
  if (slab_event(ctx, s, s->ev[3][0]) || slab_event(ctx, s, s->ev[3][1])) return 1;   // no all-reduce on this path
  tfl_grid dv = st.p;
  dv.data = s->div.get();
  Geo g;
  {
    SlabScope scope(ctx, s, planes[0], planes[1]);
    if (tfl_velocity_divergence_forward(ctx, &st.U, &st.flags, &dv)) return 1;
    if (make_geo(ctx, &st.flags, 1, &g)) return 1;
    launch_jacobi_mask(st.flags.data, s->mask.get(), g, ctx->stream);
    ctx->launches += 1;
  }
  TFL_CUDA(ctx, cudaMemsetAsync(st.p.data, 0, s->cells * 4, ctx->stream));   // generic/tfluids.cu:1854-1855
  TFL_CUDA(ctx, cudaMemsetAsync(s->p2.get(), 0, s->cells * 4, ctx->stream));
  s->jx = 0;
  s->jbytes = 0;
  s->tol_last = s->p_tol > 0.0f;
  if (s->tol_last) {
    if (slab_jacobi_tol(ctx, s, iters, planes, g)) return 1;
  } else {
    float* buf[2] = {st.p.data, s->p2.get()};
    int done = 0;
    for (int b = 0; b < nblk; b++) {
      const int32_t* o = s->jsched.data() + (size_t)b * TFL_JACOBI_BLOCK_INTS;
      if (o[1] > 0) {
        tfl_grid pc = st.p;
        pc.data = buf[done & 1];
        if (slab_exchange(ctx, s, {&pc}, o[1], kPhaseP)) return 1;
      }
      if (run_jacobi_block(ctx, s->mask.get(), s->div.get(), buf[done & 1], buf[(done + 1) & 1], g, o[2], o[3], o[4], o[5], o[0], -1) < 0)
        return 1;
      done += o[0];
    }
    if (done & 1) TFL_CUDA(ctx, cudaMemcpyAsync(st.p.data, s->p2.get(), s->cells * 4, cudaMemcpyDeviceToDevice, ctx->stream));
  }
  if (check_launch(ctx, "slab_sim_step (jacobi)")) return 1;
  SlabScope scope(ctx, s, s->own_lo, s->own_hi);
  return tfl_velocity_update_forward(ctx, &st.U, &st.flags, &st.p);
}

}  // namespace

extern "C" {

// Sweeps per p exchange.  After an exchange of width w, p is right on owned +- w planes and sweep s (1-based) of the
// block that follows on owned +- (w - s): a block of k sweeps needs one exchange of width k, or k + 1 for the last
// block, which must leave p right on the plane below the owned ones (the velocity update reads it).  p starts at
// zero everywhere, so the first block needs no exchange.  Blocks: `halo` sweeps each, the last one the rest
// (0 .. halo - 1 sweeps; with 0 it is the 1-plane exchange alone).  One rank computes everything in one block.
int tfl_slab_jacobi_schedule(int32_t gnz, int32_t world, int32_t rank, int32_t margin, int32_t max_iter,
                             int32_t planes[3], int32_t* blocks, int32_t cap) {
  if (gnz < 3 || world < 1 || rank < 0 || rank >= world || margin < 2 || max_iter < 1) return -1;
  const int halo = 2 * margin + 2;
  if (world > 1 && gnz / world < halo) return -1;
  int z0, z1;
  slab_planes(gnz, world, rank, &z0, &z1);
  const int lo_halo = std::min(halo, z0), hi_halo = std::min(halo, gnz - z1);
  const int nz = (z1 - z0) + lo_halo + hi_halo, own_lo = lo_halo, own_hi = lo_halo + (z1 - z0);
  const bool lo = rank > 0, hi = rank < world - 1;     // sides with a neighbour: the ranges shrink there
  const int nblk = world == 1 ? 1 : (max_iter + halo) / halo;
  int wmax = 0;
  for (int b = 0; b < nblk; b++) {
    const bool last = b == nblk - 1;
    const int k = world == 1 ? max_iter : (last ? max_iter - (nblk - 1) * halo : halo);
    const int w = world == 1 ? 0 : k + (last ? 1 : 0);
    wmax = std::max(wmax, w);
    if (blocks && b < cap) {
      int32_t* o = blocks + (size_t)b * TFL_JACOBI_BLOCK_INTS;
      o[0] = k;
      o[1] = b > 0 ? w : 0;
      o[2] = lo ? own_lo - (w - 1) : 0;
      o[3] = hi ? own_hi + (w - 1) : nz;
      o[4] = lo;
      o[5] = hi;
    }
  }
  if (planes) {
    planes[0] = lo ? own_lo - (wmax - 1) : 0;
    planes[1] = hi ? own_hi + (wmax - 1) : nz;
    planes[2] = world > 1 ? wmax : 0;
  }
  return nblk;
}

// The projection network's ghost depth (cnn_slab_check): 3 s + 2 planes for the coarsest bank's scale s =
// 2^(banks_num-1), i.e. a halo 2 margin + 2 from margin = ceil(3 s / 2), and never below the single-bank minimum 2.
// 2 margin + 1 of it is the U / p exchange before the projection.
int tfl_slab_cnn_margin(int32_t banks_num) {
  if (banks_num <= 1) return 2;
  if (banks_num > kTcMaxBanks) return -1;
  return std::max(2, (3 * (1 << (banks_num - 1)) + 1) / 2);
}

int tfl_jacobi_slab_block(tfl_ctx* ctx, const tfl_grid* pa, const tfl_grid* pb, const tfl_grid* flags,
                          const tfl_grid* div, int is_3d, int32_t z_lo, int32_t z_hi, int32_t shrink_lo,
                          int32_t shrink_hi, int32_t sweeps, int32_t path, int32_t* path_out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (check_scalar(ctx, flags, "flags") || check_scalar(ctx, pa, "pa") || check_scalar(ctx, pb, "pb") ||
      check_scalar(ctx, div, "div"))
    return 1;
  if (!same_spatial(flags, pa) || !same_spatial(flags, pb) || !same_spatial(flags, div)) return fail(ctx, "size mismatch");
  if (path < -1 || path > 1 || sweeps < 0 || shrink_lo < 0 || shrink_lo > 1 || shrink_hi < 0 || shrink_hi > 1)
    return fail(ctx, "jacobi_slab_block: bad arguments");
  Geo g;
  if (make_geo(ctx, flags, is_3d, &g)) return 1;
  if (z_lo < 0 || z_hi > g.nz || z_lo >= z_hi || (sweeps > 0 && z_hi - z_lo - (sweeps - 1) * (shrink_lo + shrink_hi) < 1))
    return fail(ctx, "jacobi_slab_block: planes [%d, %d) do not hold %d sweeps", z_lo, z_hi, sweeps);
  // the stencil reads one plane beyond the range: inside the local storage unless that side is a global end
  if ((z_lo < 1 && g.zoff > 0) || (z_hi > g.nz - 1 && g.zoff + g.nz < g.gnz))
    return fail(ctx, "jacobi_slab_block: planes [%d, %d) reach past the local storage", z_lo, z_hi);
  const size_t cells = (size_t)g.n * g.nb;
  if (arena_reserve(ctx, carve_bytes({cells}))) return 1;
  Carver cv(ctx);
  unsigned char* mask = cv.take<unsigned char>(cells);
  Geo gm = g;
  gm.zlo = z_lo;
  gm.zhi = z_hi;
  launch_jacobi_mask(flags->data, mask, gm, ctx->stream);
  ctx->launches += 1;
  const int used = run_jacobi_block(ctx, mask, div->data, pa->data, pb->data, g, z_lo, z_hi, shrink_lo, shrink_hi, sweeps, path);
  if (used < 0) return fail(ctx, "jacobi_slab_block: the one-launch block does not apply (3-D, nx %% 128, ny %% 8, co-residency)");
  if (path_out) *path_out = used;
  return check_launch(ctx, "jacobi_slab_block");
}

}  // extern "C"

namespace {

// What tfl_slab_sim_step refuses, before anything is launched; the messages start with `who`.
int slab_step_refusal(tfl_ctx* ctx, const tfl_slab_sim* s, const tfl_mconf* mc, tfl_cnn* cnn, const char* who) {
  if (!s || !mc) return fail(ctx, "%s: nil argument", who);
  const bool jacobi = mc->sim_method == TFL_SIM_JACOBI;
  if (mc->sim_method == TFL_SIM_PCG)
    return fail(ctx, "%s: simMethod 'pcg' is not decomposed: the IC(0) triangular solves of its "
                     "preconditioner sweep the whole domain in order and do not shard over z-slabs", who);
  if (!jacobi && mc->sim_method != TFL_SIM_CONVNET)
    return fail(ctx, "%s: mconf.simMethod (%d) is not a valid option", who, mc->sim_method);
  if (!jacobi && !cnn) return fail(ctx, "%s: simMethod 'convnet' needs a model", who);
  if (!jacobi && cnn_slab_check(ctx, cnn, s->margin, s->gnz, s->ny, s->nx, s->zoff, s->nz, s->own_lo, s->own_hi))
    return fail(ctx, "%s: %s", who, ctx->err.c_str());
  if (jacobi && mc->max_iter < 0) return fail(ctx, "%s: At least 1 iteration is needed (maxIter < 1)", who);
  if (s->world != ctx->comm_world || s->rank != ctx->comm_rank) return fail(ctx, "%s: communicator changed", who);
  if (jacobi && s->p_tol > 0.0f) {        // the direct tolerance step reads its stop word on the host
    bool capturing = false;
    if (stream_capturing(ctx, who, &capturing)) return 1;
    if (capturing)
      return fail(ctx, "%s: the stream is being captured and a step with a Jacobi tolerance waits for its stop decision "
                       "on the host; capture it with tfl_slab_graph_create instead", who);
  }
  return 0;
}

// The step of tfl_slab_sim_step after its refusals: enqueued directly or captured (tfl_slab_graph_create).
int slab_step(tfl_ctx* ctx, tfl_slab_sim* s, const tfl_mconf* mc, tfl_cnn* cnn) {
  const bool jacobi = mc->sim_method == TFL_SIM_JACOBI;
  const tfl_state& st = s->st;
  struct StepMark {                     // the flags are refreshed once per step (the two advections share them)
    tfl_ctx* c;
    explicit StepMark(tfl_ctx* cc) : c(cc) { c->in_slab_step = true; c->fcache.fresh_for = nullptr; }
    ~StepMark() { c->in_slab_step = false; c->fcache.fresh_for = nullptr; }
  } mark_(ctx);
  auto bcs = [&]() -> int {           // on the owned planes: ghost planes are always refreshed from their owners
    SlabScope scope(ctx, s, s->own_lo, s->own_hi);
    if (st.U_bc.data && tfl_apply_bc(ctx, &st.U, &st.U_bc_inv_mask, &st.U_bc)) return 1;
    if (st.density_bc.data && tfl_apply_bc(ctx, &st.density, &st.density_bc_inv_mask, &st.density_bc)) return 1;
    return 0;
  };
  if (slab_exchange(ctx, s, {&st.U, &st.density}, s->halo, 0)) return 1;
  {
    SlabScope scope(ctx, s, s->own_lo, s->own_hi);
    if (tfl_advect_scalar(ctx, mc->dt, &st.density, &st.U, &st.flags, mc->advection_method, 0, mc->maccormack_strength, nullptr)) return 1;
    if (tfl_advect_vel(ctx, mc->dt, &st.U, &st.flags, mc->advection_method, mc->maccormack_strength, nullptr)) return 1;
  }
  if (bcs()) return 1;
  if (slab_exchange(ctx, s, {&st.U, &st.density}, 4, 1)) return 1;
  const StepForces fo = step_forces(mc, s->nx, s->ny, s->gnz);
  {
    // point-wise forces also on the three ghost planes the confinement stencil reads across the cut
    SlabScope scope(ctx, s, s->own_lo - std::min(3, s->lo_halo), s->own_hi + std::min(3, s->hi_halo));
    if (fo.buoyancy && tfl_add_buoyancy(ctx, &st.U, &st.flags, &st.density, fo.buoy, mc->dt)) return 1;
    if (fo.gravity && tfl_add_gravity(ctx, &st.U, &st.flags, fo.grav, mc->dt)) return 1;
  }
  if (fo.vorticity) {
    SlabScope scope(ctx, s, s->own_lo, s->own_hi);
    if (tfl_vorticity_confinement(ctx, &st.U, &st.flags, fo.vort_amp)) return 1;
  }
  if (jacobi) {
    {
      SlabScope scope(ctx, s, s->own_lo, s->own_hi);
      if (tfl_set_wall_bcs_forward(ctx, &st.U, &st.flags)) return 1;      // :248-251
    }
    if (bcs()) return 1;                                                   // :252
    if (slab_jacobi_projection(ctx, s, mc->max_iter > 0 ? mc->max_iter : 100)) return 1;
    if (bcs()) return 1;                                                   // :321
    SlabScope scope(ctx, s, s->own_lo, s->own_hi);
    return tfl_clamp(ctx, &st.U, -1e6f, 1e6f);
  }
  if (bcs()) return 1;
  // the network input's reach across the cut (5 planes for a single bank)
  if (slab_exchange(ctx, s, {&st.U, &st.p}, 2 * tfl_slab_cnn_margin(cnn->nbanks) + 1, 2)) return 1;
  tfl_grid u1 = st.U;
  u1.data = s->U1.get();
  double* sums = s->sums.get();
  {
    SlabScope scope(ctx, s, s->own_lo, s->own_hi);
    if (tfl_cnn_stats(ctx, &st.U, &st.flags, &u1, sums)) return 1;
  }
  if (slab_event(ctx, s, s->ev[3][0])) return 1;
  if (s->world > 1 && s->peer_ok && s->all_inbox_dev) {
    k_sum_push<<<1, kMaxRanks, 0, ctx->stream>>>(sums, s->all_inbox_dev.get(), s->layout(), s->rank, s->world, s->seq.get());
    k_sum_pull<<<1, kMaxRanks, 0, ctx->stream>>>(sums, s->inbox.get(), s->layout(), s->world, s->seq.get(), ctx->counters.get());
    ctx->launches += 2;
  } else if (s->world > 1 && ctx->comm) {
    TFL_NCCL(ctx, nccl_api()->AllReduce(sums, sums, 2, ncclDouble, ncclSum, ctx->comm, ctx->stream));
  }
  if (slab_event(ctx, s, s->ev[3][1])) return 1;
  {
    SlabScope scope(ctx, s, s->own_lo, s->own_hi);
    if (tfl_cnn_project_from_sums(ctx, cnn, &st.p, &u1, &st.flags, sums, &st.p, &st.U, mc->normalize_input_threshold)) return 1;
  }
  if (bcs()) return 1;
  SlabScope scope(ctx, s, s->own_lo, s->own_hi);
  return tfl_clamp(ctx, &st.U, -1e6f, 1e6f);
}

}  // namespace

// ---------------------------------------------------------------------------------------
// The slab step as a CUDA graph: one tfl_slab_sim_step captured on the context's stream and replayed with one launch.
// The exchanges need no host: their sequence numbers are read and advanced on the device (SlabSeq), so replays and
// direct steps interleave freely, on one rank or across ranks.  Pointers and the captured step's host-side choices
// (advection tile halo, Jacobi path and block schedule) are frozen, and the graph keeps the captured step's
// exchange statistics to hand to tfl_slab_sim_exchange_stats / _jacobi_stats after each replay; its event-record
// nodes time the replay.  Buffers the library reallocates are guarded by generation, as in tfl_step_graph.
// ---------------------------------------------------------------------------------------
struct tfl_slab_graph {
  GraphPtr graph;
  GraphExecPtr exec;
  tfl_slab_sim* sim = nullptr;
  long long launches = 0;           // kernels in one replay
  BufferGens gens;
  unsigned long long peer_gen = 0;
  size_t bytes_sent[3] = {0, 0, 0};
  int jx = 0;
  size_t jbytes = 0;
  bool jacobi = false;
  bool tol = false;                 // the captured step solves to a tolerance: its statistics come from the device
  std::vector<int> tol_widths;
};

extern "C" {

// One tfluids.simulate (lib/simulate.lua:175-327; simMethod 'convnet' or 'jacobi') on this rank's slab.  Asynchronous.
int tfl_slab_sim_step(tfl_ctx* ctx, tfl_slab_sim* s, const tfl_mconf* mc, tfl_cnn* cnn) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (slab_step_refusal(ctx, s, mc, cnn, "slab_sim_step") || slab_step(ctx, s, mc, cnn)) return 1;
  if (mc->sim_method == TFL_SIM_JACOBI && s->tol_last) s->tol_stepped = true;
  s->last.done = true;
  s->last.cnn = mc->sim_method == TFL_SIM_JACOBI ? nullptr : cnn;
  s->last.sim_method = mc->sim_method;
  s->last.gens = buffer_gens(ctx, s->last.cnn);
  return 0;
}

void tfl_slab_graph_destroy(tfl_ctx* ctx, tfl_slab_graph* g) {
  DeviceGuard guard_(ctx);
  if (g && ctx) cudaStreamSynchronize(ctx->stream);
  delete g;
}

int tfl_slab_graph_create(tfl_ctx* ctx, tfl_slab_sim* s, const tfl_mconf* mc, tfl_cnn* cnn, tfl_slab_graph** out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!out) return fail(ctx, "slab_graph: nil argument");
  if (slab_step_refusal(ctx, s, mc, cnn, "slab_graph")) return 1;
  cudaStream_t st = ctx->stream;
  if (st == nullptr || st == cudaStreamLegacy || st == cudaStreamPerThread)
    return fail(ctx, "slab_graph: the default stream cannot be captured; give the context a stream (tfl_set_stream)");
  if (s->world > 1 && !s->peer_ok)
    return fail(ctx, "slab_graph: world %d without peer memory: only peer-memory exchanges (tfl_slab_sim_ipc_connect) "
                     "and one rank are captured, not NCCL; step directly (tfl_slab_sim_step)", s->world);
  const tfl_cnn* model = mc->sim_method == TFL_SIM_JACOBI ? nullptr : cnn;
  if (!s->last.done || s->last.cnn != model || s->last.sim_method != mc->sim_method)
    return fail(ctx, "slab_graph: no earlier tfl_slab_sim_step with this sim, model and simMethod; step directly once "
                     "before capturing (the step's buffers are sized then: capturing must not allocate)");
  if (const char* what = reallocated_buffer(ctx, s->last.gens))
    return fail(ctx, "slab_graph: %s reallocated since the last tfl_slab_sim_step with this sim; step directly once "
                     "more before capturing", what);
  std::unique_ptr<tfl_slab_graph> g(new tfl_slab_graph());
  TFL_CUDA(ctx, cudaStreamSynchronize(st));
  const long long l0 = ctx->launches;
  size_t bytes_sent[3];                   // the sim's statistics stay those of its last direct step or replay
  memcpy(bytes_sent, s->bytes_sent, sizeof(bytes_sent));
  const int jx = s->jx;
  const size_t jbytes = s->jbytes;
  const bool tol_last = s->tol_last;
  const std::vector<int> tol_widths = s->tol_widths;
  if (cudaStreamBeginCapture(st, cudaStreamCaptureModeRelaxed) != cudaSuccess) {
    cudaGetLastError();
    return fail(ctx, "slab_graph: cudaStreamBeginCapture failed");
  }
  s->capturing = true;
  const int rc = slab_step(ctx, s, mc, cnn);
  s->capturing = false;
  cudaGraph_t graph = nullptr;
  const cudaError_t e = cudaStreamEndCapture(st, &graph);
  g->graph.reset(graph);
  g->launches = ctx->launches - l0;
  ctx->launches = l0;
  memcpy(g->bytes_sent, s->bytes_sent, sizeof(bytes_sent));
  g->jx = s->jx;
  g->jbytes = s->jbytes;
  g->jacobi = mc->sim_method == TFL_SIM_JACOBI;
  g->tol = g->jacobi && s->tol_last;
  g->tol_widths = s->tol_widths;
  memcpy(s->bytes_sent, bytes_sent, sizeof(bytes_sent));
  s->jx = jx;
  s->jbytes = jbytes;
  s->tol_last = tol_last;
  s->tol_widths = tol_widths;
  if (rc != 0 || e != cudaSuccess || !graph) {
    cudaGetLastError();
    const std::string why = rc != 0 ? ctx->err : std::string(cudaGetErrorString(e));
    return fail(ctx, "slab_graph: capture failed (%s)", why.c_str());
  }
  cudaGraphExec_t exec = nullptr;
  if (cudaGraphInstantiate(&exec, graph, 0) != cudaSuccess) {
    cudaGetLastError();
    return fail(ctx, "slab_graph: cudaGraphInstantiate failed");
  }
  g->exec.reset(exec);
  g->sim = s;
  g->gens = buffer_gens(ctx, model);
  g->peer_gen = s->peer_gen;
  *out = g.release();
  return 0;
}

int tfl_slab_graph_launch(tfl_ctx* ctx, tfl_slab_graph* g) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!g || !g->exec) return fail(ctx, "slab_graph is nil");
  if (const char* stale = reallocated_buffer(ctx, g->gens))
    return fail(ctx, "slab_graph: stale graph: %s reallocated since the capture (a call on another grid shape or a "
                     "larger grid); replaying would touch freed memory: capture the step again", stale);
  if (g->peer_gen != g->sim->peer_gen)
    return fail(ctx, "slab_graph: stale graph: the peers' inboxes were mapped again (tfl_slab_sim_ipc_connect) since "
                     "the capture; replaying would store into the old mappings: capture the step again");
  TFL_CUDA(ctx, cudaGraphLaunch(g->exec.get(), ctx->stream));
  ctx->launches += g->launches;
  tfl_slab_sim* s = g->sim;
  memcpy(s->bytes_sent, g->bytes_sent, sizeof(s->bytes_sent));
  s->jx = g->jx;
  s->jbytes = g->jbytes;
  if (g->jacobi) s->tol_last = g->tol;
  if (g->tol) {
    s->tol_stepped = true;
    s->tol_widths = g->tol_widths;
  }
  return 0;
}

// The step leaves the ghost planes stale; the divergence on the last owned plane reads U_z one plane above it.  So one
// plane of U_z is exchanged first -- on the p exchange's inbox area and sequence, which every rank advances alike as
// long as every rank records -- without counting in the last step's Jacobi statistics.
int tfl_slab_sim_monitor_record(tfl_ctx* ctx, tfl_slab_sim* s, tfl_monitor* mon, int64_t* index_out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!ctx) return 1;
  if (index_out) *index_out = -1;
  if (!s || !mon) return fail(ctx, "slab_sim_monitor_record: nil argument");
  if (s->world != ctx->comm_world || s->rank != ctx->comm_rank) return fail(ctx, "slab_sim_monitor_record: communicator changed");
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  TFL_CUDA(ctx, cudaStreamIsCapturing(ctx->stream, &cs));
  if (cs != cudaStreamCaptureStatusNone)        // before the exchange: a refusal enqueues nothing
    return fail(ctx, "monitor_record: the context's stream is being captured into a graph; record after the graph's launch");
  if (monitor_precheck(ctx, mon, 1, s->gnz)) return 1;
  tfl_grid uz = s->st.U;
  uz.nc = 1;
  uz.data = s->st.U.data + 2 * s->cells;
  const int jx = s->jx;
  const size_t jbytes = s->jbytes;
  if (slab_exchange(ctx, s, {&uz}, 1, kPhaseP)) return 1;
  s->jx = jx;
  s->jbytes = jbytes;
  SlabScope scope(ctx, s, s->own_lo, s->own_hi);
  return tfl_monitor_record(ctx, mon, &s->st.U, &s->st.flags, index_out);
}

// Peer-memory halos: export this rank's inbox (64-byte CUDA IPC handle) ...
int tfl_slab_sim_ipc_export(tfl_ctx* ctx, tfl_slab_sim* s, char* handle_out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!s || !handle_out) return fail(ctx, "slab_sim_ipc_export: nil argument");
  if (!s->inbox) return fail(ctx, "slab_sim_ipc_export: a single rank has no neighbours");
  static_assert(sizeof(cudaIpcMemHandle_t) <= TFL_IPC_HANDLE_BYTES, "IPC handle fits the ABI buffer");
  return ipc_export(ctx, s->inbox.get(), handle_out, TFL_IPC_HANDLE_BYTES);
}

// ... and map every rank's (handles: world x TFL_IPC_HANDLE_BYTES in rank order; NULL switches back to NCCL).
// From then on tfl_slab_sim_step exchanges halos with push / pull kernels over NVLink instead of NCCL send / recv
// and reduces the two sums through the same inboxes.  Every rank must connect before any rank steps (the host
// application's barrier).
int tfl_slab_sim_ipc_connect(tfl_ctx* ctx, tfl_slab_sim* s, const char* handles) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!s || !s->inbox) return fail(ctx, "slab_sim_ipc_connect: nil argument");
  auto drop = [&]() {
    s->mapped.clear();
    s->all_inbox.clear();
    s->peer_inbox[0] = s->peer_inbox[1] = nullptr;
    s->peer_ok = false;
    s->peer_gen++;
  };
  TFL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  drop();
  if (!handles) return 0;                          // back to NCCL (e.g. another rank could not map its peers)
  if (s->world > kMaxRanks) return fail(ctx, "slab_sim_ipc_connect: more than %d ranks", kMaxRanks);
  s->mapped.resize(s->world);
  s->all_inbox.assign(s->world, nullptr);
  s->all_inbox[s->rank] = s->inbox.get();
  for (int r = 0; r < s->world; r++) {
    if (r == s->rank) continue;
    if (ipc_map(ctx, handles + (size_t)r * TFL_IPC_HANDLE_BYTES, &s->mapped[r], "slab_sim_ipc_connect",
                ("(rank " + std::to_string(r) + ")").c_str(), " (the exchanges stay on NCCL)")) {
      drop();
      return 1;
    }
    s->all_inbox[r] = s->mapped[r].get();
  }
  if (!s->all_inbox_dev) {
    void* p = nullptr;
    TFL_CUDA(ctx, cudaMalloc(&p, kMaxRanks * sizeof(float*)));
    s->all_inbox_dev.reset((float**)p);
  }
  TFL_CUDA(ctx, cudaMemcpy(s->all_inbox_dev.get(), s->all_inbox.data(), s->world * sizeof(float*), cudaMemcpyHostToDevice));
  if (s->rank > 0) s->peer_inbox[0] = s->all_inbox[s->rank - 1];
  if (s->rank < s->world - 1) s->peer_inbox[1] = s->all_inbox[s->rank + 1];
  s->peer_ok = true;
  return 0;
}

// Device time of the last step's three halo exchanges and of its all-reduce (ms) and the bytes this rank sent in
// each exchange.  Synchronises.
int tfl_slab_sim_exchange_stats(tfl_ctx* ctx, tfl_slab_sim* s, float ms[4], int64_t bytes[3]) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!s) return fail(ctx, "slab_sim is nil");
  TFL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  for (int i = 0; i < 4; i++) {
    ms[i] = 0.0f;
    if (cudaEventElapsedTime(&ms[i], s->ev[i][0].get(), s->ev[i][1].get()) != cudaSuccess) { cudaGetLastError(); ms[i] = -1.0f; }
  }
  for (int i = 0; i < 3; i++) bytes[i] = (int64_t)s->bytes_sent[i];
  return 0;
}

// The last step's p exchanges of the Jacobi projection: how many, their summed device time (ms) and the bytes this
// rank sent in them.  Synchronises.
int tfl_slab_sim_jacobi_stats(tfl_ctx* ctx, tfl_slab_sim* s, int32_t* exchanges, float* ms, int64_t* bytes) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!s) return fail(ctx, "slab_sim is nil");
  TFL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (s->tol_last) {      // the exchanges before the stopping block's and the 1-plane one; not timed inside the loop
    SlabTolState h;
    TFL_CUDA(ctx, cudaMemcpy(&h, s->tol_state.get(), sizeof(h), cudaMemcpyDeviceToHost));
    int n = 0;
    size_t planes = 0;
    const bool moved = s->world > 1 && (s->peer_ok || ctx->comm);
    for (int b = 0; moved && b <= h.stop_blk && b < (int)s->tol_widths.size(); b++)
      if (s->tol_widths[b] > 0) { n++; planes += s->tol_widths[b]; }
    if (moved && h.fix) { n++; planes += 1; }
    if (exchanges) *exchanges = n;
    if (ms) *ms = -1.0f;
    if (bytes) *bytes = (int64_t)(planes * s->plane * 4 * ((s->rank > 0) + (s->rank < s->world - 1)));
    return 0;
  }
  float total = 0.0f;
  for (int i = 0; i < s->jx; i++) {
    float t = 0.0f;
    TFL_CUDA(ctx, cudaEventElapsedTime(&t, s->jev[2 * i].get(), s->jev[2 * i + 1].get()));
    total += t;
  }
  if (exchanges) *exchanges = s->jx;
  if (ms) *ms = total;
  if (bytes) *bytes = (int64_t)s->jbytes;
  return 0;
}

int tfl_slab_sim_set_jacobi_tolerance(tfl_ctx* ctx, tfl_slab_sim* s, float p_tol) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!ctx) return 1;
  if (!s) return fail(ctx, "slab_sim_set_jacobi_tolerance: nil argument");
  if (!(p_tol >= 0.0f)) return fail(ctx, "slab_sim_set_jacobi_tolerance: pTol must be >= 0 (got %g)", p_tol);
  if (p_tol > 0.0f && !s->p_save) {             // allocated here, so that no step (and no capture) allocates
    bool capturing = false;
    if (stream_capturing(ctx, "slab_sim_set_jacobi_tolerance", &capturing)) return 1;
    if (capturing)
      return fail(ctx, "slab_sim_set_jacobi_tolerance: the stream is being captured; set the tolerance before capturing");
    const size_t nown = (size_t)(s->z1 - s->z0), tiles = (size_t)jacobi_plane_tiles(s->nx, s->ny);
    const size_t per_block = (size_t)s->halo * s->gnz;
    if (!(s->p_save = dev_zeros<float>(s->cells)) || !(s->tol_slots = dev_zeros<double>(s->halo * nown * tiles)) ||
        !(s->tol_send = dev_zeros<double>(per_block)) || !(s->tol_recv = dev_zeros<double>(per_block)) ||
        !(s->tol_state = dev_zeros<SlabTolState>(1)) || !(s->tol_rerun = dev_zeros<int>(s->halo))) {
      s->p_save.reset();
      return fail(ctx, "slab_sim_set_jacobi_tolerance: allocation failed");
    }
  }
  s->p_tol = p_tol;
  return 0;
}

int tfl_slab_sim_jacobi_status(tfl_ctx* ctx, tfl_slab_sim* s, float* residual, int32_t* iterations) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!ctx) return 1;
  if (!s) return fail(ctx, "slab_sim_jacobi_status: nil argument");
  if (!s->tol_stepped)
    return fail(ctx, "slab_sim_jacobi_status: no step has solved to a Jacobi tolerance yet "
                     "(tfl_slab_sim_set_jacobi_tolerance, then a 'jacobi' step)");
  if (!s->tol_last)
    return fail(ctx, "slab_sim_jacobi_status: the last 'jacobi' step ran the fixed count (pTol 0): it has no residual "
                     "or iteration count of its own");
  bool capturing = false;
  if (stream_capturing(ctx, "slab_sim_jacobi_status", &capturing)) return 1;
  if (capturing)
    return fail(ctx, "slab_sim_jacobi_status: the stream is being captured and this call waits for the device; read "
                     "the status after the graph's launch");
  SlabTolState h;
  TFL_CUDA(ctx, cudaMemcpyAsync(&h, s->tol_state.get(), sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
  TFL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (residual) *residual = h.res;
  if (iterations) *iterations = h.iter;
  return 0;
}

}  // extern "C"
