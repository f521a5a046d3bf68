// C ABI of the z-slab driver (include/tfl.h): the NCCL loader, the halo exchange and all-reduce kernels, and
// tfl_comm_* / tfl_slab_sim_*.
#include <dlfcn.h>
#include <string.h>
#include <algorithm>
#include <vector>

#include "tfl_api_internal.h"

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

// floats reserved behind the halo counters of an inbox for the all-reduce: [2 parities][world <= 64][2] doubles, then
// [2][64] step counters
constexpr int kSumAreaFloats = 2 * 64 * 2 * 2 + 2 * 64;

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
  // Peer-memory halo exchange (CUDA IPC over NVLink, tfl_slab_sim_ipc_*): this rank's inbox -- per phase and side a
  // receive buffer of xbuf_side floats that the neighbour's push kernel fills with remote stores, and a step counter
  // it raises afterwards -- and the neighbours' inboxes mapped into this process.
  DevPtr<float> inbox;              // exported: [3 phases][2 sides][xbuf_side] floats, then 64 counters
  std::vector<IpcPtr<float>> mapped;           // the other ranks' inboxes (cudaIpcOpenMemHandle), empty at [rank]
  float* peer_inbox[2] = {nullptr, nullptr};   // lower / upper neighbour's inbox
  std::vector<float*> all_inbox;               // every rank's inbox (own pointer at [rank]): the all-reduce's targets
  DevPtr<float*> all_inbox_dev;                // the same table on the device
  DevPtr<unsigned int> push_done;              // CTAs of the running push kernel that finished their stores
  bool peer_ok = false;
  unsigned int step_no = 0;
  EventPtr ev[4][2];
  size_t bytes_sent[3] = {0, 0, 0};
  // Jacobi projection (simMethod 'jacobi'): divergence, second p buffer and mask of the local slab; the p exchanges
  // land in their own inbox area behind the all-reduce's -- [2 parities][2 sides][p_side] floats, then
  // [2 parities][2 sides] counters -- and carry the monotone sequence number jseq instead of step_no.
  DevPtr<float> div;
  DevPtr<float> p2;
  DevPtr<unsigned char> mask;
  size_t p_side = 0;                // halo planes of one channel
  unsigned int jseq = 0;
  std::vector<int32_t> jsched;
  std::vector<EventPtr> jev;        // [2 * exchange] begin / end of the last step's p exchanges
  int jx = 0;                       // p exchanges of the last step
  size_t jbytes = 0;
};

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
      (!(s->inbox = dev_zeros<float>(6 * s->xbuf_side + 64 + kSumAreaFloats + 4 * s->p_side + 64)) ||
       !(s->push_done = dev_zeros<unsigned int>(1))))
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
};
template <bool UNPACK>
__global__ void k_slab_pack(SlabPack d) {
  const long long per_side = d.cnt * d.nchan;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < 2 * per_side; t += (long long)gridDim.x * blockDim.x) {
    const int side = t >= per_side;
    const long long r = t - side * per_side;
    const int c = (int)(r / d.cnt);
    const long long e = r - c * d.cnt;
    if (!UNPACK) {
      float* buf = side ? d.send_hi : d.send_lo;
      if (buf) buf[r] = d.chan[c][(side ? d.src_hi : d.src_lo) + e];
    } else {
      const float* buf = side ? d.recv_hi : d.recv_lo;
      if (buf) d.chan[c][(side ? d.dst_hi : d.dst_lo) + e] = buf[r];
    }
  }
}

// Peer-memory exchange, sending half: every channel's boundary planes are written straight into the neighbours'
// inboxes (remote stores over NVLink), and when the last CTA has finished, the step number is stored (system
// scope, after a system-wide fence) into the neighbours' counters.
__global__ void k_slab_push(SlabPack d, float* peer_lo_buf, float* peer_hi_buf, unsigned int* peer_lo_flag,
                            unsigned int* peer_hi_flag, unsigned int step, unsigned int* done) {
  const long long per_side = d.cnt * d.nchan;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < 2 * per_side; t += (long long)gridDim.x * blockDim.x) {
    const int side = t >= per_side;
    const long long r = t - side * per_side;
    const int c = (int)(r / d.cnt);
    const long long e = r - c * d.cnt;
    float* buf = side ? peer_hi_buf : peer_lo_buf;
    if (buf) buf[r] = d.chan[c][(side ? d.src_hi : d.src_lo) + e];
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int prev = atomicAdd(done, 1u);
    if (prev == gridDim.x - 1) {               // every CTA's stores are fenced: publish
      *done = 0u;
      __threadfence_system();
      if (peer_lo_flag) asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(peer_lo_flag), "r"(step) : "memory");
      if (peer_hi_flag) asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(peer_hi_flag), "r"(step) : "memory");
    }
  }
}
// ... receiving half: wait until the neighbours' counters have reached this step, then scatter the inbox into the
// ghost planes.  The wait is bounded (a neighbour that never arrives raises the fault counter instead of hanging
// the GPU).
__global__ void k_slab_pull(SlabPack d, const float* buf_lo, const float* buf_hi, const unsigned int* flag_lo,
                            const unsigned int* flag_hi, unsigned int step, unsigned long long* faults) {
  __shared__ int ok;
  if (threadIdx.x == 0) {
    ok = 1;
    const long long t0 = clock64();
    for (int sde = 0; sde < 2; sde++) {
      const unsigned int* f = sde ? flag_hi : flag_lo;
      if (!f) continue;
      for (;;) {
        unsigned int v;
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(f) : "memory");
        if ((int)(v - step) >= 0) break;
        if (clock64() - t0 > 4000000000LL) { ok = 0; break; }       // ~2 s
        __nanosleep(200);
      }
    }
    if (!ok && blockIdx.x == 0 && faults) atomicAdd(faults, 1ULL);
  }
  __syncthreads();
  if (!ok) return;
  const long long per_side = d.cnt * d.nchan;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < 2 * per_side; t += (long long)gridDim.x * blockDim.x) {
    const int side = t >= per_side;
    const long long r = t - side * per_side;
    const int c = (int)(r / d.cnt);
    const long long e = r - c * d.cnt;
    const float* buf = side ? buf_hi : buf_lo;
    if (buf) d.chan[c][(side ? d.dst_hi : d.dst_lo) + e] = __ldcg(buf + r);
  }
}

// All-reduce of the two partial sums over peer memory: every rank stores its pair into slot [parity][rank] of every
// rank's inbox and raises that rank's counter [parity][rank]; then waits for all counters of its own inbox and adds
// the pairs in rank order (the same order on every rank: identical results everywhere, independent of timing).
// Slots alternate with the step's parity: a rank that is still reading step s cannot be overwritten by step s + 1.
__device__ __forceinline__ double* sum_slot(float* inbox, size_t xbuf_side, int parity, int r) {
  return reinterpret_cast<double*>(inbox + 6 * xbuf_side + 64) + ((size_t)parity * 64 + r) * 2;
}
__device__ __forceinline__ unsigned int* sum_flag(float* inbox, size_t xbuf_side, int parity, int r) {
  return reinterpret_cast<unsigned int*>(inbox + 6 * xbuf_side + 64 + 2 * 64 * 2 * 2) + parity * 64 + r;
}
__global__ void k_sum_push(const double* __restrict__ mine, float* const* __restrict__ inboxes, size_t xbuf_side, int rank,
                           int world, unsigned int step) {
  const int t = threadIdx.x;
  if (t >= world) return;
  const int parity = step & 1;
  double* slot = sum_slot(inboxes[t], xbuf_side, parity, rank);
  slot[0] = mine[0];
  slot[1] = mine[1];
  __threadfence_system();
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(sum_flag(inboxes[t], xbuf_side, parity, rank)), "r"(step) : "memory");
}
__global__ void k_sum_pull(double* __restrict__ out, float* inbox, size_t xbuf_side, int world, unsigned int step,
                           unsigned long long* faults) {
  __shared__ int ok;
  const int t = threadIdx.x, parity = step & 1;
  if (t == 0) ok = 1;
  __syncthreads();
  if (t < world) {
    const long long t0 = clock64();
    for (;;) {
      unsigned int v;
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(sum_flag(inbox, xbuf_side, parity, t)) : "memory");
      if ((int)(v - step) >= 0) break;
      if (clock64() - t0 > 4000000000LL) { ok = 0; break; }
      __nanosleep(100);
    }
  }
  __syncthreads();
  if (t == 0) {
    if (!ok) { if (faults) atomicAdd(faults, 1ULL); return; }
    double s0 = 0.0, s1 = 0.0;
    for (int r = 0; r < world; r++) {
      const volatile double* slot = sum_slot(inbox, xbuf_side, parity, r);
      s0 += slot[0];
      s1 += slot[1];
    }
    out[0] = s0;
    out[1] = s1;
  }
}

// The Jacobi p exchange: several per step, so its inbox slots alternate with the parity of a sequence number (a rank
// may push exchange e + 1 while its neighbour still scatters exchange e; it cannot push e + 2 before the neighbour
// has pushed e + 1, which that neighbour does after scattering e).
constexpr int kPhaseP = 4;

// Refresh `width` ghost planes on both sides of the listed fields from the neighbours' owned planes.
int slab_exchange(tfl_ctx* ctx, tfl_slab_sim* s, std::initializer_list<const tfl_grid*> fields, int width, int phase) {
  const bool pph = phase == kPhaseP;
  if (!pph) {
    TFL_CUDA(ctx, cudaEventRecord(s->ev[phase][0].get(), ctx->stream));
    s->bytes_sent[phase] = 0;
  }
  if (s->world > 1 && width > 0 && (ctx->comm || s->peer_ok)) {
    if (width > s->halo) return fail(ctx, "slab exchange of %d planes exceeds the halo (%d)", width, s->halo);
    if (pph) {
      s->jseq += 1;
      while ((int)s->jev.size() < 2 * (s->jx + 1)) {
        cudaEvent_t e = nullptr;
        TFL_CUDA(ctx, cudaEventCreate(&e));
        s->jev.emplace_back(e);
      }
      TFL_CUDA(ctx, cudaEventRecord(s->jev[2 * s->jx].get(), ctx->stream));
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
      // inbox layout: buffer (phase, from-below = 0 / from-above = 1) at ((phase * 2 + from) * xbuf_side), counters behind;
      // the p exchange's (parity, from) buffers and counters behind the all-reduce area
      const size_t p_area = 6 * s->xbuf_side + 64 + kSumAreaFloats;
      const unsigned int seq = pph ? s->jseq : s->step_no, par = seq & 1u;
      auto buf = [&](float* base, int from) {
        return pph ? base + p_area + ((size_t)par * 2 + from) * s->p_side : base + ((size_t)phase * 2 + from) * s->xbuf_side;
      };
      auto flag = [&](float* base, int from) {
        return pph ? (unsigned int*)(base + p_area + 4 * s->p_side) + par * 2 + from
                   : (unsigned int*)(base + 6 * s->xbuf_side) + phase * 2 + from;
      };
      d.send_lo = d.send_hi = d.recv_lo = d.recv_hi = nullptr;
      // my first owned planes land in the lower neighbour's "from above" slot, my last ones in the upper neighbour's "from below"
      k_slab_push<<<blocks, 256, 0, ctx->stream>>>(d, lo ? buf(s->peer_inbox[0], 1) : nullptr, hi ? buf(s->peer_inbox[1], 0) : nullptr,
                                                   lo ? flag(s->peer_inbox[0], 1) : nullptr, hi ? flag(s->peer_inbox[1], 0) : nullptr,
                                                   seq, s->push_done.get());
      float* inbox = s->inbox.get();
      k_slab_pull<<<blocks, 256, 0, ctx->stream>>>(d, lo ? buf(inbox, 0) : nullptr, hi ? buf(inbox, 1) : nullptr,
                                                   lo ? flag(inbox, 0) : nullptr, hi ? flag(inbox, 1) : nullptr,
                                                   seq, ctx->counters.get());
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
      TFL_CUDA(ctx, cudaEventRecord(s->jev[2 * s->jx + 1].get(), ctx->stream));
      s->jx += 1;
      s->jbytes += sent;
      return 0;
    }
    s->bytes_sent[phase] = sent;
  }
  if (!pph) TFL_CUDA(ctx, cudaEventRecord(s->ev[phase][1].get(), ctx->stream));
  return 0;
}

struct SlabScope {       // slab placement of the context for the enclosed calls
  tfl_ctx* ctx;
  SlabScope(tfl_ctx* c, const tfl_slab_sim* s, int zlo, int zhi) : ctx(c) {
    c->slab = true; c->zoff = s->zoff; c->gnz = s->gnz; c->zlo = zlo; c->zhi = zhi; c->slab_margin = s->margin;
  }
  ~SlabScope() { ctx->slab = false; ctx->slab_margin = 2; }
};

// One block of sweeps on a prepared mask: the cooperative block kernel or one launch per sweep (path -1: automatic,
// 0: per sweep, 1: one launch, refused when it does not apply).  Returns the path taken, -1 on refusal.
// The automatic path takes the one-launch kernel only with 4-plane blocks (ranges up to 2.16M cells on an H100):
// measured on an H100 at 400 W, 34 / 100 sweeps of 128^3 run at 8.4 / 7.3 us per sweep in one launch against
// 8.9 / 8.2 per launch, but a 6-sweep block on an 8-rank slab of 256^3 (256^2 x 42 planes, 6-plane blocks) takes
// 154 us against 94 us in per-sweep launches.
int run_jacobi_block(tfl_ctx* ctx, const unsigned char* mask, const float* div, float* pa, float* pb, const Geo& g,
                     int z_lo, int z_hi, int shr_lo, int shr_hi, int sweeps, int path) {
  if (sweeps < 1) return 0;
  if (path != 0 && launch_jacobi_block(mask, div, pa, pb, g, z_lo, z_hi, shr_lo, shr_hi, sweeps, path == 1, ctx->stream)) {
    ctx->launches += 1;
    return 1;
  }
  if (path == 1) return -1;
  launch_jacobi_range_sweeps(mask, div, pa, pb, g, z_lo, z_hi, shr_lo, shr_hi, sweeps, ctx->stream);
  ctx->launches += sweeps;
  return 0;
}

// lib/simulate.lua:275-303 with pTol = 0 on this rank's slab: divergence, `iters` Jacobi sweeps from p = 0 in the
// blocks of tfl_slab_jacobi_schedule, velocity update on the owned planes.  Every cell sees the single-GPU sweep's
// operands, so p and U are bit-identical to tfl_simulate_step's.
int slab_jacobi_projection(tfl_ctx* ctx, tfl_slab_sim* s, int iters) {
  const tfl_state& st = s->st;
  int32_t planes[3];
  const int nblk = tfl_slab_jacobi_schedule(s->gnz, s->world, s->rank, s->margin, iters, planes, nullptr, 0);
  if (nblk < 1) return fail(ctx, "slab_sim_step: no Jacobi schedule for this slab");
  s->jsched.resize((size_t)nblk * TFL_JACOBI_BLOCK_INTS);
  tfl_slab_jacobi_schedule(s->gnz, s->world, s->rank, s->margin, iters, planes, s->jsched.data(), nblk);
  if (slab_exchange(ctx, s, {&st.U}, planes[2], 2)) return 1;
  TFL_CUDA(ctx, cudaEventRecord(s->ev[3][0].get(), ctx->stream));          // no all-reduce on this path
  TFL_CUDA(ctx, cudaEventRecord(s->ev[3][1].get(), ctx->stream));
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
  float* buf[2] = {st.p.data, s->p2.get()};
  int done = 0;
  s->jx = 0;
  s->jbytes = 0;
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

// One tfluids.simulate (lib/simulate.lua:175-327; simMethod 'convnet' or 'jacobi') on this rank's slab.  Asynchronous.
int tfl_slab_sim_step(tfl_ctx* ctx, tfl_slab_sim* s, const tfl_mconf* mc, tfl_cnn* cnn) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!s || !mc) return fail(ctx, "slab_sim_step: nil argument");
  const bool jacobi = mc->sim_method == TFL_SIM_JACOBI;
  if (mc->sim_method == TFL_SIM_PCG)
    return fail(ctx, "slab_sim_step: simMethod 'pcg' is not decomposed: the IC(0) triangular solves of its "
                     "preconditioner sweep the whole domain in order and do not shard over z-slabs");
  if (!jacobi && mc->sim_method != TFL_SIM_CONVNET)
    return fail(ctx, "slab_sim_step: mconf.simMethod (%d) is not a valid option", mc->sim_method);
  if (!jacobi && !cnn) return fail(ctx, "slab_sim_step: simMethod 'convnet' needs a model");
  if (!jacobi && cnn_slab_check(ctx, cnn, s->margin, s->gnz, s->ny, s->nx, s->zoff, s->nz, s->own_lo, s->own_hi))
    return fail(ctx, "slab_sim_step: %s", ctx->err.c_str());
  if (jacobi && mc->max_iter < 0) return fail(ctx, "slab_sim_step: At least 1 iteration is needed (maxIter < 1)");
  if (s->world != ctx->comm_world || s->rank != ctx->comm_rank) return fail(ctx, "slab_sim_step: communicator changed");
  const tfl_state& st = s->st;
  s->step_no += 1;                      // what the peers' counters must reach in this step's exchanges
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
  TFL_CUDA(ctx, cudaEventRecord(s->ev[3][0].get(), ctx->stream));
  if (s->world > 1 && s->peer_ok && s->all_inbox_dev) {
    k_sum_push<<<1, 64, 0, ctx->stream>>>(sums, s->all_inbox_dev.get(), s->xbuf_side, s->rank, s->world, s->step_no);
    k_sum_pull<<<1, 64, 0, ctx->stream>>>(sums, s->inbox.get(), s->xbuf_side, s->world, s->step_no, ctx->counters.get());
    ctx->launches += 2;
  } else if (s->world > 1 && ctx->comm) {
    TFL_NCCL(ctx, nccl_api()->AllReduce(sums, sums, 2, ncclDouble, ncclSum, ctx->comm, ctx->stream));
  }
  TFL_CUDA(ctx, cudaEventRecord(s->ev[3][1].get(), ctx->stream));
  {
    SlabScope scope(ctx, s, s->own_lo, s->own_hi);
    if (tfl_cnn_project_from_sums(ctx, cnn, &st.p, &u1, &st.flags, sums, &st.p, &st.U, mc->normalize_input_threshold)) return 1;
  }
  if (bcs()) return 1;
  SlabScope scope(ctx, s, s->own_lo, s->own_hi);
  return tfl_clamp(ctx, &st.U, -1e6f, 1e6f);
}

// Peer-memory halos: export this rank's inbox (64-byte CUDA IPC handle) ...
int tfl_slab_sim_ipc_export(tfl_ctx* ctx, tfl_slab_sim* s, char* handle_out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!s || !handle_out) return fail(ctx, "slab_sim_ipc_export: nil argument");
  if (!s->inbox) return fail(ctx, "slab_sim_ipc_export: a single rank has no neighbours");
  static_assert(sizeof(cudaIpcMemHandle_t) <= TFL_IPC_HANDLE_BYTES, "IPC handle fits the ABI buffer");
  cudaIpcMemHandle_t h;
  TFL_CUDA(ctx, cudaIpcGetMemHandle(&h, s->inbox.get()));
  memset(handle_out, 0, TFL_IPC_HANDLE_BYTES);
  memcpy(handle_out, &h, sizeof(h));
  return 0;
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
  };
  TFL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  drop();
  if (!handles) return 0;                          // back to NCCL (e.g. another rank could not map its peers)
  if (s->world > 64) return fail(ctx, "slab_sim_ipc_connect: more than 64 ranks");
  s->mapped.resize(s->world);
  s->all_inbox.assign(s->world, nullptr);
  s->all_inbox[s->rank] = s->inbox.get();
  for (int r = 0; r < s->world; r++) {
    if (r == s->rank) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, handles + (size_t)r * TFL_IPC_HANDLE_BYTES, sizeof(h));
    void* q = nullptr;
    const cudaError_t e = cudaIpcOpenMemHandle(&q, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
      cudaGetLastError();
      drop();
      return fail(ctx, "slab_sim_ipc_connect: cudaIpcOpenMemHandle(rank %d): %s (the exchanges stay on NCCL)", r, cudaGetErrorString(e));
    }
    s->mapped[r].reset((float*)q);
    s->all_inbox[r] = (float*)q;
  }
  if (!s->all_inbox_dev) {
    void* p = nullptr;
    TFL_CUDA(ctx, cudaMalloc(&p, 64 * sizeof(float*)));
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

}  // extern "C"
