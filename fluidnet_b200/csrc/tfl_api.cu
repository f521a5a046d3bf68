// C ABI of libtfl (include/tfl.h): context, scratch arena, argument checks that mirror the
// asserts of the reference's Lua wrappers (torch/tfluids/init.lua), and the operator /
// whole-step entry points that enqueue the kernels of tfl_stencils.cu, tfl_model_stages.cu
// and tfl_cnn*.cu on the context's stream.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nvtx3/nvToolsExt.h>
#include <nccl.h>      // types and prototypes only: libnccl is loaded on demand (dlopen), see NcclApi
#include <stdarg.h>
#include <stdio.h>
#include <string.h>
#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

#include "tfl_kernels.h"
#include "tfl_cnn_tc.h"

using namespace tfl;

struct tfl_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = true;
  std::string err;
  char* arena = nullptr;
  size_t arena_bytes = 0;
  size_t arena_used = 0;
  unsigned long long* counters = nullptr;   // [0] trace faults, [1] bad occupancy cells
  double* dscratch = nullptr;               // small double scratch (reductions), 256 entries
  long long launches = 0;
  bool slab = false;
  int zoff = 0, gnz = 0, zlo = 0, zhi = 0;
  int slab_margin = 2;                      // extra planes on which forward passes are evaluated
  cudaStream_t side_stream = nullptr;       // density advection runs beside velocity advection
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  // Host-buffer step (tfl_host_sim_step): copies run on their own streams and the step waits for each
  // input only where it is first read / hands each output over as soon as it is final.
  cudaStream_t copy_in = nullptr, copy_out = nullptr;
  cudaEvent_t ev_u_in = nullptr, ev_d_in = nullptr, ev_p_in = nullptr, ev_d_ready = nullptr, ev_d_out = nullptr;
  struct {
    bool active = false;
    float* density_host = nullptr;          // where the advected density goes once it is final
    size_t density_bytes = 0;
    bool density_sent = false;
  } ov;
  PcgScratch pcg;                           // grow-only buffers of the PCG solve
  // Byte copy of the step's flags and their clearance field (advection fast path), kept between steps:
  // each step re-derives the bytes, compares them with the copy on the device and rebuilds the
  // clearance only if something changed (no host round trip).
  struct {
    unsigned char* bytes = nullptr;         // [3][cells]: flags, clearance, scratch
    size_t cells = 0;
    int nb = 0, nz = 0, ny = 0, nx = 0;
    int* changed = nullptr;                 // device word
    const float* fresh_for = nullptr;       // set inside a slab step: the cache already mirrors these flags
  } fcache;
  // advectVel over shared-memory tiles (tfl_advect_tile.cu): the kernel reports the longest trace of a call
  // into a device word that is copied, asynchronously, into a pinned host word; the NEXT calls pick the tile
  // halo from it (stale by a step or two -- it only selects a code path, never a result).
  struct {
    unsigned int* dev = nullptr;
    unsigned int* host = nullptr;           // pinned
    int mode = -1;                          // -1 automatic, 0 two-kernel version, 1 / 2 forced halo
    int variant = 0;                        // tile shape (tuning)
    int calls_since_probe = 0;
    // bench.py's roofline: CUDA events right around the tile kernel's launch (off unless asked for)
    bool timed = false;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  } tile;
  // z-slab decomposition over several GPUs (tfl_comm_init / tfl_slab_sim_*): the communicator lives here
  ncclComm_t comm = nullptr;
  int comm_rank = 0, comm_world = 1;
  bool in_slab_step = false;
};

struct tfl_cnn {
  int is3d = 1;
  int n_layers = 0;
  std::vector<int> cin, cout, ks;
  std::vector<float*> w;     // device, [cin][tap][cout]
  std::vector<float*> b;     // device, [cout]
  int max_c = 0;
  // per-layer extras of the 'tog' / 'yang' graphs (lib/model.lua:164-239): the convolution emits
  // cout * up^d channels that a pixel shuffle turns into cout channels at `up` times the resolution, a
  // pooling of size `pool` follows the non-linearity.  plain = every pool / up is 1 and the non-linearity is ReLU.
  std::vector<int> pool, up;
  int pool_is_max = 0;
  int nonlin = 1;            // 1 ReLU, 2 sigmoid (activation codes of tfl_cnn.cu)
  bool plain = true;
  double max_rel = 0.0;      // largest channels x (cells relative to the input grid) of any stage
  // tensor-core path (3-D 'default' architecture only)
  int mode = 0;              // 0 fp32 FMA, 1 TF32 tensor cores, 2 3xTF32 tensor cores
  bool tc_ok = false;
  float* wB[2][3] = {{nullptr, nullptr, nullptr}, {nullptr, nullptr, nullptr}};   // [split][layer]
  float* tail = nullptr;     // w4[8][8], b4[8], w5[8], b5[1]
  float* act[3] = {nullptr, nullptr, nullptr};   // padded channels-last activation buffers
  ConvTcGeo act_geo = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
};


// Every entry point runs on the context's device whatever the caller's current device is, and leaves the
// caller's current device as it found it (a host with several contexts / GPUs in one thread).
// One NVTX range per entry point (named after the function): nsys / ncu --nvtx timelines show the operators.
// nvtx3 is header-only and costs a null-pointer test when no tool is attached.
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};

struct DeviceGuard {
  int prev = -1;
  bool switched = false;
  explicit DeviceGuard(const tfl_ctx* ctx) {
    if (!ctx) return;
    if (cudaGetDevice(&prev) == cudaSuccess && prev != ctx->device) switched = cudaSetDevice(ctx->device) == cudaSuccess;
  }
  ~DeviceGuard() { if (switched) cudaSetDevice(prev); }
};

namespace {

int fail(tfl_ctx* ctx, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  if (ctx) ctx->err = buf;
  return 1;
}

#define TFL_CUDA(ctx, call)                                                            \
  do {                                                                                 \
    cudaError_t e_ = (call);                                                           \
    if (e_ != cudaSuccess) return fail(ctx, "%s: %s", #call, cudaGetErrorString(e_));  \
  } while (0)

int check_launch(tfl_ctx* ctx, const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(ctx, "%s: launch failed: %s", what, cudaGetErrorString(e));
  return 0;
}

// Bump allocator over one growing device buffer (the reference's getTempStorage,
// tfluids/init.lua:35-64).  Growing synchronises; steady state does not allocate.
int arena_reserve(tfl_ctx* ctx, size_t bytes) {
  if (bytes <= ctx->arena_bytes) return 0;
  TFL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (ctx->arena) cudaFree(ctx->arena);
  ctx->arena = nullptr;
  ctx->arena_bytes = 0;
  void* p = nullptr;
  TFL_CUDA(ctx, cudaMalloc(&p, bytes));
  ctx->arena = (char*)p;
  ctx->arena_bytes = bytes;
  return 0;
}
struct Carver {
  tfl_ctx* ctx;
  size_t off = 0;
  explicit Carver(tfl_ctx* c) : ctx(c) {}
  template <typename T>
  T* take(size_t count) {
    const size_t a = (off + 255) & ~(size_t)255;
    off = a + count * sizeof(T);
    return (T*)(ctx->arena + a);
  }
};
size_t carve_bytes(std::initializer_list<size_t> sizes) {
  size_t off = 0;
  for (size_t s : sizes) off = ((off + 255) & ~(size_t)255) + s;
  return off + 256;
}

bool same_spatial(const tfl_grid* a, const tfl_grid* b) {
  return a->nb == b->nb && a->nz == b->nz && a->ny == b->ny && a->nx == b->nx;
}

// Mirrors the shape asserts of init.lua (e.g. :100-120, :177-191).
int check_scalar(tfl_ctx* ctx, const tfl_grid* g, const char* name) {
  if (!g || !g->data) return fail(ctx, "%s is nil", name);
  if (g->nc != 1) return fail(ctx, "%s is not scalar", name);
  if (g->nb < 1 || g->nz < 1 || g->ny < 1 || g->nx < 1) return fail(ctx, "%s: Dimension mismatch", name);
  return 0;
}
int check_vel(tfl_ctx* ctx, const tfl_grid* U, const tfl_grid* flags) {
  if (!U || !U->data) return fail(ctx, "U is nil");
  if (U->nc != 2 && U->nc != 3) return fail(ctx, "2D velocity field must have only 2 channels");
  if (U->nc == 2 && flags->nz != 1) return fail(ctx, "2D velocity field but zdepth > 1");
  if (!same_spatial(U, flags)) return fail(ctx, "Size mismatch");
  return 0;
}

int make_geo(tfl_ctx* ctx, const tfl_grid* flags, int is3d, Geo* g) {
  g->nx = flags->nx; g->ny = flags->ny; g->nz = flags->nz; g->nb = flags->nb;
  g->is3d = is3d ? 1 : 0;
  g->nc = is3d ? 3 : 2;
  g->n = (long long)flags->nx * flags->ny * flags->nz;
  g->faults = ctx->counters;
  if (ctx->slab) {
    if (!is3d) return fail(ctx, "slab decomposition needs a 3D grid");
    g->zoff = ctx->zoff; g->gnz = ctx->gnz; g->zlo = ctx->zlo; g->zhi = ctx->zhi;
    if (g->zlo < 0 || g->zhi > g->nz || g->zlo >= g->zhi || g->zoff < 0 || g->zoff + g->nz > g->gnz)
      return fail(ctx, "slab range does not fit the local grid");
  } else {
    g->zoff = 0; g->gnz = flags->nz; g->zlo = 0; g->zhi = flags->nz;
  }
  if (!is3d && flags->nz != 1) return fail(ctx, "2D grid must have zsize == 1");
  if (g->n * (long long)g->nb * 3 >= (1LL << 31) * 4) return fail(ctx, "grid too large");
  return 0;
}

// z-slab mode: the MacCormack forward pass must also cover the planes the backward traces of the
// owned planes can reach (margin), but never start a trace on a local end plane that is not a
// global end (the MAC samples reach one plane further).
void widen_for_forward_pass(const tfl_ctx* ctx, const Geo& g, Geo* gf) {
  if (!ctx->slab) { gf->zlo = 0; gf->zhi = g.nz; return; }
  const int lo_lim = (g.zoff == 0) ? 0 : 1;
  const int hi_lim = (g.zoff + g.nz == g.gnz) ? g.nz : g.nz - 1;
  gf->zlo = std::max(lo_lim, g.zlo - ctx->slab_margin);
  gf->zhi = std::min(hi_lim, g.zhi + ctx->slab_margin);
}

// (Re)allocates the flag-byte cache for this grid shape; a new cache starts "changed" (the word stays set
// until a step has rebuilt the clearance: the step resets it after the rebuild is enqueued).
int flag_cache_ensure(tfl_ctx* ctx, const Geo& g) {
  auto& fc = ctx->fcache;
  const size_t cells = (size_t)g.n * g.nb;
  if (!fc.changed) {
    void* p = nullptr;
    TFL_CUDA(ctx, cudaMalloc(&p, sizeof(int)));
    fc.changed = (int*)p;
  }
  if (fc.bytes && fc.cells == cells && fc.nb == g.nb && fc.nz == g.nz && fc.ny == g.ny && fc.nx == g.nx) {
    TFL_CUDA(ctx, cudaMemsetAsync(fc.changed, 0, sizeof(int), ctx->stream));
    return 0;
  }
  TFL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (fc.bytes) cudaFree(fc.bytes);
  fc.bytes = nullptr;
  void* p = nullptr;
  TFL_CUDA(ctx, cudaMalloc(&p, 3 * cells + 64));
  fc.bytes = (unsigned char*)p;
  fc.cells = cells; fc.nb = g.nb; fc.nz = g.nz; fc.ny = g.ny; fc.nx = g.nx;
  TFL_CUDA(ctx, cudaMemsetAsync(fc.bytes, 0, 3 * cells + 64, ctx->stream));
  TFL_CUDA(ctx, cudaMemsetAsync(fc.changed, 1, sizeof(int), ctx->stream));     // non-zero: rebuild
  return 0;
}

// Byte flags + clearance field of `flags` for this call, through the context's cache: the bytes are
// re-derived and compared on the device, the clearance is rebuilt only when one differs.
int prepare_flags(tfl_ctx* ctx, const float* flags, const Geo& g, unsigned char** fl8, unsigned char** clear) {
  const size_t cells = (size_t)g.n * g.nb;
  auto& fc = ctx->fcache;
  if (fc.fresh_for == flags && fc.bytes && fc.cells == cells && fc.nz == g.nz && fc.ny == g.ny && fc.nx == g.nx) {
    *fl8 = fc.bytes;                        // refreshed earlier in this (slab) step: nothing wrote the flags since
    *clear = fc.bytes + cells;
    return 0;
  }
  if (flag_cache_ensure(ctx, g)) return 1;
  *fl8 = ctx->fcache.bytes;
  *clear = ctx->fcache.bytes + cells;
  launch_flags_to_u8(flags, *fl8, (long long)cells, ctx->fcache.changed, ctx->stream);
  ctx->launches += 1 + launch_clearance(*fl8, *clear, *clear + cells, g, ctx->fcache.changed, ctx->stream);
  if (ctx->in_slab_step) fc.fresh_for = flags;
  return 0;
}

// Halo of the advection tile kernels for this call (0: use the per-pass kernels), from the longest trace the
// velocity kernel reported on earlier calls.
int tile_halo_choice(tfl_ctx* ctx, bool probe) {
  auto& tl = ctx->tile;
  if (tl.mode >= 0) return tl.mode;
  float longest = 0.0f;
  if (tl.host) { const unsigned int bits = *(volatile unsigned int*)tl.host; memcpy(&longest, &bits, 4); }
  int hf = longest < 0.45f ? 1 : (longest < 1.4f ? 2 : 0);
  // beyond the wide halo the per-pass kernels are faster; the velocity kernel looks again every 16th call
  if (hf == 0 && probe && ++tl.calls_since_probe >= 16) { hf = 2; tl.calls_since_probe = 0; }
  return hf;
}

// advectVel('maccormackOurs') dispatch: the tile kernel when the grid qualifies and the traces of the recent
// calls fit its halo, the two-kernel version otherwise.  Returns the launch count, < 0 for a bad method.
template <typename FT>
int advect_vel_dispatch(tfl_ctx* ctx, float dt, const float* U, const FT* flags, const unsigned char* fl8,
                        const unsigned char* clear, int method, float strength, float* dst, float* fwd, const Geo& g,
                        const Geo& gf, cudaStream_t st) {
  const bool ours = method == TFL_ADVECT_MACCORMACK_OURS || method == TFL_ADVECT_RK2_OURS || method == TFL_ADVECT_RK3_OURS;
  auto& tl = ctx->tile;
  if (ours && fl8 && clear && tl.mode != 0) {
    if (!tl.dev) {
      void* p = nullptr;
      if (cudaMalloc(&p, sizeof(unsigned int)) == cudaSuccess) tl.dev = (unsigned int*)p;
      if (cudaHostAlloc(&p, sizeof(unsigned int), cudaHostAllocDefault) == cudaSuccess) { tl.host = (unsigned int*)p; *tl.host = 0; }
    }
    const int hf = tile_halo_choice(ctx, true);
    if (hf > 0 && tl.dev && tl.host) {
      cudaMemsetAsync(tl.dev, 0, sizeof(unsigned int), st);
      if (tl.timed) cudaEventRecord(tl.ev0, st);
      const bool launched = launch_advect_vel_tile(dt, U, fl8, clear, strength, dst, g, hf, tl.variant, tl.dev, st);
      if (tl.timed) cudaEventRecord(tl.ev1, st);
      if (launched) {
        cudaMemcpyAsync(tl.host, tl.dev, sizeof(unsigned int), cudaMemcpyDeviceToHost, st);
        return 1;
      }
    }
  }
  return launch_advect_vel(dt, U, flags, clear, method, strength, dst, fwd, g, gf, st);
}

template <typename FT>
int advect_scalar_dispatch(tfl_ctx* ctx, float dt, const float* s, const float* U, const FT* flags,
                           const unsigned char* fl8, const unsigned char* clear, int method, int outside, float strength,
                           float* dst, float* fwd, float* fwd_pos, const Geo& g, const Geo& gf, cudaStream_t st) {
  if (method == TFL_ADVECT_MACCORMACK_OURS && fl8 && clear && ctx->tile.mode != 0) {
    const int hf = tile_halo_choice(ctx, false);
    if (hf > 0 && launch_advect_scalar_tile(dt, s, U, fl8, clear, outside, strength, dst, g, hf, ctx->tile.variant, st))
      return 1;
  }
  return launch_advect_scalar(dt, s, U, flags, clear, method, outside, strength, dst, fwd, fwd_pos, g, gf, st);
}

float get_dx(const Geo& g) {     // third_party/grid.cc:37-40 on the GLOBAL grid
  int m = g.nx > g.ny ? g.nx : g.ny;
  if (g.gnz > m) m = g.gnz;
  return 1.0f / (float)m;
}

}  // namespace

extern "C" {

const char* tfl_version(void) { return "libtfl 0.1 (sm_90a)"; }

int tfl_advect_method_from_string(const char* s) {
  if (!s) return -1;
  if (!strcmp(s, "euler")) return TFL_ADVECT_EULER;
  if (!strcmp(s, "maccormack")) return TFL_ADVECT_MACCORMACK;
  if (!strcmp(s, "eulerOurs")) return TFL_ADVECT_EULER_OURS;
  if (!strcmp(s, "rk2Ours")) return TFL_ADVECT_RK2_OURS;
  if (!strcmp(s, "rk3Ours")) return TFL_ADVECT_RK3_OURS;
  if (!strcmp(s, "maccormackOurs")) return TFL_ADVECT_MACCORMACK_OURS;
  return -1;
}

int tfl_create(tfl_ctx** out, int device) {
  if (!out) return 1;
  *out = nullptr;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0 || device < 0 || device >= n) return 1;
  int prev_dev = device;
  cudaGetDevice(&prev_dev);
  struct Restore { int d; ~Restore() { cudaSetDevice(d); } } restore_{prev_dev};   // caller's device stays current
  if (cudaSetDevice(device) != cudaSuccess) return 1;
  tfl_ctx* c = new tfl_ctx();
  c->device = device;
  if (cudaStreamCreate(&c->stream) != cudaSuccess) { delete c; return 1; }
  void* p = nullptr;
  if (cudaMalloc(&p, 16 * sizeof(unsigned long long)) != cudaSuccess) { delete c; return 1; }
  c->counters = (unsigned long long*)p;
  cudaMemset(c->counters, 0, 16 * sizeof(unsigned long long));
  if (cudaMalloc(&p, 256 * sizeof(double)) != cudaSuccess) { delete c; return 1; }
  c->dscratch = (double*)p;
  cudaStreamCreateWithFlags(&c->side_stream, cudaStreamNonBlocking);
  cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming);
  cudaStreamCreateWithFlags(&c->copy_in, cudaStreamNonBlocking);
  cudaStreamCreateWithFlags(&c->copy_out, cudaStreamNonBlocking);
  for (cudaEvent_t* e : {&c->ev_u_in, &c->ev_d_in, &c->ev_p_in, &c->ev_d_ready, &c->ev_d_out})
    cudaEventCreateWithFlags(e, cudaEventDisableTiming);
  *out = c;
  return 0;
}

void tfl_destroy(tfl_ctx* ctx) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  if (ctx->arena) cudaFree(ctx->arena);
  if (ctx->counters) cudaFree(ctx->counters);
  if (ctx->dscratch) cudaFree(ctx->dscratch);
  pcg_release(ctx->pcg);
  if (ctx->fcache.bytes) cudaFree(ctx->fcache.bytes);
  if (ctx->fcache.changed) cudaFree(ctx->fcache.changed);
  if (ctx->tile.dev) cudaFree(ctx->tile.dev);
  if (ctx->tile.host) cudaFreeHost(ctx->tile.host);
  if (ctx->tile.ev0) { cudaEventDestroy(ctx->tile.ev0); cudaEventDestroy(ctx->tile.ev1); }
  tfl_comm_destroy(ctx);
  if (ctx->side_stream) { cudaStreamSynchronize(ctx->side_stream); cudaStreamDestroy(ctx->side_stream); }
  if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
  if (ctx->ev_join) cudaEventDestroy(ctx->ev_join);
  for (cudaStream_t q : {ctx->copy_in, ctx->copy_out}) if (q) { cudaStreamSynchronize(q); cudaStreamDestroy(q); }
  for (cudaEvent_t e : {ctx->ev_u_in, ctx->ev_d_in, ctx->ev_p_in, ctx->ev_d_ready, ctx->ev_d_out}) if (e) cudaEventDestroy(e);
  if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
}

const char* tfl_last_error(const tfl_ctx* ctx) { return ctx ? ctx->err.c_str() : "no context"; }

int tfl_set_stream(tfl_ctx* ctx, void* s) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!ctx) return 1;
  TFL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (s == nullptr) {
    if (!ctx->own_stream) {
      TFL_CUDA(ctx, cudaStreamCreate(&ctx->stream));
      ctx->own_stream = true;
    }
    return 0;
  }
  if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
  ctx->stream = (cudaStream_t)s;
  ctx->own_stream = false;
  return 0;
}
void* tfl_get_stream(tfl_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }
int tfl_sync(tfl_ctx* ctx) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  TFL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return 0;
}
int64_t tfl_launch_count(const tfl_ctx* ctx) { return ctx ? ctx->launches : 0; }

int tfl_trace_faults(tfl_ctx* ctx, int64_t* count, int reset) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  unsigned long long v = 0;
  TFL_CUDA(ctx, cudaMemcpyAsync(&v, ctx->counters, sizeof(v), cudaMemcpyDeviceToHost, ctx->stream));
  TFL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (count) *count = (int64_t)v;
  if (reset) TFL_CUDA(ctx, cudaMemsetAsync(ctx->counters, 0, sizeof(v), ctx->stream));
  return 0;
}

int tfl_set_slab(tfl_ctx* ctx, int32_t z_offset, int32_t global_nz, int32_t z_lo, int32_t z_hi) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (global_nz <= 0) { ctx->slab = false; return 0; }
  ctx->slab = true;
  ctx->zoff = z_offset; ctx->gnz = global_nz; ctx->zlo = z_lo; ctx->zhi = z_hi;
  return 0;
}

int tfl_set_slab_margin(tfl_ctx* ctx, int32_t planes) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (planes < 0) return fail(ctx, "slab margin must be >= 0");
  ctx->slab_margin = planes;
  return 0;
}

int tfl_alloc(tfl_ctx* ctx, size_t bytes, void** p) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  TFL_CUDA(ctx, cudaMalloc(p, bytes));
  return 0;
}
int tfl_free(tfl_ctx* ctx, void* p) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  TFL_CUDA(ctx, cudaFree(p));
  return 0;
}
int tfl_alloc_host(tfl_ctx* ctx, size_t bytes, void** p) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  TFL_CUDA(ctx, cudaMallocHost(p, bytes));
  return 0;
}
int tfl_free_host(tfl_ctx* ctx, void* p) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  TFL_CUDA(ctx, cudaFreeHost(p));
  return 0;
}
int tfl_memcpy_h2d(tfl_ctx* ctx, void* d, const void* h, size_t bytes) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  TFL_CUDA(ctx, cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, ctx->stream));
  return 0;
}
int tfl_memcpy_d2h(tfl_ctx* ctx, void* h, const void* d, size_t bytes) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  TFL_CUDA(ctx, cudaMemcpyAsync(h, d, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  return 0;
}
int tfl_memcpy_d2d(tfl_ctx* ctx, void* dst, const void* src, size_t bytes) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  TFL_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, ctx->stream));
  return 0;
}

// ---------------------------------------------------------------------------------------
// Operators
// ---------------------------------------------------------------------------------------
int tfl_empty_domain(tfl_ctx* ctx, const tfl_grid* flags, int is_3d, int bnd) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (check_scalar(ctx, flags, "flags")) return 1;
  if (!((!is_3d || (ctx->slab ? ctx->gnz : flags->nz) >= bnd * 2 + 1) && flags->ny >= bnd * 2 + 1 &&
        flags->nx >= bnd * 2 + 1))
    return fail(ctx, "simulation domain not big enough!");       // init.lua:549-551
  Geo g;
  if (make_geo(ctx, flags, is_3d, &g)) return 1;
  launch_empty_domain(flags->data, g, bnd, ctx->stream);
  ctx->launches += 1;
  return check_launch(ctx, "emptyDomain");
}

int tfl_flags_to_occupancy(tfl_ctx* ctx, const tfl_grid* flags, const tfl_grid* occ, int64_t* bad) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (check_scalar(ctx, flags, "flags") || check_scalar(ctx, occ, "occupancy")) return 1;
  if (!same_spatial(flags, occ)) return fail(ctx, "Size mismatch");
  const long long n = (long long)flags->nb * flags->nz * flags->ny * flags->nx;
  TFL_CUDA(ctx, cudaMemsetAsync(ctx->counters + 1, 0, sizeof(unsigned long long), ctx->stream));
  launch_flags_to_occupancy(flags->data, occ->data, n, ctx->counters + 1, ctx->stream);
  ctx->launches += 1;
  if (check_launch(ctx, "flagsToOccupancy")) return 1;
  if (bad) {
    unsigned long long v = 0;
    TFL_CUDA(ctx, cudaMemcpyAsync(&v, ctx->counters + 1, sizeof(v), cudaMemcpyDeviceToHost, ctx->stream));
    TFL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *bad = (int64_t)v;
  }
  return 0;
}

int tfl_set_wall_bcs_forward(tfl_ctx* ctx, const tfl_grid* U, const tfl_grid* flags) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (check_scalar(ctx, flags, "flags") || check_vel(ctx, U, flags)) return 1;
  Geo g;
  if (make_geo(ctx, flags, U->nc == 3, &g)) return 1;
  launch_set_wall_bcs(U->data, flags->data, g, 0, ctx->stream);
  ctx->launches += 1;
  return check_launch(ctx, "setWallBcsForward");
}

int tfl_velocity_divergence_forward(tfl_ctx* ctx, const tfl_grid* U, const tfl_grid* flags,
                                    const tfl_grid* div) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (check_scalar(ctx, flags, "flags") || check_vel(ctx, U, flags) || check_scalar(ctx, div, "UDiv")) return 1;
  if (!same_spatial(flags, div)) return fail(ctx, "Size mismatch");
  Geo g;
  if (make_geo(ctx, flags, U->nc == 3, &g)) return 1;
  launch_divergence(U->data, flags->data, div->data, g, ctx->stream);
  ctx->launches += 1;
  return check_launch(ctx, "velocityDivergenceForward");
}

int tfl_velocity_update_forward(tfl_ctx* ctx, const tfl_grid* U, const tfl_grid* flags, const tfl_grid* p) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (check_scalar(ctx, flags, "flags") || check_vel(ctx, U, flags) || check_scalar(ctx, p, "p")) return 1;
  if (!same_spatial(flags, p)) return fail(ctx, "Size mismatch");
  Geo g;
  if (make_geo(ctx, flags, U->nc == 3, &g)) return 1;
  launch_velocity_update(U->data, flags->data, p->data, g, ctx->stream);
  ctx->launches += 1;
  return check_launch(ctx, "velocityUpdateForward");
}

int tfl_add_buoyancy(tfl_ctx* ctx, const tfl_grid* U, const tfl_grid* flags, const tfl_grid* density,
                     const float gravity[3], float dt) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (check_scalar(ctx, flags, "flags") || check_vel(ctx, U, flags) || check_scalar(ctx, density, "density"))
    return 1;
  if (!same_spatial(flags, density)) return fail(ctx, "Size mismatch");
  if (!gravity) return fail(ctx, "gravity must be a 3D vector (even in 2D).");
  Geo g;
  if (make_geo(ctx, flags, U->nc == 3, &g)) return 1;
  // strength = (-g) * (dt / dx), third_party/tfluids.cc:1190-1191.
  const float scale = dt / get_dx(g);
  const float s[3] = {(-gravity[0]) * scale, (-gravity[1]) * scale, (-gravity[2]) * scale};
  launch_add_buoyancy(U->data, flags->data, density->data, s, g, ctx->stream);
  ctx->launches += 1;
  return check_launch(ctx, "addBuoyancy");
}

int tfl_add_gravity(tfl_ctx* ctx, const tfl_grid* U, const tfl_grid* flags, const float gravity[3], float dt) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (check_scalar(ctx, flags, "flags") || check_vel(ctx, U, flags)) return 1;
  if (!gravity) return fail(ctx, "gravity must be a 3D vector (even in 2D).");
  Geo g;
  if (make_geo(ctx, flags, U->nc == 3, &g)) return 1;
  const float scale = dt / get_dx(g);                 // third_party/tfluids.cc:1259-1260
  const float f[3] = {gravity[0] * scale, gravity[1] * scale, gravity[2] * scale};
  launch_add_gravity(U->data, flags->data, f, g, ctx->stream);
  ctx->launches += 1;
  return check_launch(ctx, "addGravity");
}

int tfl_vorticity_confinement(tfl_ctx* ctx, const tfl_grid* U, const tfl_grid* flags, float strength) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (check_scalar(ctx, flags, "flags") || check_vel(ctx, U, flags)) return 1;
  Geo g;
  if (make_geo(ctx, flags, U->nc == 3, &g)) return 1;
  const size_t cells = (size_t)g.n * g.nb;
  if (arena_reserve(ctx, carve_bytes({cells * 3 * 4, cells * 4, cells * 3 * 4}))) return 1;
  Carver cv(ctx);
  float* curl = cv.take<float>(cells * 3);
  float* cnorm = cv.take<float>(cells);
  float* force = cv.take<float>(cells * 3);
  ctx->launches += launch_vorticity(U->data, flags->data, strength, curl, cnorm, force, g, ctx->stream);
  return check_launch(ctx, "vorticityConfinement");
}

int tfl_advect_scalar(tfl_ctx* ctx, float dt, const tfl_grid* s, const tfl_grid* U, const tfl_grid* flags,
                      int method, int sample_outside_fluid, float strength, const tfl_grid* s_dst) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (check_scalar(ctx, flags, "flags") || check_scalar(ctx, s, "s") || check_vel(ctx, U, flags)) return 1;
  if (!same_spatial(flags, s)) return fail(ctx, "Size mismatch");
  if (s_dst && (check_scalar(ctx, s_dst, "sDst") || !same_spatial(s_dst, s))) return fail(ctx, "Size mismatch");
  if (method < 0 || method > 5)
    return fail(ctx, "advection method not supported (options are: euler, maccormack, rk2Ours, rk3Ours, "
                     "eulerOurs, maccormackOurs)");
  Geo g;
  if (make_geo(ctx, flags, U->nc == 3, &g)) return 1;
  const size_t cells = (size_t)g.n * g.nb;
  const bool in_place = (s_dst == nullptr) || (s_dst->data == s->data);
  if (arena_reserve(ctx, carve_bytes({cells * 4, cells * 4 * g.nc, cells * 4}))) return 1;
  Carver cv(ctx);
  float* fwd = cv.take<float>(cells);
  float* fwd_pos = cv.take<float>(cells * g.nc);
  float* tmp = cv.take<float>(cells);
  unsigned char *fl8 = nullptr, *clear = nullptr;
  float* dst = in_place ? tmp : s_dst->data;
  Geo gf = g;     // forward pass on a wider range: its halo planes feed the backward pass
  widen_for_forward_pass(ctx, g, &gf);
  const bool traced = method == TFL_ADVECT_EULER_OURS || method == TFL_ADVECT_MACCORMACK_OURS;
  if (traced && prepare_flags(ctx, flags->data, g, &fl8, &clear)) return 1;
  const int nl = advect_scalar_dispatch(ctx, dt, s->data, U->data, flags->data, fl8, traced ? clear : nullptr, method,
                                        sample_outside_fluid, strength, dst, fwd, fwd_pos, g, gf, ctx->stream);
  if (nl < 0) return fail(ctx, "advectScalar: bad method");
  ctx->launches += nl;
  if (check_launch(ctx, "advectScalar")) return 1;
  if (in_place) {
    // s:copy(tmp) (init.lua:145-148); only the computed planes in slab mode.
    for (int b = 0; b < g.nb; b++) {
      const size_t off = (size_t)b * g.n + (size_t)g.zlo * g.ny * g.nx;
      const size_t cnt = (size_t)(g.zhi - g.zlo) * g.ny * g.nx;
      TFL_CUDA(ctx, cudaMemcpyAsync(s->data + off, tmp + off, cnt * 4, cudaMemcpyDeviceToDevice, ctx->stream));
    }
  }
  return 0;
}

int tfl_advect_vel(tfl_ctx* ctx, float dt, const tfl_grid* U, const tfl_grid* flags, int method,
                   float strength, const tfl_grid* U_dst) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (check_scalar(ctx, flags, "flags") || check_vel(ctx, U, flags)) return 1;
  if (U_dst && (check_vel(ctx, U_dst, flags) || U_dst->nc != U->nc)) return fail(ctx, "Size mismatch");
  if (method < 0 || method > 5) return fail(ctx, "advection method not supported");
  Geo g;
  if (make_geo(ctx, flags, U->nc == 3, &g)) return 1;
  const size_t cells = (size_t)g.n * g.nb;
  const bool in_place = (U_dst == nullptr) || (U_dst->data == U->data);
  if (arena_reserve(ctx, carve_bytes({cells * 4 * g.nc, cells * 4 * g.nc}))) return 1;
  Carver cv(ctx);
  float* fwd = cv.take<float>(cells * g.nc);
  float* tmp = cv.take<float>(cells * g.nc);
  unsigned char *fl8 = nullptr, *clear = nullptr;
  float* dst = in_place ? tmp : U_dst->data;
  Geo gf = g;
  widen_for_forward_pass(ctx, g, &gf);
  const bool traced = method != TFL_ADVECT_EULER && method != TFL_ADVECT_MACCORMACK;
  if (traced && prepare_flags(ctx, flags->data, g, &fl8, &clear)) return 1;
  const int nl = advect_vel_dispatch(ctx, dt, U->data, flags->data, fl8, traced ? clear : nullptr, method, strength, dst,
                                     fwd, g, gf, ctx->stream);
  if (nl < 0) return fail(ctx, "advectVel: bad method");
  ctx->launches += nl;
  if (check_launch(ctx, "advectVel")) return 1;
  if (in_place) {
    for (int b = 0; b < g.nb; b++)
      for (int c = 0; c < g.nc; c++) {
        const size_t off = ((size_t)b * g.nc + c) * g.n + (size_t)g.zlo * g.ny * g.nx;
        const size_t cnt = (size_t)(g.zhi - g.zlo) * g.ny * g.nx;
        TFL_CUDA(ctx, cudaMemcpyAsync(U->data + off, tmp + off, cnt * 4, cudaMemcpyDeviceToDevice, ctx->stream));
      }
  }
  return 0;
}

int tfl_solve_linear_system_jacobi(tfl_ctx* ctx, const tfl_grid* p, const tfl_grid* flags,
                                   const tfl_grid* div, int is_3d, float p_tol, int max_iter,
                                   float* residual, int* iterations) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (check_scalar(ctx, flags, "flags") || check_scalar(ctx, p, "p") || check_scalar(ctx, div, "div")) return 1;
  if (!same_spatial(flags, p) || !same_spatial(flags, div)) return fail(ctx, "size mismatch");
  if (!is_3d && flags->nz != 1) return fail(ctx, "d > 1 for a 2D domain");
  if (max_iter < 1) return fail(ctx, "At least 1 iteration is needed (maxIter < 1)");
  if (ctx->slab) return fail(ctx, "Jacobi on a z-slab goes through the multi-GPU driver (halo exchange per sweep)");
  Geo g;
  if (make_geo(ctx, flags, is_3d, &g)) return 1;
  const size_t cells = (size_t)g.n * g.nb;
  if (arena_reserve(ctx, carve_bytes({cells * 4, cells}))) return 1;
  Carver cv(ctx);
  float* p_prev = cv.take<float>(cells);
  unsigned char* mask = cv.take<unsigned char>(cells);
  cudaStream_t st = ctx->stream;
  launch_jacobi_mask(flags->data, mask, g, st);
  ctx->launches += 1;
  // p <- 0, pPrev <- 0 (generic/tfluids.cu:1854-1855).
  TFL_CUDA(ctx, cudaMemsetAsync(p->data, 0, cells * 4, st));
  TFL_CUDA(ctx, cudaMemsetAsync(p_prev, 0, cells * 4, st));
  float* cur = p->data;
  float* prev = p_prev;
  float res = 0.0f;
  int iter = 0;
  const bool need_every = p_tol > 0.0f;     // residual < pTol can only trigger for pTol > 0
  std::vector<double> h(g.nb);
  // A fixed number of sweeps on an L2-resident grid: all but the last inside one cooperative kernel (sweep 0
  // reads p_prev and writes p, as the loop below does); the loop then runs the last sweep and the residual.
  if (!need_every && max_iter > 2) {
    const int fused = max_iter - 1;
    if (launch_jacobi_sweeps(mask, div->data, p_prev, p->data, g, fused, st)) {
      ctx->launches += 1;
      iter = fused;
      if (fused & 1) { cur = p_prev; prev = p->data; }        // the last fused sweep wrote p
    }
  }
  for (;;) {
    launch_jacobi_iter(mask, div->data, prev, cur, g, st);
    ctx->launches += 1;
    const bool last = (iter + 1 >= max_iter);
    if (need_every || (last && residual)) {
      TFL_CUDA(ctx, cudaMemsetAsync(ctx->dscratch, 0, sizeof(double) * g.nb, st));
      launch_sqdiff(p->data, p_prev, g.n, g.nb, ctx->dscratch, st);
      ctx->launches += 1;
      TFL_CUDA(ctx, cudaMemcpyAsync(h.data(), ctx->dscratch, sizeof(double) * g.nb, cudaMemcpyDeviceToHost, st));
      TFL_CUDA(ctx, cudaStreamSynchronize(st));
      double worst = 0.0;
      for (int b = 0; b < g.nb; b++) { const double nr = sqrt(h[b]); if (nr > worst) worst = nr; }
      res = (float)worst;
      if (res < p_tol) break;
    }
    iter++;
    if (iter >= max_iter) break;
    float* t = cur; cur = prev; prev = t;
  }
  if (cur == p_prev) TFL_CUDA(ctx, cudaMemcpyAsync(p->data, p_prev, cells * 4, cudaMemcpyDeviceToDevice, st));
  if (check_launch(ctx, "solveLinearSystemJacobi")) return 1;
  if (residual) *residual = res;
  if (iterations) *iterations = iter;
  return 0;
}

int tfl_precond_from_string(const char* name) {
  if (!name) return -1;
  if (!strcmp(name, "none")) return TFL_PRECOND_NONE;
  if (!strcmp(name, "ilu0")) return TFL_PRECOND_ILU0;
  if (!strcmp(name, "ic0")) return TFL_PRECOND_IC0;
  return -1;
}

int tfl_solve_linear_system_pcg(tfl_ctx* ctx, const tfl_grid* p, const tfl_grid* flags, const tfl_grid* div,
                                int is_3d, int precond, float tol, int max_iter, float* residual,
                                int* iterations) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (check_scalar(ctx, flags, "flags") || check_scalar(ctx, p, "p") || check_scalar(ctx, div, "div")) return 1;
  if (!same_spatial(flags, p) || !same_spatial(flags, div)) return fail(ctx, "size mismatch");
  if (!is_3d && flags->nz != 1) return fail(ctx, "d > 1 for a 2D domain");
  if (precond < TFL_PRECOND_NONE || precond > TFL_PRECOND_IC0)
    return fail(ctx, "Incorrect preconType ('none', 'ic0', 'ilu0')");      // generic/tfluids.cu:1551
  if (ctx->slab) return fail(ctx, "PCG does not shard (triangular solves): single GPU only");
  if ((long long)flags->nb * flags->nz * flags->ny * flags->nx >= (1ll << 31)) return fail(ctx, "PCG: grid too large");
  if (arena_reserve(ctx, pcg_workspace_bytes(flags->nb, flags->nz, flags->ny, flags->nx))) return 1;
  const int rc = pcg_solve(ctx->pcg, ctx->arena, p->data, flags->data, div->data, flags->nb, flags->nz, flags->ny,
                           flags->nx, is_3d, precond, tol, max_iter, residual, iterations, &ctx->launches,
                           ctx->stream);
  if (rc == 3) { cudaError_t e = cudaGetLastError(); return fail(ctx, "solveLinearSystemPCG: %s", cudaGetErrorString(e)); }
  if (rc) return fail(ctx, "%s", pcg_status_string(rc));
  return check_launch(ctx, "solveLinearSystemPCG");
}

int tfl_normalize_pressure_mean(tfl_ctx* ctx, const tfl_grid* p, const tfl_grid* flags, int is_3d) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (check_scalar(ctx, flags, "flags") || check_scalar(ctx, p, "p")) return 1;
  if (!same_spatial(flags, p)) return fail(ctx, "size mismatch");
  if (!is_3d && flags->nz != 1) return fail(ctx, "d > 1 for a 2D domain");
  if (ctx->slab) return fail(ctx, "normalizePressureMean: single GPU only (connected components span the slabs)");
  if ((long long)flags->nb * flags->nz * flags->ny * flags->nx >= (1ll << 31)) return fail(ctx, "grid too large");
  if (arena_reserve(ctx, pcg_workspace_bytes(flags->nb, flags->nz, flags->ny, flags->nx))) return 1;
  if (normalize_pressure_mean(ctx->arena, p->data, flags->data, flags->nb, flags->nz, flags->ny, flags->nx, is_3d,
                              &ctx->launches, ctx->stream))
    return fail(ctx, "normalizePressureMean: %s", cudaGetErrorString(cudaGetLastError()));
  return check_launch(ctx, "normalizePressureMean");
}

int tfl_volumetric_up_sampling_nearest_forward(tfl_ctx* ctx, int ratio, const tfl_grid* in, const tfl_grid* out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!in || !out || !in->data || !out->data) return fail(ctx, "ERROR: input and output must be dim 5");
  if (ratio < 1) return fail(ctx, "ratio must be a positive integer");
  if (out->nb != in->nb || out->nc != in->nc || out->nz != in->nz * ratio || out->ny != in->ny * ratio ||
      out->nx != in->nx * ratio)
    return fail(ctx, "ERROR: input : output size mismatch.");             // generic/tfluids.cc:528-532
  launch_upsample_nearest(in->data, out->data, in->nb * in->nc, in->nz, in->ny, in->nx, ratio, ctx->stream);
  ctx->launches += 1;
  return check_launch(ctx, "volumetricUpSamplingNearestForward");
}

int tfl_rectangular_blur(tfl_ctx* ctx, const tfl_grid* src, int blur_rad, int is_3d, const tfl_grid* dst) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!src || !dst || !src->data || !dst->data) return fail(ctx, "ERROR: src and dst must be dim 5");
  if (!same_spatial(src, dst) || src->nc != dst->nc) return fail(ctx, "size mismatch");
  if (blur_rad <= 0) return fail(ctx, "blurRad must be a positive, non-zero integer");   // init.lua:586-587
  if (src->data == dst->data) return fail(ctx, "rectangularBlur: dst must not alias src");
  const size_t cells = (size_t)src->nb * src->nc * src->nz * src->ny * src->nx;
  if (arena_reserve(ctx, carve_bytes({cells * 4}))) return 1;
  Carver cv(ctx);
  float* tmp = cv.take<float>(cells);
  const int nbf = src->nb * src->nc;
  cudaStream_t st = ctx->stream;
  // generic/tfluids.cc:700-757: z into dst (3-D), y into tmp, x into dst.
  const float* cur = src->data;
  if (is_3d) {
    launch_blur_axis(cur, dst->data, nbf, src->nz, src->ny, src->nx, 2, blur_rad, st);
    cur = dst->data;
    ctx->launches += 1;
  }
  launch_blur_axis(cur, tmp, nbf, src->nz, src->ny, src->nx, 1, blur_rad, st);
  launch_blur_axis(tmp, dst->data, nbf, src->nz, src->ny, src->nx, 0, blur_rad, st);
  ctx->launches += 2;
  return check_launch(ctx, "rectangularBlur");
}

int tfl_signed_distance_field(tfl_ctx* ctx, const tfl_grid* flags, int search_rad, int is_3d, const tfl_grid* dst) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (check_scalar(ctx, flags, "flags") || check_scalar(ctx, dst, "dst")) return 1;
  if (!same_spatial(flags, dst)) return fail(ctx, "size mismatch");
  if (search_rad <= 0) return fail(ctx, "searchRad must be a positive, non-zero integer");   // init.lua:609-610
  if (!is_3d && flags->nz != 1) return fail(ctx, "d > 1 for a 2D domain");
  launch_signed_distance_field(flags->data, dst->data, flags->nb, flags->nz, flags->ny, flags->nx, search_rad,
                               ctx->stream);
  ctx->launches += 1;
  return check_launch(ctx, "signedDistanceField");
}

int tfl_velocity_divergence_backward(tfl_ctx* ctx, const tfl_grid* U, const tfl_grid* flags, const tfl_grid* go,
                                     const tfl_grid* gU) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (check_scalar(ctx, flags, "flags") || check_vel(ctx, U, flags) || check_scalar(ctx, go, "gradOutput")) return 1;
  if (!gU || !gU->data || gU->nc != U->nc || !same_spatial(gU, U) || !same_spatial(go, flags)) return fail(ctx, "Size mismatch");
  if (ctx->slab) return fail(ctx, "backward operators: single GPU only");
  launch_velocity_divergence_backward(flags->data, go->data, gU->data, flags->nb, flags->nz, flags->ny, flags->nx,
                                      U->nc == 3, ctx->stream);
  ctx->launches += 1;
  return check_launch(ctx, "velocityDivergenceBackward");
}

int tfl_velocity_update_backward(tfl_ctx* ctx, const tfl_grid* U, const tfl_grid* flags, const tfl_grid* p,
                                 const tfl_grid* go, const tfl_grid* gp) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (check_scalar(ctx, flags, "flags") || check_vel(ctx, U, flags) || check_scalar(ctx, p, "p") ||
      check_scalar(ctx, gp, "gradP"))
    return 1;
  if (!go || !go->data || go->nc != U->nc || !same_spatial(go, U) || !same_spatial(gp, p) || !same_spatial(p, flags))
    return fail(ctx, "Size mismatch");
  if (ctx->slab) return fail(ctx, "backward operators: single GPU only");
  launch_velocity_update_backward(flags->data, go->data, gp->data, flags->nb, flags->nz, flags->ny, flags->nx,
                                  U->nc == 3, ctx->stream);
  ctx->launches += 1;
  return check_launch(ctx, "velocityUpdateBackward");
}

int tfl_volumetric_up_sampling_nearest_backward(tfl_ctx* ctx, int ratio, const tfl_grid* in, const tfl_grid* go,
                                                const tfl_grid* gi) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!in || !go || !gi || !in->data || !go->data || !gi->data)
    return fail(ctx, "ERROR: input, gradOutput and gradInput must be dim 5");
  if (ratio < 1) return fail(ctx, "ratio must be a positive integer");
  if (go->nb != in->nb || go->nc != in->nc || go->nz != in->nz * ratio || go->ny != in->ny * ratio ||
      go->nx != in->nx * ratio)
    return fail(ctx, "ERROR: input : gradOutput size mismatch.");          // generic/tfluids.cc:584-590
  if (!same_spatial(gi, in) || gi->nc != in->nc) return fail(ctx, "ERROR: input : gradInput size mismatch.");
  launch_upsample_nearest_backward(go->data, gi->data, in->nb * in->nc, in->nz, in->ny, in->nx, ratio, ctx->stream);
  ctx->launches += 1;
  return check_launch(ctx, "volumetricUpSamplingNearestBackward");
}

// Debug hook (not in include/tfl.h): planes per CTA of the PCG sweep pipeline.
extern "C" int tfl_debug_pcg_groups(tfl_ctx* ctx, int groups) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!ctx) return 1;
  ctx->pcg.groups_override = groups;
  return 0;
}

extern "C" int tfl_debug_pcg_timing(tfl_ctx* ctx, void* dev_buf) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!ctx) return 1;
  ctx->pcg.debug_timing = dev_buf;
  return 0;
}

int tfl_apply_bc(tfl_ctx* ctx, const tfl_grid* x, const tfl_grid* inv_mask, const tfl_grid* bc) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!x || !inv_mask || !bc || !x->data || !inv_mask->data || !bc->data) return fail(ctx, "applyBC: nil tensor");
  if (!same_spatial(x, inv_mask) || !same_spatial(x, bc) || x->nc != inv_mask->nc || x->nc != bc->nc)
    return fail(ctx, "Size mismatch");
  if (ctx->slab) {                // the planes this rank computes; ghost planes come from the neighbours
    if (ctx->zlo < 0 || ctx->zhi > x->nz || ctx->zlo >= ctx->zhi) return fail(ctx, "applyBC: slab range does not fit");
    const long long plane = (long long)x->ny * x->nx, cnt = (long long)(ctx->zhi - ctx->zlo) * plane;
    for (int bc_i = 0; bc_i < x->nb * x->nc; bc_i++) {
      const long long off = ((long long)bc_i * x->nz + ctx->zlo) * plane;
      launch_apply_bc(x->data + off, inv_mask->data + off, bc->data + off, cnt, ctx->stream);
    }
    ctx->launches += x->nb * x->nc;
    return check_launch(ctx, "applyBC");
  }
  const long long n = (long long)x->nb * x->nc * x->nz * x->ny * x->nx;
  launch_apply_bc(x->data, inv_mask->data, bc->data, n, ctx->stream);
  ctx->launches += 1;
  return check_launch(ctx, "applyBC");
}

int tfl_clamp(tfl_ctx* ctx, const tfl_grid* x, float lo, float hi) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!x || !x->data) return fail(ctx, "clamp: nil tensor");
  if (ctx->slab) {
    if (ctx->zlo < 0 || ctx->zhi > x->nz || ctx->zlo >= ctx->zhi) return fail(ctx, "clamp: slab range does not fit");
    const long long plane = (long long)x->ny * x->nx, cnt = (long long)(ctx->zhi - ctx->zlo) * plane;
    for (int bc_i = 0; bc_i < x->nb * x->nc; bc_i++)
      launch_clamp(x->data + ((long long)bc_i * x->nz + ctx->zlo) * plane, lo, hi, cnt, ctx->stream);
    ctx->launches += x->nb * x->nc;
    return check_launch(ctx, "clamp");
  }
  const long long n = (long long)x->nb * x->nc * x->nz * x->ny * x->nx;
  launch_clamp(x->data, lo, hi, n, ctx->stream);
  ctx->launches += 1;
  return check_launch(ctx, "clamp");
}

// ---------------------------------------------------------------------------------------
// CNN projection
// ---------------------------------------------------------------------------------------
int tfl_cnn_create(tfl_ctx* ctx, int is_3d, int n_layers, const int32_t* cin, const int32_t* cout,
                   const int32_t* ksize, const float* const* weights, const float* const* biases,
                   tfl_cnn** out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  return tfl_cnn_create_graph(ctx, is_3d, n_layers, cin, cout, ksize, nullptr, nullptr, 0, 0, weights, biases, out);
}

int tfl_cnn_create_graph(tfl_ctx* ctx, int is_3d, int n_layers, const int32_t* cin, const int32_t* cout_logical,
                         const int32_t* ksize, const int32_t* pool, const int32_t* up, int pool_is_max,
                         int nonlin_sigmoid, const float* const* weights, const float* const* biases,
                         tfl_cnn** out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!out || n_layers < 1) return fail(ctx, "cnn: bad arguments");
  // Channels the convolution of layer l really emits: cout * up^d (ConvolutionUpsample, model_utils.lua:74-76).
  std::vector<int32_t> cout_conv(n_layers);
  bool plain = !nonlin_sigmoid;
  for (int l = 0; l < n_layers; l++) {
    const int u = up ? up[l] : 1, pl = pool ? pool[l] : 1;
    if (u < 1 || pl < 1) return fail(ctx, "cnn: pooling / upsampling sizes must be >= 1");
    if (u > 1 && pl > 1) return fail(ctx, "Pooling and upsampling in the same layer!");          // model.lua:326
    if (l == n_layers - 1 && pl != 1) return fail(ctx, "Pooling is not allowed in the last layer");  // model.lua:245
    cout_conv[l] = cout_logical[l] * u * u * (is_3d ? u : 1);
    if (u != 1 || pl != 1) plain = false;
  }
  const int32_t* cout = cout_conv.data();
  if (cout_logical[n_layers - 1] != 1) return fail(ctx, "Last layer osize must be 1 (pressure)");   // model.lua:244
  if (cin[0] != 3) return fail(ctx, "cnn: the first layer must take 3 channels (pDiv, div, occupancy)");
  tfl_cnn* m = new tfl_cnn();
  m->plain = plain;
  m->pool_is_max = pool_is_max ? 1 : 0;
  m->nonlin = nonlin_sigmoid ? 2 : 1;
  m->is3d = is_3d ? 1 : 0;
  m->n_layers = n_layers;
  for (int l = 0; l < n_layers; l++) {
    if (l > 0 && cin[l] != cout_logical[l - 1]) { delete m; return fail(ctx, "cnn: channel mismatch at layer %d", l); }
    m->pool.push_back(pool ? pool[l] : 1);
    m->up.push_back(up ? up[l] : 1);
    if (ksize[l] % 2 != 1) { delete m; return fail(ctx, "convolution size must be odd"); }   // model_utils.lua:70
    const int kz = is_3d ? ksize[l] : 1;
    const int taps = kz * ksize[l] * ksize[l];
    std::vector<float> relaid((size_t)cin[l] * taps * cout[l]);
    for (int o = 0; o < cout[l]; o++)
      for (int c = 0; c < cin[l]; c++)
        for (int t = 0; t < taps; t++)
          relaid[((size_t)c * taps + t) * cout[l] + o] = weights[l][((size_t)o * cin[l] + c) * taps + t];
    float *dw = nullptr, *db = nullptr;
    if (cudaMalloc((void**)&dw, relaid.size() * 4) != cudaSuccess ||
        cudaMalloc((void**)&db, cout[l] * 4) != cudaSuccess) { delete m; return fail(ctx, "cnn: cudaMalloc failed"); }
    cudaMemcpy(dw, relaid.data(), relaid.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(db, biases[l], cout[l] * 4, cudaMemcpyHostToDevice);
    m->cin.push_back(cin[l]); m->cout.push_back(cout[l]); m->ks.push_back(ksize[l]);
    m->w.push_back(dw); m->b.push_back(db);
    if (cout[l] > m->max_c) m->max_c = cout[l];
  }
  {   // largest activation of the graph, in channels x cells-of-the-input-grid
    double rel = 1.0;
    m->max_rel = 3.0;
    for (int l = 0; l < n_layers; l++) {
      m->max_rel = std::max(m->max_rel, rel * cout[l]);                          // convolution output
      const int u = m->up[l], pl = m->pool[l];
      rel *= (double)u * u * (is_3d ? u : 1);
      m->max_rel = std::max(m->max_rel, rel * cout_logical[l]);                  // after the pixel shuffle
      rel /= (double)pl * pl * (is_3d ? pl : 1);
    }
    if (rel != 1.0) { tfl_cnn_destroy(ctx, m); return fail(ctx, "cnn: pooling and upsampling do not return to the input resolution"); }
    if ((double)m->max_c < m->max_rel) m->max_c = (int)std::ceil(m->max_rel);
  }
  // Tensor-core eligibility: the 3-D 'default' graph (lib/model.lua:219-226).
  static const int want[5][3] = {{3, 8, 3}, {8, 8, 3}, {8, 8, 3}, {8, 8, 1}, {8, 1, 1}};
  m->tc_ok = plain && is_3d && n_layers == 5;
  for (int l = 0; m->tc_ok && l < 5; l++)
    m->tc_ok = cin[l] == want[l][0] && cout[l] == want[l][1] && ksize[l] == want[l][2];
  if (m->tc_ok) {
    for (int split = 0; split < 2; split++)
      for (int l = 0; l < 3; l++) {
        std::vector<float> packed(conv_tc_b_floats(split));
        conv_tc_pack_weights(weights[l], cin[l], split, packed.data());
        cudaMalloc((void**)&m->wB[split][l], packed.size() * 4);
        cudaMemcpy(m->wB[split][l], packed.data(), packed.size() * 4, cudaMemcpyHostToDevice);
      }
    std::vector<float> tail(64 + 8 + 8 + 1);
    memcpy(tail.data(), weights[3], 64 * 4);
    memcpy(tail.data() + 64, biases[3], 8 * 4);
    memcpy(tail.data() + 72, weights[4], 8 * 4);
    tail[80] = biases[4][0];
    cudaMalloc((void**)&m->tail, tail.size() * 4);
    cudaMemcpy(m->tail, tail.data(), tail.size() * 4, cudaMemcpyHostToDevice);
    m->mode = 2;
  }
  *out = m;
  return 0;
}

int tfl_cnn_set_mode(tfl_ctx* ctx, tfl_cnn* m, int mode) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!m || mode < 0 || mode > 2) return fail(ctx, "cnn_set_mode: bad arguments");
  if (mode > 0 && !m->tc_ok)
    return fail(ctx, "cnn_set_mode: the tensor-core path covers the 3-D 'default' architecture only");
  m->mode = mode;
  return 0;
}
int tfl_cnn_get_mode(const tfl_cnn* m) { return m ? m->mode : -1; }
// Undocumented debugging hook.
// mode: -1 automatic, 0 two-kernel advectVel, 1 / 2 tile kernel with that halo; variant: tile shape.
int tfl_debug_advect_tile(tfl_ctx* ctx, int mode, int variant) {
  if (!ctx) return 1;
  ctx->tile.mode = mode;
  ctx->tile.variant = variant;
  return 0;
}

// Events around the advectVel tile kernel alone (bench.py's roofline).  on: start recording; the getter
// synchronises and returns the duration of the last recorded launch in ms (< 0 if none).
int tfl_debug_time_advect_kernel(tfl_ctx* ctx, int on) {
  if (!ctx) return 1;
  DeviceGuard guard_(ctx);
  auto& tl = ctx->tile;
  if (on && !tl.ev0) { cudaEventCreate(&tl.ev0); cudaEventCreate(&tl.ev1); }
  tl.timed = on != 0 && tl.ev0 && tl.ev1;
  return 0;
}
float tfl_debug_last_advect_kernel_ms(tfl_ctx* ctx) {
  if (!ctx || !ctx->tile.ev0) return -1.0f;
  DeviceGuard guard_(ctx);
  float ms = -1.0f;
  if (cudaEventSynchronize(ctx->tile.ev1) != cudaSuccess || cudaEventElapsedTime(&ms, ctx->tile.ev0, ctx->tile.ev1) != cudaSuccess) {
    cudaGetLastError();
    return -1.0f;
  }
  return ms;
}

// Undocumented debugging hook (not in tfl.h): per-CTA phase timestamps of the tensor-core conv.
int tfl_debug_conv_timestamps(void* dev_buf) { conv_tc_set_debug((long long*)dev_buf); return 0; }

void tfl_cnn_destroy(tfl_ctx* ctx, tfl_cnn* m) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!m) return;
  if (ctx) cudaStreamSynchronize(ctx->stream);
  for (float* p : m->w) cudaFree(p);
  for (float* p : m->b) cudaFree(p);
  for (int sp = 0; sp < 2; sp++)
    for (int l = 0; l < 3; l++)
      if (m->wB[sp][l]) cudaFree(m->wB[sp][l]);
  if (m->tail) cudaFree(m->tail);
  for (float* p : m->act)
    if (p) cudaFree(p);
  delete m;
}

// Tensor-core path: padded channels-last activations owned by the model (their zero borders
// must survive between calls, so they do not live in the shared arena).
static int cnn_ensure_act(tfl_ctx* ctx, tfl_cnn* m, const Geo& g) {
  if (m->act_geo.nb == g.nb && m->act_geo.nz == g.nz && m->act_geo.ny == g.ny && m->act_geo.nx == g.nx) return 0;
  TFL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  m->act_geo = make_conv_tc_geo(g.nb, g.nz, g.ny, g.nx);
  for (int i = 0; i < 3; i++) {
    if (m->act[i]) cudaFree(m->act[i]);
    m->act[i] = nullptr;
    TFL_CUDA(ctx, cudaMalloc((void**)&m->act[i], conv_tc_act_bytes(m->act_geo)));
    TFL_CUDA(ctx, cudaMemset(m->act[i], 0, conv_tc_act_bytes(m->act_geo)));
  }
  return 0;
}

// The three 3x3x3 layers (+ fused 1x1x1 tail) on tensor cores: act[0] -> act[1] -> act[2] -> p_net.
// p_lo / p_hi: planes on which p_net is wanted (default all).  Layer l then only has to produce the planes the
// later layers' 3x3x3 stencils reach from there; on a z-slab that spares most of the ghost planes.
static void run_conv_stack(tfl_cnn* m, float* p_net, cudaStream_t st, int p_lo = 0, int p_hi = -1) {
  const ConvTcGeo& tg = m->act_geo;
  if (p_hi < 0) p_hi = tg.nz;
  const int split = m->mode == 2 ? 1 : 0;
  ConvTcGeo g1 = tg, g2 = tg, g3 = tg;
  g3.z_lo = std::max(0, p_lo);     g3.z_hi = std::min(tg.nz, p_hi);
  g2.z_lo = std::max(0, p_lo - 1); g2.z_hi = std::min(tg.nz, p_hi + 1);
  g1.z_lo = std::max(0, p_lo - 2); g1.z_hi = std::min(tg.nz, p_hi + 2);
  launch_conv3_tc(m->act[0], m->act[1], nullptr, m->wB[split][0], m->b[0], nullptr, 1, 0, split, g1, st);
  launch_conv3_tc(m->act[1], m->act[2], nullptr, m->wB[split][1], m->b[1], nullptr, 2, 0, split, g2, st);
  launch_conv3_tc(m->act[2], nullptr, p_net, m->wB[split][2], m->b[2], m->tail, 2, 1, split, g3, st);
}

static int cnn_project_impl(tfl_ctx* ctx, tfl_cnn* m, const float* p_div, const float* U_div,
                            const float* flags, float* p_out, float* U_out, float threshold, const Geo& g,
                            char* scratch, float** scale_dev_out) {
  // scratch layout (caller reserved): U1 [nc], x0 [3], actA [max_c], actB [max_c], scale [nb]
  const size_t cells = (size_t)g.n * g.nb;
  size_t off = 0;
  auto take = [&](size_t bytes) { char* p = scratch + off; off = (off + bytes + 255) & ~(size_t)255; return p; };
  float* U1 = (float*)take(cells * 4 * g.nc);
  float* x0 = (float*)take(cells * 4 * 3);
  float* actA = (float*)take(cells * 4 * m->max_c);      // max_c covers max_rel (set at creation)
  float* actB = (float*)take(cells * 4 * m->max_c);
  float* scale = (float*)take(sizeof(float) * g.nb);
  double* sums = ctx->dscratch + 64;
  cudaStream_t st = ctx->stream;
  TFL_CUDA(ctx, cudaMemsetAsync(sums, 0, sizeof(double) * 2 * g.nb, st));
  launch_cnn_mask_stats(U_div, flags, U1, sums, g.zlo, g.zhi, g, st);
  launch_cnn_scale(sums, scale, g.nb, (long long)g.nc * g.n, threshold, st);
  if (m->mode > 0 && m->tc_ok && !ctx->slab) {
    if (cnn_ensure_act(ctx, m, g)) return 1;
    const ConvTcGeo& tg = m->act_geo;
    launch_cnn_inputs_padded(p_div, U1, flags, scale, m->act[0], tg.px, tg.py, g, st);
    float* p_net = actA;      // plain [b][z][y][x]
    run_conv_stack(m, p_net, st);
    launch_cnn_finish(p_net, U1, flags, scale, p_out, U_out, g, st);
    ctx->launches += 7;
    if (scale_dev_out) *scale_dev_out = scale;
    return check_launch(ctx, "cnn_project (tensor cores)");
  }
  launch_cnn_inputs(p_div, U1, flags, scale, x0, g, st);
  ctx->launches += 3;
  const float* in = x0;
  if (m->plain) {
    float* bufs[2] = {actA, actB};
    for (int l = 0; l < m->n_layers; l++) {
      float* o = bufs[l & 1];
      const int act = (l < m->n_layers - 1) ? 1 : 0;
      if (launch_conv_direct(in, o, m->w[l], m->b[l], m->cin[l], m->cout[l], m->ks[l], act, g, st) < 0)
        return fail(ctx, "cnn: unsupported layer shape cout=%d k=%d", m->cout[l], m->ks[l]);
      ctx->launches += 1;
      in = o;
    }
  } else {
    // 'tog' / 'yang' graphs: conv (+ pixel shuffle) -> non-linearity -> pooling, layer by layer, on grids
    // whose resolution follows the pooling / upsampling sizes (lib/model.lua:262-340, single bank).
    if (ctx->slab) return fail(ctx, "cnn: pooled / upsampled graphs run on whole grids only");
    float* bufs[3] = {actA, actB, (float*)take((size_t)((double)cells * m->max_rel + 64) * 4)};
    auto other = [&](const float* a, const float* b2) {
      for (float* c : bufs) if (c != a && c != b2) return c;
      return bufs[0];
    };
    Geo gl = g;
    for (int l = 0; l < m->n_layers; l++) {
      const int u = m->up[l], pl = m->pool[l];
      const int act = (l < m->n_layers - 1) ? m->nonlin : 0;     // element-wise: commutes with the shuffle
      float* o = other(in, nullptr);
      if (launch_conv_direct(in, o, m->w[l], m->b[l], m->cin[l], m->cout[l], m->ks[l], act, gl, st) < 0)
        return fail(ctx, "cnn: unsupported layer shape cout=%d k=%d", m->cout[l], m->ks[l]);
      ctx->launches += 1;
      const float* cur = o;
      int chans = m->cout[l];
      if (u > 1) {
        chans = m->cout[l] / (u * u * (gl.is3d ? u : 1));
        float* sh = other(cur, nullptr);
        launch_pixel_shuffle(cur, sh, gl.nb, chans, gl.nz, gl.ny, gl.nx, u, gl.is3d, st);
        ctx->launches += 1;
        gl.nx *= u; gl.ny *= u; if (gl.is3d) gl.nz *= u;
        cur = sh;
      }
      if (pl > 1) {
        if (gl.nx % pl || gl.ny % pl || (gl.is3d && gl.nz % pl))
          return fail(ctx, "cnn: grid %dx%dx%d is not divisible by the pooling size %d", gl.nx, gl.ny, gl.nz, pl);
        float* po = other(cur, nullptr);
        launch_pool(cur, po, gl.nb * chans, gl.nz, gl.ny, gl.nx, pl, gl.is3d, m->pool_is_max, st);
        ctx->launches += 1;
        gl.nx /= pl; gl.ny /= pl; if (gl.is3d) gl.nz /= pl;
        cur = po;
      }
      gl.n = (long long)gl.nx * gl.ny * gl.nz;
      gl.gnz = gl.nz; gl.zlo = 0; gl.zhi = gl.nz;
      in = cur;
    }
    if (gl.nx != g.nx || gl.ny != g.ny || gl.nz != g.nz) return fail(ctx, "cnn: graph does not return to the input resolution");
  }
  launch_cnn_finish(in, U1, flags, scale, p_out, U_out, g, st);
  ctx->launches += 1;
  if (scale_dev_out) *scale_dev_out = scale;
  return check_launch(ctx, "cnn_project");
}

static size_t cnn_scratch_bytes(const tfl_cnn* m, const Geo& g) {
  const size_t cells = (size_t)g.n * g.nb;
  size_t bytes = cells * 4 * (g.nc + 3 + 2 * (size_t)m->max_c) + 4 * g.nb + 8 * 256;
  if (!m->plain) bytes += (size_t)((double)cells * m->max_rel + 64) * 4 + 256;     // third rotating buffer
  return bytes;
}

int tfl_cnn_project(tfl_ctx* ctx, tfl_cnn* m, const tfl_grid* p_div, const tfl_grid* U_div,
                    const tfl_grid* flags, const tfl_grid* p_out, const tfl_grid* U_out, float threshold,
                    float* scale_out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!m) return fail(ctx, "cnn is nil");
  if (check_scalar(ctx, flags, "flags") || check_scalar(ctx, p_div, "pDiv") || check_vel(ctx, U_div, flags) ||
      check_scalar(ctx, p_out, "p") || check_vel(ctx, U_out, flags))
    return 1;
  if (!same_spatial(flags, p_div) || !same_spatial(flags, p_out) || U_out->nc != U_div->nc)
    return fail(ctx, "Size mismatch");
  if ((U_div->nc == 3) != (m->is3d != 0)) return fail(ctx, "model / data dimensionality mismatch");
  if (ctx->slab) return fail(ctx, "cnn_project on a z-slab goes through the multi-GPU driver");
  Geo g;
  if (make_geo(ctx, flags, m->is3d, &g)) return 1;
  if (arena_reserve(ctx, cnn_scratch_bytes(m, g))) return 1;
  float* scale_dev = nullptr;
  if (cnn_project_impl(ctx, m, p_div->data, U_div->data, flags->data, p_out->data, U_out->data, threshold, g,
                       ctx->arena, &scale_dev))
    return 1;
  if (scale_out) {
    TFL_CUDA(ctx, cudaMemcpyAsync(scale_out, scale_dev, sizeof(float) * g.nb, cudaMemcpyDeviceToHost, ctx->stream));
    TFL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  return 0;
}

// z-slab variant of model:forward, split around the one global reduction (the input scale):
//   tfl_cnn_stats              U1 = SetWallBcs mask * U on every local plane where the mask is
//                              computable, and (sum, sum of squares) over the OWNED planes into
//                              dev_sums[2 * nb] (device doubles the caller all-reduces, e.g. with NCCL);
//   tfl_cnn_project_from_sums  everything after the reduction.  The conv stack runs on the whole
//                              local slab (halo planes included), so results are valid on planes at
//                              least 4 planes away from a local end that is not a global end.
int tfl_cnn_stats(tfl_ctx* ctx, const tfl_grid* U_div, const tfl_grid* flags, const tfl_grid* U1,
                  double* dev_sums) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (check_scalar(ctx, flags, "flags") || check_vel(ctx, U_div, flags) || check_vel(ctx, U1, flags)) return 1;
  if (!dev_sums) return fail(ctx, "cnn_stats: nil sums");
  Geo g;
  if (make_geo(ctx, flags, U_div->nc == 3, &g)) return 1;
  Geo gw = g;
  if (ctx->slab) {
    gw.zlo = (g.zoff == 0) ? 0 : 1;
    gw.zhi = (g.zoff + g.nz == g.gnz) ? g.nz : g.nz - 1;
  }
  TFL_CUDA(ctx, cudaMemsetAsync(dev_sums, 0, sizeof(double) * 2 * g.nb, ctx->stream));
  launch_cnn_mask_stats(U_div->data, flags->data, U1->data, dev_sums, g.zlo, g.zhi, gw, ctx->stream);
  ctx->launches += 1;
  return check_launch(ctx, "cnn_stats");
}

int tfl_cnn_project_from_sums(tfl_ctx* ctx, tfl_cnn* m, const tfl_grid* p_div, const tfl_grid* U1,
                              const tfl_grid* flags, const double* dev_sums, const tfl_grid* p_out,
                              const tfl_grid* U_out, float threshold) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!m) return fail(ctx, "cnn is nil");
  if (!m->tc_ok || m->mode == 0) return fail(ctx, "cnn_project_from_sums needs the tensor-core path (3-D default net)");
  if (check_scalar(ctx, flags, "flags") || check_scalar(ctx, p_div, "pDiv") || check_vel(ctx, U1, flags) ||
      check_scalar(ctx, p_out, "p") || check_vel(ctx, U_out, flags))
    return 1;
  Geo g;
  if (make_geo(ctx, flags, 1, &g)) return 1;
  if (cnn_ensure_act(ctx, m, g)) return 1;
  const size_t cells = (size_t)g.n * g.nb;
  if (arena_reserve(ctx, carve_bytes({cells * 4, 4 * (size_t)g.nb}))) return 1;
  Carver cv(ctx);
  float* p_net = cv.take<float>(cells);
  float* scale = cv.take<float>(g.nb);
  cudaStream_t st = ctx->stream;
  // scale from the (already reduced) sums; the sample count is that of the GLOBAL grid.
  launch_cnn_scale(dev_sums, scale, g.nb, (long long)g.nc * g.nx * g.ny * g.gnz, threshold, st);
  Geo gi = g;            // the divergence reads U1 one plane up
  if (ctx->slab) {
    gi.zlo = (g.zoff == 0) ? 0 : 1;
    gi.zhi = (g.zoff + g.nz == g.gnz) ? g.nz : g.nz - 2;
  }
  const ConvTcGeo& tg = m->act_geo;
  launch_cnn_inputs_padded(p_div->data, U1->data, flags->data, scale, m->act[0], tg.px, tg.py, gi, st);
  // the velocity update of the computed planes [zlo, zhi) reads p on [zlo - 1, zhi)
  if (ctx->slab) run_conv_stack(m, p_net, st, g.zlo - 1, g.zhi);
  else run_conv_stack(m, p_net, st);
  launch_cnn_finish(p_net, U1->data, flags->data, scale, p_out->data, U_out->data, g, st);
  ctx->launches += 6;
  return check_launch(ctx, "cnn_project_from_sums");
}

// ---------------------------------------------------------------------------------------
// tfluids.simulate (lib/simulate.lua:175-327)
// ---------------------------------------------------------------------------------------
static int set_const_vals(tfl_ctx* ctx, const tfl_state* s) {       // lib/simulate.lua:130-160
  if (s->p_bc.data && s->p_bc_inv_mask.data && tfl_apply_bc(ctx, &s->p, &s->p_bc_inv_mask, &s->p_bc)) return 1;
  if (s->U_bc.data && s->U_bc_inv_mask.data && tfl_apply_bc(ctx, &s->U, &s->U_bc_inv_mask, &s->U_bc)) return 1;
  if (s->density.data && s->density_bc.data && s->density_bc_inv_mask.data &&
      tfl_apply_bc(ctx, &s->density, &s->density_bc_inv_mask, &s->density_bc))
    return 1;
  return 0;
}

// Fused pipeline for the convnet path with the tensor-core conv stack: 12 launches, every
// field crosses memory once per stage.  Bit-identical to the operator sequence below.
static int simulate_step_fused(tfl_ctx* ctx, const tfl_state* s, const tfl_mconf* mc, tfl_cnn* m, const Geo& g) {
  const size_t cells = (size_t)g.n * g.nb;
  const bool has_density = s->density.data != nullptr;
  if (cnn_ensure_act(ctx, m, g)) return 1;
  if (arena_reserve(ctx, carve_bytes({cells * 4, cells * 4 * g.nc, cells * 4, cells * 4 * g.nc, cells * 4 * g.nc,
                                      cells * 12, cells * 4, cells * 4, 4 * (size_t)g.nb, cells * 12, cells / 4 + 64})))
    return 1;
  Carver cv(ctx);
  float* fwd_s = cv.take<float>(cells);
  float* fwd_pos = cv.take<float>(cells * g.nc);
  float* tmp_s = cv.take<float>(cells);
  float* fwd_u = cv.take<float>(cells * g.nc);
  float* tmp_u = cv.take<float>(cells * g.nc);
  float* curl = cv.take<float>(cells * 3);
  float* cnorm = cv.take<float>(cells);
  float* p_net = cv.take<float>(cells);
  float* scale = cv.take<float>(g.nb);
  float* force = cv.take<float>(cells * 3);
  unsigned char* qmask_buf = cv.take<unsigned char>(cells / 4 + 64);
  cudaStream_t st = ctx->stream;
  // Byte copy of the flags for this step (every bit the kernels test is below 256) and, when a byte
  // differs from the previous step's copy, the clearance field of the advection fast path.
  unsigned char *fl8 = nullptr, *clear = nullptr;
  if (prepare_flags(ctx, s->flags.data, g, &fl8, &clear)) return 1;
  const bool ov = ctx->ov.active;
  if (ov) TFL_CUDA(ctx, cudaStreamWaitEvent(st, ctx->ev_u_in, 0));          // U has arrived from the host
  // Which quads of the BC arrays are the identity pair (the point-wise stages then skip their loads): rebuilt
  // every step from the arrays, beside the advection (on the side stream when there is one).
  const unsigned char* qmask = nullptr;
  const bool u_bc0 = s->U_bc.data && s->U_bc_inv_mask.data;
  const bool d_bc0 = has_density && s->density_bc.data && s->density_bc_inv_mask.data;
  bool qmask_on_side = false;
  if (has_density) {
    // Density and velocity advection are independent (both read the old U): run the density
    // kernels on a side stream so the two latency-bound kernel pairs overlap.
    TFL_CUDA(ctx, cudaEventRecord(ctx->ev_fork, st));
    TFL_CUDA(ctx, cudaStreamWaitEvent(ctx->side_stream, ctx->ev_fork, 0));
    if (launch_bc_quad_mask(u_bc0 ? s->U_bc_inv_mask.data : nullptr, u_bc0 ? s->U_bc.data : nullptr,
                            d_bc0 ? s->density_bc_inv_mask.data : nullptr, d_bc0 ? s->density_bc.data : nullptr,
                            qmask_buf, g, ctx->side_stream)) {
      qmask = qmask_buf;
      qmask_on_side = true;
      ctx->launches += 1;
    }
    if (ov) TFL_CUDA(ctx, cudaStreamWaitEvent(ctx->side_stream, ctx->ev_d_in, 0));
    const int nl = advect_scalar_dispatch(ctx, mc->dt, s->density.data, s->U.data, fl8, fl8, clear, mc->advection_method,
                                          0, mc->maccormack_strength, tmp_s, fwd_s, fwd_pos, g, g, ctx->side_stream);
    if (nl < 0) return fail(ctx, "advectScalar: bad method");
    ctx->launches += nl;
    TFL_CUDA(ctx, cudaEventRecord(ctx->ev_join, ctx->side_stream));
  }
  {
    const int nl = advect_vel_dispatch(ctx, mc->dt, s->U.data, fl8, fl8, clear, mc->advection_method,
                                       mc->maccormack_strength, tmp_u, fwd_u, g, g, st);
    if (nl < 0) return fail(ctx, "advectVel: bad method");
    ctx->launches += nl;
  }
  if (has_density) TFL_CUDA(ctx, cudaStreamWaitEvent(st, ctx->ev_join, 0));
  if (!qmask_on_side && launch_bc_quad_mask(u_bc0 ? s->U_bc_inv_mask.data : nullptr, u_bc0 ? s->U_bc.data : nullptr, nullptr,
                                            nullptr, qmask_buf, g, st)) {
    qmask = qmask_buf;
    ctx->launches += 1;
  }
  const int dmax = std::max(g.nx, std::max(g.ny, g.gnz));
  const double dx = 1.0 / (double)dmax;
  const bool u_bc = s->U_bc.data && s->U_bc_inv_mask.data;
  const bool d_bc = has_density && s->density_bc.data && s->density_bc_inv_mask.data;
  float bs[3] = {0.0f, 0.0f, 0.0f};
  const int do_buoy = has_density && mc->buoyancy_scale > 0.0;
  if (do_buoy) {
    const float k = (float)(-(dx / 4.0) * mc->buoyancy_scale);
    const float scale_dt = mc->dt / get_dx(g);
    for (int a = 0; a < 3; a++) bs[a] = (-(mc->gravity[a] * k)) * scale_dt;
  }
  launch_post_advect(has_density ? tmp_s : nullptr, tmp_u, fl8, has_density ? s->density.data : nullptr,
                     s->U.data, u_bc ? s->U_bc_inv_mask.data : nullptr, u_bc ? s->U_bc.data : nullptr,
                     d_bc ? s->density_bc_inv_mask.data : nullptr, d_bc ? s->density_bc.data : nullptr, qmask, do_buoy, bs,
                     g, st);
  ctx->launches += 1;
  if (ov && has_density && ctx->ov.density_host) {
    // The density is final here (nothing later in the step writes it): send it home while the
    // vorticity / projection kernels run.
    TFL_CUDA(ctx, cudaEventRecord(ctx->ev_d_ready, st));
    TFL_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_out, ctx->ev_d_ready, 0));
    TFL_CUDA(ctx, cudaMemcpyAsync(ctx->ov.density_host, s->density.data, ctx->ov.density_bytes, cudaMemcpyDeviceToHost,
                                  ctx->copy_out));
    TFL_CUDA(ctx, cudaEventRecord(ctx->ev_d_out, ctx->copy_out));
    ctx->ov.density_sent = true;
  }
  if (mc->gravity_scale > 0.0) {
    const float k = (float)((-dx / 4.0) * mc->gravity_scale);
    const float scale_dt = mc->dt / get_dx(g);
    const float f[3] = {(mc->gravity[0] * k) * scale_dt, (mc->gravity[1] * k) * scale_dt, (mc->gravity[2] * k) * scale_dt};
    launch_add_gravity(s->U.data, fl8, f, g, st);
    ctx->launches += 1;
  }
  const int do_vort = mc->vorticity_confinement_amp > 0.0;
  const float amp = (float)(dx * mc->vorticity_confinement_amp);
  if (do_vort) {
    launch_vort_curl(s->U.data, curl, cnorm, force, amp, g, st);
    ctx->launches += 2;
  }
  double* sums = ctx->dscratch + 64;
  TFL_CUDA(ctx, cudaMemsetAsync(sums, 0, sizeof(double) * 2 * g.nb, st));
  launch_vort_bc_mask(s->U.data, fl8, force, do_vort, u_bc ? s->U_bc_inv_mask.data : nullptr,
                      u_bc ? s->U_bc.data : nullptr, qmask, 1, sums, g, st);
  const ConvTcGeo& tg = m->act_geo;
  if (ov) TFL_CUDA(ctx, cudaStreamWaitEvent(st, ctx->ev_p_in, 0));          // pDiv is first read here
  launch_cnn_inputs_fused(s->p.data, s->U.data, fl8, sums, mc->normalize_input_threshold, scale, m->act[0],
                          tg.px, tg.py, g, st);
  run_conv_stack(m, p_net, st);
  launch_cnn_finish_fused(p_net, s->U.data, fl8, scale, s->p.data, u_bc ? s->U_bc_inv_mask.data : nullptr,
                          u_bc ? s->U_bc.data : nullptr, qmask, -1e6f, 1e6f, g, st);
  ctx->launches += 6;
  return check_launch(ctx, "simulate_step (fused)");
}

int tfl_simulate_step(tfl_ctx* ctx, const tfl_state* s, const tfl_mconf* mc, tfl_cnn* cnn) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!s || !mc) return fail(ctx, "simulate: nil state / mconf");
  if (check_scalar(ctx, &s->flags, "flags") || check_scalar(ctx, &s->p, "pDiv") || check_vel(ctx, &s->U, &s->flags))
    return 1;
  const int is3d = s->U.nc == 3;
  Geo g;
  if (make_geo(ctx, &s->flags, is3d, &g)) return 1;
  const bool has_density = s->density.data != nullptr;
  if (mc->sim_method == TFL_SIM_CONVNET && cnn && cnn->tc_ok && cnn->mode > 0 && !ctx->slab && g.nb == 1 &&
      !s->p_bc.data && mc->advection_method >= 0 && mc->advection_method <= 5) {
    if (has_density && (check_scalar(ctx, &s->density, "density") || !same_spatial(&s->density, &s->flags)))
      return fail(ctx, "Size mismatch");
    return simulate_step_fused(ctx, s, mc, cnn, g);
  }
  // 1-2. advect scalars then velocity (lib/simulate.lua:183-199).
  if (has_density && tfl_advect_scalar(ctx, mc->dt, &s->density, &s->U, &s->flags, mc->advection_method, 0,
                                       mc->maccormack_strength, nullptr))
    return 1;
  if (tfl_advect_vel(ctx, mc->dt, &s->U, &s->flags, mc->advection_method, mc->maccormack_strength, nullptr))
    return 1;
  if (set_const_vals(ctx, s)) return 1;                               // :202
  const int dmax = std::max(g.nx, std::max(g.ny, g.gnz));
  const double dx = 1.0 / (double)dmax;                              // tfluids.getDx, init.lua:560-564
  // gravity:mul(scalar) is a float tensor op: the Lua double is cast to float first.
  if (has_density && mc->buoyancy_scale > 0.0) {                     // :216-226
    const float k = (float)(-(dx / 4.0) * mc->buoyancy_scale);
    const float gv[3] = {mc->gravity[0] * k, mc->gravity[1] * k, mc->gravity[2] * k};
    if (tfl_add_buoyancy(ctx, &s->U, &s->flags, &s->density, gv, mc->dt)) return 1;
  }
  if (mc->gravity_scale > 0.0) {                                     // :229-233
    const float k = (float)((-dx / 4.0) * mc->gravity_scale);
    const float gv[3] = {mc->gravity[0] * k, mc->gravity[1] * k, mc->gravity[2] * k};
    if (tfl_add_gravity(ctx, &s->U, &s->flags, gv, mc->dt)) return 1;
  }
  if (mc->vorticity_confinement_amp > 0.0) {                         // :236-239
    const float amp = (float)(dx * mc->vorticity_confinement_amp);
    if (tfl_vorticity_confinement(ctx, &s->U, &s->flags, amp)) return 1;
  }
  if (mc->sim_method != TFL_SIM_CONVNET && tfl_set_wall_bcs_forward(ctx, &s->U, &s->flags)) return 1;  // :248-251
  if (set_const_vals(ctx, s)) return 1;                               // :252
  if (mc->sim_method == TFL_SIM_CONVNET) {                            // :262-272
    if (!cnn) return fail(ctx, "simulate: simMethod 'convnet' needs a model");
    if (tfl_cnn_project(ctx, cnn, &s->p, &s->U, &s->flags, &s->p, &s->U, mc->normalize_input_threshold, nullptr))
      return 1;
  } else if (mc->sim_method == TFL_SIM_JACOBI) {                      // :275-303
    if (!s->div.data) return fail(ctx, "simulate: state.div scratch is required for jacobi/pcg");
    if (tfl_velocity_divergence_forward(ctx, &s->U, &s->flags, &s->div)) return 1;
    const int iters = mc->max_iter > 0 ? mc->max_iter : 100;
    if (tfl_solve_linear_system_jacobi(ctx, &s->p, &s->flags, &s->div, is3d, 0.0f, iters, nullptr, nullptr))
      return 1;
    if (tfl_velocity_update_forward(ctx, &s->U, &s->flags, &s->p)) return 1;
  } else if (mc->sim_method == TFL_SIM_PCG) {                         // :280-286: tol 1e-4, 'ic0'
    if (!s->div.data) return fail(ctx, "simulate: state.div scratch is required for jacobi/pcg");
    if (tfl_velocity_divergence_forward(ctx, &s->U, &s->flags, &s->div)) return 1;
    const int iters = mc->max_iter > 0 ? mc->max_iter : 100;
    if (tfl_solve_linear_system_pcg(ctx, &s->p, &s->flags, &s->div, is3d, TFL_PRECOND_IC0, 1e-4f, iters, nullptr,
                                    nullptr))
      return 1;
    if (tfl_velocity_update_forward(ctx, &s->U, &s->flags, &s->p)) return 1;
  } else {
    return fail(ctx, "mconf.simMethod (%d) is not a valid option", mc->sim_method);
  }
  if (set_const_vals(ctx, s)) return 1;                               // :321
  return tfl_clamp(ctx, &s->U, -1e6f, 1e6f);                          // :326
}

// ---------------------------------------------------------------------------------------
// Host-buffer driver for the same step.
// ---------------------------------------------------------------------------------------
struct tfl_host_sim {
  tfl_state st;
  std::vector<void*> owned;
  size_t cells = 0;
  int nc = 3;
};

int tfl_host_sim_create(tfl_ctx* ctx, int32_t nb, int32_t nz, int32_t ny, int32_t nx, int is_3d,
                        const float* flags, const float* U_bc, const float* U_bc_inv, const float* d_bc,
                        const float* d_bc_inv, tfl_host_sim** out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!out || !flags) return fail(ctx, "host_sim: bad arguments");
  tfl_host_sim* hs = new tfl_host_sim();
  memset(&hs->st, 0, sizeof(hs->st));
  hs->nc = is_3d ? 3 : 2;
  hs->cells = (size_t)nb * nz * ny * nx;
  auto mk = [&](tfl_grid* g, int nc, const float* host) -> int {
    g->nb = nb; g->nc = nc; g->nz = nz; g->ny = ny; g->nx = nx;
    void* p = nullptr;
    if (cudaMalloc(&p, hs->cells * nc * 4) != cudaSuccess) return 1;
    hs->owned.push_back(p);
    g->data = (float*)p;
    if (host) cudaMemcpy(p, host, hs->cells * nc * 4, cudaMemcpyHostToDevice);
    else cudaMemset(p, 0, hs->cells * nc * 4);
    return 0;
  };
  int bad = 0;
  bad |= mk(&hs->st.flags, 1, flags);
  bad |= mk(&hs->st.p, 1, nullptr);
  bad |= mk(&hs->st.U, hs->nc, nullptr);
  bad |= mk(&hs->st.density, 1, nullptr);
  bad |= mk(&hs->st.div, 1, nullptr);
  if (U_bc && U_bc_inv) { bad |= mk(&hs->st.U_bc, hs->nc, U_bc); bad |= mk(&hs->st.U_bc_inv_mask, hs->nc, U_bc_inv); }
  if (d_bc && d_bc_inv) { bad |= mk(&hs->st.density_bc, 1, d_bc); bad |= mk(&hs->st.density_bc_inv_mask, 1, d_bc_inv); }
  if (bad) { tfl_host_sim_destroy(ctx, hs); return fail(ctx, "host_sim: cudaMalloc failed"); }
  *out = hs;
  return 0;
}

void tfl_host_sim_destroy(tfl_ctx* ctx, tfl_host_sim* hs) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!hs) return;
  if (ctx) cudaStreamSynchronize(ctx->stream);
  for (void* p : hs->owned) cudaFree(p);
  delete hs;
}

int tfl_host_sim_step(tfl_ctx* ctx, tfl_host_sim* hs, float* p, float* U, float* density,
                      const tfl_mconf* mc, tfl_cnn* cnn) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!hs || !p || !U) return fail(ctx, "host_sim_step: nil buffer");
  cudaStream_t st = ctx->stream;
  tfl_state s = hs->st;
  if (!density) s.density.data = nullptr;
  // Inputs in the order the step reads them: U (both advections), density (density advection), pDiv
  // (network input, much later).  One copy stream keeps them in that order on the PCIe link.
  TFL_CUDA(ctx, cudaEventRecord(ctx->ev_fork, st));                      // earlier work on the step stream
  TFL_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_in, ctx->ev_fork, 0));
  TFL_CUDA(ctx, cudaMemcpyAsync(s.U.data, U, hs->cells * 4 * hs->nc, cudaMemcpyHostToDevice, ctx->copy_in));
  TFL_CUDA(ctx, cudaEventRecord(ctx->ev_u_in, ctx->copy_in));
  if (density) TFL_CUDA(ctx, cudaMemcpyAsync(s.density.data, density, hs->cells * 4, cudaMemcpyHostToDevice, ctx->copy_in));
  TFL_CUDA(ctx, cudaEventRecord(ctx->ev_d_in, ctx->copy_in));
  TFL_CUDA(ctx, cudaMemcpyAsync(s.p.data, p, hs->cells * 4, cudaMemcpyHostToDevice, ctx->copy_in));
  TFL_CUDA(ctx, cudaEventRecord(ctx->ev_p_in, ctx->copy_in));
  const bool fused = mc->sim_method == TFL_SIM_CONVNET && cnn && cnn->tc_ok && cnn->mode > 0 && !ctx->slab &&
                     hs->st.flags.nb == 1 && mc->advection_method >= 0 && mc->advection_method <= 5;
  ctx->ov.active = fused;
  ctx->ov.density_host = density;
  ctx->ov.density_bytes = hs->cells * 4;
  ctx->ov.density_sent = false;
  if (!fused) {                                                           // operator-by-operator path: no overlap
    TFL_CUDA(ctx, cudaStreamWaitEvent(st, ctx->ev_p_in, 0));
  }
  const int rc = tfl_simulate_step(ctx, &s, mc, cnn);
  const bool density_sent = ctx->ov.density_sent;
  ctx->ov.active = false;
  if (rc) { cudaStreamSynchronize(ctx->copy_in); cudaStreamSynchronize(ctx->copy_out); return 1; }
  TFL_CUDA(ctx, cudaMemcpyAsync(U, s.U.data, hs->cells * 4 * hs->nc, cudaMemcpyDeviceToHost, st));
  TFL_CUDA(ctx, cudaMemcpyAsync(p, s.p.data, hs->cells * 4, cudaMemcpyDeviceToHost, st));
  if (density && !density_sent)
    TFL_CUDA(ctx, cudaMemcpyAsync(density, s.density.data, hs->cells * 4, cudaMemcpyDeviceToHost, st));
  if (density_sent) TFL_CUDA(ctx, cudaStreamWaitEvent(st, ctx->ev_d_out, 0));
  TFL_CUDA(ctx, cudaStreamSynchronize(st));
  return 0;
}

}  // extern "C"

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
  tfl_state st;
  float* U1 = nullptr;
  double* sums = nullptr;
  float* xbuf = nullptr;            // [send down | send up | recv from below | recv from above], xbuf_side floats each
  size_t xbuf_side = 0;
  // Peer-memory halo exchange (CUDA IPC over NVLink, tfl_slab_sim_ipc_*): this rank's inbox -- per phase and side a
  // receive buffer of xbuf_side floats that the neighbour's push kernel fills with remote stores, and a step counter
  // it raises afterwards -- and the neighbours' inboxes mapped into this process.
  float* inbox = nullptr;           // cudaMalloc'ed, exported: [3 phases][2 sides][xbuf_side] floats, then 64 counters
  float* peer_inbox[2] = {nullptr, nullptr};   // lower / upper neighbour's inbox (cudaIpcOpenMemHandle)
  std::vector<float*> all_inbox;               // every rank's inbox (own pointer at [rank]): the all-reduce's targets
  float** all_inbox_dev = nullptr;             // the same table on the device
  unsigned int* push_done = nullptr;           // CTAs of the running push kernel that finished their stores
  bool peer_ok = false;
  unsigned int step_no = 0;
  std::vector<void*> owned;
  cudaEvent_t ev[4][2] = {{nullptr, nullptr}, {nullptr, nullptr}, {nullptr, nullptr}, {nullptr, nullptr}};
  size_t bytes_sent[3] = {0, 0, 0};
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
  if (!s) return;
  if (ctx) cudaStreamSynchronize(ctx->stream);
  for (int r = 0; r < (int)s->all_inbox.size(); r++) if (r != s->rank && s->all_inbox[r]) cudaIpcCloseMemHandle(s->all_inbox[r]);
  for (void* p : s->owned) cudaFree(p);
  for (auto& pr : s->ev) for (cudaEvent_t e : pr) if (e) cudaEventDestroy(e);
  delete s;
}

// All host arrays are GLOBAL [c][gnz][ny][nx] fields, identical on every rank; each rank keeps its slab.
int tfl_slab_sim_create(tfl_ctx* ctx, int32_t gnz, int32_t ny, int32_t nx, int32_t margin, const float* flags,
                        const float* U_bc, const float* U_bc_inv, const float* d_bc, const float* d_bc_inv,
                        tfl_slab_sim** out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!out || !flags || gnz < 3 || ny < 3 || nx < 3 || margin < 2) return fail(ctx, "slab_sim: bad arguments (margin >= 2)");
  tfl_slab_sim* s = new tfl_slab_sim();
  memset(&s->st, 0, sizeof(s->st));
  s->gnz = gnz; s->ny = ny; s->nx = nx; s->margin = margin; s->halo = 2 * margin + 2;
  s->rank = ctx->comm_rank; s->world = ctx->comm_world;
  const int base = gnz / s->world, rem = gnz % s->world;
  if (s->world > 1 && base < s->halo) { delete s; return fail(ctx, "slab_sim: slabs of %d planes are thinner than the halo (%d)", base, s->halo); }
  s->z0 = s->rank * base + std::min(s->rank, rem);
  s->z1 = s->z0 + base + (s->rank < rem ? 1 : 0);
  s->lo_halo = std::min(s->halo, s->z0);
  s->hi_halo = std::min(s->halo, gnz - s->z1);
  s->zoff = s->z0 - s->lo_halo;
  s->nz = (s->z1 - s->z0) + s->lo_halo + s->hi_halo;
  s->own_lo = s->lo_halo;
  s->own_hi = s->lo_halo + (s->z1 - s->z0);
  s->plane = (size_t)ny * nx;
  s->cells = s->plane * s->nz;
  const size_t gcells = s->plane * gnz;
  auto mk = [&](tfl_grid* g, int nc, const float* host) -> int {
    g->nb = 1; g->nc = nc; g->nz = s->nz; g->ny = ny; g->nx = nx;
    void* p = nullptr;
    if (cudaMalloc(&p, s->cells * nc * 4) != cudaSuccess) return 1;
    s->owned.push_back(p);
    g->data = (float*)p;
    if (!host) return cudaMemset(p, 0, s->cells * nc * 4) != cudaSuccess;
    for (int c = 0; c < nc; c++)
      if (cudaMemcpy((float*)p + c * s->cells, host + c * gcells + (size_t)s->zoff * s->plane, s->cells * 4,
                     cudaMemcpyHostToDevice) != cudaSuccess)
        return 1;
    return 0;
  };
  int bad = 0;
  bad |= mk(&s->st.flags, 1, flags);
  bad |= mk(&s->st.p, 1, nullptr);
  bad |= mk(&s->st.U, 3, nullptr);
  bad |= mk(&s->st.density, 1, nullptr);
  if (U_bc && U_bc_inv) { bad |= mk(&s->st.U_bc, 3, U_bc); bad |= mk(&s->st.U_bc_inv_mask, 3, U_bc_inv); }
  if (d_bc && d_bc_inv) { bad |= mk(&s->st.density_bc, 1, d_bc); bad |= mk(&s->st.density_bc_inv_mask, 1, d_bc_inv); }
  void* p = nullptr;
  bad |= cudaMalloc(&p, s->cells * 3 * 4) != cudaSuccess;
  if (!bad) { s->owned.push_back(p); s->U1 = (float*)p; }
  bad |= cudaMalloc(&p, 2 * sizeof(double)) != cudaSuccess;
  if (!bad) { s->owned.push_back(p); s->sums = (double*)p; }
  s->xbuf_side = (size_t)s->halo * s->plane * 4;          // the widest exchange: halo planes of 4 channels
  bad |= cudaMalloc(&p, 4 * s->xbuf_side * sizeof(float)) != cudaSuccess;
  if (!bad) { s->owned.push_back(p); s->xbuf = (float*)p; }
  if (s->world > 1) {
    const size_t inbox_bytes = (6 * s->xbuf_side + 64 + kSumAreaFloats) * sizeof(float);
    bad |= cudaMalloc(&p, inbox_bytes) != cudaSuccess;
    if (!bad) { s->owned.push_back(p); s->inbox = (float*)p; bad |= cudaMemset(p, 0, inbox_bytes) != cudaSuccess; }
    bad |= cudaMalloc(&p, sizeof(unsigned int)) != cudaSuccess;
    if (!bad) { s->owned.push_back(p); s->push_done = (unsigned int*)p; bad |= cudaMemset(p, 0, sizeof(unsigned int)) != cudaSuccess; }
  }
  for (auto& pr : s->ev) for (cudaEvent_t& e : pr) bad |= cudaEventCreate(&e) != cudaSuccess;
  if (bad) { tfl_slab_sim_destroy(ctx, s); return fail(ctx, "slab_sim: allocation failed"); }
  *out = s;
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

// Refresh `width` ghost planes on both sides of the listed fields from the neighbours' owned planes.
int slab_exchange(tfl_ctx* ctx, tfl_slab_sim* s, std::initializer_list<const tfl_grid*> fields, int width, int phase) {
  TFL_CUDA(ctx, cudaEventRecord(s->ev[phase][0], ctx->stream));
  s->bytes_sent[phase] = 0;
  if (s->world > 1 && width > 0 && (ctx->comm || s->peer_ok)) {
    if (width > s->halo) return fail(ctx, "slab exchange of %d planes exceeds the halo (%d)", width, s->halo);
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
    if (side > s->xbuf_side) return fail(ctx, "slab exchange buffer too small");
    const bool lo = s->rank > 0, hi = s->rank < s->world - 1;
    const int blocks = (int)std::min<size_t>((2 * side + 255) / 256, 132 * 4);
    if (s->peer_ok) {
      // inbox layout: buffer (phase, from-below = 0 / from-above = 1) at ((phase * 2 + from) * xbuf_side), counters behind
      auto buf = [&](float* base, int from) { return base + ((size_t)phase * 2 + from) * s->xbuf_side; };
      auto flag = [&](float* base, int from) { return (unsigned int*)(base + 6 * s->xbuf_side) + phase * 2 + from; };
      d.send_lo = d.send_hi = d.recv_lo = d.recv_hi = nullptr;
      // my first owned planes land in the lower neighbour's "from above" slot, my last ones in the upper neighbour's "from below"
      k_slab_push<<<blocks, 256, 0, ctx->stream>>>(d, lo ? buf(s->peer_inbox[0], 1) : nullptr, hi ? buf(s->peer_inbox[1], 0) : nullptr,
                                                   lo ? flag(s->peer_inbox[0], 1) : nullptr, hi ? flag(s->peer_inbox[1], 0) : nullptr,
                                                   s->step_no, s->push_done);
      k_slab_pull<<<blocks, 256, 0, ctx->stream>>>(d, lo ? buf(s->inbox, 0) : nullptr, hi ? buf(s->inbox, 1) : nullptr,
                                                   lo ? flag(s->inbox, 0) : nullptr, hi ? flag(s->inbox, 1) : nullptr,
                                                   s->step_no, ctx->counters);
      s->bytes_sent[phase] = (size_t)(lo + hi) * side * 4;
      ctx->launches += 2;
    } else {
      NcclApi* nc = nccl_api();
      d.send_lo = lo ? s->xbuf : nullptr;
      d.send_hi = hi ? s->xbuf + s->xbuf_side : nullptr;
      d.recv_lo = lo ? s->xbuf + 2 * s->xbuf_side : nullptr;
      d.recv_hi = hi ? s->xbuf + 3 * s->xbuf_side : nullptr;
      k_slab_pack<false><<<blocks, 256, 0, ctx->stream>>>(d);
      TFL_NCCL(ctx, nc->GroupStart());
      if (lo) {                                       // lower neighbour: my first owned planes go down
        TFL_NCCL(ctx, nc->Send(d.send_lo, side, ncclFloat, s->rank - 1, ctx->comm, ctx->stream));
        TFL_NCCL(ctx, nc->Recv(d.recv_lo, side, ncclFloat, s->rank - 1, ctx->comm, ctx->stream));
        s->bytes_sent[phase] += side * 4;
      }
      if (hi) {                                       // upper neighbour
        TFL_NCCL(ctx, nc->Send(d.send_hi, side, ncclFloat, s->rank + 1, ctx->comm, ctx->stream));
        TFL_NCCL(ctx, nc->Recv(d.recv_hi, side, ncclFloat, s->rank + 1, ctx->comm, ctx->stream));
        s->bytes_sent[phase] += side * 4;
      }
      TFL_NCCL(ctx, nc->GroupEnd());
      k_slab_pack<true><<<blocks, 256, 0, ctx->stream>>>(d);
      ctx->launches += 2;
    }
  }
  TFL_CUDA(ctx, cudaEventRecord(s->ev[phase][1], ctx->stream));
  return 0;
}

struct SlabScope {       // slab placement of the context for the enclosed calls
  tfl_ctx* ctx;
  SlabScope(tfl_ctx* c, const tfl_slab_sim* s, int zlo, int zhi) : ctx(c) {
    c->slab = true; c->zoff = s->zoff; c->gnz = s->gnz; c->zlo = zlo; c->zhi = zhi; c->slab_margin = s->margin;
  }
  ~SlabScope() { ctx->slab = false; ctx->slab_margin = 2; }
};

}  // namespace

extern "C" {

// One tfluids.simulate (convnet path, lib/simulate.lua:175-327) on this rank's slab.  Asynchronous.
int tfl_slab_sim_step(tfl_ctx* ctx, tfl_slab_sim* s, const tfl_mconf* mc, tfl_cnn* cnn) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!s || !mc || !cnn) return fail(ctx, "slab_sim_step: nil argument");
  if (mc->sim_method != TFL_SIM_CONVNET) return fail(ctx, "slab_sim_step: only simMethod 'convnet' is decomposed");
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
  const int dmax = std::max(s->nx, std::max(s->ny, s->gnz));
  const double dx = 1.0 / (double)dmax;
  {
    // point-wise forces also on the three ghost planes the confinement stencil reads across the cut
    SlabScope scope(ctx, s, s->own_lo - std::min(3, s->lo_halo), s->own_hi + std::min(3, s->hi_halo));
    if (mc->buoyancy_scale > 0.0) {
      const float k = (float)(-(dx / 4.0) * mc->buoyancy_scale);
      const float gv[3] = {mc->gravity[0] * k, mc->gravity[1] * k, mc->gravity[2] * k};
      if (tfl_add_buoyancy(ctx, &st.U, &st.flags, &st.density, gv, mc->dt)) return 1;
    }
    if (mc->gravity_scale > 0.0) {
      const float k = (float)((-dx / 4.0) * mc->gravity_scale);
      const float gv[3] = {mc->gravity[0] * k, mc->gravity[1] * k, mc->gravity[2] * k};
      if (tfl_add_gravity(ctx, &st.U, &st.flags, gv, mc->dt)) return 1;
    }
  }
  if (mc->vorticity_confinement_amp > 0.0) {
    SlabScope scope(ctx, s, s->own_lo, s->own_hi);
    if (tfl_vorticity_confinement(ctx, &st.U, &st.flags, (float)(dx * mc->vorticity_confinement_amp))) return 1;
  }
  if (bcs()) return 1;
  if (slab_exchange(ctx, s, {&st.U, &st.p}, 5, 2)) return 1;
  tfl_grid u1 = st.U;
  u1.data = s->U1;
  {
    SlabScope scope(ctx, s, s->own_lo, s->own_hi);
    if (tfl_cnn_stats(ctx, &st.U, &st.flags, &u1, s->sums)) return 1;
  }
  TFL_CUDA(ctx, cudaEventRecord(s->ev[3][0], ctx->stream));
  if (s->world > 1 && s->peer_ok && s->all_inbox_dev) {
    k_sum_push<<<1, 64, 0, ctx->stream>>>(s->sums, s->all_inbox_dev, s->xbuf_side, s->rank, s->world, s->step_no);
    k_sum_pull<<<1, 64, 0, ctx->stream>>>(s->sums, s->inbox, s->xbuf_side, s->world, s->step_no, ctx->counters);
    ctx->launches += 2;
  } else if (s->world > 1 && ctx->comm) {
    TFL_NCCL(ctx, nccl_api()->AllReduce(s->sums, s->sums, 2, ncclDouble, ncclSum, ctx->comm, ctx->stream));
  }
  TFL_CUDA(ctx, cudaEventRecord(s->ev[3][1], ctx->stream));
  {
    SlabScope scope(ctx, s, s->own_lo, s->own_hi);
    if (tfl_cnn_project_from_sums(ctx, cnn, &st.p, &u1, &st.flags, s->sums, &st.p, &st.U, mc->normalize_input_threshold)) return 1;
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
  TFL_CUDA(ctx, cudaIpcGetMemHandle(&h, s->inbox));
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
    for (int r = 0; r < (int)s->all_inbox.size(); r++)
      if (r != s->rank && s->all_inbox[r]) cudaIpcCloseMemHandle(s->all_inbox[r]);
    s->all_inbox.clear();
    s->peer_inbox[0] = s->peer_inbox[1] = nullptr;
    s->peer_ok = false;
  };
  TFL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  drop();
  if (!handles) return 0;                          // back to NCCL (e.g. another rank could not map its peers)
  if (s->world > 64) return fail(ctx, "slab_sim_ipc_connect: more than 64 ranks");
  s->all_inbox.assign(s->world, nullptr);
  s->all_inbox[s->rank] = s->inbox;
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
    s->all_inbox[r] = (float*)q;
  }
  if (!s->all_inbox_dev) {
    void* p = nullptr;
    TFL_CUDA(ctx, cudaMalloc(&p, 64 * sizeof(float*)));
    s->owned.push_back(p);
    s->all_inbox_dev = (float**)p;
  }
  TFL_CUDA(ctx, cudaMemcpy(s->all_inbox_dev, s->all_inbox.data(), s->world * sizeof(float*), cudaMemcpyHostToDevice));
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
    if (cudaEventElapsedTime(&ms[i], s->ev[i][0], s->ev[i][1]) != cudaSuccess) { cudaGetLastError(); ms[i] = -1.0f; }
  }
  for (int i = 0; i < 3; i++) bytes[i] = (int64_t)s->bytes_sent[i];
  return 0;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------
// The step as a CUDA graph: tfl_simulate_step captured once on the context's stream (both streams of the
// fused step, their fork / join events, the memsets and the telemetry copy become graph nodes) and replayed
// with one launch.  Pointers and every host-side choice of the captured call (fused or per-operator path,
// advection tile halo) are frozen into the graph; results equal tfl_simulate_step's.
// ---------------------------------------------------------------------------------------
struct tfl_step_graph {
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t exec = nullptr;
  long long launches = 0;       // kernels in one replay
};

extern "C" {

void tfl_step_graph_destroy(tfl_ctx* ctx, tfl_step_graph* g) {
  DeviceGuard guard_(ctx);
  if (!g) return;
  if (ctx) cudaStreamSynchronize(ctx->stream);
  if (g->exec) cudaGraphExecDestroy(g->exec);
  if (g->graph) cudaGraphDestroy(g->graph);
  delete g;
}

// Preconditions: the context runs on a non-default stream (tfl_set_stream; the legacy default stream cannot be
// captured) and one tfl_simulate_step with the same state shapes has already run (scratch buffers are sized
// then: capturing must not allocate).
int tfl_step_graph_create(tfl_ctx* ctx, const tfl_state* state, const tfl_mconf* mc, tfl_cnn* cnn, tfl_step_graph** out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!out || !state || !mc) return fail(ctx, "step_graph: nil argument");
  cudaStream_t st = ctx->stream;
  if (st == nullptr || st == cudaStreamLegacy || st == cudaStreamPerThread)
    return fail(ctx, "step_graph: the default stream cannot be captured; give the context a stream (tfl_set_stream)");
  TFL_CUDA(ctx, cudaStreamSynchronize(st));
  const long long l0 = ctx->launches;
  if (cudaStreamBeginCapture(st, cudaStreamCaptureModeRelaxed) != cudaSuccess) {
    cudaGetLastError();
    return fail(ctx, "step_graph: cudaStreamBeginCapture failed");
  }
  const int rc = tfl_simulate_step(ctx, state, mc, cnn);
  tfl_step_graph* g = new tfl_step_graph();
  const cudaError_t e = cudaStreamEndCapture(st, &g->graph);
  if (rc != 0 || e != cudaSuccess || !g->graph) {
    cudaGetLastError();
    const std::string why = rc != 0 ? ctx->err : std::string(cudaGetErrorString(e));
    tfl_step_graph_destroy(ctx, g);
    return fail(ctx, "step_graph: capture failed (%s); run tfl_simulate_step once before capturing", why.c_str());
  }
  g->launches = ctx->launches - l0;
  ctx->launches = l0;
  if (cudaGraphInstantiate(&g->exec, g->graph, 0) != cudaSuccess) {
    cudaGetLastError();
    tfl_step_graph_destroy(ctx, g);
    return fail(ctx, "step_graph: cudaGraphInstantiate failed");
  }
  *out = g;
  return 0;
}

int tfl_step_graph_launch(tfl_ctx* ctx, tfl_step_graph* g) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!g || !g->exec) return fail(ctx, "step_graph is nil");
  TFL_CUDA(ctx, cudaGraphLaunch(g->exec, ctx->stream));
  ctx->launches += g->launches;
  return 0;
}

}  // extern "C"
