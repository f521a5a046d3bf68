// Internal interface of the C ABI units: tfl_api.cu (context, memory, operators, step drivers), tfl_api_cnn.cu
// (projection network: creation and entry points), tfl_cnn_forward.cu (its forward drivers), tfl_api_cnn_debug.cu (its
// test hooks) and tfl_api_slab.cu (z-slab driver).
#pragma once
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <nvtx3/nvToolsExt.h>
#include <nccl.h>      // types and prototypes only: libnccl is loaded on demand (dlopen), see tfl_api_slab.cu
#include <algorithm>
#include <initializer_list>
#include <memory>
#include <string>
#include <vector>

#include "tfl_kernels.h"
#include "tfl_cnn_tc.h"

using namespace tfl;

constexpr char kConvZStalled[] =
    "internal error, the z-streaming tensor-core convolution's pipeline stalled (a bounded wait ran out)";

struct tfl_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;            // where work is enqueued: own_stream, or a stream the caller adopted
  StreamPtr own_stream;                     // the stream the context made (empty while an adopted one is current)
  std::string err;
  DevPtr<char> arena;
  size_t arena_bytes = 0;
  size_t arena_used = 0;
  // Generation counters of the buffers a step graph captures: bumped whenever the buffer is freed and allocated
  // again, so that tfl_step_graph_launch can refuse a graph that would replay freed memory.
  unsigned long long arena_gen = 0;
  DevPtr<unsigned long long> counters;      // [0] trace faults, [1] bad occupancy cells
  long long launches = 0;
  bool slab = false;
  int zoff = 0, gnz = 0, zlo = 0, zhi = 0;
  int slab_margin = 2;                      // extra planes on which forward passes are evaluated
  StreamPtr side_stream;                    // density advection runs beside velocity advection
  EventPtr ev_fork, ev_join;
  // Host-buffer step (tfl_host_sim_step): copies run on their own streams and the step waits for each
  // input only where it is first read / hands each output over as soon as it is final.
  StreamPtr copy_in, copy_out;
  EventPtr ev_u_in, ev_d_in, ev_p_in, ev_d_ready, ev_d_out;
  struct {
    bool active = false;
    float* density_host = nullptr;          // where the advected density goes once it is final
    size_t density_bytes = 0;
    bool density_sent = false;
  } ov;
  PcgScratch pcg;                           // grow-only buffers of the PCG solve
  StreamPtr loop_body;                      // captures the body of a WHILE node (capture_while)
  PinnedPtr<int> done_host;                 // host copy of a device-stopped loop's done word (run_until_done)
  PcgGraphScratch* pcg_graph = nullptr;     // set while tfl_step_graph_create captures: PCG solves are captured there
  // Byte copy of the step's flags and their clearance field (advection fast path), kept between steps:
  // each step re-derives the bytes, compares them with the copy on the device and rebuilds the
  // clearance only if something changed (no host round trip).
  struct {
    DevPtr<unsigned char> bytes;            // [3][cells]: flags, clearance, scratch
    size_t cells = 0;
    int nb = 0, nz = 0, ny = 0, nx = 0;
    DevPtr<int> changed;                    // device word
    const float* fresh_for = nullptr;       // set inside a slab step: the cache already mirrors these flags
    unsigned long long gen = 0;             // bumped on every reallocation of `bytes` (see arena_gen)
  } fcache;
  // advectVel over shared-memory tiles (tfl_advect_tile.cu): the kernel reports the longest trace of a call
  // into a device word that is copied, asynchronously, into a pinned host word; the NEXT calls pick the tile
  // halo from it (stale by a step or two -- it only selects a code path, never a result).
  struct {
    DevPtr<unsigned int> dev;
    PinnedPtr<unsigned int> host;
    int mode = -1;                          // -1 automatic, 0 two-kernel version, 1 / 2 forced halo
    int calls_since_probe = 0;
    int last_vel_halo = 0, last_scalar_halo = 0;   // halo of the last dispatches' tile kernels (0: none ran)
    // bench.py's roofline: CUDA events right around the tile kernel's launch (off unless asked for)
    bool timed = false;
    EventPtr ev0, ev1;
  } tile;
  // z-slab decomposition over several GPUs (tfl_comm_init / tfl_slab_sim_*): the communicator lives here
  ncclComm_t comm = nullptr;
  int comm_rank = 0, comm_world = 1;
  bool in_slab_step = false;
};

struct tfl_cnn {
  int is3d = 1;
  int n_layers = 0;
  std::vector<int> cin, cout, ks;   // per convolution (= per stage unless banked)
  std::vector<DevPtr<float>> w;     // device, [cin][tap][cout]
  std::vector<DevPtr<float>> b;     // device, [cout]
  // multi-resolution banks (lib/model.lua:252-361): stages [split, join) (0-based here) hold one convolution
  // per bank; conv0[l] is the index of stage l's first convolution.  nbanks == 1: single bank.
  int nbanks = 1, split = 0, join = 0, bank_add = 0;
  // banksType 'dilate' (nbanks > 1 only): no pyramid, bank i's convolutions in [split, join) dilated by 2^i (0-based
  // i), every bank at bank 1's resolution, no upsampling at the join.  On the tensor cores bank i's buffers hold its
  // phase sub-grids (make_conv_tc_phase_geo).
  int bank_dilate = 0;
  std::vector<int> conv0;
  int max_c = 0;
  // per-layer extras of the 'tog' / 'yang' graphs (lib/model.lua:164-239): the convolution emits
  // cout * up^d channels that a pixel shuffle turns into cout channels at `up` times the resolution, a
  // pooling of size `pool` follows the non-linearity.  plain = every pool / up is 1 and the non-linearity is ReLU.
  std::vector<int> pool, up;
  int pool_is_max = 0;
  int nonlin = 1;            // 1 ReLU, 2 sigmoid, 3 ReLU6 (activation codes of tfl_cnn.cu)
  // batch normalization (tfl_cnn_norm) after every convolution but the last, on its stage's output: per convolution,
  // bn_wb [2][c] (weight, bias) and eps for batch statistics, or bn_ac [2][c] (a, c of y = a x + c, computed at
  // creation from the running statistics).  bn_max_c: the most channels of one BN module (sizes the scratch).
  bool bn = false, bn_batch = false;
  std::vector<DevPtr<float>> bn_wb, bn_ac;
  std::vector<float> bn_eps;
  int bn_max_c = 0;
  // batch statistics on the tensor cores (run_conv_stack): the partials of one module and the (a, c) of BN1..BN4
  DevPtr<double> bn_part;
  DevPtr<float> bn_tcac;
  bool plain = true;
  double max_rel = 0.0;      // largest channels x (cells relative to the input grid) of any stage
  double bank_rel = 0.0;     // the same over one bank's activations in the banked stages (conv output, pooled)
  // input block (tfl_cnn_inputs): in_sel the kCnnIn* channels, in_ch = cin[0]; norm_func a kCnnScale* code (kCnnScaleOne
  // when normalizeInput is off), norm_chan the kCnnStat* field.  With the pressure skip the last convolution keeps
  // its hidden channels and w_skip, its pDiv weight, is added by launch_cnn_skip.
  int in_sel = kCnnInPDiv | kCnnInDiv, in_ch = 3;
  int norm_func = kCnnScaleStd, norm_chan = kCnnStatU;
  bool skip = false;
  float w_skip = 0.0f;
  bool default_inputs = true;
  int tc_planes = 1;         // float4 planes of the tensor-core input (2 when UDiv is an input)
  // tensor-core path (3-D 'default' architecture, single-bank or with banks split at stage 1 and joined at stage 3)
  int mode = 0;              // 0 fp32 FMA, 1 TF32 tensor cores, 2 3xTF32 tensor cores
  bool tc_ok = false;
  DevPtr<float> tail;        // w4[8][8], b4[8], w5[8], b5[1]
  DevPtr<float> act[3];      // padded channels-last activation buffers
  ConvTcGeo act_geo = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  int act_zoff = 0;          // global plane of act's local plane 0 (z-slab; 0 on whole grids)
  unsigned long long act_gen = 0;   // bumped whenever act / bact / part are reallocated (see tfl_ctx::arena_gen)
  // Packed weights per split: layers 1 / 2 of bank i at wBk[2 i] / wBk[2 i + 1]; the join layer's weights (one for
  // 'add', bank i's 8-channel slice at wBj[i] for 'concat', which for one bank is the whole layer 3).  Banks 2..N
  // own three padded buffers each (pyramid input, layer 1, layer 2) at their resolution; 'concat' with N > 1 adds
  // an fp32 partial sum.  On a z-slab, bank i's local plane 0 is its global coarse plane borg[i - 1] =
  // ceil(act_zoff / 2^i), and it holds the coarse planes whose 2^i fine planes all lie in the local slab.
  std::vector<DevPtr<float>> wBk[2], wBj[2];
  std::vector<DevPtr<float>> bact;
  std::vector<ConvTcGeo> bgeo;
  std::vector<int> borg;
  DevPtr<float> part;
};

// The generations of the library-owned buffers a step graph holds pointers into (the context's scratch arena and flag
// cache, the model's activation buffers), taken at capture and compared before every replay.
struct BufferGens {
  unsigned long long arena = 0, fcache = 0, act = 0;
  const tfl_cnn* cnn = nullptr;     // the captured model (its act_gen is compared), or null
};
inline BufferGens buffer_gens(const tfl_ctx* ctx, const tfl_cnn* cnn) {
  BufferGens g;
  g.arena = ctx->arena_gen;
  g.fcache = ctx->fcache.gen;
  g.cnn = cnn;
  g.act = cnn ? cnn->act_gen : 0;
  return g;
}
// The first of those buffers reallocated since `then`, by name, or null.
inline const char* reallocated_buffer(const tfl_ctx* ctx, const BufferGens& then) {
  return then.arena != ctx->arena_gen            ? "the context's scratch arena"
         : then.fcache != ctx->fcache.gen        ? "the context's flag cache"
         : then.cnn && then.act != then.cnn->act_gen ? "the model's activation buffers"
                                                  : nullptr;
}

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

inline int fail(tfl_ctx* ctx, const char* fmt, ...) {
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

// Whether the context's stream is being captured into a graph (*capturing), or fails naming `who`.
int stream_capturing(tfl_ctx* ctx, const char* who, bool* capturing);

// A loop of `total` units that stops on the device by setting *done, run directly: enqueue(k, n) enqueues units
// [k, k + n) on the context's stream (0, or nonzero when it failed), in chunks of first, 2 first, ... up to `most`
// units.  After each chunk but the one that reaches total, the host reads *done and stops once it is set.  0, or 1
// when enqueue or a CUDA call failed (fails naming `who` when the pinned host word cannot be allocated).
template <typename Enqueue>
int run_until_done(tfl_ctx* ctx, const char* who, const int* done, int total, int first, int most, Enqueue&& enqueue) {
  if (!ctx->done_host && !(ctx->done_host = pinned_alloc<int>(1))) return fail(ctx, "%s: cudaMallocHost failed", who);
  for (int k = 0, chunk = first; k < total; chunk = std::min(2 * chunk, most)) {
    const int n = std::min(chunk, total - k);
    if (enqueue(k, n)) return 1;
    k += n;
    if (k >= total) break;
    TFL_CUDA(ctx, cudaMemcpyAsync(ctx->done_host.get(), done, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    TFL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (*ctx->done_host) break;
  }
  return 0;
}

// One block of Jacobi sweeps on a prepared mask, for the whole-grid and z-slab drivers: the cooperative block kernel or
// one launch per sweep (path -1: automatic, 0: per sweep, 1: one launch, refused when it does not apply).  Returns the
// path taken, -1 on refusal.
// The automatic path takes the one-launch kernel only with 4-plane blocks (ranges up to 2.16M cells on an H100):
// measured on an H100 at 400 W, 34 / 100 sweeps of 128^3 run at 8.4 / 7.3 us per sweep in one launch against
// 8.9 / 8.2 per launch, but a 6-sweep block on an 8-rank slab of 256^3 (256^2 x 42 planes, 6-plane blocks) takes
// 154 us against 94 us in per-sweep launches.
inline int run_jacobi_block(tfl_ctx* ctx, const unsigned char* mask, const float* div, float* pa, float* pb,
                            const Geo& g, int z_lo, int z_hi, int shr_lo, int shr_hi, int sweeps, int path) {
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

inline int check_launch(tfl_ctx* ctx, const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(ctx, "%s: launch failed: %s", what, cudaGetErrorString(e));
  return 0;
}

// Bump allocator over one growing device buffer (the reference's getTempStorage,
// tfluids/init.lua:35-64).  Growing synchronises; steady state does not allocate.
inline int arena_reserve(tfl_ctx* ctx, size_t bytes) {
  if (bytes <= ctx->arena_bytes) return 0;
  TFL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  ctx->arena.reset();                       // before the larger one is allocated
  ctx->arena_bytes = 0;
  ctx->arena_gen++;
  void* p = nullptr;
  TFL_CUDA(ctx, cudaMalloc(&p, bytes));
  ctx->arena.reset((char*)p);
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
    return (T*)(ctx->arena.get() + a);
  }
};
inline size_t carve_bytes(std::initializer_list<size_t> sizes) {
  size_t off = 0;
  for (size_t s : sizes) off = ((off + 255) & ~(size_t)255) + s;
  return off + 256;
}

inline bool same_spatial(const tfl_grid* a, const tfl_grid* b) {
  return a->nb == b->nb && a->nz == b->nz && a->ny == b->ny && a->nx == b->nx;
}

// Mirrors the shape asserts of init.lua (e.g. :100-120, :177-191).
inline int check_scalar(tfl_ctx* ctx, const tfl_grid* g, const char* name) {
  if (!g || !g->data) return fail(ctx, "%s is nil", name);
  if (g->nc != 1) return fail(ctx, "%s is not scalar", name);
  if (g->nb < 1 || g->nz < 1 || g->ny < 1 || g->nx < 1) return fail(ctx, "%s: Dimension mismatch", name);
  return 0;
}
inline int check_vel(tfl_ctx* ctx, const tfl_grid* U, const tfl_grid* flags) {
  if (!U || !U->data) return fail(ctx, "U is nil");
  if (U->nc != 2 && U->nc != 3) return fail(ctx, "2D velocity field must have only 2 channels");
  if (U->nc == 2 && flags->nz != 1) return fail(ctx, "2D velocity field but zdepth > 1");
  if (!same_spatial(U, flags)) return fail(ctx, "Size mismatch");
  return 0;
}

// cell() (tfl_device.cuh) indexes one (batch, channel) block of n cells in 32 bits; the second bound keeps the whole
// velocity field within 2^33 cells.
inline bool grid_too_large(long long n, int nb) { return n >= (1LL << 31) || n * (long long)nb * 3 >= (1LL << 31) * 4; }

// CUDA launches at most 65535 blocks along gridDim.y and along gridDim.z, and the launchers put the batch's planes and
// the rows there:
//  * planes (z): launch_dims, quad_dims, conv_launch and k_jacobi_iter4 give a block two planes of a grid with nz > 1
//    and one plane otherwise, over all nb entries: nb nz <= 2 x 65535 (nz > 1), nb <= 65535 (nz = 1).  The launchers
//    that give a block more planes (the advection tiles 8, the box convolution 5 or 6, k_jacobi_march at least 4)
//    stay below that, and so does nb <= 65535 for k_sqdiff (y) and k_monitor_chunks (z), one block per entry.
//  * rows (y): launch_dims gives a block two rows of a grid with nz > 1 (rows of a multiple of 64 cells) and four
//    otherwise; every other launcher more: ny <= 2 x 65535 (nz > 1), ny <= 4 x 65535 (nz = 1).
// Two launchers go further: k_monitor_chunks puts one block per plane on y (tfl_monitor_create refuses gnz > 65535)
// and the recorder's k_pack_vbox one per row on z (tfl_recorder_create refuses ny > 65535).
constexpr long long kMaxGridYZ = 65535;
inline long long max_batch_planes(int nz) { return nz > 1 ? 2 * kMaxGridYZ : kMaxGridYZ; }
inline long long max_rows(int nz) { return nz > 1 ? 2 * kMaxGridYZ : 4 * kMaxGridYZ; }
// 0 if every launcher a call on an nb x nz x ny grid can reach fits CUDA's grid, else fails naming the limit.
inline int check_launch_grid(tfl_ctx* ctx, const char* who, int nb, int nz, int ny) {
  if ((long long)nb * nz > max_batch_planes(nz))
    return fail(ctx, "%s: grid too large for one launch: nb x nz = %lld planes, at most %lld (65535 blocks along "
                     "gridDim.z, %d plane(s) each)", who, (long long)nb * nz, max_batch_planes(nz), nz > 1 ? 2 : 1);
  if (ny > max_rows(nz))
    return fail(ctx, "%s: grid too large for one launch: ny = %d rows, at most %lld (65535 blocks along gridDim.y, "
                     "%d rows each)", who, ny, max_rows(nz), nz > 1 ? 2 : 4);
  return 0;
}

// The global planes [*z0, *z1) z-slab rank `rank` of `world` owns in a domain of gnz planes: gnz / world each, one more
// for the first gnz % world ranks.  The slab simulator, its Jacobi schedule and the slab recorder all use this rule.
inline void slab_planes(int gnz, int world, int rank, int* z0, int* z1) {
  const int base = gnz / world, rem = gnz % world;
  *z0 = rank * base + (rank < rem ? rank : rem);
  *z1 = *z0 + base + (rank < rem ? 1 : 0);
}

// CUDA IPC for the peer-memory exchanges (tfl_api_slab.cu).  ipc_export: the handle of device allocation `dev` into an
// ABI buffer of `bytes`, zero-filled behind the handle.  ipc_map: maps the allocation whose handle starts at `handle`
// into *out; on failure it clears the CUDA error and fails as "<who>: <the CUDA call><which>: <error><tail>".
int ipc_export(tfl_ctx* ctx, void* dev, char* out, size_t bytes);
int ipc_map(tfl_ctx* ctx, const char* handle, IpcPtr<float>* out, const char* who, const char* which, const char* tail);

inline int make_geo(tfl_ctx* ctx, const tfl_grid* flags, int is3d, Geo* g) {
  g->nx = flags->nx; g->ny = flags->ny; g->nz = flags->nz; g->nb = flags->nb;
  g->is3d = is3d ? 1 : 0;
  g->nc = is3d ? 3 : 2;
  g->n = (long long)flags->nx * flags->ny * flags->nz;
  g->faults = ctx->counters.get();
  if (ctx->slab) {
    if (!is3d) return fail(ctx, "slab decomposition needs a 3D grid");
    g->zoff = ctx->zoff; g->gnz = ctx->gnz; g->zlo = ctx->zlo; g->zhi = ctx->zhi;
    if (g->zlo < 0 || g->zhi > g->nz || g->zlo >= g->zhi || g->zoff < 0 || g->zoff + g->nz > g->gnz)
      return fail(ctx, "slab range does not fit the local grid");
  } else {
    g->zoff = 0; g->gnz = flags->nz; g->zlo = 0; g->zhi = flags->nz;
  }
  if (!is3d && flags->nz != 1) return fail(ctx, "2D grid must have zsize == 1");
  if (grid_too_large(g->n, g->nb)) return fail(ctx, "grid too large");
  return check_launch_grid(ctx, "grid", g->nb, g->nz, g->ny);
}

// The step's body forces (lib/simulate.lua:216-239) for a grid of global extent nx x ny x gnz: the vectors that
// tfl_add_buoyancy / tfl_add_gravity take, the vorticity confinement amplitude, and whether each one runs
// (buoyancy also needs a density).
struct StepForces {
  bool buoyancy, gravity, vorticity;
  float buoy[3], grav[3];
  float vort_amp;
};
StepForces step_forces(const tfl_mconf* mc, int nx, int ny, int gnz);

constexpr int kMaxBanks = kMaxBankPtrs;     // banks a join kernel takes
constexpr int kTailFloats = 64 + 8 + 8 + 1;     // the fused 1x1x1 tail: w4[8][8], b4[8], w5[8], b5[1]

// Appends p to v; false (and v unchanged) if p is empty, its upload having failed.
inline bool keep(std::vector<DevPtr<float>>& v, DevPtr<float> p) {
  if (!p) return false;
  v.push_back(std::move(p));
  return true;
}

// Weight layouts of the projection network (tfl_api_cnn.cu).
// Packs a [8][cin][3][3][3] weight for launch_conv3_tc / launch_conv3_tc_join and uploads it.
DevPtr<float> upload_tc_weights(const float* w, int cin, int split);
// A convolution weight in Torch layout [cout][cin][taps] re-laid out as the [cin][tap][cout] that
// launch_conv_direct and launch_conv_any read.
std::vector<float> relayout_conv_weights(const float* w, int cin, int cout, int taps);
// Bank i's 8-channel slice of a 'concat' join weight [8][8 nbanks][3][3][3] (one bank: the whole weight).
std::vector<float> concat_slice(const float* w, int nbanks, int i);

// The projection network's forward pass (tfl_cnn_forward.cu).  What enqueues kernels returns how many it enqueued.
// Tensor-core path: padded channels-last activations owned by the model (their zero borders
// must survive between calls, so they do not live in the shared arena).
// z-slab (g.zoff, g.gnz): bank i holds the global coarse planes [ceil(zoff / 2^i), floor((zoff + nz) / 2^i)).
// Dilated banks: bank i's buffers hold its 8^i phase sub-grids per batch entry (make_conv_tc_phase_geo).
int cnn_ensure_act(tfl_ctx* ctx, tfl_cnn* m, const Geo& g);
// The three 3x3x3 layers (+ fused 1x1x1 tail) on tensor cores: act[0] -> act[1] -> act[2] -> p_net.
// p_lo / p_hi: planes on which p_net is wanted (default all).  Layer l then only has to produce the planes the
// later layers' 3x3x3 stencils reach from there; on a z-slab that spares most of the ghost planes.
int run_conv_stack(tfl_cnn* m, float* p_net, cudaStream_t st, int p_lo = 0, int p_hi = -1);
// The join layer of a banked stack (split 1, join 3) -> p_net on the output planes [g.z_lo, g.z_hi), reading bank
// i's layer-2 output l2[i] (geometry geo[i], 2^-i of bank 1's resolution) with nearest indexing.  z-slab: local
// full-resolution plane 0 is global plane zoff, bank i's local plane 0 its global coarse plane org[i] (whole grids:
// all 0).  'add': one launch summing the banks, weights wj[0]; 'concat': one launch per bank with its slice wj[i],
// banks N..2 writing / adding the fp32 partial sum `part`, bank 1 last adding it before the bias, ReLU and tail (one
// bank: no partial sum).  phases: banks 2..N are dilated banks held as phase sub-grids (geo[i] =
// make_conv_tc_phase_geo(.., i)) rather than multi-resolution banks.
int launch_tc_join(const float* const* l2, const ConvTcGeo* geo, const int* org, int zoff, int nbanks, bool add,
                   float* part, float* p_net, const std::vector<DevPtr<float>>& wj, const float* bias,
                   const float* tail, int split, const ConvTcGeo& g, cudaStream_t st, bool phases = false,
                   const TcEpi& ep = TcEpi());
// Device fields of one forward: pDiv, the velocity (UDiv, or on a z-slab the wall-masked U1 of tfl_cnn_stats), the
// flags, and the p and U the forward writes.
struct CnnFields {
  const float *p_div, *U, *flags;
  float *p_out, *U_out;
};
// model:forward on the whole grid g; scale_out (host, may be null) receives the input scale of every batch entry.
int cnn_project(tfl_ctx* ctx, tfl_cnn* m, const CnnFields& f, float threshold, const Geo& g, float* scale_out);
// Everything after the one global reduction, from the reduced sums of tfl_cnn_stats (tensor-core path only).
int cnn_project_from_sums(tfl_ctx* ctx, tfl_cnn* m, const CnnFields& f, const double* dev_sums, float threshold,
                          const Geo& g);
// Whether the model runs on a z-slab of a [gnz][ny][nx] domain with this margin whose local planes [0, nz) start at
// global plane zoff and own [own_lo, own_hi): the tensor-core path, and for banked models the margin of
// tfl_slab_cnn_margin, ghost planes that deep and a global grid divisible by 2^(banksNum-1).  Fails naming the
// z-slab; launches nothing.
int cnn_slab_check(tfl_ctx* ctx, const tfl_cnn* m, int margin, int gnz, int ny, int nx, int zoff, int nz, int own_lo,
                   int own_hi);

// The step monitor's refusals that do not need the grid (tfl_monitor.cu): a full ring, another nb or gnz.
int monitor_precheck(tfl_ctx* ctx, const tfl_monitor* m, int nb, int gnz);
