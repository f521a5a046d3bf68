// C ABI of libtfl (include/tfl.h): context, scratch arena, argument checks that mirror the
// asserts of the reference's Lua wrappers (torch/tfluids/init.lua), and the operator /
// whole-step entry points that enqueue the kernels of tfl_stencils.cu, tfl_model_stages.cu
// and tfl_cnn*.cu on the context's stream.  The projection network's entry points are in
// tfl_api_cnn.cu, the z-slab driver's in tfl_api_slab.cu.
#include <string.h>
#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

#include "tfl_api_internal.h"

namespace {

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
  void* p = nullptr;
  if (!fc.changed) {
    TFL_CUDA(ctx, cudaMalloc(&p, sizeof(int)));
    fc.changed.reset((int*)p);
  }
  if (fc.bytes && fc.cells == cells && fc.nb == g.nb && fc.nz == g.nz && fc.ny == g.ny && fc.nx == g.nx) {
    TFL_CUDA(ctx, cudaMemsetAsync(fc.changed.get(), 0, sizeof(int), ctx->stream));
    return 0;
  }
  TFL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  fc.bytes.reset();                         // before the new one is allocated
  fc.gen++;
  TFL_CUDA(ctx, cudaMalloc(&p, 3 * cells + 64));
  fc.bytes.reset((unsigned char*)p);
  fc.cells = cells; fc.nb = g.nb; fc.nz = g.nz; fc.ny = g.ny; fc.nx = g.nx;
  TFL_CUDA(ctx, cudaMemsetAsync(fc.bytes.get(), 0, 3 * cells + 64, ctx->stream));
  TFL_CUDA(ctx, cudaMemsetAsync(fc.changed.get(), 1, sizeof(int), ctx->stream));     // non-zero: rebuild
  return 0;
}

// Byte flags + clearance field of `flags` for this call, through the context's cache: the bytes are
// re-derived and compared on the device, the clearance is rebuilt only when one differs.
int prepare_flags(tfl_ctx* ctx, const float* flags, const Geo& g, unsigned char** fl8, unsigned char** clear) {
  const size_t cells = (size_t)g.n * g.nb;
  auto& fc = ctx->fcache;
  if (fc.fresh_for == flags && fc.bytes && fc.cells == cells && fc.nz == g.nz && fc.ny == g.ny && fc.nx == g.nx) {
    *fl8 = fc.bytes.get();                  // refreshed earlier in this (slab) step: nothing wrote the flags since
    *clear = fc.bytes.get() + cells;
    return 0;
  }
  if (flag_cache_ensure(ctx, g)) return 1;
  *fl8 = fc.bytes.get();
  *clear = fc.bytes.get() + cells;
  launch_flags_to_u8(flags, *fl8, (long long)cells, fc.changed.get(), ctx->stream);
  ctx->launches += 1 + launch_clearance(*fl8, *clear, *clear + cells, g, fc.changed.get(), ctx->stream);
  if (ctx->in_slab_step) fc.fresh_for = flags;
  return 0;
}

// Halo of the advection tile kernels for this call (0: use the per-pass kernels), from the longest trace the
// velocity kernel reported on earlier calls.
int tile_halo_choice(tfl_ctx* ctx, bool probe) {
  auto& tl = ctx->tile;
  if (tl.mode >= 0) return tl.mode;
  float longest = 0.0f;
  if (tl.host) { const unsigned int bits = *(volatile unsigned int*)tl.host.get(); memcpy(&longest, &bits, 4); }
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
  tl.last_vel_halo = 0;
  if (ours && fl8 && clear && tl.mode != 0) {
    if (!tl.dev || !tl.host) {
      if (!tl.dev) tl.dev = dev_alloc<unsigned int>(1);
      if (!tl.host && (tl.host = pinned_alloc<unsigned int>(1))) *tl.host = 0;
      if (!tl.dev || !tl.host) cudaGetLastError();    // no telemetry: the two-kernel version runs, nothing fails
    }
    const int hf = tile_halo_choice(ctx, true);
    if (hf > 0 && tl.dev && tl.host) {
      cudaMemsetAsync(tl.dev.get(), 0, sizeof(unsigned int), st);
      if (tl.timed) cudaEventRecord(tl.ev0.get(), st);
      const bool launched = launch_advect_vel_tile(dt, U, fl8, clear, strength, dst, g, hf, tl.variant, tl.dev.get(), st);
      if (tl.timed) cudaEventRecord(tl.ev1.get(), st);
      if (launched) {
        cudaMemcpyAsync(tl.host.get(), tl.dev.get(), sizeof(unsigned int), cudaMemcpyDeviceToHost, st);
        tl.last_vel_halo = hf;
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
  ctx->tile.last_scalar_halo = 0;
  if (method == TFL_ADVECT_MACCORMACK_OURS && fl8 && clear && ctx->tile.mode != 0) {
    const int hf = tile_halo_choice(ctx, false);
    if (hf > 0 && launch_advect_scalar_tile(dt, s, U, fl8, clear, outside, strength, dst, g, hf, ctx->tile.variant, st)) {
      ctx->tile.last_scalar_halo = hf;
      return 1;
    }
  }
  return launch_advect_scalar(dt, s, U, flags, clear, method, outside, strength, dst, fwd, fwd_pos, g, gf, st);
}

float get_dx(const Geo& g) {     // third_party/grid.cc:37-40 on the GLOBAL grid
  int m = g.nx > g.ny ? g.nx : g.ny;
  if (g.gnz > m) m = g.gnz;
  return 1.0f / (float)m;
}

// dst <- src on the planes [zlo, zhi) of each of `fields` consecutive [nz][ny][nx] fields: s:copy(tmp)
// (init.lua:145-148), only the computed planes in slab mode.
int copy_planes(tfl_ctx* ctx, float* dst, const float* src, int fields, const Geo& g) {
  for (int f = 0; f < fields; f++) {
    const size_t off = (size_t)f * g.n + (size_t)g.zlo * g.ny * g.nx;
    const size_t cnt = (size_t)(g.zhi - g.zlo) * g.ny * g.nx;
    TFL_CUDA(ctx, cudaMemcpyAsync(dst + off, src + off, cnt * 4, cudaMemcpyDeviceToDevice, ctx->stream));
  }
  return 0;
}

// An element-wise kernel over x: one launch(offset, count) over all of x, or in slab mode one per [b][c] field
// over the planes this rank computes (ghost planes come from the neighbours).
template <typename Launch>
int for_computed_planes(tfl_ctx* ctx, const tfl_grid* x, const char* what, Launch launch) {
  if (ctx->slab) {
    if (ctx->zlo < 0 || ctx->zhi > x->nz || ctx->zlo >= ctx->zhi) return fail(ctx, "%s: slab range does not fit", what);
    const long long plane = (long long)x->ny * x->nx, cnt = (long long)(ctx->zhi - ctx->zlo) * plane;
    for (int bc_i = 0; bc_i < x->nb * x->nc; bc_i++) launch(((long long)bc_i * x->nz + ctx->zlo) * plane, cnt);
    ctx->launches += x->nb * x->nc;
    return check_launch(ctx, what);
  }
  launch(0LL, (long long)x->nb * x->nc * x->nz * x->ny * x->nx);
  ctx->launches += 1;
  return check_launch(ctx, what);
}

}  // namespace

StepForces step_forces(const tfl_mconf* mc, int nx, int ny, int gnz) {
  const int dmax = std::max(nx, std::max(ny, gnz));
  const double dx = 1.0 / (double)dmax;                              // tfluids.getDx, init.lua:560-564
  StepForces f;
  f.buoyancy = mc->buoyancy_scale > 0.0;
  f.gravity = mc->gravity_scale > 0.0;
  f.vorticity = mc->vorticity_confinement_amp > 0.0;
  // gravity:mul(scalar) is a float tensor op: the Lua double is cast to float first.
  const float kb = (float)(-(dx / 4.0) * mc->buoyancy_scale);
  const float kg = (float)((-dx / 4.0) * mc->gravity_scale);
  for (int a = 0; a < 3; a++) {
    f.buoy[a] = mc->gravity[a] * kb;
    f.grav[a] = mc->gravity[a] * kg;
  }
  f.vort_amp = (float)(dx * mc->vorticity_confinement_amp);
  return f;
}

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
  // Declared after restore_: on a failure below, what was made is released while `device` is still current.
  std::unique_ptr<tfl_ctx> c(new tfl_ctx());
  c->device = device;
  if (!(c->own_stream = new_stream(cudaStreamDefault))) return 1;
  c->stream = c->own_stream.get();
  if (!(c->counters = dev_zeros<unsigned long long>(16)) || !(c->dscratch = dev_alloc<double>(256))) return 1;
  for (StreamPtr* q : {&c->side_stream, &c->copy_in, &c->copy_out})
    if (!(*q = new_stream(cudaStreamNonBlocking))) return 1;
  for (EventPtr* e : {&c->ev_fork, &c->ev_join, &c->ev_u_in, &c->ev_d_in, &c->ev_p_in, &c->ev_d_ready, &c->ev_d_out})
    if (!(*e = new_event(cudaEventDisableTiming))) return 1;
  *out = c.release();
  return 0;
}

void tfl_destroy(tfl_ctx* ctx) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!ctx) return;
  for (cudaStream_t q : {ctx->stream, ctx->side_stream.get(), ctx->copy_in.get(), ctx->copy_out.get()})
    cudaStreamSynchronize(q);
  tfl_comm_destroy(ctx);
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
      cudaStream_t q = nullptr;
      TFL_CUDA(ctx, cudaStreamCreate(&q));
      ctx->own_stream.reset(q);
      ctx->stream = q;
    }
    return 0;
  }
  if ((cudaStream_t)s == ctx->own_stream.get()) return 0;
  ctx->own_stream.reset();                  // an adopted stream is the caller's: never destroyed here
  ctx->stream = (cudaStream_t)s;
  return 0;
}
void* tfl_get_stream(tfl_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }
int tfl_sync(tfl_ctx* ctx) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  TFL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (conv_tc_take_z_fault(ctx->stream)) return fail(ctx, "%s", kConvZStalled);
  return 0;
}
int64_t tfl_launch_count(const tfl_ctx* ctx) { return ctx ? ctx->launches : 0; }

int tfl_trace_faults(tfl_ctx* ctx, int64_t* count, int reset) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  unsigned long long v = 0;
  TFL_CUDA(ctx, cudaMemcpyAsync(&v, ctx->counters.get(), sizeof(v), cudaMemcpyDeviceToHost, ctx->stream));
  TFL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (count) *count = (int64_t)v;
  if (reset) TFL_CUDA(ctx, cudaMemsetAsync(ctx->counters.get(), 0, sizeof(v), ctx->stream));
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
  TFL_CUDA(ctx, cudaMemsetAsync(ctx->counters.get() + 1, 0, sizeof(unsigned long long), ctx->stream));
  launch_flags_to_occupancy(flags->data, occ->data, n, ctx->counters.get() + 1, ctx->stream);
  ctx->launches += 1;
  if (check_launch(ctx, "flagsToOccupancy")) return 1;
  if (bad) {
    unsigned long long v = 0;
    TFL_CUDA(ctx, cudaMemcpyAsync(&v, ctx->counters.get() + 1, sizeof(v), cudaMemcpyDeviceToHost, ctx->stream));
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
  return in_place ? copy_planes(ctx, s->data, tmp, g.nb, g) : 0;
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
  return in_place ? copy_planes(ctx, U->data, tmp, g.nb * g.nc, g) : 0;
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
  // Larger grids are bandwidth-bound per sweep and do not fit the SMs.
  if (!need_every && max_iter > 2 && g.is3d && g.nz >= 4 && g.n * g.nb <= (3LL << 20)) {
    const int fused = max_iter - 1;
    if (launch_jacobi_block(mask, div->data, p_prev, p->data, g, 0, g.nz, 0, 0, fused, /*deep=*/false, st)) {
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
      TFL_CUDA(ctx, cudaMemsetAsync(ctx->dscratch.get(), 0, sizeof(double) * g.nb, st));
      launch_sqdiff(p->data, p_prev, g.n, g.nb, ctx->dscratch.get(), st);
      ctx->launches += 1;
      TFL_CUDA(ctx, cudaMemcpyAsync(h.data(), ctx->dscratch.get(), sizeof(double) * g.nb, cudaMemcpyDeviceToHost, st));
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

// Arguments and workspace of the PCG entry points (the solve and the preconditioner hook): out and rhs are the
// scalar grids written and read beside flags.
static int pcg_check_args(tfl_ctx* ctx, const tfl_grid* out, const char* out_name, const tfl_grid* flags,
                          const tfl_grid* rhs, const char* rhs_name, int is_3d, int precond) {
  if (check_scalar(ctx, flags, "flags") || check_scalar(ctx, out, out_name) || check_scalar(ctx, rhs, rhs_name)) return 1;
  if (!same_spatial(flags, out) || !same_spatial(flags, rhs)) return fail(ctx, "size mismatch");
  if (!is_3d && flags->nz != 1) return fail(ctx, "d > 1 for a 2D domain");
  if (precond < TFL_PRECOND_NONE || precond > TFL_PRECOND_IC0)
    return fail(ctx, "Incorrect preconType ('none', 'ic0', 'ilu0')");      // generic/tfluids.cu:1551
  if (ctx->slab) return fail(ctx, "PCG does not shard (triangular solves): single GPU only");
  if ((long long)flags->nb * flags->nz * flags->ny * flags->nx >= (1ll << 31)) return fail(ctx, "PCG: grid too large");
  return arena_reserve(ctx, pcg_workspace_bytes(flags->nb, flags->nz, flags->ny, flags->nx)) ? 1 : 0;
}

static int pcg_report(tfl_ctx* ctx, int rc, const char* what) {
  if (rc == 3) return fail(ctx, "%s: %s", what, cudaGetErrorString(cudaGetLastError()));
  if (rc) return fail(ctx, "%s", pcg_status_string(rc));
  return check_launch(ctx, what);
}

int tfl_solve_linear_system_pcg(tfl_ctx* ctx, const tfl_grid* p, const tfl_grid* flags, const tfl_grid* div,
                                int is_3d, int precond, float tol, int max_iter, float* residual,
                                int* iterations) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (pcg_check_args(ctx, p, "p", flags, div, "div", is_3d, precond)) return 1;
  const int rc =
      ctx->pcg_graph
          ? pcg_solve_graph(*ctx->pcg_graph, ctx->pcg, ctx->arena.get(), p->data, flags->data, div->data, flags->nb,
                            flags->nz, flags->ny, flags->nx, is_3d, precond, tol, max_iter, &ctx->launches, ctx->stream)
          : pcg_solve(ctx->pcg, ctx->arena.get(), p->data, flags->data, div->data, flags->nb, flags->nz, flags->ny,
                      flags->nx, is_3d, precond, tol, max_iter, residual, iterations, &ctx->launches, ctx->stream);
  return pcg_report(ctx, rc, "solveLinearSystemPCG");
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
  if (normalize_pressure_mean(ctx->arena.get(), p->data, flags->data, flags->nb, flags->nz, flags->ny, flags->nx, is_3d,
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

// Debug hook: the PCG preconditioner alone, z = M^-1 r (0 outside every system of two or more cells),
// through the labelling, system build and sweeps of tfl_solve_linear_system_pcg.  geometry (4 ints, may be
// null): NYP, planes per CTA, plane chunks, cooperative grid of the sweeps.
extern "C" int tfl_debug_pcg_precond(tfl_ctx* ctx, const tfl_grid* z, const tfl_grid* flags, const tfl_grid* r,
                                     int is_3d, int precond, int* geometry) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (pcg_check_args(ctx, z, "z", flags, r, "r", is_3d, precond)) return 1;
  const int rc = pcg_precond(ctx->pcg, ctx->arena.get(), z->data, flags->data, r->data, flags->nb, flags->nz, flags->ny,
                             flags->nx, is_3d, precond, geometry, &ctx->launches, ctx->stream);
  return pcg_report(ctx, rc, "pcg precond");
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
  return for_computed_planes(ctx, x, "applyBC", [&](long long off, long long n) {
    launch_apply_bc(x->data + off, inv_mask->data + off, bc->data + off, n, ctx->stream);
  });
}

int tfl_clamp(tfl_ctx* ctx, const tfl_grid* x, float lo, float hi) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!x || !x->data) return fail(ctx, "clamp: nil tensor");
  return for_computed_planes(ctx, x, "clamp",
                             [&](long long off, long long n) { launch_clamp(x->data + off, lo, hi, n, ctx->stream); });
}
// Debug hook: the grid checks every operator makes on its flags descriptor (make_geo), alone.  The data pointer
// is never read and nothing is launched, so any extent can be asked about without allocating it.
int tfl_debug_make_geo(tfl_ctx* ctx, const tfl_grid* flags, int is_3d) {
  if (!ctx || !flags) return 1;
  Geo g;
  return make_geo(ctx, flags, is_3d, &g);
}

// Undocumented debugging hook.
// mode: -1 automatic, 0 two-kernel advectVel, 1 / 2 tile kernel with that halo; variant: tile shape.
int tfl_debug_advect_tile(tfl_ctx* ctx, int mode, int variant) {
  if (!ctx) return 1;
  ctx->tile.mode = mode;
  ctx->tile.variant = variant;
  return 0;
}

// Undocumented debugging hook, read-only: the tile halo the last advectVel and advectScalar dispatches launched
// (0: the per-pass kernels ran) and the longest trace in the pinned telemetry word, which the next automatic choice
// reads (synchronise first for the last call's value).  Launches nothing.
int tfl_debug_advect_tile_used(tfl_ctx* ctx, int32_t* vel_halo, int32_t* scalar_halo, float* longest) {
  if (!ctx || !vel_halo || !scalar_halo || !longest) return 1;
  *vel_halo = ctx->tile.last_vel_halo;
  *scalar_halo = ctx->tile.last_scalar_halo;
  *longest = 0.0f;
  if (ctx->tile.host) {
    const unsigned int bits = *(volatile unsigned int*)ctx->tile.host.get();
    memcpy(longest, &bits, 4);
  }
  return 0;
}

// Events around the advectVel tile kernel alone (bench.py's roofline).  on: start recording; the getter
// synchronises and returns the duration of the last recorded launch in ms (< 0 if none).
int tfl_debug_time_advect_kernel(tfl_ctx* ctx, int on) {
  if (!ctx) return 1;
  DeviceGuard guard_(ctx);
  auto& tl = ctx->tile;
  if (on && !(tl.ev0 && tl.ev1)) {
    tl.ev0 = new_event(cudaEventDefault);
    tl.ev1 = new_event(cudaEventDefault);
    if (!tl.ev0 || !tl.ev1) cudaGetLastError();     // untimed: the getter reports -1, nothing else fails
  }
  tl.timed = on != 0 && tl.ev0 && tl.ev1;
  return 0;
}
float tfl_debug_last_advect_kernel_ms(tfl_ctx* ctx) {
  if (!ctx || !ctx->tile.ev0 || !ctx->tile.ev1) return -1.0f;
  DeviceGuard guard_(ctx);
  float ms = -1.0f;
  cudaEvent_t e0 = ctx->tile.ev0.get(), e1 = ctx->tile.ev1.get();
  if (cudaEventSynchronize(e1) != cudaSuccess || cudaEventElapsedTime(&ms, e0, e1) != cudaSuccess) {
    cudaGetLastError();
    return -1.0f;
  }
  return ms;
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

// Fused pipeline for the convnet path with the tensor-core conv stack: 12 launches with a single-bank
// stack, every field crosses memory once per stage.  Bit-identical to the operator sequence below.
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
  if (ov) TFL_CUDA(ctx, cudaStreamWaitEvent(st, ctx->ev_u_in.get(), 0));          // U has arrived from the host
  // Which quads of the BC arrays are the identity pair (the point-wise stages then skip their loads): rebuilt
  // every step from the arrays, beside the advection (on the side stream when there is one).
  const unsigned char* qmask = nullptr;
  const bool u_bc0 = s->U_bc.data && s->U_bc_inv_mask.data;
  const bool d_bc0 = has_density && s->density_bc.data && s->density_bc_inv_mask.data;
  bool qmask_on_side = false;
  if (has_density) {
    // Density and velocity advection are independent (both read the old U): run the density
    // kernels on a side stream so the two latency-bound kernel pairs overlap.
    TFL_CUDA(ctx, cudaEventRecord(ctx->ev_fork.get(), st));
    TFL_CUDA(ctx, cudaStreamWaitEvent(ctx->side_stream.get(), ctx->ev_fork.get(), 0));
    if (launch_bc_quad_mask(u_bc0 ? s->U_bc_inv_mask.data : nullptr, u_bc0 ? s->U_bc.data : nullptr,
                            d_bc0 ? s->density_bc_inv_mask.data : nullptr, d_bc0 ? s->density_bc.data : nullptr,
                            qmask_buf, g, ctx->side_stream.get())) {
      qmask = qmask_buf;
      qmask_on_side = true;
      ctx->launches += 1;
    }
    if (ov) TFL_CUDA(ctx, cudaStreamWaitEvent(ctx->side_stream.get(), ctx->ev_d_in.get(), 0));
    const int nl = advect_scalar_dispatch(ctx, mc->dt, s->density.data, s->U.data, fl8, fl8, clear, mc->advection_method,
                                          0, mc->maccormack_strength, tmp_s, fwd_s, fwd_pos, g, g, ctx->side_stream.get());
    if (nl < 0) return fail(ctx, "advectScalar: bad method");
    ctx->launches += nl;
    TFL_CUDA(ctx, cudaEventRecord(ctx->ev_join.get(), ctx->side_stream.get()));
  }
  {
    const int nl = advect_vel_dispatch(ctx, mc->dt, s->U.data, fl8, fl8, clear, mc->advection_method,
                                       mc->maccormack_strength, tmp_u, fwd_u, g, g, st);
    if (nl < 0) return fail(ctx, "advectVel: bad method");
    ctx->launches += nl;
  }
  if (has_density) TFL_CUDA(ctx, cudaStreamWaitEvent(st, ctx->ev_join.get(), 0));
  if (!qmask_on_side && launch_bc_quad_mask(u_bc0 ? s->U_bc_inv_mask.data : nullptr, u_bc0 ? s->U_bc.data : nullptr, nullptr,
                                            nullptr, qmask_buf, g, st)) {
    qmask = qmask_buf;
    ctx->launches += 1;
  }
  const StepForces fo = step_forces(mc, g.nx, g.ny, g.gnz);
  const float scale_dt = mc->dt / get_dx(g);          // as tfl_add_buoyancy / tfl_add_gravity scale their vectors
  const bool u_bc = s->U_bc.data && s->U_bc_inv_mask.data;
  const bool d_bc = has_density && s->density_bc.data && s->density_bc_inv_mask.data;
  float bs[3] = {0.0f, 0.0f, 0.0f};
  const int do_buoy = has_density && fo.buoyancy;
  if (do_buoy)
    for (int a = 0; a < 3; a++) bs[a] = (-fo.buoy[a]) * scale_dt;
  launch_post_advect(has_density ? tmp_s : nullptr, tmp_u, fl8, has_density ? s->density.data : nullptr,
                     s->U.data, u_bc ? s->U_bc_inv_mask.data : nullptr, u_bc ? s->U_bc.data : nullptr,
                     d_bc ? s->density_bc_inv_mask.data : nullptr, d_bc ? s->density_bc.data : nullptr, qmask, do_buoy, bs,
                     g, st);
  ctx->launches += 1;
  if (ov && has_density && ctx->ov.density_host) {
    // The density is final here (nothing later in the step writes it): send it home while the
    // vorticity / projection kernels run.
    TFL_CUDA(ctx, cudaEventRecord(ctx->ev_d_ready.get(), st));
    TFL_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_out.get(), ctx->ev_d_ready.get(), 0));
    TFL_CUDA(ctx, cudaMemcpyAsync(ctx->ov.density_host, s->density.data, ctx->ov.density_bytes, cudaMemcpyDeviceToHost,
                                  ctx->copy_out.get()));
    TFL_CUDA(ctx, cudaEventRecord(ctx->ev_d_out.get(), ctx->copy_out.get()));
    ctx->ov.density_sent = true;
  }
  if (fo.gravity) {
    const float f[3] = {fo.grav[0] * scale_dt, fo.grav[1] * scale_dt, fo.grav[2] * scale_dt};
    launch_add_gravity(s->U.data, fl8, f, g, st);
    ctx->launches += 1;
  }
  if (fo.vorticity) {
    launch_vort_curl(s->U.data, curl, cnorm, force, fo.vort_amp, g, st);
    ctx->launches += 2;
  }
  double* sums = ctx->dscratch.get() + 64;
  TFL_CUDA(ctx, cudaMemsetAsync(sums, 0, sizeof(double) * 2 * g.nb, st));
  launch_vort_bc_mask(s->U.data, fl8, force, fo.vorticity, u_bc ? s->U_bc_inv_mask.data : nullptr,
                      u_bc ? s->U_bc.data : nullptr, qmask, 1, sums, g, st);
  const ConvTcGeo& tg = m->act_geo;
  if (ov) TFL_CUDA(ctx, cudaStreamWaitEvent(st, ctx->ev_p_in.get(), 0));          // pDiv is first read here
  launch_cnn_inputs_fused(s->p.data, s->U.data, fl8, sums, mc->normalize_input_threshold, scale, m->act[0].get(),
                          tg.px, tg.py, g, st);
  const int stack = run_conv_stack(m, p_net, st);
  launch_cnn_finish_fused(p_net, s->U.data, fl8, scale, s->p.data, u_bc ? s->U_bc_inv_mask.data : nullptr,
                          u_bc ? s->U_bc.data : nullptr, qmask, -1e6f, 1e6f, g, st);
  ctx->launches += 3 + stack;     // launch_vort_bc_mask, the fused input and finish, and the stack's own
  return check_launch(ctx, "simulate_step (fused)");
}

// Whether tfl_simulate_step takes the fused pipeline for this state, configuration and model.
static bool fused_step_applies(const tfl_ctx* ctx, const tfl_state* s, const tfl_mconf* mc, const tfl_cnn* cnn) {
  return mc->sim_method == TFL_SIM_CONVNET && cnn && cnn->tc_ok && cnn->mode > 0 && cnn->default_inputs && !ctx->slab &&
         s->flags.nb == 1 &&
         !s->p_bc.data && mc->advection_method >= 0 && mc->advection_method <= 5;
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
  if (fused_step_applies(ctx, s, mc, cnn)) {
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
  const StepForces fo = step_forces(mc, g.nx, g.ny, g.gnz);
  if (has_density && fo.buoyancy && tfl_add_buoyancy(ctx, &s->U, &s->flags, &s->density, fo.buoy, mc->dt))  // :216-226
    return 1;
  if (fo.gravity && tfl_add_gravity(ctx, &s->U, &s->flags, fo.grav, mc->dt)) return 1;                      // :229-233
  if (fo.vorticity && tfl_vorticity_confinement(ctx, &s->U, &s->flags, fo.vort_amp)) return 1;              // :236-239
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
  tfl_state st;                     // views of the buffers below
  DevPtr<float> flags, p, U, density, div, U_bc, U_bc_inv, d_bc, d_bc_inv;
  size_t cells = 0;
  int nc = 3;
};

int tfl_host_sim_create(tfl_ctx* ctx, int32_t nb, int32_t nz, int32_t ny, int32_t nx, int is_3d,
                        const float* flags, const float* U_bc, const float* U_bc_inv, const float* d_bc,
                        const float* d_bc_inv, tfl_host_sim** out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!out || !flags) return fail(ctx, "host_sim: bad arguments");
  *out = nullptr;
  if (nb < 1 || nz < 1 || ny < 1 || nx < 1) return fail(ctx, "host_sim: every grid extent must be >= 1");
  if (!is_3d && nz != 1) return fail(ctx, "host_sim: 2D grid must have zsize == 1");
  if (grid_too_large((long long)nz * ny * nx, nb)) return fail(ctx, "host_sim: grid too large");
  std::unique_ptr<tfl_host_sim> hs(new tfl_host_sim());
  memset(&hs->st, 0, sizeof(hs->st));
  hs->nc = is_3d ? 3 : 2;
  hs->cells = (size_t)nb * nz * ny * nx;
  // d <- a device copy of host (zeros without one) of nc channels; g views it
  auto mk = [&](DevPtr<float>& d, tfl_grid* g, int nc, const float* host) {
    d = host ? upload(host, hs->cells * nc) : dev_zeros<float>(hs->cells * nc);
    *g = {d.get(), nb, nc, nz, ny, nx};
    return d != nullptr;
  };
  tfl_state& st = hs->st;
  const int nc = hs->nc;
  if (!mk(hs->flags, &st.flags, 1, flags) || !mk(hs->p, &st.p, 1, nullptr) || !mk(hs->U, &st.U, nc, nullptr) ||
      !mk(hs->density, &st.density, 1, nullptr) || !mk(hs->div, &st.div, 1, nullptr) ||
      (U_bc && U_bc_inv && (!mk(hs->U_bc, &st.U_bc, nc, U_bc) || !mk(hs->U_bc_inv, &st.U_bc_inv_mask, nc, U_bc_inv))) ||
      (d_bc && d_bc_inv && (!mk(hs->d_bc, &st.density_bc, 1, d_bc) || !mk(hs->d_bc_inv, &st.density_bc_inv_mask, 1, d_bc_inv))))
    return fail(ctx, "host_sim: cudaMalloc failed");
  *out = hs.release();
  return 0;
}

void tfl_host_sim_destroy(tfl_ctx* ctx, tfl_host_sim* hs) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (hs && ctx) cudaStreamSynchronize(ctx->stream);
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
  TFL_CUDA(ctx, cudaEventRecord(ctx->ev_fork.get(), st));                      // earlier work on the step stream
  TFL_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_in.get(), ctx->ev_fork.get(), 0));
  TFL_CUDA(ctx, cudaMemcpyAsync(s.U.data, U, hs->cells * 4 * hs->nc, cudaMemcpyHostToDevice, ctx->copy_in.get()));
  TFL_CUDA(ctx, cudaEventRecord(ctx->ev_u_in.get(), ctx->copy_in.get()));
  if (density) TFL_CUDA(ctx, cudaMemcpyAsync(s.density.data, density, hs->cells * 4, cudaMemcpyHostToDevice, ctx->copy_in.get()));
  TFL_CUDA(ctx, cudaEventRecord(ctx->ev_d_in.get(), ctx->copy_in.get()));
  TFL_CUDA(ctx, cudaMemcpyAsync(s.p.data, p, hs->cells * 4, cudaMemcpyHostToDevice, ctx->copy_in.get()));
  TFL_CUDA(ctx, cudaEventRecord(ctx->ev_p_in.get(), ctx->copy_in.get()));
  const bool fused = fused_step_applies(ctx, &s, mc, cnn);
  ctx->ov.active = fused;
  ctx->ov.density_host = density;
  ctx->ov.density_bytes = hs->cells * 4;
  ctx->ov.density_sent = false;
  if (!fused) {                                                           // operator-by-operator path: no overlap
    TFL_CUDA(ctx, cudaStreamWaitEvent(st, ctx->ev_p_in.get(), 0));
  }
  const int rc = tfl_simulate_step(ctx, &s, mc, cnn);
  const bool density_sent = ctx->ov.density_sent;
  ctx->ov.active = false;
  if (rc) { cudaStreamSynchronize(ctx->copy_in.get()); cudaStreamSynchronize(ctx->copy_out.get()); return 1; }
  TFL_CUDA(ctx, cudaMemcpyAsync(U, s.U.data, hs->cells * 4 * hs->nc, cudaMemcpyDeviceToHost, st));
  TFL_CUDA(ctx, cudaMemcpyAsync(p, s.p.data, hs->cells * 4, cudaMemcpyDeviceToHost, st));
  if (density && !density_sent)
    TFL_CUDA(ctx, cudaMemcpyAsync(density, s.density.data, hs->cells * 4, cudaMemcpyDeviceToHost, st));
  if (density_sent) TFL_CUDA(ctx, cudaStreamWaitEvent(st, ctx->ev_d_out.get(), 0));
  TFL_CUDA(ctx, cudaStreamSynchronize(st));
  return 0;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------
// The step as a CUDA graph: tfl_simulate_step captured once on the context's stream (both streams of the
// fused step, their fork / join events, the memsets and the telemetry copy become graph nodes) and replayed
// with one launch.  Pointers and every host-side choice of the captured call (fused or per-operator path,
// advection tile halo) are frozen into the graph; results equal tfl_simulate_step's.
// The graph also holds pointers into buffers the library owns: the context's scratch arena and flag cache, and
// the model's activation buffers.  Each carries a generation counter; a launch after any of them was reallocated
// is refused (the replay would read and write freed memory).
// A PCG step's solve is captured by pcg_solve_graph: its iteration loop is a conditional node the device re-arms,
// and its per-component scalars, progress words and result words are the graph's own (PcgGraphScratch), allocated
// before the capture for the most components the grid can hold.
// ---------------------------------------------------------------------------------------
struct tfl_step_graph {
  PcgGraphScratch pcg;          // declared first: released after the executable graph that uses it
  GraphPtr graph;
  GraphExecPtr exec;
  long long launches = 0;       // kernels in one replay outside the PCG loop
  unsigned long long arena_gen = 0, fcache_gen = 0, act_gen = 0;   // generations of the captured buffers
  tfl_cnn* cnn = nullptr;       // the captured model (its act_gen is checked), or null
};

extern "C" {

void tfl_step_graph_destroy(tfl_ctx* ctx, tfl_step_graph* g) {
  DeviceGuard guard_(ctx);
  if (g && ctx) cudaStreamSynchronize(ctx->stream);
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
  std::unique_ptr<tfl_step_graph> g(new tfl_step_graph());
  const bool pcg = mc->sim_method == TFL_SIM_PCG;
  if (pcg) {              // the limits of the direct solve, by name, before anything is allocated or captured
    if (check_scalar(ctx, &state->flags, "flags")) return 1;
    if (ctx->slab) return fail(ctx, "step_graph: PCG does not shard (triangular solves): single GPU only");
    const tfl_grid& f = state->flags;
    const int prc = pcg_graph_alloc(g->pcg, ctx->pcg, f.nb, f.nz, f.ny, f.nx, state->U.nc == 3);
    if (prc == 4) return fail(ctx, "step_graph: %s", pcg_status_string(prc));
    if (prc) return fail(ctx, "step_graph: PCG buffers: %s", cudaGetErrorString(cudaGetLastError()));
  }
  TFL_CUDA(ctx, cudaStreamSynchronize(st));
  const long long l0 = ctx->launches;
  if (cudaStreamBeginCapture(st, cudaStreamCaptureModeRelaxed) != cudaSuccess) {
    cudaGetLastError();
    return fail(ctx, "step_graph: cudaStreamBeginCapture failed");
  }
  ctx->pcg_graph = pcg ? &g->pcg : nullptr;
  const int rc = tfl_simulate_step(ctx, state, mc, cnn);
  ctx->pcg_graph = nullptr;
  cudaGraph_t graph = nullptr;
  const cudaError_t e = cudaStreamEndCapture(st, &graph);
  g->graph.reset(graph);
  if (rc != 0 || e != cudaSuccess || !graph) {
    cudaGetLastError();
    const std::string why = rc != 0 ? ctx->err : std::string(cudaGetErrorString(e));
    return fail(ctx, "step_graph: capture failed (%s); run tfl_simulate_step once before capturing", why.c_str());
  }
  g->launches = ctx->launches - l0;
  ctx->launches = l0;
  cudaGraphExec_t exec = nullptr;
  if (cudaGraphInstantiate(&exec, graph, 0) != cudaSuccess) {
    cudaGetLastError();
    return fail(ctx, "step_graph: cudaGraphInstantiate failed");
  }
  g->exec.reset(exec);
  g->arena_gen = ctx->arena_gen;
  g->fcache_gen = ctx->fcache.gen;
  g->cnn = cnn;
  g->act_gen = cnn ? cnn->act_gen : 0;
  *out = g.release();
  return 0;
}

int tfl_step_graph_launch(tfl_ctx* ctx, tfl_step_graph* g) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!g || !g->exec) return fail(ctx, "step_graph is nil");
  const char* stale = g->arena_gen != ctx->arena_gen      ? "the context's scratch arena"
                      : g->fcache_gen != ctx->fcache.gen  ? "the context's flag cache"
                      : g->cnn && g->act_gen != g->cnn->act_gen ? "the model's activation buffers"
                                                                : nullptr;
  if (stale)
    return fail(ctx, "step_graph: stale graph: %s reallocated since the capture (a call on another grid shape or a "
                     "larger grid); replaying would touch freed memory: capture the step again", stale);
  TFL_CUDA(ctx, cudaGraphLaunch(g->exec.get(), ctx->stream));
  ctx->launches += g->launches;
  return 0;
}

int tfl_step_graph_pcg_status(tfl_ctx* ctx, tfl_step_graph* g, float* residual, int32_t* iterations) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!g || !g->exec) return fail(ctx, "step_graph is nil");
  if (!g->pcg.captured) {
    if (iterations) *iterations = -1;
    return 0;
  }
  int w[8];
  cudaStream_t st = ctx->stream;
  TFL_CUDA(ctx, cudaMemcpyAsync(w, g->pcg.words.get(), sizeof(w), cudaMemcpyDeviceToHost, st));
  // the error has been read and the passes counted: both start again from here
  TFL_CUDA(ctx, cudaMemsetAsync(g->pcg.words.get(), 0, sizeof(int), st));
  TFL_CUDA(ctx, cudaMemsetAsync(g->pcg.words.get() + 4, 0, sizeof(unsigned long long), st));
  TFL_CUDA(ctx, cudaStreamSynchronize(st));
  unsigned long long passes = 0;
  memcpy(&passes, w + 4, sizeof(passes));
  ctx->launches += (long long)passes * g->pcg.body_launches;
  if (w[0]) return fail(ctx, "%s", pcg_status_string(w[0]));
  float res;
  memcpy(&res, w + 2, sizeof(res));
  if (residual) *residual = res;
  if (iterations) *iterations = w[1];
  return 0;
}

}  // extern "C"
