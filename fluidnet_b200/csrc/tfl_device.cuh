// Device-side building blocks shared by the stencil kernels: grid geometry, flag tests,
// MAC-grid sampling, Manta-style trilinear interpolation and the obstacle-aware line
// trace.  Written for sm_90a; every translation unit that includes this header for a
// parity-critical kernel is compiled with -fmad=false (the CPU reference has no FMA
// contraction), IEEE division / sqrt (nvcc defaults, no --use_fast_math).
//
// Semantics follow the reference CPU path (paths relative to /root/reference/torch/tfluids):
//   flag bits        third_party/cell_type.h:22-33, third_party/grid.h:103-141
//   buildIndex       third_party/grid.cc:82-130   (truncation, clamp-after-weights)
//   interpol         third_party/grid.cc:182-202, :435-456 (fixed evaluation order)
//   interpolWithFluid third_party/grid.cc:204-332
//   getCentered / getAtMAC{X,Y,Z}  third_party/grid.cc:346-417
//   calcLineTrace    generic/calc_line_trace.cc:101-503
//
// Coordinates are GLOBAL: a grid may be a z-slab [zoff, zoff+nz) of a domain with gnz
// planes; border tests and traces behave as in the undivided domain.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <float.h>

namespace tfl {

struct Geo {
  int nx, ny, nz;        // local extents of every grid
  int gnz;               // global z extent
  int zoff;              // global index of local plane 0
  int zlo, zhi;          // local planes this launch computes
  int nb;                // batch
  int is3d;
  int nc;                // velocity channels (3 or 2)
  long long n;           // cells per (batch, channel) = nx*ny*nz
  unsigned long long* faults;   // device counter (trace faults / slab overruns)
  // Local planes out of reach at the low / high end, on top of the storage bounds: an access there is a fault.
  // Non-zero only for the backward pass of a z-slab's MacCormack advection, whose forward field holds just the
  // planes the forward pass computed (the slab margin around the owned ones).
  int skip_lo = 0, skip_hi = 0;
};

struct V3 { float x, y, z; };

// Kernels are specialised on the dimensionality: copying the geometry and overwriting the two
// fields with compile-time constants lets the compiler prune 2-D/3-D branches and unroll the
// per-component loops.
template <bool IS3D>
__device__ __forceinline__ Geo static_geo(const Geo& gin) {
  Geo g = gin;
  g.is3d = IS3D ? 1 : 0;
  g.nc = IS3D ? 3 : 2;
  return g;
}

enum : int { kFluid = 1, kObstacle = 2, kEmpty = 4, kOutflow = 16, kStick = 128 };

// Offsets inside one (batch, channel) block fit 32 bits (n < 2^31, checked on the host).
__device__ __forceinline__ int cell(const Geo& g, int k, int j, int i) {
  return (k * g.ny + j) * g.nx + i;
}
// Flags come either as the API's float bit codes or as the byte copy the fused step makes
// once per step (same low 8 bits: every bit the kernels test is below 256).
__device__ __forceinline__ int flag_at(const float* __restrict__ fl, int o) { return (int)__ldg(fl + o); }
__device__ __forceinline__ int flag_at(const unsigned char* __restrict__ fl, int o) { return (int)__ldg(fl + o); }
template <typename FT>
__device__ __forceinline__ int flag_i(const FT* __restrict__ fl, const Geo& g, int k, int j, int i) {
  return flag_at(fl, cell(g, k, j, i));
}
// k is LOCAL here; the border is defined on the global grid.
__device__ __forceinline__ bool on_border(const Geo& g, int k, int j, int i) {
  const int kg = k + g.zoff;
  return i < 1 || i > g.nx - 2 || j < 1 || j > g.ny - 2 ||
         (g.is3d && (kg < 1 || kg > g.gnz - 2));
}
__device__ __forceinline__ float std_min(float a, float b) { return (b < a) ? b : a; }
__device__ __forceinline__ float std_max(float a, float b) { return (a < b) ? b : a; }
__device__ __forceinline__ float clamp_f(float v, float lo, float hi) {
  return std_min(hi, std_max(lo, v));
}
__device__ __forceinline__ int clamp_i(int x, int lo, int hi) {
  const int m = x < hi ? x : hi;
  return m > lo ? m : lo;
}
__device__ __forceinline__ void note_fault(const Geo& g) {
  if (g.faults) atomicAdd(g.faults, 1ULL);
}
// Local plane of a global z index; records a fault (and clamps) if the slab halo, or the
// planes in reach (skip_lo / skip_hi), are too small for the access.
// Clearance of a cell on local plane k, capped at its distance to the planes out of reach as the clearance field
// is capped at the ends of the local storage: the fast path of a cell with clearance never reads past them.
__device__ __forceinline__ int clear_in_reach(const Geo& g, int clr, int k) {
  if ((g.skip_lo | g.skip_hi) == 0) return clr;
  const int lo = k - g.skip_lo, hi = g.nz - 1 - g.skip_hi - k;
  return clr < lo ? (clr < hi ? clr : hi) : (lo < hi ? lo : hi);
}
__device__ __forceinline__ int local_z(const Geo& g, int kg) {
  int k = kg - g.zoff;
  if (k < g.skip_lo || k >= g.nz - g.skip_hi) {
    note_fault(g);
    k = k < g.skip_lo ? g.skip_lo : g.nz - g.skip_hi - 1;
  }
  return k;
}

__device__ __forceinline__ float norm3(V3 a) {       // vec3::norm, generic/vec3.h:119-127
  const float l2 = a.x * a.x + a.y * a.y + a.z * a.z;
  return (l2 > 1e-6f) ? sqrtf(l2) : 0.0f;
}
__device__ __forceinline__ V3 scale3(V3 a, float s) { return V3{a.x * s, a.y * s, a.z * s}; }

// ---------------------------------------------------------------------------------------
// Interpolation (positions are global; `blk` is the [z][y][x] block of one channel).
// ---------------------------------------------------------------------------------------
struct Lerp { int xi, yi, zi; float s0, s1, t0, t1, f0, f1; };

__device__ __forceinline__ Lerp build_index(const Geo& g, V3 pos) {
  Lerp q;
  const float px = pos.x - 0.5f, py = pos.y - 0.5f, pz = pos.z - 0.5f;
  q.xi = (int)px; q.yi = (int)py; q.zi = (int)pz;
  q.s1 = px - (float)q.xi; q.s0 = 1.0f - q.s1;
  q.t1 = py - (float)q.yi; q.t0 = 1.0f - q.t1;
  q.f1 = pz - (float)q.zi; q.f0 = 1.0f - q.f1;
  if (px < 0.0f) { q.xi = 0; q.s0 = 1.0f; q.s1 = 0.0f; }
  if (py < 0.0f) { q.yi = 0; q.t0 = 1.0f; q.t1 = 0.0f; }
  if (pz < 0.0f) { q.zi = 0; q.f0 = 1.0f; q.f1 = 0.0f; }
  if (q.xi >= g.nx - 1) { q.xi = g.nx - 2; q.s0 = 0.0f; q.s1 = 1.0f; }
  if (q.yi >= g.ny - 1) { q.yi = g.ny - 2; q.t0 = 0.0f; q.t1 = 1.0f; }
  if (g.gnz > 1 && q.zi >= g.gnz - 1) { q.zi = g.gnz - 2; q.f0 = 0.0f; q.f1 = 1.0f; }
  return q;
}

// Address of the (xi, yi, zi) corner in local storage; faults if the 2-plane footprint
// leaves the slab.
__device__ __forceinline__ int corner(const Geo& g, const Lerp& q) {
  int kl = q.zi - g.zoff;
  if (g.is3d) {
    if (kl < g.skip_lo || kl + 1 >= g.nz - g.skip_hi) {
      note_fault(g);
      kl = kl < g.skip_lo ? g.skip_lo : g.nz - g.skip_hi - 2;
    }
  } else {
    kl = 0;
  }
  return cell(g, kl, q.yi, q.xi);
}

__device__ __forceinline__ float lerp_at(const float* __restrict__ blk, const Geo& g,
                                         const Lerp& q, int o) {
  const int sy = g.nx, sz = g.nx * g.ny;
  const float* a = blk + o;
  if (g.is3d) {
    const float lo = ((__ldg(a) * q.t0 + __ldg(a + sy) * q.t1) * q.s0 +
                      (__ldg(a + 1) * q.t0 + __ldg(a + sy + 1) * q.t1) * q.s1) * q.f0;
    const float hi = ((__ldg(a + sz) * q.t0 + __ldg(a + sz + sy) * q.t1) * q.s0 +
                      (__ldg(a + sz + 1) * q.t0 + __ldg(a + sz + sy + 1) * q.t1) * q.s1) * q.f1;
    return lo + hi;
  }
  return (__ldg(a) * q.t0 + __ldg(a + sy) * q.t1) * q.s0 +
         (__ldg(a + 1) * q.t0 + __ldg(a + sy + 1) * q.t1) * q.s1;
}
__device__ __forceinline__ float lerp_block(const float* __restrict__ blk, const Geo& g, V3 pos) {
  const Lerp q = build_index(g, pos);
  return lerp_at(blk, g, q, corner(g, q));
}

struct FluidVal { float v; bool ok; };
__device__ __forceinline__ FluidVal pair_fluid(FluidVal a, FluidVal b, float ta, float tb) {
  FluidVal r;
  if (!a.ok && !b.ok) { r.v = 0.0f; r.ok = false; }
  else if (!a.ok) { r.v = b.v; r.ok = true; }
  else if (!b.ok) { r.v = a.v; r.ok = true; }
  else { r.v = a.v * ta + b.v * tb; r.ok = true; }
  return r;
}
template <typename FT>
__device__ __forceinline__ FluidVal fluid_val(const float* __restrict__ blk,
                                              const FT* __restrict__ fl, int o) {
  return FluidVal{__ldg(blk + o), (flag_at(fl, o) & kFluid) != 0};
}
template <typename FT>
__device__ __forceinline__ float lerp_fluid_at(const float* __restrict__ blk, const FT* __restrict__ fl,
                                               const Geo& g, const Lerp& q, int o) {
  const int sy = g.nx, sz = g.nx * g.ny;
  FluidVal all;
  const FluidVal ab = pair_fluid(fluid_val(blk, fl, o), fluid_val(blk, fl, o + sy), q.t0, q.t1);
  const FluidVal cd = pair_fluid(fluid_val(blk, fl, o + 1), fluid_val(blk, fl, o + sy + 1), q.t0, q.t1);
  const FluidVal abcd = pair_fluid(ab, cd, q.s0, q.s1);
  if (g.is3d) {
    const FluidVal ef = pair_fluid(fluid_val(blk, fl, o + sz), fluid_val(blk, fl, o + sz + sy), q.t0, q.t1);
    const FluidVal gh = pair_fluid(fluid_val(blk, fl, o + sz + 1), fluid_val(blk, fl, o + sz + sy + 1), q.t0, q.t1);
    const FluidVal efgh = pair_fluid(ef, gh, q.s0, q.s1);
    all = pair_fluid(abcd, efgh, q.f0, q.f1);
  } else {
    all = abcd;
  }
  return all.ok ? all.v : lerp_at(blk, g, q, o);
}
template <typename FT>
__device__ __forceinline__ float lerp_block_fluid(const float* __restrict__ blk,
                                                  const FT* __restrict__ fl, const Geo& g,
                                                  V3 pos) {
  const Lerp q = build_index(g, pos);
  return lerp_fluid_at(blk, fl, g, q, corner(g, q));
}

// ---------------------------------------------------------------------------------------
// MAC-grid samples at cell (i, j, k) (k local).  Ub points at channel 0 of one batch.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ V3 mac_centered(const float* __restrict__ Ub, const Geo& g, int k, int j, int i) {
  const int c = cell(g, k, j, i);
  const int sy = g.nx, sz = g.nx * g.ny;
  V3 r;
  r.x = 0.5f * (__ldg(Ub + c) + __ldg(Ub + c + 1));
  r.y = 0.5f * (__ldg(Ub + g.n + c) + __ldg(Ub + g.n + c + sy));
  r.z = g.is3d ? 0.5f * (__ldg(Ub + 2 * g.n + c) + __ldg(Ub + 2 * g.n + c + sz)) : 0.0f;
  return r;
}
__device__ __forceinline__ V3 mac_at_x(const float* __restrict__ Ub, const Geo& g, int k, int j, int i) {
  const int c = cell(g, k, j, i);
  const int sy = g.nx, sz = g.nx * g.ny;
  const float* uy = Ub + g.n;
  const float* uz = Ub + 2 * g.n;
  V3 r;
  r.x = __ldg(Ub + c);
  r.y = 0.25f * (__ldg(uy + c) + __ldg(uy + c - 1) + __ldg(uy + c + sy) + __ldg(uy + c + sy - 1));
  r.z = g.is3d ? 0.25f * (__ldg(uz + c) + __ldg(uz + c - 1) + __ldg(uz + c + sz) + __ldg(uz + c + sz - 1))
               : 0.0f;
  return r;
}
__device__ __forceinline__ V3 mac_at_y(const float* __restrict__ Ub, const Geo& g, int k, int j, int i) {
  const int c = cell(g, k, j, i);
  const int sy = g.nx, sz = g.nx * g.ny;
  const float* uy = Ub + g.n;
  const float* uz = Ub + 2 * g.n;
  V3 r;
  r.x = 0.25f * (__ldg(Ub + c) + __ldg(Ub + c - sy) + __ldg(Ub + c + 1) + __ldg(Ub + c - sy + 1));
  r.y = __ldg(uy + c);
  r.z = g.is3d ? 0.25f * (__ldg(uz + c) + __ldg(uz + c - sy) + __ldg(uz + c + sz) + __ldg(uz + c + sz - sy))
               : 0.0f;
  return r;
}
__device__ __forceinline__ V3 mac_at_z(const float* __restrict__ Ub, const Geo& g, int k, int j, int i) {
  const int c = cell(g, k, j, i);
  const int sy = g.nx, sz = g.nx * g.ny;
  const float* uy = Ub + g.n;
  const float* uz = Ub + 2 * g.n;
  V3 r;
  r.x = 0.25f * (__ldg(Ub + c) + __ldg(Ub + c - sz) + __ldg(Ub + c + 1) + __ldg(Ub + c - sz + 1));
  r.y = 0.25f * (__ldg(uy + c) + __ldg(uy + c - sz) + __ldg(uy + c + sy) + __ldg(uy + c - sz + sy));
  r.z = __ldg(uz + c);
  return r;
}

// ---------------------------------------------------------------------------------------
// Line trace.
// ---------------------------------------------------------------------------------------
#define TFL_HIT_MARGIN 1e-5f
#define TFL_TRACE_EPS 1e-12f

__device__ __forceinline__ bool out_of_domain(const Geo& g, V3 p) {
  return p.x <= 0.0f || p.x >= (float)g.nx || p.y <= 0.0f || p.y >= (float)g.ny ||
         p.z <= 0.0f || p.z >= (float)g.gnz;
}
template <typename FT>
__device__ __forceinline__ bool blocked_at(const FT* __restrict__ fl, const Geo& g, V3 p) {
  const int k = local_z(g, (int)p.z);
  return (flag_i(fl, g, k, (int)p.y, (int)p.x) & kFluid) == 0;
}

__device__ inline bool ray_hits_box(const float lo[3], const float hi[3], const float org[3],
                                    const float dir[3], float out[3]) {
  bool inside = true;
  int side[3];
  float plane[3] = {0.0f, 0.0f, 0.0f}, tmax[3];
#pragma unroll
  for (int a = 0; a < 3; a++) {
    if (org[a] < lo[a]) { side[a] = 1; plane[a] = lo[a]; inside = false; }
    else if (org[a] > hi[a]) { side[a] = 0; plane[a] = hi[a]; inside = false; }
    else side[a] = 2;
  }
  if (inside) { out[0] = org[0]; out[1] = org[1]; out[2] = org[2]; return true; }
#pragma unroll
  for (int a = 0; a < 3; a++)
    tmax[a] = (side[a] != 2 && dir[a] != 0.0f) ? (plane[a] - org[a]) / dir[a] : -1.0f;
  int w = 0;
  if (tmax[w] < tmax[1]) w = 1;
  if (tmax[w] < tmax[2]) w = 2;
  const float tw = tmax[w];
  if (tw < 0.0f) return false;
  const float tol = 1e-6f;
#pragma unroll
  for (int a = 0; a < 3; a++) {
    if (a != w) {
      out[a] = org[a] + tw * dir[a];
      if (out[a] < (lo[a] - tol) || out[a] > (hi[a] + tol)) return false;
    } else {
      out[a] = plane[a];
    }
  }
  return true;
}

__device__ inline bool ray_border(const Geo& g, V3 pos, V3 next, V3* ip) {
  const float m = TFL_HIT_MARGIN;
  float step = FLT_MAX;
  const float p[3] = {pos.x, pos.y, pos.z}, n[3] = {next.x, next.y, next.z};
  const float ext[3] = {(float)g.nx, (float)g.ny, (float)g.gnz};
#pragma unroll
  for (int a = 0; a < 3; a++) {
    if (n[a] <= m) {
      const float dl = n[a] - p[a];
      if (fabsf(dl) >= TFL_TRACE_EPS) step = std_min(step, (m - p[a]) / dl);
    }
  }
#pragma unroll
  for (int a = 0; a < 3; a++) {
    if (n[a] >= (ext[a] - m)) {
      const float dl = n[a] - p[a];
      if (fabsf(dl) >= TFL_TRACE_EPS) step = std_min(step, (ext[a] - m - p[a]) / dl);
    }
  }
  if (step < 0.0f || step >= FLT_MAX) return false;
  ip->x = step * (next.x - pos.x) + pos.x;
  ip->y = step * (next.y - pos.y) + pos.y;
  ip->z = step * (next.z - pos.z) + pos.z;
  return true;
}

// Returns true if the trace was cut short (geometry or domain border).
// Out of line on purpose: the kernels that trace keep their common (clear-space) path compact enough
// for the instruction cache, and only cells near solids / the border pay for the call.
template <typename FT>
__device__ __noinline__ bool line_trace(const FT* __restrict__ fl, const Geo& g, V3 pos, V3 delta,
                                        V3* out) {
  *out = pos;
  const float length = norm3(delta);
  if (length <= TFL_TRACE_EPS) return false;
  const V3 dir = {delta.x / length, delta.y / length, delta.z / length};
  float travelled = 0.0f;
  while (travelled < (length - TFL_HIT_MARGIN)) {
    const float step = std_min(length - travelled, 1.0f);
    V3 next = {out->x + dir.x * step, out->y + dir.y * step, out->z + dir.z * step};
    if (out_of_domain(g, next)) {
      V3 ip;
      if (!ray_border(g, *out, next, &ip)) {
        ip.x = std_min(std_max(next.x, TFL_HIT_MARGIN), (float)g.nx - TFL_HIT_MARGIN);
        ip.y = std_min(std_max(next.y, TFL_HIT_MARGIN), (float)g.ny - TFL_HIT_MARGIN);
        ip.z = std_min(std_max(next.z, TFL_HIT_MARGIN), (float)g.gnz - TFL_HIT_MARGIN);
      }
      if (out_of_domain(g, ip)) { note_fault(g); return true; }
      if (!blocked_at(fl, g, ip)) { *out = ip; return true; }
      next = ip;
    }
    if (blocked_at(fl, g, next)) {
      for (int tries = 0; tries <= 4; tries++) {
        if (!blocked_at(fl, g, next)) break;
        if (tries == 4) { note_fault(g); return true; }
        const float ctr[3] = {(float)((int)next.x) + 0.5f, (float)((int)next.y) + 0.5f,
                              (float)((int)next.z) + 0.5f};
        const float lo[3] = {ctr[0] - 0.5f - TFL_HIT_MARGIN, ctr[1] - 0.5f - TFL_HIT_MARGIN,
                             ctr[2] - 0.5f - TFL_HIT_MARGIN};
        const float hi[3] = {ctr[0] + 0.5f + TFL_HIT_MARGIN, ctr[1] + 0.5f + TFL_HIT_MARGIN,
                             ctr[2] + 0.5f + TFL_HIT_MARGIN};
        const float o[3] = {out->x, out->y, out->z}, dr[3] = {dir.x, dir.y, dir.z};
        float hitp[3];
        if (!ray_hits_box(lo, hi, o, dr, hitp)) return true;
        next = V3{hitp[0], hitp[1], hitp[2]};
      }
      *out = next;
      return true;
    }
    *out = next;
    travelled += step;
  }
  return false;
}

// ---------------------------------------------------------------------------------------
// Clear-space fast path.  clear[c] = Chebyshev distance (in cells, capped at kClearMax + 1) from cell c to
// the nearest cell that is not fluid or lies on an end of the LOCAL storage; 0 for such cells themselves
// (2-D grids ignore z).  A trace of length < clear - 0.5 that starts at the centre of c stays inside
// fluid cells of the domain interior (the nearest solid face is clear - 0.5 away), the 2x2x2
// interpolation footprint of its end point and the MacCormack clamp boxes lie inside the storage without
// any index clamp, and a trace shorter than clear - 1 only has fluid cells in that footprint.  The code
// below is line_trace / build_index / lerp_at with the branches that then cannot fire removed -- the
// arithmetic, and its order, are unchanged (bit-identical).
// ---------------------------------------------------------------------------------------
constexpr int kClearMax = 7;
#define TFL_CLEAR_SLACK 0.01f      // covers |dir| <= 1 + ulps and the accumulated step rounding
// longest trace that stays in clear space / whose interpolation footprint is all fluid
__device__ __forceinline__ float clear_reach(int clr) { return (float)clr - (0.5f + TFL_CLEAR_SLACK); }
__device__ __forceinline__ float clear_reach_fluid(int clr) { return (float)clr - (1.0f + TFL_CLEAR_SLACK); }

__device__ __forceinline__ V3 line_trace_clear(V3 pos, V3 delta, float length) {
  V3 out = pos;
  if (length <= TFL_TRACE_EPS) return out;
  const V3 dir = {delta.x / length, delta.y / length, delta.z / length};
  float travelled = 0.0f;
  while (travelled < (length - TFL_HIT_MARGIN)) {
    const float step = std_min(length - travelled, 1.0f);
    out = V3{out.x + dir.x * step, out.y + dir.y * step, out.z + dir.z * step};
    travelled += step;
  }
  return out;
}
// build_index + corner without the clamps (positions at least one cell away from every end of the
// local storage, guaranteed by the clearance test).
__device__ __forceinline__ int build_index_clear(const Geo& g, V3 pos, Lerp& q) {
  const float px = pos.x - 0.5f, py = pos.y - 0.5f, pz = pos.z - 0.5f;
  q.xi = (int)px; q.yi = (int)py; q.zi = (int)pz;
  q.s1 = px - (float)q.xi; q.s0 = 1.0f - q.s1;
  q.t1 = py - (float)q.yi; q.t0 = 1.0f - q.t1;
  q.f1 = pz - (float)q.zi; q.f0 = 1.0f - q.f1;
  return cell(g, g.is3d ? q.zi - g.zoff : 0, q.yi, q.xi);
}
// interpolWithFluid on a footprint that needs no index clamp (flags still decide which corners count)
template <typename FT>
__device__ __forceinline__ float lerp_block_fluid_noclamp(const float* __restrict__ blk, const FT* __restrict__ fl,
                                                          const Geo& g, V3 pos);
__device__ __forceinline__ float lerp_block_clear(const float* __restrict__ blk, const Geo& g, V3 pos) {
  Lerp q;
  const int o = build_index_clear(g, pos, q);
  return lerp_at(blk, g, q, o);
}
template <typename FT>
__device__ __forceinline__ float lerp_block_fluid_noclamp(const float* __restrict__ blk, const FT* __restrict__ fl,
                                                          const Geo& g, V3 pos) {
  Lerp q;
  const int o = build_index_clear(g, pos, q);
  return lerp_fluid_at(blk, fl, g, q, o);
}

// ---------------------------------------------------------------------------------------
// Launch geometry shared by the per-cell kernels.
// ---------------------------------------------------------------------------------------
// (b, k, j, i) of this thread; returns false if outside the launch range.
__device__ __forceinline__ bool thread_cell(const Geo& g, int& b, int& k, int& j, int& i) {
  i = blockIdx.x * blockDim.x + threadIdx.x;
  j = blockIdx.y * blockDim.y + threadIdx.y;
  const int zz = blockIdx.z * blockDim.z + threadIdx.z;
  const int nzr = g.zhi - g.zlo;
  if (zz < nzr) {                       // first (usually only) batch element: no integer division
    b = 0;
    k = g.zlo + zz;
  } else {
    b = zz / nzr;
    k = g.zlo + (zz - b * nzr);
  }
  return i < g.nx && j < g.ny && b < g.nb;
}

static inline void launch_dims(const Geo& g, dim3& grid, dim3& block) {
  const int nzr = g.zhi - g.zlo;
  if (g.nz == 1) block = dim3(32, 8, 1);
  else block = dim3(32, 4, 2);
  if (g.nx > 32 && g.nx % 64 == 0) { block.x = 64; block.y = (g.nz == 1) ? 4 : 2; }
  grid = dim3((g.nx + block.x - 1) / block.x, (g.ny + block.y - 1) / block.y,
              ((long long)g.nb * nzr + block.z - 1) / block.z);
}


// Which velocity components setWallBcsForward zeroes at (i, j, k)
// (third_party/tfluids.cc:926-1002).
template <typename FT>
__device__ __forceinline__ void wall_bc_zero_mask(const FT* __restrict__ fl, const Geo& g, int k,
                                                  int j, int i, bool z[3]) {
  z[0] = z[1] = z[2] = false;
  const int fc = flag_i(fl, g, k, j, i);
  const bool cf = fc & kFluid, co = fc & kObstacle;
  if (!cf && !co) return;
  const int kg = k + g.zoff;
  if (i > 0) {
    const int f = flag_i(fl, g, k, j, i - 1);
    if ((f & kObstacle) || (co && (f & kFluid))) z[0] = true;
  }
  if (j > 0) {
    const int f = flag_i(fl, g, k, j - 1, i);
    if ((f & kObstacle) || (co && (f & kFluid))) z[1] = true;
  }
  if (kg > 0) {
    const int f = flag_i(fl, g, local_z(g, kg - 1), j, i);
    if ((f & kObstacle) || (co && (f & kFluid))) z[2] = true;
  }
  if (cf) {
    if ((i > 0 && (flag_i(fl, g, k, j, i - 1) & kStick)) ||
        (i < g.nx - 1 && (flag_i(fl, g, k, j, i + 1) & kStick))) { z[1] = true; if (g.is3d) z[2] = true; }
    if ((j > 0 && (flag_i(fl, g, k, j - 1, i) & kStick)) ||
        (j < g.ny - 1 && (flag_i(fl, g, k, j + 1, i) & kStick))) { z[0] = true; if (g.is3d) z[2] = true; }
    if (g.is3d && ((kg > 0 && (flag_i(fl, g, local_z(g, kg - 1), j, i) & kStick)) ||
                   (kg < g.gnz - 1 && (flag_i(fl, g, local_z(g, kg + 1), j, i) & kStick)))) {
      z[0] = true; z[1] = true;
    }
  }
}


// Vorticity-confinement force at one cell from the stored curl / |curl| fields
// (third_party/tfluids.cc:1411-1439).
__device__ __forceinline__ V3 conf_force(const float* __restrict__ cb, const float* __restrict__ cn,
                                         const Geo& g, int k, int j, int i, float strength) {
  if (on_border(g, k, j, i)) return V3{0.0f, 0.0f, 0.0f};
  const int c = cell(g, k, j, i);
  const int sy = g.nx, sz = g.nx * g.ny;
  V3 gr = {0.0f, 0.0f, 0.0f};
  gr.x = 0.5f * (__ldg(cn + c + 1) - __ldg(cn + c - 1));
  gr.y = 0.5f * (__ldg(cn + c + sy) - __ldg(cn + c - sy));
  if (g.is3d) gr.z = 0.5f * (__ldg(cn + c + sz) - __ldg(cn + c - sz));
  const float gn = norm3(gr);
  if (gn > 1e-6f) { gr.x /= gn; gr.y /= gn; gr.z /= gn; } else { gr.x = gr.y = gr.z = 0.0f; }
  const V3 w = {__ldg(cb + c), __ldg(cb + g.n + c), __ldg(cb + 2 * g.n + c)};
  V3 f;
  f.x = ((gr.y * w.z) - (gr.z * w.y)) * strength;
  f.y = ((gr.z * w.x) - (gr.x * w.z)) * strength;
  f.z = ((gr.x * w.y) - (gr.y * w.x)) * strength;
  return f;
}


// nn.StandardDeviation + nn.Clamp on the accumulated sums (lib/modules/variance.lua:44-76).
__device__ __forceinline__ float scale_from_sums(const double* __restrict__ sums, int b, long long n,
                                                 float threshold) {
  const float sum = (float)sums[2 * b], sumsq = (float)sums[2 * b + 1];
  float out = sumsq * (float)n;
  out = out + (-1.0f) * (sum * sum);
  out = out / (float)((double)n * (double)(n - 1));
  out = sqrtf(out);
  return (out < threshold) ? threshold : out;
}

// Block-wide sum of (s, ss) -> two atomics per block.  All threads of the block must call.
__device__ __forceinline__ void block_accumulate(double s, double ss, double* __restrict__ dst) {
  __shared__ double sh[2][32];
  const int tid = (threadIdx.z * blockDim.y + threadIdx.y) * blockDim.x + threadIdx.x;
  const int lane = tid & 31, w = tid >> 5;
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_down_sync(0xffffffffu, s, o);
    ss += __shfl_down_sync(0xffffffffu, ss, o);
  }
  if (lane == 0) { sh[0][w] = s; sh[1][w] = ss; }
  __syncthreads();
  if (w == 0) {
    const int nw = (blockDim.x * blockDim.y * blockDim.z + 31) >> 5;
    s = lane < nw ? sh[0][lane] : 0.0;
    ss = lane < nw ? sh[1][lane] : 0.0;
    for (int o = 16; o > 0; o >>= 1) {
      s += __shfl_down_sync(0xffffffffu, s, o);
      ss += __shfl_down_sync(0xffffffffu, ss, o);
    }
    if (lane == 0) {
      atomicAdd(dst, s);
      atomicAdd(dst + 1, ss);
    }
  }
}

}  // namespace tfl
