// MAC-grid stencil kernels of the Eulerian step (everything except the conv stack).
// Compiled with -fmad=false: results are bit-identical to the reference CPU operators
// (see oracle/ and tests/).  One thread per cell, x fastest (coalesced rows); neighbour
// reuse comes from L1/L2.  Launchers at the bottom are called by tfl_api.cu.
//
// Reference operators restated here (paths relative to /root/reference/torch/tfluids):
//   advectScalar   third_party/tfluids.cc:23-588     advectVel   third_party/tfluids.cc:594-920
//   setWallBcs     third_party/tfluids.cc:926-1002   divergence  third_party/tfluids.cc:1008-1066
//   velocityUpdate third_party/tfluids.cc:1072-1156  buoyancy    third_party/tfluids.cc:1162-1233
//   addGravity     third_party/tfluids.cc:1239-1306  vorticity   third_party/tfluids.cc:1312-1458
//   Jacobi         generic/tfluids.cu:1765-1927      emptyDomain generic/tfluids.cc:136-172
//   flagsToOccupancy generic/tfluids.cu:355-401
#include <algorithm>
#include <cstdlib>
#include <cooperative_groups.h>
#include "tfl_device.cuh"
#include "tfl_advect.cuh"
#include "tfl_kernels.h"

namespace tfl {

// ---------------------------------------------------------------------------------------
// emptyDomain / flagsToOccupancy
// ---------------------------------------------------------------------------------------
template <bool IS3D, typename FT>
__global__ void k_empty_domain(float* __restrict__ flags, Geo gin, int bnd) {
  const Geo g = static_geo<IS3D>(gin);
  int b, k, j, i;
  if (!thread_cell(g, b, k, j, i)) return;
  const int kg = k + g.zoff;
  const bool border = i < bnd || i > g.nx - 1 - bnd || j < bnd || j > g.ny - 1 - bnd ||
                      (g.is3d && (kg < bnd || kg > g.gnz - 1 - bnd));
  flags[b * g.n + cell(g, k, j, i)] = border ? (float)kObstacle : (float)kFluid;
}

__global__ void k_flags_to_occupancy(const float* __restrict__ flags, float* __restrict__ occ,
                                     long long n, unsigned long long* bad) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const int f = (int)flags[t];
  float o;
  if (f == kFluid) o = 0.0f;
  else if (f == kObstacle) o = 1.0f;
  else { o = -1.0f; atomicAdd(bad, 1ULL); }     // CUDA reference writes -1 (generic/tfluids.cu:362-370)
  occ[t] = o;
}

// ---------------------------------------------------------------------------------------
// setWallBcsForward
// ---------------------------------------------------------------------------------------
template <bool IS3D, typename FT>
__global__ void k_set_wall_bcs(float* __restrict__ U, const FT* __restrict__ flags, Geo gin,
                               int as_mask) {
  const Geo g = static_geo<IS3D>(gin);
  int b, k, j, i;
  if (!thread_cell(g, b, k, j, i)) return;
  bool z[3];
  wall_bc_zero_mask(flags + b * g.n, g, k, j, i, z);
  float* ub = U + (long long)b * g.nc * g.n + cell(g, k, j, i);
  for (int c = 0; c < g.nc; c++)
    if (z[c]) ub[c * g.n] = as_mask ? ub[c * g.n] * 0.0f : 0.0f;
}

// ---------------------------------------------------------------------------------------
// velocityDivergenceForward  (returns u(i)-u(i+1)+..., i.e. minus the divergence)
// ---------------------------------------------------------------------------------------
template <bool IS3D, typename FT>
__global__ void k_divergence(const float* __restrict__ U, const FT* __restrict__ flags,
                             float* __restrict__ div, Geo gin) {
  const Geo g = static_geo<IS3D>(gin);
  int b, k, j, i;
  if (!thread_cell(g, b, k, j, i)) return;
  const int c = cell(g, k, j, i);
  const float* ub = U + (long long)b * g.nc * g.n;
  float r = 0.0f;
  if (!on_border(g, k, j, i) && (flag_i(flags + b * g.n, g, k, j, i) & kFluid)) {
    r = __ldg(ub + c) - __ldg(ub + c + 1) + __ldg(ub + g.n + c) - __ldg(ub + g.n + c + g.nx);
    if (g.is3d) r += (__ldg(ub + 2 * g.n + c) - __ldg(ub + 2 * g.n + c + (long long)g.nx * g.ny));
  }
  div[b * g.n + c] = r;
}

// ---------------------------------------------------------------------------------------
// velocityUpdateForward
// ---------------------------------------------------------------------------------------
template <bool IS3D, typename FT>
__global__ void k_velocity_update(float* __restrict__ U, const FT* __restrict__ flags,
                                  const float* __restrict__ p, Geo gin) {
  const Geo g = static_geo<IS3D>(gin);
  int b, k, j, i;
  if (!thread_cell(g, b, k, j, i)) return;
  if (on_border(g, k, j, i)) return;
  const FT* fl = flags + b * g.n;
  const float* pb = p + b * g.n;
  float* ub = U + (long long)b * g.nc * g.n;
  const int c = cell(g, k, j, i);
  const int st[3] = {1, g.nx, g.nx * g.ny};
  const int fc = flag_i(fl, g, k, j, i);
  int fn[3];
  fn[0] = flag_i(fl, g, k, j, i - 1);
  fn[1] = flag_i(fl, g, k, j - 1, i);
  fn[2] = g.is3d ? flag_i(fl, g, k - 1, j, i) : 0;
  const float pc = __ldg(pb + c);
  if (fc & kFluid) {
    for (int a = 0; a < g.nc; a++) {
      float u = ub[a * g.n + c];
      if (fn[a] & kFluid) u -= (pc - __ldg(pb + c - st[a]));
      if (fn[a] & kEmpty) u -= pc;
      ub[a * g.n + c] = u;
    }
  } else if ((fc & kEmpty) && !(fc & kOutflow)) {
    for (int a = 0; a < g.nc; a++) {
      float u = ub[a * g.n + c];
      if (fn[a] & kFluid) u += __ldg(pb + c - st[a]);
      else u = 0.0f;
      ub[a * g.n + c] = u;
    }
  }
}

// ---------------------------------------------------------------------------------------
// addBuoyancy / addGravity
// ---------------------------------------------------------------------------------------
template <bool IS3D, typename FT>
__global__ void k_add_buoyancy(float* __restrict__ U, const FT* __restrict__ flags,
                               const float* __restrict__ rho, float sx, float sy_, float sz_, Geo gin) {
  const Geo g = static_geo<IS3D>(gin);
  int b, k, j, i;
  if (!thread_cell(g, b, k, j, i)) return;
  if (on_border(g, k, j, i)) return;
  const FT* fl = flags + b * g.n;
  if (!(flag_i(fl, g, k, j, i) & kFluid)) return;
  const float* rb = rho + b * g.n;
  float* ub = U + (long long)b * g.nc * g.n;
  const int c = cell(g, k, j, i);
  const float rc = __ldg(rb + c);
  if (flag_i(fl, g, k, j, i - 1) & kFluid) ub[c] += (0.5f * sx * (rc + __ldg(rb + c - 1)));
  if (flag_i(fl, g, k, j - 1, i) & kFluid) ub[g.n + c] += (0.5f * sy_ * (rc + __ldg(rb + c - g.nx)));
  if (g.is3d && (flag_i(fl, g, k - 1, j, i) & kFluid))
    ub[2 * g.n + c] += (0.5f * sz_ * (rc + __ldg(rb + c - (long long)g.nx * g.ny)));
}

template <bool IS3D, typename FT>
__global__ void k_add_gravity(float* __restrict__ U, const FT* __restrict__ flags, float fx,
                              float fy, float fz, Geo gin) {
  const Geo g = static_geo<IS3D>(gin);
  int b, k, j, i;
  if (!thread_cell(g, b, k, j, i)) return;
  if (on_border(g, k, j, i)) return;
  const FT* fl = flags + b * g.n;
  const int fc = flag_i(fl, g, k, j, i);
  const bool cf = fc & kFluid, ce = fc & kEmpty;
  if (!cf && !ce) return;
  float* ub = U + (long long)b * g.nc * g.n;
  const int c = cell(g, k, j, i);
  int f = flag_i(fl, g, k, j, i - 1);
  if ((f & kFluid) || (cf && (f & kEmpty))) ub[c] += fx;
  f = flag_i(fl, g, k, j - 1, i);
  if ((f & kFluid) || (cf && (f & kEmpty))) ub[g.n + c] += fy;
  if (g.is3d) {
    f = flag_i(fl, g, k - 1, j, i);
    if ((f & kFluid) || (cf && (f & kEmpty))) ub[2 * g.n + c] += fz;
  }
}

// ---------------------------------------------------------------------------------------
// vorticityConfinement: two kernels instead of the reference's four passes.
//   (1) curl + |curl| straight from the face velocities (centred velocities are
//       recomputed per neighbour, bit-identical to storing them);
//   (2) confinement force recomputed at the 4 cells each face needs, then applied.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ V3 centered_or_zero(const float* __restrict__ Ub, const Geo& g, int k,
                                               int j, int i) {
  if (on_border(g, k, j, i)) return V3{0.0f, 0.0f, 0.0f};
  return mac_centered(Ub, g, k, j, i);
}

template <bool IS3D, typename FT>
__global__ void k_vort_curl(const float* __restrict__ U, float* __restrict__ curl,
                            float* __restrict__ cnorm, Geo gin) {
  const Geo g = static_geo<IS3D>(gin);
  int b, k, j, i;
  if (!thread_cell(g, b, k, j, i)) return;
  const float* ub = U + (long long)b * g.nc * g.n;
  const int c = cell(g, k, j, i);
  V3 w = {0.0f, 0.0f, 0.0f};
  float nrm = 0.0f;
  if (!on_border(g, k, j, i)) {
    const V3 xm = centered_or_zero(ub, g, k, j, i - 1), xp = centered_or_zero(ub, g, k, j, i + 1);
    const V3 ym = centered_or_zero(ub, g, k, j - 1, i), yp = centered_or_zero(ub, g, k, j + 1, i);
    w.z = 0.5f * ((xp.y - xm.y) - (yp.x - ym.x));
    if (g.is3d) {
      const V3 zm = centered_or_zero(ub, g, k - 1, j, i), zp = centered_or_zero(ub, g, k + 1, j, i);
      w.x = 0.5f * ((yp.z - ym.z) - (zp.y - zm.y));
      w.y = 0.5f * ((zp.x - zm.x) - (xp.z - xm.z));
    }
    nrm = norm3(w);
  }
  float* cb = curl + (long long)b * 3 * g.n;
  cb[c] = w.x; cb[g.n + c] = w.y; cb[2 * g.n + c] = w.z;
  cnorm[b * g.n + c] = nrm;
}

// Confinement force per cell (zero on the border), third_party/tfluids.cc:1411-1439.
template <bool IS3D, typename FT>
__global__ void k_vort_force(const float* __restrict__ curl, const float* __restrict__ cnorm,
                             float* __restrict__ force, float strength, Geo gin) {
  const Geo g = static_geo<IS3D>(gin);
  int b, k, j, i;
  if (!thread_cell(g, b, k, j, i)) return;
  const V3 f = conf_force(curl + (long long)b * 3 * g.n, cnorm + b * g.n, g, k, j, i, strength);
  float* fb = force + (long long)b * 3 * g.n + cell(g, k, j, i);
  fb[0] = f.x; fb[g.n] = f.y; fb[2 * g.n] = f.z;
}

// AddForceField, third_party/tfluids.cc:1312-1339 (CPU caller guards the border, :1443-1451).
template <bool IS3D, typename FT>
__global__ void k_vort_apply(float* __restrict__ U, const FT* __restrict__ flags,
                             const float* __restrict__ force, Geo gin) {
  const Geo g = static_geo<IS3D>(gin);
  int b, k, j, i;
  if (!thread_cell(g, b, k, j, i)) return;
  if (on_border(g, k, j, i)) return;
  const FT* fl = flags + b * g.n;
  const int fc = flag_i(fl, g, k, j, i);
  const bool cf = fc & kFluid, ce = fc & kEmpty;
  if (!cf && !ce) return;
  const float* fb = force + (long long)b * 3 * g.n;
  float* ub = U + (long long)b * g.nc * g.n;
  const int c = cell(g, k, j, i);
  int f = flag_i(fl, g, k, j, i - 1);
  if ((f & kFluid) || (cf && (f & kEmpty))) ub[c] += (0.5f * (__ldg(fb + c - 1) + __ldg(fb + c)));
  f = flag_i(fl, g, k, j - 1, i);
  if ((f & kFluid) || (cf && (f & kEmpty)))
    ub[g.n + c] += (0.5f * (__ldg(fb + g.n + c - g.nx) + __ldg(fb + g.n + c)));
  if (g.is3d) {
    f = flag_i(fl, g, k - 1, j, i);
    if ((f & kFluid) || (cf && (f & kEmpty)))
      ub[2 * g.n + c] += (0.5f * (__ldg(fb + 2 * g.n + c - g.nx * g.ny) + __ldg(fb + 2 * g.n + c)));
  }
}

// ---------------------------------------------------------------------------------------
// advectScalar
// ---------------------------------------------------------------------------------------
template <typename FT>
__device__ __forceinline__ float sample_scalar(const float* __restrict__ src, const FT* __restrict__ fl,
                                               const Geo& g, V3 pos, bool outside) {
  return outside ? lerp_block(src, g, pos) : lerp_block_fluid(src, fl, g, pos);
}
__device__ __forceinline__ V3 sample_vel(const float* __restrict__ ub, const Geo& g, V3 pos) {
  const Lerp q = build_index(g, pos);
  const long long o = corner(g, q);
  V3 r;
  r.x = lerp_at(ub, g, q, o);
  r.y = lerp_at(ub + g.n, g, q, o);
  r.z = g.is3d ? lerp_at(ub + 2 * g.n, g, q, o) : 0.0f;
  return r;
}

// One semi-Lagrangian pass for an interior cell.  `pos_out` receives the trace end
// point ("SavePos" variants) when non-null.
template <int METHOD, typename FT>
__device__ __forceinline__ float advect_scalar_cell(const FT* __restrict__ fl, const float* __restrict__ ub,
                                                    const float* __restrict__ src, const Geo& g, float dt,
                                                    int k, int j, int i, bool outside, V3* pos_out) {
  const V3 start = {(float)i + 0.5f, (float)j + 0.5f, (float)(k + g.zoff) + 0.5f};
  if (METHOD == TFL_ADVECT_EULER || METHOD == TFL_ADVECT_MACCORMACK) {
    const V3 c = mac_centered(ub, g, k, j, i);
    const V3 p = {start.x - c.x * dt, start.y - c.y * dt, start.z - c.z * dt};
    return lerp_block(src, g, p);
  }
  if (!(flag_i(fl, g, k, j, i) & kFluid)) {
    if (pos_out) *pos_out = start;
    return __ldg(src + cell(g, k, j, i));
  }
  const V3 c = mac_centered(ub, g, k, j, i);
  if (METHOD == TFL_ADVECT_EULER_OURS || METHOD == TFL_ADVECT_MACCORMACK_OURS) {
    V3 back;
    line_trace(fl, g, start, scale3(c, -dt), &back);
    if (pos_out) *pos_out = back;
    return sample_scalar(src, fl, g, back, outside);
  }
  if (METHOD == TFL_ADVECT_RK2_OURS) {
    V3 half, back;
    if (line_trace(fl, g, start, scale3(c, -dt * 0.5f), &half)) return sample_scalar(src, fl, g, half, outside);
    const V3 v = sample_vel(ub, g, half);
    line_trace(fl, g, start, scale3(v, -dt), &back);
    return sample_scalar(src, fl, g, back, outside);
  }
  // RK3 (CPU behaviour: a third-stage hit samples at the third-stage position,
  // third_party/tfluids.cc:117-126).
  V3 p2, p3, back;
  if (line_trace(fl, g, start, scale3(c, -dt * 0.5f), &p2)) return sample_scalar(src, fl, g, p2, outside);
  const V3 k2 = sample_vel(ub, g, p2);
  if (line_trace(fl, g, start, scale3(k2, -dt * 0.75f), &p3)) return sample_scalar(src, fl, g, p3, outside);
  const V3 k3 = sample_vel(ub, g, p3);
  const float w1 = -dt * (float)(2.0 / 9.0), w2 = -dt * (float)(3.0 / 9.0), w3 = -dt * (float)(4.0 / 9.0);
  const V3 a1 = scale3(c, w1), a2 = scale3(k2, w2), a3 = scale3(k3, w3);
  const V3 disp = {(a1.x + a2.x) + a3.x, (a1.y + a2.y) + a3.y, (a1.z + a2.z) + a3.z};
  line_trace(fl, g, start, disp, &back);
  return sample_scalar(src, fl, g, back, outside);
}

// eulerOurs / maccormackOurs pass for a cell with clearance (fluid, interior): trace + sample with the
// branches that cannot fire removed; every corner of the footprint is fluid, so interpolWithFluid is the
// plain trilinear expression (same products, same order).
template <typename FT>
__device__ __forceinline__ float advect_scalar_cell_clear(const FT* __restrict__ fl, const float* __restrict__ ub,
                                                          const float* __restrict__ src, const Geo& g, float dt,
                                                          int k, int j, int i, bool outside, int clr,
                                                          V3* pos_out) {
  const V3 start = {(float)i + 0.5f, (float)j + 0.5f, (float)(k + g.zoff) + 0.5f};
  const V3 delta = scale3(mac_centered(ub, g, k, j, i), -dt);
  const float length = norm3(delta);
  if (length < clear_reach(clr)) {
    const V3 back = line_trace_clear(start, delta, length);
    if (pos_out) *pos_out = back;
    if (outside || length < clear_reach_fluid(clr)) return lerp_block_clear(src, g, back);
    return lerp_block_fluid_noclamp(src, fl, g, back);       // a solid cell may be in the footprint
  }
  V3 back;
  line_trace(fl, g, start, delta, &back);
  if (pos_out) *pos_out = back;
  return sample_scalar(src, fl, g, back, outside);
}

template <bool IS3D, typename FT, int METHOD>
__global__ void k_advect_scalar_pass1(const float* __restrict__ s, const float* __restrict__ U,
                                      const FT* __restrict__ flags, const unsigned char* __restrict__ clear,
                                      float* __restrict__ out, float* __restrict__ pos_out, float dt,
                                      int outside, Geo gin) {
  const Geo g = static_geo<IS3D>(gin);
  int b, k, j, i;
  if (!thread_cell(g, b, k, j, i)) return;
  const int c = cell(g, k, j, i);
  float v = 0.0f;
  V3 pos = {(float)i + 0.5f, (float)j + 0.5f, (float)(k + g.zoff) + 0.5f};
  constexpr bool kTraced = METHOD == TFL_ADVECT_EULER_OURS || METHOD == TFL_ADVECT_MACCORMACK_OURS;
  const int clr = (kTraced && clear) ? (int)__ldg(clear + b * g.n + c) : 0;
  if (clr > 0) {
    v = advect_scalar_cell_clear(flags + b * g.n, U + (long long)b * g.nc * g.n, s + b * g.n, g, dt, k, j, i,
                                 outside != 0, clr, pos_out ? &pos : nullptr);
  } else if (!on_border(g, k, j, i)) {
    v = advect_scalar_cell<METHOD>(flags + b * g.n, U + (long long)b * g.nc * g.n, s + b * g.n, g, dt, k,
                                   j, i, outside != 0, pos_out ? &pos : nullptr);
  }
  out[b * g.n + c] = v;
  if (pos_out) {
    float* pp = pos_out + (long long)b * g.nc * g.n + c;
    pp[0] = pos.x; pp[g.n] = pos.y;
    if (g.is3d) pp[2 * g.n] = pos.z;
  }
}

// MacCormack (ours): backward trace on the forward field + correction + clamp to the
// fluid neighbourhood of the forward trace position, fused
// (third_party/tfluids.cc:521-583, 222-234, 331-413).
template <bool IS3D, typename FT>
__global__ void k_advect_scalar_pass2_ours(const float* __restrict__ s, const float* __restrict__ fwd,
                                           const float* __restrict__ fwd_pos, const float* __restrict__ U,
                                           const FT* __restrict__ flags, const unsigned char* __restrict__ clear,
                                           float* __restrict__ dst, float dt, float strength, int outside, Geo gin) {
  const Geo g = static_geo<IS3D>(gin);
  int b, k, j, i;
  if (!thread_cell(g, b, k, j, i)) return;
  const int c = cell(g, k, j, i);
  const FT* fl = flags + b * g.n;
  const unsigned char* cl = clear ? clear + b * g.n : nullptr;
  const float* sb = s + b * g.n;
  const float* fb = fwd + b * g.n;
  const float fw = __ldg(fb + c);
  const int clr = cl ? (int)__ldg(cl + c) : 0;
  const bool border = clr > 0 ? false : on_border(g, k, j, i);
  float bw = 0.0f;
  if (clr > 0)
    bw = advect_scalar_cell_clear(fl, U + (long long)b * g.nc * g.n, fb, g, -dt, k, j, i, outside != 0,
                                  clr, nullptr);
  else if (!border)
    bw = advect_scalar_cell<TFL_ADVECT_MACCORMACK_OURS>(fl, U + (long long)b * g.nc * g.n, fb, g, -dt, k,
                                                        j, i, outside != 0, nullptr);
  float v = fw;
  if (clr > 0 || (flag_i(fl, g, k, j, i) & kFluid)) {
    const float diff = __ldg(sb + c) - bw;
    v = (float)((double)v + ((double)strength * 0.5) * (double)diff);
  }
  if (!border) {
    const float* pp = fwd_pos + (long long)b * g.nc * g.n + c;
    const float px = __ldg(pp), py = __ldg(pp + g.n), pz = g.is3d ? __ldg(pp + 2 * g.n) : 0.0f;
    v = clamp_scalar_ours(sb, fl, cl, g, v, fw, px, py, pz, outside != 0);
  }
  dst[b * g.n + c] = v;
}

// MacCormack (Manta): third_party/tfluids.cc:249-325.
template <bool IS3D, typename FT>
__global__ void k_advect_scalar_pass2_manta(const float* __restrict__ s, const float* __restrict__ fwd,
                                            const float* __restrict__ U, const FT* __restrict__ flags,
                                            float* __restrict__ dst, float dt, float strength, Geo gin) {
  const Geo g = static_geo<IS3D>(gin);
  int b, k, j, i;
  if (!thread_cell(g, b, k, j, i)) return;
  const int c = cell(g, k, j, i);
  const FT* fl = flags + b * g.n;
  const float* sb = s + b * g.n;
  const float* fb = fwd + b * g.n;
  const float* ub = U + (long long)b * g.nc * g.n;
  const float fw = __ldg(fb + c);
  const bool border = on_border(g, k, j, i);
  float bw = 0.0f;
  if (!border) bw = advect_scalar_cell<TFL_ADVECT_MACCORMACK>(fl, ub, fb, g, -dt, k, j, i, true, nullptr);
  float v = fw;
  if (flag_i(fl, g, k, j, i) & kFluid) {
    const float diff = __ldg(sb + c) - bw;
    v = (float)((double)v + ((double)strength * 0.5) * (double)diff);
  }
  if (!border) {
    const V3 vel = scale3(mac_centered(ub, g, k, j, i), dt);
    const float fi = (float)i, fj = (float)j, fk = (float)(k + g.zoff);
    float lo = FLT_MAX, hi = -FLT_MAX;
    bool bail = false;
    for (int l = 0; l < 2 && !bail; l++) {
      const int px = l == 0 ? (int)(fi - vel.x) : (int)(fi + vel.x);
      const int py = l == 0 ? (int)(fj - vel.y) : (int)(fj + vel.y);
      const int pz = l == 0 ? (int)(fk - vel.z) : (int)(fk + vel.z);
      const int i0 = clamp_i(px, 0, g.nx - 2), j0 = clamp_i(py, 0, g.ny - 2);
      const int k0 = clamp_i(pz, 0, g.is3d ? g.gnz - 2 : 1);
      const int i1 = i0 + 1, j1 = j0 + 1, k1 = g.is3d ? k0 + 1 : k0;
      bool inb = i0 >= 0 && j0 >= 0 && i1 < g.nx && j1 < g.ny;
      if (g.is3d) inb = inb && k0 >= 0 && k1 < g.gnz; else inb = inb && k0 == 0 && k1 == 0;
      if (!inb) { bail = true; break; }
      const int kl0 = local_z(g, k0), kl1 = g.is3d ? local_z(g, k1) : kl0;
// The eight corners sit at fixed offsets from the first one (same visiting order as the reference).
      const float* a0 = sb + cell(g, kl0, j0, i0);
      const int dzo = (kl1 - kl0) * g.ny * g.nx;
#define TFL_MM(off) { const float t = __ldg(a0 + (off)); if (t < lo) lo = t; if (t > hi) hi = t; }
      TFL_MM(0) TFL_MM(1) TFL_MM(g.nx) TFL_MM(g.nx + 1)
      if (g.is3d) { TFL_MM(dzo) TFL_MM(dzo + 1) TFL_MM(dzo + g.nx) TFL_MM(dzo + g.nx + 1) }
#undef TFL_MM
    }
    v = bail ? fw : clamp_f(v, lo, hi);
    const int fx = (int)((fi + 0.5f) - vel.x), fy = (int)((fj + 0.5f) - vel.y), fz = (int)((fk + 0.5f) - vel.z);
    const int bx = (int)((fi + 0.5f) + vel.x), by = (int)((fj + 0.5f) + vel.y), bz = (int)((fk + 0.5f) + vel.z);
    const int ux = g.nx - 1, uy = g.ny - 1, uz = g.gnz - 1;
    if (fx < 0 || fy < 0 || fz < 0 || bx < 0 || by < 0 || bz < 0 || fx > ux || fy > uy ||
        (fz > uz && g.is3d) || bx > ux || by > uy || (bz > uz && g.is3d) ||
        (flag_i(fl, g, local_z(g, fz), fy, fx) & kObstacle) ||
        (flag_i(fl, g, local_z(g, bz), by, bx) & kObstacle)) {
      v = fw;
    }
  }
  dst[b * g.n + c] = v;
}

// ---------------------------------------------------------------------------------------
// advectVel
// ---------------------------------------------------------------------------------------
// vel[c]: velocity at the centre of face c of this cell (mac_at_x/y/z of the advecting field), computed
// by the caller because the MacCormack clamp of the same cell needs the same three vectors.
template <bool OURS, typename FT>
__device__ __forceinline__ V3 advect_mac_cell(const FT* __restrict__ fl, const V3 (&vel)[3],
                                              const float* __restrict__ src, const Geo& g, float dt, int k,
                                              int j, int i) {
  V3 r;
  if (OURS && !(flag_i(fl, g, k, j, i) & kFluid)) {
    const int c = cell(g, k, j, i);
    r.x = __ldg(src + c); r.y = __ldg(src + g.n + c); r.z = g.is3d ? __ldg(src + 2 * g.n + c) : 0.0f;
    return r;
  }
  const V3 start = {(float)i + 0.5f, (float)j + 0.5f, (float)(k + g.zoff) + 0.5f};
  V3 p;
  if (OURS) {
    line_trace(fl, g, start, scale3(vel[0], -dt), &p);
    r.x = lerp_block(src, g, p);
    line_trace(fl, g, start, scale3(vel[1], -dt), &p);
    r.y = lerp_block(src + g.n, g, p);
    if (g.is3d) {
      line_trace(fl, g, start, scale3(vel[2], -dt), &p);
      r.z = lerp_block(src + 2 * g.n, g, p);
    } else {
      r.z = 0.0f;
    }
  } else {
    V3 v = scale3(vel[0], dt);
    p = V3{start.x - v.x, start.y - v.y, start.z - v.z};
    r.x = lerp_block(src, g, p);
    v = scale3(vel[1], dt);
    p = V3{start.x - v.x, start.y - v.y, start.z - v.z};
    r.y = lerp_block(src + g.n, g, p);
    if (g.is3d) {
      v = scale3(vel[2], dt);
      p = V3{start.x - v.x, start.y - v.y, start.z - v.z};
      r.z = lerp_block(src + 2 * g.n, g, p);
    } else {
      r.z = 0.0f;
    }
  }
  return r;
}
// The "Ours" back-trace of one face component in clear space (see tfl_device.cuh): `reach` is the
// cell's clearance minus the slack; a longer trace takes the general code.
template <typename FT>
__device__ __forceinline__ float advect_mac_component_clear(const FT* __restrict__ fl, V3 vel,
                                                            const float* __restrict__ src_c, const Geo& g,
                                                            float dt, V3 start, float reach) {
  const V3 delta = scale3(vel, -dt);
  const float length = norm3(delta);
  if (length < reach) return lerp_block_clear(src_c, g, line_trace_clear(start, delta, length));
  V3 p;
  line_trace(fl, g, start, delta, &p);
  return lerp_block(src_c, g, p);
}
template <typename FT>
__device__ __forceinline__ V3 advect_mac_cell_clear(const FT* __restrict__ fl, const V3 (&vel)[3],
                                                    const float* __restrict__ src, const Geo& g, float dt,
                                                    int k, int j, int i, float reach) {
  const V3 start = {(float)i + 0.5f, (float)j + 0.5f, (float)(k + g.zoff) + 0.5f};
  V3 r;
  r.x = advect_mac_component_clear(fl, vel[0], src, g, dt, start, reach);
  r.y = advect_mac_component_clear(fl, vel[1], src + g.n, g, dt, start, reach);
  r.z = g.is3d ? advect_mac_component_clear(fl, vel[2], src + 2 * g.n, g, dt, start, reach) : 0.0f;
  return r;
}
// Resident CTAs per SM the advectVel kernels are compiled for (register budget 65536 / 256 / N).
#ifndef TFL_ADVECT_MINB1
#define TFL_ADVECT_MINB1 4
#endif
#ifndef TFL_ADVECT_MINB2
#define TFL_ADVECT_MINB2 4
#endif

template <bool IS3D, typename FT, bool OURS>
__global__ void __launch_bounds__(256, TFL_ADVECT_MINB1) k_advect_vel_pass1(const float* __restrict__ U, const FT* __restrict__ flags,
                                   const unsigned char* __restrict__ clear, float* __restrict__ out, float dt, Geo gin) {
  const Geo g = static_geo<IS3D>(gin);
  int b, k, j, i;
  if (!thread_cell(g, b, k, j, i)) return;
  const int c = cell(g, k, j, i);
  const float* ub = U + (long long)b * g.nc * g.n;
  V3 v = {0.0f, 0.0f, 0.0f};
  const int clr = (OURS && clear) ? (int)__ldg(clear + b * g.n + c) : 0;
  if (clr > 0) {                            // fluid cell of the interior
    V3 vel[3];
    mac_face_velocities(ub, g, k, j, i, vel);
    v = advect_mac_cell_clear(flags + b * g.n, vel, ub, g, dt, k, j, i, clear_reach(clr));
  } else if (!on_border(g, k, j, i)) {
    V3 vel[3];
    mac_face_velocities(ub, g, k, j, i, vel);
    v = advect_mac_cell<OURS>(flags + b * g.n, vel, ub, g, dt, k, j, i);
  }
  float* ob = out + (long long)b * g.nc * g.n + c;
  ob[0] = v.x; ob[g.n] = v.y;
  if (g.is3d) ob[2 * g.n] = v.z;
}

// The same clamp where the cell's clearance exceeds |vel|: both 2x2x2 boxes lie inside the local
// storage, so the index clamps and the bounds test cannot fire.
__device__ __forceinline__ float clamp_component_mac_clear(const float* __restrict__ orig_c, const Geo& g,
                                                           float val, int kloc, int j, int i, V3 vel) {
  const float fi = (float)i, fj = (float)j, fk = (float)(kloc + g.zoff);
  float lo = FLT_MAX, hi = -FLT_MAX;
  const int sy = g.nx, sz = g.nx * g.ny;
#pragma unroll
  for (int l = 0; l < 2; l++) {
    const int i0 = l == 0 ? (int)(fi - vel.x) : (int)(fi + vel.x);
    const int j0 = l == 0 ? (int)(fj - vel.y) : (int)(fj + vel.y);
    const int k0 = g.is3d ? (l == 0 ? (int)(fk - vel.z) : (int)(fk + vel.z)) - g.zoff : 0;
    const float* a0 = orig_c + cell(g, k0, j0, i0);
    const float* a1 = a0 + sy;
#define TFL_MM(ptr, off) { const float t = __ldg((ptr) + (off)); if (t < lo) lo = t; if (t > hi) hi = t; }
    TFL_MM(a0, 0) TFL_MM(a0, 1) TFL_MM(a1, 0) TFL_MM(a1, 1)
    if (g.is3d) {
      const float* b0 = a0 + sz;
      const float* b1 = b0 + sy;
      TFL_MM(b0, 0) TFL_MM(b0, 1) TFL_MM(b1, 0) TFL_MM(b1, 1)
    }
#undef TFL_MM
  }
  return clamp_f(val, lo, hi);
}

// Backward pass on the forward field + MacCormackCorrectMAC + MacCormackClampMAC, fused
// (third_party/tfluids.cc:859-915, 660-774).
template <bool IS3D, typename FT, bool OURS>
__global__ void __launch_bounds__(256, TFL_ADVECT_MINB2) k_advect_vel_pass2(const float* __restrict__ U, const float* __restrict__ fwd,
                                   const FT* __restrict__ flags, const unsigned char* __restrict__ clear,
                                   float* __restrict__ dst, float dt, float strength, Geo gin) {
  const Geo g = static_geo<IS3D>(gin);
  int b, k, j, i;
  if (!thread_cell(g, b, k, j, i)) return;
  const int c = cell(g, k, j, i);
  const FT* fl = flags + b * g.n;
  const float* ub = U + (long long)b * g.nc * g.n;
  const float* fb = fwd + (long long)b * g.nc * g.n;
  float* db = dst + (long long)b * g.nc * g.n + c;
  const int clr = (OURS && clear) ? (int)__ldg(clear + b * g.n + c) : 0;
  if (clr > 0) {
    // Fluid cell of the interior.  clr >= 2: its 26 neighbours are fluid, no face is skipped by the
    // correction; clr == 1: the three lower neighbours decide.
    const float reach = clear_reach(clr);
    V3 vel[3];
    mac_face_velocities(ub, g, k, j, i, vel);
    const V3 bw = advect_mac_cell_clear(fl, vel, fb, g, -dt, k, j, i, reach);
    const float bwv[3] = {bw.x, bw.y, bw.z};
    bool skip[3] = {false, false, false};
    if (clr == 1) {
      skip[0] = !(flag_at(fl, c - 1) & kFluid);
      skip[1] = !(flag_at(fl, c - g.nx) & kFluid);
      skip[2] = g.is3d && !(flag_at(fl, c - g.nx * g.ny) & kFluid);
    }
#pragma unroll
    for (int a = 0; a < 3; a++) {
      if (a < g.nc) {
        const float fw = __ldg(fb + a * g.n + c);
        float v = fw;
        if (!skip[a]) {
          const float diff = __ldg(ub + a * g.n + c) - bwv[a];
          v = (float)((double)fw + ((double)strength * 0.5) * (double)diff);
        }
        const V3 d = scale3(vel[a], dt);
        // |d| is the trace length of this component (the trace displacement is -d)
        if (norm3(d) < reach) v = clamp_component_mac_clear(ub + a * g.n, g, v, k, j, i, d);
        else v = clamp_component_mac(ub + a * g.n, g, v, fw, k + g.zoff, j, i, d);
        db[a * g.n] = v;
      }
    }
    return;
  }
  const bool border = on_border(g, k, j, i);
  V3 bw = {0.0f, 0.0f, 0.0f};
  V3 vel[3];
  if (!border) {
    mac_face_velocities(ub, g, k, j, i, vel);
    bw = advect_mac_cell<OURS>(fl, vel, fb, g, -dt, k, j, i);
  }
  const int kg = k + g.zoff;
  const bool cf = flag_i(fl, g, k, j, i) & kFluid;
  bool skip[3] = {!cf, !cf, !cf};
  if (i > 0 && !(flag_i(fl, g, k, j, i - 1) & kFluid)) skip[0] = true;
  if (j > 0 && !(flag_i(fl, g, k, j - 1, i) & kFluid)) skip[1] = true;
  if (g.is3d && kg > 0 && !(flag_i(fl, g, local_z(g, kg - 1), j, i) & kFluid)) skip[2] = true;
  const float bwv[3] = {bw.x, bw.y, bw.z};
  float val[3], fwv[3];
  for (int a = 0; a < g.nc; a++) {
    fwv[a] = __ldg(fb + a * g.n + c);
    float v = fwv[a];
    if (!skip[a]) {
      const float diff = __ldg(ub + a * g.n + c) - bwv[a];
      v = (float)((double)v + ((double)strength * 0.5) * (double)diff);
    }
    val[a] = v;
  }
  if (!border) {
    val[0] = clamp_component_mac(ub, g, val[0], fwv[0], kg, j, i, scale3(vel[0], dt));
    val[1] = clamp_component_mac(ub + g.n, g, val[1], fwv[1], kg, j, i, scale3(vel[1], dt));
    if (g.is3d)
      val[2] = clamp_component_mac(ub + 2 * g.n, g, val[2], fwv[2], kg, j, i,
                                   scale3(vel[2], dt));
  }
  for (int a = 0; a < g.nc; a++) db[a * g.n] = val[a];
}

// ---------------------------------------------------------------------------------------
// Jacobi.  The obstacle tests of the 7-point stencil are folded once per solve into one
// byte per cell; iterations then read p(7) + div + 1 byte and stay bit-identical to
// generic/tfluids.cu:1765-1821 in IEEE arithmetic.
//   bit0: cell is border-or-obstacle (p = 0); bits1..6: neighbour -x,+x,-y,+y,-z,+z is obstacle.
// ---------------------------------------------------------------------------------------
template <bool IS3D, typename FT>
__global__ void k_jacobi_mask(const FT* __restrict__ flags, unsigned char* __restrict__ mask, Geo gin) {
  const Geo g = static_geo<IS3D>(gin);
  int b, k, j, i;
  if (!thread_cell(g, b, k, j, i)) return;
  const FT* fl = flags + b * g.n;
  unsigned m = 0;
  if (on_border(g, k, j, i) || (flag_i(fl, g, k, j, i) & kObstacle)) {
    m = 1;
  } else {
    if (flag_i(fl, g, k, j, i - 1) & kObstacle) m |= 2;
    if (flag_i(fl, g, k, j, i + 1) & kObstacle) m |= 4;
    if (flag_i(fl, g, k, j - 1, i) & kObstacle) m |= 8;
    if (flag_i(fl, g, k, j + 1, i) & kObstacle) m |= 16;
    if (g.is3d) {
      if (flag_i(fl, g, k - 1, j, i) & kObstacle) m |= 32;
      if (flag_i(fl, g, k + 1, j, i) & kObstacle) m |= 64;
    }
  }
  mask[b * g.n + cell(g, k, j, i)] = (unsigned char)m;
}

template <bool IS3D, typename FT>
__global__ void k_jacobi_iter(const unsigned char* __restrict__ mask, const float* __restrict__ div,
                              const float* __restrict__ prev, float* __restrict__ cur, Geo gin) {
  const Geo g = static_geo<IS3D>(gin);
  int b, k, j, i;
  if (!thread_cell(g, b, k, j, i)) return;
  const long long c = b * g.n + cell(g, k, j, i);
  const unsigned m = mask[c];
  if (m & 1) { cur[c] = 0.0f; return; }
  const int sy = g.nx, sz = g.nx * g.ny;
  const float pc = __ldg(prev + c);
  float p1 = (m & 2) ? pc : __ldg(prev + c - 1);
  float p2 = (m & 4) ? pc : __ldg(prev + c + 1);
  float p3 = (m & 8) ? pc : __ldg(prev + c - sy);
  float p4 = (m & 16) ? pc : __ldg(prev + c + sy);
  float p5 = 0.0f, p6 = 0.0f;
  if (g.is3d) {
    p5 = (m & 32) ? pc : __ldg(prev + c - sz);
    p6 = (m & 64) ? pc : __ldg(prev + c + sz);
  }
  const float denom = g.is3d ? 6.0f : 4.0f;
  cur[c] = (p1 + p2 + p3 + p4 + p5 + p6 + __ldg(div + c)) / denom;
}

// Same update, 4 consecutive x cells per thread (float4 rows, one 32-bit load for the 4 mask
// bytes): 8 memory instructions per 4 cells instead of 40.  Requires nx % 4 == 0.
template <bool IS3D, typename FT>
__global__ void __launch_bounds__(256)
k_jacobi_iter4(const unsigned char* __restrict__ mask, const float* __restrict__ div,
               const float* __restrict__ prev, float* __restrict__ cur, Geo gin) {
  const Geo g = static_geo<IS3D>(gin);
  const int i0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  const int j = blockIdx.y * blockDim.y + threadIdx.y;
  const int zz = blockIdx.z * blockDim.z + threadIdx.z;
  const int nzr = g.zhi - g.zlo;
  const int b = zz / nzr;
  const int k = g.zlo + (zz - b * nzr);
  if (i0 >= g.nx || j >= g.ny || b >= g.nb) return;
  const long long c = b * g.n + cell(g, k, j, i0);
  const unsigned m4 = __ldg((const unsigned*)(mask + c));
  float out[4] = {0.0f, 0.0f, 0.0f, 0.0f};
  if ((m4 & 0x01010101u) != 0x01010101u) {          // at least one cell of the quad is live
    const int sy = g.nx, sz = g.nx * g.ny;
    const float4 pc = __ldg((const float4*)(prev + c));
    const float4 dv = __ldg((const float4*)(div + c));
    const float4 ym = __ldg((const float4*)(prev + c - sy));   // a live cell is never on the border,
    const float4 yp = __ldg((const float4*)(prev + c + sy));   // so these rows exist
    float4 zm = make_float4(0.f, 0.f, 0.f, 0.f), zp = zm;
    if (g.is3d) {
      zm = __ldg((const float4*)(prev + c - sz));
      zp = __ldg((const float4*)(prev + c + sz));
    }
    const float left = i0 > 0 ? __ldg(prev + c - 1) : 0.0f;
    const float right = i0 + 4 < g.nx ? __ldg(prev + c + 4) : 0.0f;
    const float pcv[4] = {pc.x, pc.y, pc.z, pc.w};
    const float xm[4] = {left, pc.x, pc.y, pc.z};
    const float xp[4] = {pc.y, pc.z, pc.w, right};
    const float ymv[4] = {ym.x, ym.y, ym.z, ym.w}, ypv[4] = {yp.x, yp.y, yp.z, yp.w};
    const float zmv[4] = {zm.x, zm.y, zm.z, zm.w}, zpv[4] = {zp.x, zp.y, zp.z, zp.w};
    const float dvv[4] = {dv.x, dv.y, dv.z, dv.w};
    const float denom = g.is3d ? 6.0f : 4.0f;
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const unsigned m = (m4 >> (8 * q)) & 0xFFu;
      if (m & 1) continue;
      const float p1 = (m & 2) ? pcv[q] : xm[q];
      const float p2 = (m & 4) ? pcv[q] : xp[q];
      const float p3 = (m & 8) ? pcv[q] : ymv[q];
      const float p4 = (m & 16) ? pcv[q] : ypv[q];
      float p5 = 0.0f, p6 = 0.0f;
      if (g.is3d) {
        p5 = (m & 32) ? pcv[q] : zmv[q];
        p6 = (m & 64) ? pcv[q] : zpv[q];
      }
      out[q] = (p1 + p2 + p3 + p4 + p5 + p6 + dvv[q]) / denom;
    }
  }
  *(float4*)(cur + c) = make_float4(out[0], out[1], out[2], out[3]);
}

// 2.5-D variant: a CTA owns a 128 x 8 (x, y) patch and marches over a chunk of z planes keeping the
// previous / current / next plane of p in registers, so every p value is read from L2/HBM once per
// sweep (plus the patch's y halo rows) instead of five times; y neighbours inside the patch are
// exchanged through shared memory, x neighbours with warp shuffles.  Per-cell arithmetic is the
// same expression as above (bit-identical).  Requires 3-D, nx % 128 == 0, ny % 8 == 0.
constexpr int kJY = 8;
__global__ void __launch_bounds__(256)
k_jacobi_march(const unsigned char* __restrict__ mask, const float* __restrict__ div,
               const float* __restrict__ prev, float* __restrict__ cur, Geo g, int zchunk) {
  __shared__ float4 rows[2][kJY][32];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int i0 = (blockIdx.x * 32 + tx) * 4;
  const int j = blockIdx.y * kJY + ty;
  const int nchunks = (g.nz + zchunk - 1) / zchunk;
  const int b = blockIdx.z / nchunks;
  const int k0 = (blockIdx.z % nchunks) * zchunk;
  const int k1 = min(k0 + zchunk, g.nz);
  const int sy = g.nx, sz = g.nx * g.ny;
  const long long base = b * g.n + (long long)j * sy + i0;
  const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
  // Everything plane k needs is requested while plane k-1 is being computed (software pipelining
  // by one plane; p itself by two planes).
  struct PlaneIn { float4 dv, ym, yp; unsigned m4; float left, right; };
  auto fetch = [&](int k, PlaneIn& in) {
    const long long c = base + (long long)k * sz;
    in.m4 = __ldg((const unsigned*)(mask + c));
    in.dv = __ldg((const float4*)(div + c));
    in.ym = (ty == 0 && j > 0) ? __ldg((const float4*)(prev + c - sy)) : zero4;
    in.yp = (ty == kJY - 1 && j + 1 < g.ny) ? __ldg((const float4*)(prev + c + sy)) : zero4;
    in.left = (tx == 0 && i0 > 0) ? __ldg(prev + c - 1) : 0.0f;
    in.right = (tx == 31 && i0 + 4 < g.nx) ? __ldg(prev + c + 4) : 0.0f;
  };
  float4 pm = k0 > 0 ? __ldg((const float4*)(prev + base + (long long)(k0 - 1) * sz)) : zero4;
  float4 pc = __ldg((const float4*)(prev + base + (long long)k0 * sz));
  float4 pp = k0 + 1 < g.nz ? __ldg((const float4*)(prev + base + (long long)(k0 + 1) * sz)) : zero4;
  PlaneIn in;
  fetch(k0, in);
  for (int k = k0; k < k1; k++) {
    const long long c = base + (long long)k * sz;
    const float4 pq = k + 2 < g.nz ? __ldg((const float4*)(prev + c + 2 * (long long)sz)) : zero4;
    PlaneIn nx_in = in;
    if (k + 1 < k1) fetch(k + 1, nx_in);
    const int buf = k & 1;
    rows[buf][ty][tx] = pc;
    float left = __shfl_up_sync(0xffffffffu, pc.w, 1);
    float right = __shfl_down_sync(0xffffffffu, pc.x, 1);
    if (tx == 0) left = in.left;
    if (tx == 31) right = in.right;
    __syncthreads();
    const float4 ym = ty > 0 ? rows[buf][ty - 1][tx] : in.ym;
    const float4 yp = ty < kJY - 1 ? rows[buf][ty + 1][tx] : in.yp;
    const unsigned m4 = in.m4;
    float out[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    if ((m4 & 0x01010101u) != 0x01010101u) {
      const float pcv[4] = {pc.x, pc.y, pc.z, pc.w};
      const float xm[4] = {left, pc.x, pc.y, pc.z};
      const float xp[4] = {pc.y, pc.z, pc.w, right};
      const float ymv[4] = {ym.x, ym.y, ym.z, ym.w}, ypv[4] = {yp.x, yp.y, yp.z, yp.w};
      const float zmv[4] = {pm.x, pm.y, pm.z, pm.w}, zpv[4] = {pp.x, pp.y, pp.z, pp.w};
      const float dvv[4] = {in.dv.x, in.dv.y, in.dv.z, in.dv.w};
#pragma unroll
      for (int q = 0; q < 4; q++) {
        const unsigned m = (m4 >> (8 * q)) & 0xFFu;
        if (m & 1) continue;
        const float p1 = (m & 2) ? pcv[q] : xm[q];
        const float p2 = (m & 4) ? pcv[q] : xp[q];
        const float p3 = (m & 8) ? pcv[q] : ymv[q];
        const float p4 = (m & 16) ? pcv[q] : ypv[q];
        const float p5 = (m & 32) ? pcv[q] : zmv[q];
        const float p6 = (m & 64) ? pcv[q] : zpv[q];
        out[q] = (p1 + p2 + p3 + p4 + p5 + p6 + dvv[q]) / 6.0f;
      }
    }
    *(float4*)(cur + c) = make_float4(out[0], out[1], out[2], out[3]);
    pm = pc;
    pc = pp;
    pp = pq;
    in = nx_in;
  }
}

// All sweeps in ONE kernel with the CTA's cells resident on the SM.  A CTA owns a 128 x 8 x kJZ block for the
// whole solve (cooperative launch: every CTA stays resident): its p values live in registers from sweep to
// sweep, div and the block's y-rows in shared memory, and per sweep only the block's halo (two z planes, two
// y rows per plane, the x neighbours of wider grids) is read from L2 -- written there by the neighbouring CTAs
// before the grid-wide barrier that separates the sweeps.  For grids whose fields sit in L2 (128^3: 8 MB per
// field) the one-kernel-per-sweep version spent most of a sweep on the launch boundary and on L2 latency in
// its plane-by-plane march; here a sweep is one halo round trip, ~500 instructions per thread and the barrier.
// p is read with ld.global.cg (L1 is not coherent across CTAs).  Same per-cell expression (bit-identical).
constexpr int kJZ = 4;
constexpr int kJG = 4;        // blocks per CTA: fewer, fatter CTAs make the grid-wide barrier (one atomic per CTA) cheaper
__global__ void __launch_bounds__(256 * kJG, 1)
k_jacobi_resident(const unsigned char* __restrict__ mask, const float* __restrict__ div, float* pa, float* pb, Geo g,
                  int sweeps, int nblocks) {
  cooperative_groups::grid_group grid = cooperative_groups::this_grid();
  extern __shared__ float4 jsm[];
  // thread group threadIdx.z of the CTA owns block blockIdx.x * kJG + threadIdx.z (x tile fastest, then y, then z chunk)
  constexpr int kGroupF4 = kJZ * (kJY + 2) * 32 + kJZ * kJY * 32;
  float4* gsm = jsm + threadIdx.z * kGroupF4;
  float4 (*rows)[kJY + 2][32] = reinterpret_cast<float4 (*)[kJY + 2][32]>(gsm);               // [kJZ][kJY + 2][32]
  float4 (*dvs)[kJY][32] = reinterpret_cast<float4 (*)[kJY][32]>(gsm + kJZ * (kJY + 2) * 32);   // [kJZ][kJY][32]
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int blk = blockIdx.x * kJG + threadIdx.z;
  const bool live = blk < nblocks;                         // a group without a block only takes part in the barriers
  const int nxt = g.nx / 128, nyt = g.ny / kJY;
  const int bx = blk % nxt, by = (blk / nxt) % nyt, bz = blk / (nxt * nyt);
  const int i0 = (bx * 32 + tx) * 4;
  const int j = by * kJY + ty;
  const int nchunks = (g.nz + kJZ - 1) / kJZ;
  const int b = live ? bz / nchunks : 0;
  const int k0 = live ? (bz % nchunks) * kJZ : 0;
  const int np = live ? min(kJZ, g.nz - k0) : 0;           // planes of this block
  const int sy = g.nx, sz = g.nx * g.ny;
  const long long base = live ? b * g.n + (long long)k0 * sz + (long long)j * sy + i0 : 0;
  const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
  const bool has_left = tx == 0 && i0 > 0, has_right = tx == 31 && i0 + 4 < g.nx;
  unsigned m4[kJZ];
  float4 pc[kJZ];
#pragma unroll
  for (int k = 0; k < kJZ; k++) {
    const bool in = k < np;
    m4[k] = in ? __ldg((const unsigned*)(mask + base + (long long)k * sz)) : 0x01010101u;
    dvs[k][ty][tx] = in ? __ldg((const float4*)(div + base + (long long)k * sz)) : zero4;
    pc[k] = in ? __ldcg((const float4*)(pa + base + (long long)k * sz)) : zero4;
  }
  for (int s = 0; s < sweeps; s++) {
    const float* prev = (s & 1) ? pb : pa;                 // sweep 0 reads pa and writes pb
    float* cur = (s & 1) ? pa : pb;
    // halo of the block, all requests in flight together
    const float4 zlo = (live && k0 > 0) ? __ldcg((const float4*)(prev + base - sz)) : zero4;
    const float4 zhi = (live && k0 + np < g.nz) ? __ldcg((const float4*)(prev + base + (long long)np * sz)) : zero4;
    float left[kJZ], right[kJZ];
#pragma unroll
    for (int k = 0; k < kJZ; k++) {
      const long long c = base + (long long)k * sz;
      const bool in = k < np;
      if (ty == 0) rows[k][0][tx] = (in && j > 0) ? __ldcg((const float4*)(prev + c - sy)) : zero4;
      if (ty == kJY - 1) rows[k][kJY + 1][tx] = (in && j + 1 < g.ny) ? __ldcg((const float4*)(prev + c + sy)) : zero4;
      left[k] = (in && has_left) ? __ldcg(prev + c - 1) : 0.0f;
      right[k] = (in && has_right) ? __ldcg(prev + c + 4) : 0.0f;
      rows[k][ty + 1][tx] = pc[k];
    }
    asm volatile("bar.sync %0, 256;" ::"r"(1 + (int)threadIdx.z) : "memory");      // this group's rows are in place
    float4 below = zlo;
#pragma unroll
    for (int k = 0; k < kJZ; k++) {
      const float4 ctr = pc[k];
      const float4 above = k + 1 < kJZ ? (k + 1 < np ? pc[k + 1] : zhi) : zhi;
      float out[4] = {0.0f, 0.0f, 0.0f, 0.0f};
      const unsigned mm = m4[k];
      float lf = __shfl_up_sync(0xffffffffu, ctr.w, 1);        // every lane takes part, whatever its mask
      float rt = __shfl_down_sync(0xffffffffu, ctr.x, 1);
      if (tx == 0) lf = left[k];
      if (tx == 31) rt = right[k];
      if ((mm & 0x01010101u) != 0x01010101u) {
        const float4 ym = rows[k][ty][tx], yp = rows[k][ty + 2][tx], dv = dvs[k][ty][tx];
        const float pcv[4] = {ctr.x, ctr.y, ctr.z, ctr.w};
        const float xm[4] = {lf, ctr.x, ctr.y, ctr.z};
        const float xp[4] = {ctr.y, ctr.z, ctr.w, rt};
        const float ymv[4] = {ym.x, ym.y, ym.z, ym.w}, ypv[4] = {yp.x, yp.y, yp.z, yp.w};
        const float zmv[4] = {below.x, below.y, below.z, below.w}, zpv[4] = {above.x, above.y, above.z, above.w};
        const float dvv[4] = {dv.x, dv.y, dv.z, dv.w};
#pragma unroll
        for (int q = 0; q < 4; q++) {
          const unsigned m = (mm >> (8 * q)) & 0xFFu;
          if (m & 1) continue;
          const float p1 = (m & 2) ? pcv[q] : xm[q];
          const float p2 = (m & 4) ? pcv[q] : xp[q];
          const float p3 = (m & 8) ? pcv[q] : ymv[q];
          const float p4 = (m & 16) ? pcv[q] : ypv[q];
          const float p5 = (m & 32) ? pcv[q] : zmv[q];
          const float p6 = (m & 64) ? pcv[q] : zpv[q];
          out[q] = (p1 + p2 + p3 + p4 + p5 + p6 + dvv[q]) / 6.0f;
        }
      }
      const float4 o4 = make_float4(out[0], out[1], out[2], out[3]);
      if (k < np) *(float4*)(cur + base + (long long)k * sz) = o4;
      pc[k] = o4;
      below = ctr;
    }
    grid.sync();                                           // also orders the shared rows against the next sweep
  }
}

// sum over one batch element of (a - b)^2, accumulated in double: out[b] += ...
__global__ void k_sqdiff(const float* __restrict__ a, const float* __restrict__ bb, long long n,
                         double* __restrict__ out) {
  const int b = blockIdx.y;
  const float* pa = a + b * n;
  const float* pb = bb + b * n;
  double acc = 0.0;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n;
       t += (long long)gridDim.x * blockDim.x) {
    const float d = pa[t] - pb[t];
    acc += (double)d * (double)d;
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
  __shared__ double warp_sums[32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) warp_sums[w] = acc;
  __syncthreads();
  if (w == 0) {
    acc = (lane < (blockDim.x >> 5)) ? warp_sums[lane] : 0.0;
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
    if (lane == 0) atomicAdd(out + b, acc);
  }
}

// ---------------------------------------------------------------------------------------
// Flat element-wise helpers (the cutorch calls lib/simulate.lua makes on the step).
// ---------------------------------------------------------------------------------------
__global__ void k_apply_bc(float* __restrict__ x, const float* __restrict__ inv, const float* __restrict__ bc,
                           long long n) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const float v = x[t] * __ldg(inv + t);
  x[t] = v + __ldg(bc + t);
}
__global__ void k_clamp(float* __restrict__ x, float lo, float hi, long long n) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const float v = x[t];
  x[t] = (v < lo) ? lo : ((v > hi) ? hi : v);
}

// ---------------------------------------------------------------------------------------
// Launchers
// ---------------------------------------------------------------------------------------
// Launch `kernel<IS3D, FT, extra...>` with IS3D picked from the geometry.
#define TFL_LAUNCH3(kernel, FT, g, st, ...)                      \
  do {                                                           \
    dim3 grid_, block_;                                          \
    launch_dims(g, grid_, block_);                               \
    if ((g).is3d) kernel<true, FT><<<grid_, block_, 0, st>>>(__VA_ARGS__);   \
    else kernel<false, FT><<<grid_, block_, 0, st>>>(__VA_ARGS__);           \
  } while (0)
#define TFL_LAUNCH3X(kernel, FT, X, g, st, ...)                  \
  do {                                                           \
    dim3 grid_, block_;                                          \
    launch_dims(g, grid_, block_);                               \
    if ((g).is3d) kernel<true, FT, X><<<grid_, block_, 0, st>>>(__VA_ARGS__);   \
    else kernel<false, FT, X><<<grid_, block_, 0, st>>>(__VA_ARGS__);           \
  } while (0)

void launch_empty_domain(float* flags, const Geo& g, int bnd, cudaStream_t st) {
  TFL_LAUNCH3(k_empty_domain, float, g, st, flags, g, bnd);
}
void launch_flags_to_occupancy(const float* flags, float* occ, long long n, unsigned long long* bad,
                               cudaStream_t st) {
  k_flags_to_occupancy<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(flags, occ, n, bad);
}
template <typename FT>
void launch_set_wall_bcs(float* U, const FT* flags, const Geo& g, int as_mask, cudaStream_t st) {
  TFL_LAUNCH3(k_set_wall_bcs, FT, g, st, U, flags, g, as_mask);
}
template <typename FT>
void launch_divergence(const float* U, const FT* flags, float* div, const Geo& g, cudaStream_t st) {
  TFL_LAUNCH3(k_divergence, FT, g, st, U, flags, div, g);
}
template <typename FT>
void launch_velocity_update(float* U, const FT* flags, const float* p, const Geo& g, cudaStream_t st) {
  TFL_LAUNCH3(k_velocity_update, FT, g, st, U, flags, p, g);
}
template <typename FT>
void launch_add_buoyancy(float* U, const FT* flags, const float* rho, const float s[3], const Geo& g,
                         cudaStream_t st) {
  TFL_LAUNCH3(k_add_buoyancy, FT, g, st, U, flags, rho, s[0], s[1], s[2], g);
}
template <typename FT>
void launch_add_gravity(float* U, const FT* flags, const float f[3], const Geo& g, cudaStream_t st) {
  TFL_LAUNCH3(k_add_gravity, FT, g, st, U, flags, f[0], f[1], f[2], g);
}
// curl + |curl| on [zlo-2, zhi+1), then the force on [zlo-1, zhi) (what AddForceField on
// [zlo, zhi) reads).  force always has 3 channels.
void launch_vort_curl(const float* U, float* curl, float* cnorm, float* force, float strength, const Geo& g,
                      cudaStream_t st) {
  if (g.zlo == 0 && g.zhi == g.nz && g.zoff == 0 && g.gnz == g.nz &&
      launch_vort_curl_quad(U, curl, cnorm, force, strength, g, st))
    return;                                              // whole grid on one GPU: 4 voxels per thread
  Geo g1 = g;
  g1.zlo = g.zlo - 2 < 0 ? 0 : g.zlo - 2;
  g1.zhi = g.zhi + 1 > g.nz ? g.nz : g.zhi + 1;
  TFL_LAUNCH3(k_vort_curl, float, g1, st, U, curl, cnorm, g1);
  Geo g2 = g;
  g2.zlo = g.zlo - 1 < 0 ? 0 : g.zlo - 1;
  TFL_LAUNCH3(k_vort_force, float, g2, st, curl, cnorm, force, strength, g2);
}
template <typename FT>
int launch_vorticity(float* U, const FT* flags, float strength, float* curl, float* cnorm, float* force,
                     const Geo& g, cudaStream_t st) {
  launch_vort_curl(U, curl, cnorm, force, strength, g, st);
  TFL_LAUNCH3(k_vort_apply, FT, g, st, U, flags, force, g);
  return 3;
}

template <typename FT>
int launch_advect_scalar(float dt, const float* s, const float* U, const FT* flags, const unsigned char* clear,
                         int method, int outside, float strength, float* dst, float* fwd, float* fwd_pos,
                         const Geo& g, const Geo& g_fwd, cudaStream_t st) {
  switch (method) {
    case TFL_ADVECT_EULER:
      TFL_LAUNCH3X(k_advect_scalar_pass1, FT, TFL_ADVECT_EULER, g, st, s, U, flags, clear, dst, nullptr, dt, outside, g);
      return 1;
    case TFL_ADVECT_EULER_OURS:
      TFL_LAUNCH3X(k_advect_scalar_pass1, FT, TFL_ADVECT_EULER_OURS, g, st, s, U, flags, clear, dst, nullptr, dt, outside, g);
      return 1;
    case TFL_ADVECT_RK2_OURS:
      TFL_LAUNCH3X(k_advect_scalar_pass1, FT, TFL_ADVECT_RK2_OURS, g, st, s, U, flags, clear, dst, nullptr, dt, outside, g);
      return 1;
    case TFL_ADVECT_RK3_OURS:
      TFL_LAUNCH3X(k_advect_scalar_pass1, FT, TFL_ADVECT_RK3_OURS, g, st, s, U, flags, clear, dst, nullptr, dt, outside, g);
      return 1;
    case TFL_ADVECT_MACCORMACK:
      TFL_LAUNCH3X(k_advect_scalar_pass1, FT, TFL_ADVECT_MACCORMACK, g_fwd, st, s, U, flags, clear, fwd, nullptr, dt, outside, g_fwd);
      TFL_LAUNCH3(k_advect_scalar_pass2_manta, FT, g, st, s, fwd, U, flags, dst, dt, strength, g);
      return 2;
    case TFL_ADVECT_MACCORMACK_OURS:
      TFL_LAUNCH3X(k_advect_scalar_pass1, FT, TFL_ADVECT_MACCORMACK_OURS, g_fwd, st, s, U, flags, clear, fwd, fwd_pos, dt, outside, g_fwd);
      TFL_LAUNCH3(k_advect_scalar_pass2_ours, FT, g, st, s, fwd, fwd_pos, U, flags, clear, dst, dt, strength, outside, g);
      return 2;
  }
  return -1;
}

template <typename FT>
int launch_advect_vel(float dt, const float* U, const FT* flags, const unsigned char* clear, int method,
                      float strength, float* dst, float* fwd, const Geo& g, const Geo& g_fwd, cudaStream_t st) {
  if (method == TFL_ADVECT_RK2_OURS || method == TFL_ADVECT_RK3_OURS) method = TFL_ADVECT_MACCORMACK_OURS;
  switch (method) {
    case TFL_ADVECT_EULER:
      TFL_LAUNCH3X(k_advect_vel_pass1, FT, false, g, st, U, flags, clear, dst, dt, g);
      return 1;
    case TFL_ADVECT_EULER_OURS:
      TFL_LAUNCH3X(k_advect_vel_pass1, FT, true, g, st, U, flags, clear, dst, dt, g);
      return 1;
    case TFL_ADVECT_MACCORMACK:
      TFL_LAUNCH3X(k_advect_vel_pass1, FT, false, g_fwd, st, U, flags, clear, fwd, dt, g_fwd);
      TFL_LAUNCH3X(k_advect_vel_pass2, FT, false, g, st, U, fwd, flags, clear, dst, dt, strength, g);
      return 2;
    case TFL_ADVECT_MACCORMACK_OURS:
      TFL_LAUNCH3X(k_advect_vel_pass1, FT, true, g_fwd, st, U, flags, clear, fwd, dt, g_fwd);
      TFL_LAUNCH3X(k_advect_vel_pass2, FT, true, g, st, U, fwd, flags, clear, dst, dt, strength, g);
      return 2;
  }
  return -1;
}

template <typename FT>
void launch_jacobi_mask(const FT* flags, unsigned char* mask, const Geo& g, cudaStream_t st) {
  TFL_LAUNCH3(k_jacobi_mask, FT, g, st, flags, mask, g);
}
void launch_jacobi_iter(const unsigned char* mask, const float* div, const float* prev, float* cur,
                        const Geo& g, cudaStream_t st) {
  const bool aligned = ((uintptr_t)mask % 4 == 0) && ((uintptr_t)div % 16 == 0) && ((uintptr_t)prev % 16 == 0) &&
                       ((uintptr_t)cur % 16 == 0);
  // The marching kernel pays off once the fields no longer fit L2 (>= 4M cells); smaller grids keep
  // more CTAs in flight with the flat float4 kernel.  (Tests force it through nx == 128 / 256 shapes
  // with few planes, where both kernels are selected by shape alone.)
  const bool big = g.n * g.nb >= (4LL << 20) || g.nz < 16;
  if (g.is3d && aligned && big && g.nx % 128 == 0 && g.ny % kJY == 0 && g.zlo == 0 && g.zhi == g.nz && g.nz >= 8) {
    // enough CTAs to fill the machine (>= ~4 per SM), chunks of at least 4 planes
    const int xy_ctas = (g.nx / 128) * (g.ny / kJY) * g.nb;
    int zchunk = 32;
    while (zchunk > 4 && (long long)xy_ctas * ((g.nz + zchunk - 1) / zchunk) < 592) zchunk >>= 1;
    dim3 block(32, kJY, 1);
    dim3 grid(g.nx / 128, g.ny / kJY, ((g.nz + zchunk - 1) / zchunk) * g.nb);
    k_jacobi_march<<<grid, block, 0, st>>>(mask, div, prev, cur, g, zchunk);
    return;
  }
  if (g.nx % 4 == 0 && aligned) {
    const int nzr = g.zhi - g.zlo;
    const int qx = g.nx / 4;
    dim3 block(qx >= 32 ? 32 : qx, 1, 1);
    block.y = g.nz == 1 ? 8 : 4;
    block.z = g.nz == 1 ? 1 : 2;
    dim3 grid((qx + block.x - 1) / block.x, (g.ny + block.y - 1) / block.y,
              ((long long)g.nb * nzr + block.z - 1) / block.z);
    if (g.is3d) k_jacobi_iter4<true, float><<<grid, block, 0, st>>>(mask, div, prev, cur, g);
    else k_jacobi_iter4<false, float><<<grid, block, 0, st>>>(mask, div, prev, cur, g);
    return;
  }
  TFL_LAUNCH3(k_jacobi_iter, float, g, st, mask, div, prev, cur, g);
}
// `sweeps` Jacobi sweeps in ONE cooperative launch: sweep 0 reads pa and writes pb, sweep 1 the other way, ...
// (the result is in pb for an odd count).  Returns false when the shape / device does not qualify (the caller
// then launches one kernel per sweep).
bool launch_jacobi_sweeps(const unsigned char* mask, const float* div, float* pa, float* pb, const Geo& g, int sweeps,
                          cudaStream_t st) {
  const bool aligned = ((uintptr_t)mask % 4 == 0) && ((uintptr_t)div % 16 == 0) && ((uintptr_t)pa % 16 == 0) &&
                       ((uintptr_t)pb % 16 == 0);
  // fields that sit in L2; larger grids are bandwidth-bound per sweep and do not fit the SMs
  if (!g.is3d || !aligned || g.nx % 128 != 0 || g.ny % kJY != 0 || g.nz < 4 || g.zlo != 0 || g.zhi != g.nz ||
      g.n * g.nb > (3LL << 20) || sweeps < 2)
    return false;
  const int smem = kJG * (kJZ * (kJY + 2) * 32 + kJZ * kJY * 32) * (int)sizeof(float4);
  static int capacities[64];         // resident CTAs of this kernel, per device (0: not asked yet, -1: cannot)
  int dev = 0;
  cudaGetDevice(&dev);
  int& capacity = capacities[dev & 63];
  if (capacity == 0) {
    int sms = 0, per_sm = 0, coop = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
    capacity = -1;
    if (coop && cudaFuncSetAttribute(k_jacobi_resident, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) == cudaSuccess &&
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_jacobi_resident, 256 * kJG, smem) == cudaSuccess &&
        sms * per_sm > 0)
      capacity = sms * per_sm;
    cudaGetLastError();
  }
  const int nch = (g.nz + kJZ - 1) / kJZ;
  int nblocks = (g.nx / 128) * (g.ny / kJY) * nch * g.nb;
  const int ctas = (nblocks + kJG - 1) / kJG;
  if (ctas > capacity) return false;
  dim3 block(32, kJY, kJG), grid(ctas, 1, 1);
  Geo gg = g;
  void* args[] = {(void*)&mask, (void*)&div, (void*)&pa, (void*)&pb, (void*)&gg, (void*)&sweeps, (void*)&nblocks};
  if (cudaLaunchCooperativeKernel((const void*)k_jacobi_resident, grid, block, args, smem, st) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return true;
}
void launch_sqdiff(const float* a, const float* b, long long n, int nb, double* out, cudaStream_t st) {
  long long blocks = (n + 1023) / 1024;
  if (blocks > 592) blocks = 592;
  k_sqdiff<<<dim3((unsigned)blocks, nb), 256, 0, st>>>(a, b, n, out);
}
void launch_apply_bc(float* x, const float* inv, const float* bc, long long n, cudaStream_t st) {
  k_apply_bc<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(x, inv, bc, n);
}
void launch_clamp(float* x, float lo, float hi, long long n, cudaStream_t st) {
  k_clamp<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(x, lo, hi, n);
}


// Explicit instantiations: float flags (operator-level API) and byte flags (fused step).
#define TFL_INSTANTIATE(FT)                                                                                   \
  template void launch_set_wall_bcs<FT>(float*, const FT*, const Geo&, int, cudaStream_t);                    \
  template void launch_divergence<FT>(const float*, const FT*, float*, const Geo&, cudaStream_t);            \
  template void launch_velocity_update<FT>(float*, const FT*, const float*, const Geo&, cudaStream_t);       \
  template void launch_add_buoyancy<FT>(float*, const FT*, const float*, const float*, const Geo&, cudaStream_t); \
  template void launch_add_gravity<FT>(float*, const FT*, const float*, const Geo&, cudaStream_t);           \
  template int launch_vorticity<FT>(float*, const FT*, float, float*, float*, float*, const Geo&, cudaStream_t); \
  template int launch_advect_scalar<FT>(float, const float*, const float*, const FT*, const unsigned char*, int, int, \
                                        float, float*, float*, float*, const Geo&, const Geo&, cudaStream_t);  \
  template int launch_advect_vel<FT>(float, const float*, const FT*, const unsigned char*, int, float, float*, \
                                     float*, const Geo&, const Geo&, cudaStream_t);                          \
  template void launch_jacobi_mask<FT>(const FT*, unsigned char*, const Geo&, cudaStream_t);
TFL_INSTANTIATE(float)
TFL_INSTANTIATE(unsigned char)
#undef TFL_INSTANTIATE

// ---------------------------------------------------------------------------------------
// Clearance field of the advection fast path (tfl_device.cuh): three separable passes over the LOCAL
// storage.  x: run of usable cells around the cell; y, z: largest r such that the previous pass' value
// is >= r on every line cell within r (the box of radius r is all usable <=> the distance is r + 1).
// ---------------------------------------------------------------------------------------
// Grid-stride kernels on a fixed small grid: a launch whose gate word is 0 (flags unchanged) costs almost nothing.
__device__ __forceinline__ bool clear_cell(const Geo& g, long long t, int& b, int& k, int& j, int& i) {
  const long long total = g.n * g.nb;
  if (t >= total) return false;
  b = (int)(t / g.n);
  int r = (int)(t - b * g.n);
  k = r / (g.nx * g.ny);
  r -= k * g.nx * g.ny;
  j = r / g.nx;
  i = r - j * g.nx;
  return true;
}
template <typename FT>
__global__ void k_clear_x(const FT* __restrict__ flags, unsigned char* __restrict__ out, Geo g,
                          const int* __restrict__ gate) {
  if (gate && *gate == 0) return;          // flags unchanged since the cached field was built
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;; t += (long long)gridDim.x * blockDim.x) {
    int b, k, j, i;
    if (!clear_cell(g, t, b, k, j, i)) return;
    const FT* row = flags + b * g.n + cell(g, k, j, 0);
    // usable = fluid and not on an end of the storage (whole row if j / k sit on one)
    const bool row_ok = j > 0 && j < g.ny - 1 && (!g.is3d || (k > 0 && k < g.nz - 1));
    int r = -1;
    if (row_ok && i > 0 && i < g.nx - 1 && (flag_at(row, i) & kFluid)) {
      r = 0;
      for (int d = 1; d <= kClearMax; d++) {
        if (i - d < 1 || i + d > g.nx - 2 || !(flag_at(row, i - d) & kFluid) || !(flag_at(row, i + d) & kFluid)) break;
        r = d;
      }
    }
    out[t] = (unsigned char)(r < 0 ? 255 : r);      // 255 marks an unusable cell for the next pass
  }
}
// AXIS 1: y, 2: z.  `in` holds the previous pass (255 = unusable cell), `out` the combined radius r of the
// all-usable box; the last pass writes the distance r + 1, and 0 for unusable cells.
template <int AXIS, bool LAST>
__global__ void k_clear_axis(const unsigned char* __restrict__ in, unsigned char* __restrict__ out, Geo g,
                             const int* __restrict__ gate) {
  if (gate && *gate == 0) return;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;; t += (long long)gridDim.x * blockDim.x) {
    int b, k, j, i;
    if (!clear_cell(g, t, b, k, j, i)) return;
    const int stride = AXIS == 1 ? g.nx : g.nx * g.ny;
    const int pos = AXIS == 1 ? j : k, ext = AXIS == 1 ? g.ny : g.nz;
    const int self = in[t];
    int r;
    if (self == 255) {
      r = LAST ? 0 : 255;
    } else {
      r = 0;
      int m = self;
      for (int d = 1; d <= kClearMax; d++) {
        if (pos - d < 0 || pos + d >= ext) break;
        const int a = in[t - d * stride], bb = in[t + d * stride];
        if (a == 255 || bb == 255) break;
        m = min(m, min(a, bb));
        if (m < d) break;
        r = d;
      }
      if (LAST) r += 1;
    }
    out[t] = (unsigned char)r;
  }
}
template <typename FT>
int launch_clearance(const FT* flags, unsigned char* clear, unsigned char* tmp, const Geo& g, const int* gate,
                     cudaStream_t st) {
  const long long total = g.n * g.nb;
  const int block = 256;
  const int grid = (int)std::min<long long>((total + block - 1) / block, 132 * 8);
  if (g.is3d) {                            // (a 3-D grid with fewer than 3 planes gets clearance 0)
    k_clear_x<FT><<<grid, block, 0, st>>>(flags, clear, g, gate);
    k_clear_axis<1, false><<<grid, block, 0, st>>>(clear, tmp, g, gate);
    k_clear_axis<2, true><<<grid, block, 0, st>>>(tmp, clear, g, gate);
    return 3;
  }
  k_clear_x<FT><<<grid, block, 0, st>>>(flags, tmp, g, gate);
  k_clear_axis<1, true><<<grid, block, 0, st>>>(tmp, clear, g, gate);
  return 2;
}
template int launch_clearance<float>(const float*, unsigned char*, unsigned char*, const Geo&, const int*, cudaStream_t);
template int launch_clearance<unsigned char>(const unsigned char*, unsigned char*, unsigned char*, const Geo&, const int*,
                                             cudaStream_t);

// float flags -> byte flags (once per fused step).  With `changed` the kernel also reports whether any
// byte differs from what the destination held (the step keeps its byte copy and the clearance field
// between calls and rebuilds the latter only then).
__global__ void k_flags_to_u8(const float* __restrict__ f, unsigned char* __restrict__ o, long long n,
                              int* __restrict__ changed) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const unsigned char v = (unsigned char)(((int)f[t]) & 0xFF);
  if (changed && o[t] != v) *changed = 1;
  o[t] = v;
}
// 16 cells per thread: four 16-byte loads, one 16-byte store.
__global__ void k_flags_to_u8_x16(const float4* __restrict__ f, uint4* __restrict__ o, long long n16,
                                  int* __restrict__ changed) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n16) return;
  unsigned w[4];
#pragma unroll
  for (int q = 0; q < 4; q++) {
    const float4 v = __ldg(f + 4 * t + q);
    w[q] = (unsigned)(((int)v.x) & 0xFF) | ((unsigned)(((int)v.y) & 0xFF) << 8) |
           ((unsigned)(((int)v.z) & 0xFF) << 16) | ((unsigned)(((int)v.w) & 0xFF) << 24);
  }
  if (changed) {
    const uint4 old = o[t];
    if (old.x != w[0] || old.y != w[1] || old.z != w[2] || old.w != w[3]) *changed = 1;
  }
  o[t] = make_uint4(w[0], w[1], w[2], w[3]);
}
void launch_flags_to_u8(const float* f, unsigned char* o, long long n, int* changed, cudaStream_t st) {
  if (n % 16 == 0 && ((size_t)f % 16) == 0 && ((size_t)o % 16) == 0) {
    const long long n16 = n / 16;
    k_flags_to_u8_x16<<<(unsigned)((n16 + 255) / 256), 256, 0, st>>>((const float4*)f, (uint4*)o, n16, changed);
    return;
  }
  k_flags_to_u8<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(f, o, n, changed);
}

}  // namespace tfl
