// Fused variants of the point-wise stages of tfluids.simulate (torch/lib/simulate.lua:175-327)
// used by tfl_simulate_step on the convnet path.  Each kernel performs, per cell and in the
// SAME floating-point order, what a run of separate operators / cutorch calls does in the
// reference loop, so results are bit-identical to the operator-by-operator sequence while
// the velocity / density fields cross HBM once instead of once per operator.
// Compiled with -fmad=false.  The fused step runs the 3-D tensor-core stack only, so these stages are
// 3-D kernels on the step's byte flags; the curl / force quads also serve the 2-D vorticity confinement.
//
//   k_post_advect        s:copy(tmp) ; U:copy(tmp)            (tfluids/init.lua:145-148, :215-218)
//                        setConstVals (U, density)            (lib/simulate.lua:202, :130-160)
//                        tfluids.addBuoyancy                  (lib/simulate.lua:216-226)
//   k_vort_bc_mask       vorticityConfinement's AddForceField (third_party/tfluids.cc:1312-1339)
//                        setConstVals (U)                     (lib/simulate.lua:252)
//                        tfluids.SetWallBcs mask multiply + the sums behind the input scale of the field
//                        normalizeInputChan names, U or pDiv  (lib/model.lua:81-117)
//   k_cnn_div_stats_fused the same sums of div(U1), normalizeInputChan 'div' (lib/model.lua:108-116)
//   k_cnn_inputs_fused   scale (std, 'norm' or 1), ApplyScale of the inputChannels set (pDiv, UDiv, div),
//                        VelocityDivergence, FlagsToOccupancy, into one or two float4 planes
//                                                             (lib/model.lua:86-150)
//   (launch_cnn_skip)    addPressureSkip, between the convolution stack and the finish (lib/model.lua:357-361)
//   k_cnn_finish_fused   VelocityUpdate, ApplyScale, SetWallBcs (lib/model.lua:380-390)
//                        setConstVals (U) ; U:clamp(-1e6, 1e6) (lib/simulate.lua:321, :326)
// The input block is a template argument of the kernels that depend on it, so the default block (pDiv, div,
// occupancy; std of U) compiles to the code it has on its own.
#include <initializer_list>
#include "tfl_device.cuh"
#include "tfl_kernels.h"

namespace tfl {

struct BcPtrs {
  const float* u_inv; const float* u_bc;        // may be null (no velocity BC)
  const float* d_inv; const float* d_bc;        // may be null (no density BC)
  // Quad kernels only, may be null: one byte per 4 cells, bit 0 = the velocity BC of the quad is the identity pair
  // (invMask bits == 1.0f and bc bits == +0.0f on all 4 cells of all channels), bit 1 = the same for the density
  // BC.  Such a quad applies x * 1.0f + 0.0f without loading the arrays (k_bc_quad_mask rebuilds the bytes every
  // step from the arrays themselves: nothing is assumed about the caller keeping them unchanged).
  const unsigned char* qmask;
};
// x * 1.0f is x; x + (+0.0f) is x except that it turns -0 into +0: kept, so that skipping the loads changes nothing.
__device__ __forceinline__ float bc_identity(float x) { return (x * 1.0f) + 0.0f; }

__device__ __forceinline__ float bc_apply(float x, const float* __restrict__ inv, const float* __restrict__ bc,
                                          long long o) {
  if (inv == nullptr) return x;
  const float t = x * __ldg(inv + o);
  return t + __ldg(bc + o);
}

// density = BC(tmp_s); U = BC(tmp_U) (+ buoyancy with the NEW density).
__global__ void k_post_advect(const float* __restrict__ tmp_s, const float* __restrict__ tmp_u,
                              const unsigned char* __restrict__ flags, float* __restrict__ density,
                              float* __restrict__ U, BcPtrs bc, int do_buoy, float sx, float sy_, float sz_,
                              Geo gin) {
  const Geo g = static_geo<true>(gin);
  int b, k, j, i;
  if (!thread_cell(g, b, k, j, i)) return;
  const int c = cell(g, k, j, i);
  const long long sb = b * g.n, ub = (long long)b * g.nc * g.n;
  float rc = 0.0f;
  if (density) {
    rc = bc_apply(__ldg(tmp_s + sb + c), bc.d_inv, bc.d_bc, sb + c);
    // The loop applies setConstVals to the density two more times before the step ends
    // (lib/simulate.lua:252, :321) and nothing else writes it: store the final value (equal to rc for
    // idempotent BCs such as the plume's), the buoyancy below reads the first application.
    density[sb + c] = bc_apply(bc_apply(rc, bc.d_inv, bc.d_bc, sb + c), bc.d_inv, bc.d_bc, sb + c);
  }
  float u[3];
  for (int a = 0; a < g.nc; a++) u[a] = bc_apply(__ldg(tmp_u + ub + a * g.n + c), bc.u_inv, bc.u_bc, ub + a * g.n + c);
  if (do_buoy && density && !on_border(g, k, j, i)) {
    const unsigned char* fl = flags + sb;
    if (flag_i(fl, g, k, j, i) & kFluid) {
      const int st[3] = {1, g.nx, g.nx * g.ny};
      const float str[3] = {sx, sy_, sz_};
      int fn[3];
      fn[0] = flag_i(fl, g, k, j, i - 1);
      fn[1] = flag_i(fl, g, k, j - 1, i);
      fn[2] = g.is3d ? flag_i(fl, g, k - 1, j, i) : 0;
      for (int a = 0; a < g.nc; a++) {
        if (fn[a] & kFluid) {
          const float rn = bc_apply(__ldg(tmp_s + sb + c - st[a]), bc.d_inv, bc.d_bc, sb + c - st[a]);
          u[a] += (0.5f * str[a] * (rc + rn));
        }
      }
    }
  }
  for (int a = 0; a < g.nc; a++) U[ub + a * g.n + c] = u[a];
}

// U += confinement force; U = BC(U); then (mask_mode 1) U *= wall mask and accumulate the
// sums for the input scale: of the masked U (STAT kCnnStatU), of p_div (kCnnStatPDiv), or none (kCnnStatNone).
// BATCH (nb > 1): the sums go to each thread's own entry (add_entry_sums); nb = 1 compiles without that branch.
template <bool BATCH, int STAT>
__global__ void k_vort_bc_mask(float* __restrict__ U, const unsigned char* __restrict__ flags,
                               const float* __restrict__ force, int do_vort, BcPtrs bc, int mask_mode,
                               double* __restrict__ sums, Geo gin, const float* __restrict__ p_div) {
  const Geo g = static_geo<true>(gin);
  int b, k, j, i;
  const bool live = thread_cell(g, b, k, j, i);
  double s = 0.0, ss = 0.0;
  if (live) {
    const int c = cell(g, k, j, i);
    const long long ub = (long long)b * g.nc * g.n;
    const unsigned char* fl = flags + b * g.n;
    float u[3];
    for (int a = 0; a < g.nc; a++) u[a] = U[ub + a * g.n + c];
    if (do_vort && !on_border(g, k, j, i)) {
      const int fc = flag_i(fl, g, k, j, i);
      const bool cf = fc & kFluid, ce = fc & kEmpty;
      if (cf || ce) {
        const float* fb = force + (long long)b * 3 * g.n;
        int f = flag_i(fl, g, k, j, i - 1);
        if ((f & kFluid) || (cf && (f & kEmpty))) u[0] += (0.5f * (__ldg(fb + c - 1) + __ldg(fb + c)));
        f = flag_i(fl, g, k, j - 1, i);
        if ((f & kFluid) || (cf && (f & kEmpty))) u[1] += (0.5f * (__ldg(fb + g.n + c - g.nx) + __ldg(fb + g.n + c)));
        if (g.is3d) {
          f = flag_i(fl, g, k - 1, j, i);
          if ((f & kFluid) || (cf && (f & kEmpty)))
            u[2] += (0.5f * (__ldg(fb + 2 * g.n + c - g.nx * g.ny) + __ldg(fb + 2 * g.n + c)));
        }
      }
    }
    for (int a = 0; a < g.nc; a++) u[a] = bc_apply(u[a], bc.u_inv, bc.u_bc, ub + a * g.n + c);
    if (mask_mode) {
      bool z[3];
      wall_bc_zero_mask(fl, g, k, j, i, z);
      for (int a = 0; a < g.nc; a++) {
        if (z[a]) u[a] = u[a] * 0.0f;
        if (STAT == kCnnStatU) {
          const float sq = u[a] * u[a];
          s += (double)u[a];
          ss += (double)sq;
        }
      }
      if (STAT == kCnnStatPDiv) {
        const float v = __ldg(p_div + b * g.n + c);
        const float sq = v * v;
        s += (double)v;
        ss += (double)sq;
      }
    }
    for (int a = 0; a < g.nc; a++) U[ub + a * g.n + c] = u[a];
  }
  if (STAT != kCnnStatNone && mask_mode) {
    if (BATCH) add_entry_sums(s, ss, sums, live, b, g);         // a block may straddle two entries
    else block_accumulate(s, ss, sums + 2 * (live ? b : 0));
  }
}

// tfluids.VelocityDivergence of U1 at cell c (flag f) of a 3-D grid.
__device__ __forceinline__ float fused_div(const float* __restrict__ ub, int f, const Geo& g, int k, int j, int i,
                                           int c) {
  float dv = 0.0f;
  if (!on_border(g, k, j, i) && (f & kFluid)) {
    dv = __ldg(ub + c) - __ldg(ub + c + 1) + __ldg(ub + g.n + c) - __ldg(ub + g.n + c + g.nx);
    if (g.is3d) dv += (__ldg(ub + 2 * g.n + c) - __ldg(ub + 2 * g.n + c + (long long)g.nx * g.ny));
  }
  return dv;
}

// normalizeInputChan 'div': sums[b] += (sum div(U1), sum div(U1)^2), k_cnn_div_stats on the step's byte flags, once
// k_vort_bc_mask has left U1 in U.
template <bool BATCH>
__global__ void k_cnn_div_stats_fused(const float* __restrict__ U1, const unsigned char* __restrict__ flags,
                                      double* __restrict__ sums, Geo gin) {
  const Geo g = static_geo<true>(gin);
  int b, k, j, i;
  const bool live = thread_cell(g, b, k, j, i);
  double s = 0.0, ss = 0.0;
  if (live) {
    const int c = cell(g, k, j, i);
    const float dv = fused_div(U1 + (long long)b * g.nc * g.n, flag_i(flags + b * g.n, g, k, j, i), g, k, j, i, c);
    const float sq = dv * dv;
    s += (double)dv;
    ss += (double)sq;
  }
  if (BATCH) add_entry_sums(s, ss, sums, live, b, g);
  else block_accumulate(s, ss, sums + 2 * (live ? b : 0));
}

// The input scale of entry b from the sums (k_cnn_scale's expressions): SCALE kFusedStdU (nn.StandardDeviation over
// the nc n values of U), kFusedStdN (over the n values of pDiv or div), kFusedNorm ('norm') or kFusedOne
// (normalizeInput off: exactly 1).
enum : int { kFusedStdU = 0, kFusedStdN = 1, kFusedNorm = 2, kFusedOne = 3 };
template <int SCALE>
__device__ __forceinline__ float fused_scale(const double* __restrict__ sums, int b, const Geo& g, float threshold) {
  if (SCALE == kFusedStdU) return scale_from_sums(sums, b, (long long)g.nc * g.n, threshold);
  if (SCALE == kFusedStdN) return scale_from_sums(sums, b, g.n, threshold);
  if (SCALE == kFusedNorm) {
    const float out = sqrtf((float)sums[2 * b + 1]);
    return (out < threshold) ? threshold : out;
  }
  return 1.0f;
}

// Channel `slot` of the input set SEL (kCnnIn* bits), of the values at one voxel: pDiv/s, U1/s (3), div/s, occupancy in
// that order (cnn_input_channels), then zeros up to 8.
template <int SEL, int SLOT>
__device__ __forceinline__ float input_channel(float p, float u0, float u1, float u2, float d, float occ) {
  constexpr int kU = (SEL & kCnnInPDiv) ? 1 : 0;
  constexpr int kD = kU + ((SEL & kCnnInUDiv) ? 3 : 0);
  constexpr int kOcc = kD + ((SEL & kCnnInDiv) ? 1 : 0);
  if constexpr ((SEL & kCnnInPDiv) && SLOT == 0) return p;
  else if constexpr ((SEL & kCnnInUDiv) && SLOT == kU) return u0;
  else if constexpr ((SEL & kCnnInUDiv) && SLOT == kU + 1) return u1;
  else if constexpr ((SEL & kCnnInUDiv) && SLOT == kU + 2) return u2;
  else if constexpr ((SEL & kCnnInDiv) && SLOT == kD) return d;
  else if constexpr (SLOT == kOcc) return occ;
  else return 0.0f;
}

// The conv input of the set SEL at one voxel, channels-last: channels 0-3 on the first float4 plane, 4-7 on the
// second (written only with UDiv), as k_cnn_inputs_padded lays them out.  U1 is the already masked velocity left in U
// by k_vort_bc_mask.
template <int SEL>
__device__ __forceinline__ void put_inputs(float4* __restrict__ x0, long long o, int v, long long plane, float pd,
                                           float u0, float u1, float u2, float dv, int f, float sc) {
  const float p = pd / sc, d = dv / sc;
  const float occ = (f == kFluid) ? 0.0f : ((f == kObstacle) ? 1.0f : -1.0f);
  float us[3] = {0.0f, 0.0f, 0.0f};
  if (SEL & kCnnInUDiv) {
    us[0] = u0 / sc;
    us[1] = u1 / sc;
    us[2] = u2 / sc;
  }
#define TFL_CHANNEL(q) input_channel<SEL, q>(p, us[0], us[1], us[2], d, occ)
  x0[o + v] = make_float4(TFL_CHANNEL(0), TFL_CHANNEL(1), TFL_CHANNEL(2), TFL_CHANNEL(3));
  if (SEL & kCnnInUDiv) x0[o + v + plane] = make_float4(TFL_CHANNEL(4), TFL_CHANNEL(5), TFL_CHANNEL(6), TFL_CHANNEL(7));
#undef TFL_CHANNEL
}

template <int SEL, int SCALE>
__global__ void k_cnn_inputs_fused(const float* __restrict__ p_div, const float* __restrict__ U1,
                                   const unsigned char* __restrict__ flags, const double* __restrict__ sums,
                                   float threshold, float* __restrict__ scale_out, float4* __restrict__ x0,
                                   int px, int py, Geo gin) {
  const Geo g = static_geo<true>(gin);
  int b, k, j, i;
  if (!thread_cell(g, b, k, j, i)) return;
  const int c = cell(g, k, j, i);
  const float sc = fused_scale<SCALE>(sums, b, g, threshold);
  if (c == 0) scale_out[b] = sc;
  const float* ub = U1 + (long long)b * g.nc * g.n;
  const int f = flag_i(flags + b * g.n, g, k, j, i);
  const float dv = fused_div(ub, f, g, k, j, i, c);
  const long long plane = (long long)(g.nz + 2) * py * px;
  const long long o = (long long)b * 2 * plane + ((long long)(k + 1) * py + (j + 1)) * px + (i + 1);
  float u[3] = {0.0f, 0.0f, 0.0f};
  if (SEL & kCnnInUDiv)
    for (int a = 0; a < 3; a++) u[a] = __ldg(ub + a * g.n + c);
  put_inputs<SEL>(x0, o, 0, plane, (SEL & kCnnInPDiv) ? __ldg(p_div + b * g.n + c) : 0.0f, u[0], u[1], u[2], dv, f, sc);
}

// U = clamp(BC(setWallBcs(velocityUpdate(U1 / s, p_net) * s)));  p = p_net * s.  In place on U.
__global__ void k_cnn_finish_fused(const float* __restrict__ p_net, float* __restrict__ U,
                                   const unsigned char* __restrict__ flags, const float* __restrict__ scale,
                                   float* __restrict__ p_out, BcPtrs bc, float lo, float hi, Geo gin) {
  const Geo g = static_geo<true>(gin);
  int b, k, j, i;
  if (!thread_cell(g, b, k, j, i)) return;
  const int c = cell(g, k, j, i);
  const float sc = __ldg(scale + b);
  const unsigned char* fl = flags + b * g.n;
  const float* pb = p_net + b * g.n;
  const long long ub = (long long)b * g.nc * g.n;
  const float pc = __ldg(pb + c);
  float u[3];
  for (int a = 0; a < g.nc; a++) u[a] = U[ub + a * g.n + c] / sc;
  if (!on_border(g, k, j, i)) {
    const int st[3] = {1, g.nx, g.nx * g.ny};
    const int fc = flag_i(fl, g, k, j, i);
    int fn[3];
    fn[0] = flag_i(fl, g, k, j, i - 1);
    fn[1] = flag_i(fl, g, k, j - 1, i);
    fn[2] = g.is3d ? flag_i(fl, g, k - 1, j, i) : 0;
    if (fc & kFluid) {
      for (int a = 0; a < g.nc; a++) {
        if (fn[a] & kFluid) u[a] -= (pc - __ldg(pb + c - st[a]));
        if (fn[a] & kEmpty) u[a] -= pc;
      }
    } else if ((fc & kEmpty) && !(fc & kOutflow)) {
      for (int a = 0; a < g.nc; a++) {
        if (fn[a] & kFluid) u[a] += __ldg(pb + c - st[a]);
        else u[a] = 0.0f;
      }
    }
  }
  bool z[3];
  wall_bc_zero_mask(fl, g, k, j, i, z);
  for (int a = 0; a < g.nc; a++) {
    float v = u[a] * sc;
    if (z[a]) v = v * 0.0f;
    v = bc_apply(v, bc.u_inv, bc.u_bc, ub + a * g.n + c);
    v = (v < lo) ? lo : ((v > hi) ? hi : v);
    U[ub + a * g.n + c] = v;
  }
  p_out[b * g.n + c] = pc * sc;
}

// ---------------------------------------------------------------------------------------
// Four voxels along x per thread (rows with nx % 4 == 0): the same per-voxel arithmetic as the
// kernels above, in the same order, behind 16-byte loads / stores and one flag word per row --
// these stages are bound by instruction issue and load latency, not by HBM bandwidth, so fewer,
// wider memory instructions and fewer index computations per voxel are what pays.
// ---------------------------------------------------------------------------------------
struct Flags4 { int c[4]; };
__device__ __forceinline__ Flags4 flags4(const unsigned char* __restrict__ p, bool valid) {
  Flags4 f;
  if (valid) {
    const uchar4 v = __ldg(reinterpret_cast<const uchar4*>(p));
    f.c[0] = v.x; f.c[1] = v.y; f.c[2] = v.z; f.c[3] = v.w;
  } else {
    f.c[0] = f.c[1] = f.c[2] = f.c[3] = 0;
  }
  return f;
}
__device__ __forceinline__ void ld4(const float* __restrict__ p, float (&o)[4]) {
  const float4 v = __ldg(reinterpret_cast<const float4*>(p));
  o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
}
__device__ __forceinline__ void ld4_rw(const float* p, float (&o)[4]) {      // data this kernel also writes
  const float4 v = *reinterpret_cast<const float4*>(p);
  o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
}
__device__ __forceinline__ void st4(float* p, const float (&v)[4]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}
__device__ __forceinline__ void zero4(float (&o)[4]) { o[0] = o[1] = o[2] = o[3] = 0.0f; }

// wall_bc_zero_mask (tfl_device.cuh) on flag values of a 3-D grid; a neighbour outside the grid is passed as 0.
__device__ __forceinline__ void wall_mask_from_flags(int fc, int fxm, int fxp, int fym, int fyp, int fzm, int fzp,
                                                     bool z[3]) {
  z[0] = z[1] = z[2] = false;
  const bool cf = fc & kFluid, co = fc & kObstacle;
  if (!cf && !co) return;
  if ((fxm & kObstacle) || (co && (fxm & kFluid))) z[0] = true;
  if ((fym & kObstacle) || (co && (fym & kFluid))) z[1] = true;
  if ((fzm & kObstacle) || (co && (fzm & kFluid))) z[2] = true;
  if (cf) {
    if ((fxm & kStick) || (fxp & kStick)) { z[1] = true; z[2] = true; }
    if ((fym & kStick) || (fyp & kStick)) { z[0] = true; z[2] = true; }
    if ((fzm & kStick) || (fzp & kStick)) { z[0] = true; z[1] = true; }
  }
}

// (b, k, j, i0 .. i0 + 3) of this thread.  The fused step never runs on a slab (zlo = 0, zhi = nz).
__device__ __forceinline__ bool thread_cell4(const Geo& g, int& b, int& k, int& j, int& i0) {
  i0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  j = blockIdx.y * blockDim.y + threadIdx.y;
  const int zz = blockIdx.z * blockDim.z + threadIdx.z;
  b = zz / g.nz;
  k = zz - b * g.nz;
  return i0 < g.nx && j < g.ny && b < g.nb;
}

// The flag values around a quad of a 3-D grid: centre row, the scalars left / right of it, and the four rows around.
struct QuadFlags {
  Flags4 c, ym, yp, zm, zp;
  int left, right;
  __device__ __forceinline__ int xm(int v) const { return v == 0 ? left : c.c[v - 1]; }
  __device__ __forceinline__ int xp(int v) const { return v == 3 ? right : c.c[v + 1]; }
};
__device__ __forceinline__ QuadFlags quad_flags(const unsigned char* __restrict__ fl, const Geo& g, int c0, int k, int j,
                                                int i0, bool need_plus) {
  QuadFlags q;
  const int sy = g.nx, sz = g.nx * g.ny;
  q.c = flags4(fl + c0, true);
  q.left = i0 > 0 ? (int)__ldg(fl + c0 - 1) : 0;
  q.ym = flags4(fl + c0 - sy, j > 0);
  q.zm = flags4(fl + c0 - sz, k > 0);
  q.right = (need_plus && i0 + 4 < g.nx) ? (int)__ldg(fl + c0 + 4) : 0;
  q.yp = flags4(fl + c0 + sy, need_plus && j < g.ny - 1);
  q.zp = flags4(fl + c0 + sz, need_plus && k < g.nz - 1);
  return q;
}

__global__ void __launch_bounds__(256) k_post_advect4(const float* __restrict__ tmp_s, const float* __restrict__ tmp_u,
                                                      const unsigned char* __restrict__ flags, float* __restrict__ density,
                                                      float* __restrict__ U, BcPtrs bc, int do_buoy, float sx, float sy_,
                                                      float sz_, Geo gin) {
  const Geo g = static_geo<true>(gin);
  int b, k, j, i0;
  if (!thread_cell4(g, b, k, j, i0)) return;
  const int c0 = cell(g, k, j, i0);
  const int sy = g.nx, sz = g.nx * g.ny;
  const long long sb = b * g.n, ub = (long long)b * g.nc * g.n;
  float rc[4];
  zero4(rc);
  auto quad_bits = [&](long long o) { return bc.qmask ? (int)__ldg(bc.qmask + (o >> 2)) : 0; };
  const int qm = quad_bits(sb + c0);
  auto dens_bc = [&](long long o, float (&out)[4]) {          // BC(tmp_s) of the quad at offset o
    ld4(tmp_s + o, out);
    if (bc.d_inv) {
      if (quad_bits(o) & 2) {
#pragma unroll
        for (int v = 0; v < 4; v++) out[v] = bc_identity(out[v]);
        return;
      }
      float iv[4], bv[4];
      ld4(bc.d_inv + o, iv);
      ld4(bc.d_bc + o, bv);
#pragma unroll
      for (int v = 0; v < 4; v++) { const float t = out[v] * iv[v]; out[v] = t + bv[v]; }
    }
  };
  if (density) {
    dens_bc(sb + c0, rc);
    float fin[4] = {rc[0], rc[1], rc[2], rc[3]};
    if (bc.d_inv) {        // second and third setConstVals of the step (lib/simulate.lua:252, :321)
      if (qm & 2) {
#pragma unroll
        for (int v = 0; v < 4; v++) fin[v] = bc_identity(bc_identity(fin[v]));
      } else {
        float iv[4], bv[4];
        ld4(bc.d_inv + sb + c0, iv);
        ld4(bc.d_bc + sb + c0, bv);
#pragma unroll
        for (int v = 0; v < 4; v++) {
          float t = fin[v] * iv[v];
          t = t + bv[v];
          t = t * iv[v];
          fin[v] = t + bv[v];
        }
      }
    }
    st4(density + sb + c0, fin);
  }
  float u[3][4];
#pragma unroll
  for (int a = 0; a < 3; a++) {
    if (a < g.nc) {
      ld4(tmp_u + ub + a * g.n + c0, u[a]);
      if (bc.u_inv) {
        if (qm & 1) {
#pragma unroll
          for (int v = 0; v < 4; v++) u[a][v] = bc_identity(u[a][v]);
        } else {
          float iv[4], bv[4];
          ld4(bc.u_inv + ub + a * g.n + c0, iv);
          ld4(bc.u_bc + ub + a * g.n + c0, bv);
#pragma unroll
          for (int v = 0; v < 4; v++) { const float t = u[a][v] * iv[v]; u[a][v] = t + bv[v]; }
        }
      }
    }
  }
  if (do_buoy && density) {
    const QuadFlags q = quad_flags(flags + sb, g, c0, k, j, i0, false);
    // density (after its BC) of the -x / -y / -z neighbours
    float rl = 0.0f, ry[4], rz[4];
    zero4(ry); zero4(rz);
    if (i0 > 0) {
      rl = __ldg(tmp_s + sb + c0 - 1);
      if (bc.d_inv) {
        if (quad_bits(sb + c0 - 4) & 2) rl = bc_identity(rl);
        else { const float t = rl * __ldg(bc.d_inv + sb + c0 - 1); rl = t + __ldg(bc.d_bc + sb + c0 - 1); }
      }
    }
    if (j > 0) dens_bc(sb + c0 - sy, ry);
    if (k > 0) dens_bc(sb + c0 - sz, rz);
#pragma unroll
    for (int v = 0; v < 4; v++) {
      if (on_border(g, k, j, i0 + v) || !(q.c.c[v] & kFluid)) continue;
      if (q.xm(v) & kFluid) u[0][v] += (0.5f * sx * (rc[v] + (v == 0 ? rl : rc[v - 1])));
      if (q.ym.c[v] & kFluid) u[1][v] += (0.5f * sy_ * (rc[v] + ry[v]));
      if (q.zm.c[v] & kFluid) u[2][v] += (0.5f * sz_ * (rc[v] + rz[v]));
    }
  }
#pragma unroll
  for (int a = 0; a < 3; a++) if (a < g.nc) st4(U + ub + a * g.n + c0, u[a]);
}

template <bool BATCH, int STAT>
__global__ void __launch_bounds__(256) k_vort_bc_mask4(float* __restrict__ U, const unsigned char* __restrict__ flags,
                                                       const float* __restrict__ force, int do_vort, BcPtrs bc,
                                                       int mask_mode, double* __restrict__ sums, Geo gin,
                                                       const float* __restrict__ p_div) {
  const Geo g = static_geo<true>(gin);
  int b, k, j, i0;
  const bool live = thread_cell4(g, b, k, j, i0);
  double s = 0.0, ss = 0.0;
  if (live) {
    const int c0 = cell(g, k, j, i0);
    const int sy = g.nx, sz = g.nx * g.ny;
    const long long ub = (long long)b * g.nc * g.n;
    const QuadFlags q = quad_flags(flags + b * g.n, g, c0, k, j, i0, mask_mode != 0);
    float u[3][4];
#pragma unroll
    for (int a = 0; a < 3; a++) if (a < g.nc) ld4_rw(U + ub + a * g.n + c0, u[a]);
    if (do_vort) {
      const float* fb = force + (long long)b * 3 * g.n;
      float fx[4], fy[4], fyl[4], fz[4], fzl[4];
      ld4(fb + c0, fx);
      const float fxl = i0 > 0 ? __ldg(fb + c0 - 1) : 0.0f;
      ld4(fb + g.n + c0, fy);
      zero4(fyl); zero4(fz); zero4(fzl);
      if (j > 0) ld4(fb + g.n + c0 - sy, fyl);
      ld4(fb + 2 * g.n + c0, fz);
      if (k > 0) ld4(fb + 2 * g.n + c0 - sz, fzl);
#pragma unroll
      for (int v = 0; v < 4; v++) {
        if (on_border(g, k, j, i0 + v)) continue;
        const int fc = q.c.c[v];
        const bool cf = fc & kFluid, ce = fc & kEmpty;
        if (!(cf || ce)) continue;
        int f = q.xm(v);
        if ((f & kFluid) || (cf && (f & kEmpty))) u[0][v] += (0.5f * ((v == 0 ? fxl : fx[v - 1]) + fx[v]));
        f = q.ym.c[v];
        if ((f & kFluid) || (cf && (f & kEmpty))) u[1][v] += (0.5f * (fyl[v] + fy[v]));
        f = q.zm.c[v];
        if ((f & kFluid) || (cf && (f & kEmpty))) u[2][v] += (0.5f * (fzl[v] + fz[v]));
      }
    }
    if (bc.u_inv) {
      const bool identity = bc.qmask && (__ldg(bc.qmask + ((b * g.n + c0) >> 2)) & 1);
#pragma unroll
      for (int a = 0; a < 3; a++) {
        if (a < g.nc) {
          if (identity) {
#pragma unroll
            for (int v = 0; v < 4; v++) u[a][v] = bc_identity(u[a][v]);
          } else {
            float iv[4], bv[4];
            ld4(bc.u_inv + ub + a * g.n + c0, iv);
            ld4(bc.u_bc + ub + a * g.n + c0, bv);
#pragma unroll
            for (int v = 0; v < 4; v++) { const float t = u[a][v] * iv[v]; u[a][v] = t + bv[v]; }
          }
        }
      }
    }
    if (mask_mode) {
      float pd[4];
      if (STAT == kCnnStatPDiv) ld4(p_div + b * g.n + c0, pd);
#pragma unroll
      for (int v = 0; v < 4; v++) {
        bool z[3];
        wall_mask_from_flags(q.c.c[v], q.xm(v), q.xp(v), q.ym.c[v], q.yp.c[v], q.zm.c[v], q.zp.c[v], z);
#pragma unroll
        for (int a = 0; a < 3; a++) {
          if (a < g.nc) {
            if (z[a]) u[a][v] = u[a][v] * 0.0f;
            if (STAT == kCnnStatU) {
              const float sq = u[a][v] * u[a][v];
              s += (double)u[a][v];
              ss += (double)sq;
            }
          }
        }
        if (STAT == kCnnStatPDiv) {
          const float sq = pd[v] * pd[v];
          s += (double)pd[v];
          ss += (double)sq;
        }
      }
    }
#pragma unroll
    for (int a = 0; a < 3; a++) if (a < g.nc) st4(U + ub + a * g.n + c0, u[a]);
  }
  if (STAT != kCnnStatNone && mask_mode) {
    if (BATCH) add_entry_sums(s, ss, sums, live, b, g);         // thread_cell4's z range is [0, nz), as thread_cell's
    else block_accumulate(s, ss, sums + 2 * (live ? b : 0));
  }
}

// U1 around a quad of a 3-D grid: the x / y / z components of the quad, the x component right of it and the y / z
// components one row / plane up (0 outside the grid).
struct QuadU {
  float ux[4], uy[4], uyp[4], uz[4], uzp[4], uxr;
};
__device__ __forceinline__ QuadU quad_u(const float* __restrict__ ub, const Geo& g, int c0, int k, int j, int i0) {
  const int sy = g.nx, sz = g.nx * g.ny;
  QuadU q;
  ld4(ub + c0, q.ux);
  q.uxr = i0 + 4 < g.nx ? __ldg(ub + c0 + 4) : 0.0f;
  ld4(ub + g.n + c0, q.uy);
  zero4(q.uyp); zero4(q.uz); zero4(q.uzp);
  if (j < g.ny - 1) ld4(ub + g.n + c0 + sy, q.uyp);
  ld4(ub + 2 * g.n + c0, q.uz);
  if (k < g.nz - 1) ld4(ub + 2 * g.n + c0 + sz, q.uzp);
  return q;
}
// tfluids.VelocityDivergence at voxel v of the quad (flag f).
__device__ __forceinline__ float quad_div(const QuadU& q, int f, const Geo& g, int k, int j, int i0, int v) {
  float dv = 0.0f;
  if (!on_border(g, k, j, i0 + v) && (f & kFluid)) {
    dv = q.ux[v] - (v == 3 ? q.uxr : q.ux[v + 1]) + q.uy[v] - q.uyp[v];
    dv += (q.uz[v] - q.uzp[v]);
  }
  return dv;
}

template <bool BATCH>
__global__ void __launch_bounds__(256) k_cnn_div_stats_fused4(const float* __restrict__ U1,
                                                              const unsigned char* __restrict__ flags,
                                                              double* __restrict__ sums, Geo gin) {
  const Geo g = static_geo<true>(gin);
  int b, k, j, i0;
  const bool live = thread_cell4(g, b, k, j, i0);
  double s = 0.0, ss = 0.0;
  if (live) {
    const int c0 = cell(g, k, j, i0);
    const Flags4 fc = flags4(flags + b * g.n + c0, true);
    const QuadU q = quad_u(U1 + (long long)b * g.nc * g.n, g, c0, k, j, i0);
#pragma unroll
    for (int v = 0; v < 4; v++) {
      const float dv = quad_div(q, fc.c[v], g, k, j, i0, v);
      const float sq = dv * dv;
      s += (double)dv;
      ss += (double)sq;
    }
  }
  if (BATCH) add_entry_sums(s, ss, sums, live, b, g);
  else block_accumulate(s, ss, sums + 2 * (live ? b : 0));
}

template <int SEL, int SCALE>
__global__ void __launch_bounds__(256) k_cnn_inputs_fused4(const float* __restrict__ p_div, const float* __restrict__ U1,
                                                           const unsigned char* __restrict__ flags,
                                                           const double* __restrict__ sums, float threshold,
                                                           float* __restrict__ scale_out, float4* __restrict__ x0, int px,
                                                           int py, Geo gin) {
  const Geo g = static_geo<true>(gin);
  int b, k, j, i0;
  if (!thread_cell4(g, b, k, j, i0)) return;
  const int c0 = cell(g, k, j, i0);
  const float sc = fused_scale<SCALE>(sums, b, g, threshold);
  if (c0 == 0) scale_out[b] = sc;
  const float* ub = U1 + (long long)b * g.nc * g.n;
  const Flags4 fc = flags4(flags + b * g.n + c0, true);
  const QuadU q = quad_u(ub, g, c0, k, j, i0);
  float pd[4];
  if (SEL & kCnnInPDiv) ld4(p_div + b * g.n + c0, pd);
  else zero4(pd);
  const long long plane = (long long)(g.nz + 2) * py * px;
  const long long o = (long long)b * 2 * plane + ((long long)(k + 1) * py + (j + 1)) * px + (i0 + 1);
#pragma unroll
  for (int v = 0; v < 4; v++) {
    const int f = fc.c[v];
    float dv = 0.0f;
    if (!on_border(g, k, j, i0 + v) && (f & kFluid)) {
      dv = q.ux[v] - (v == 3 ? q.uxr : q.ux[v + 1]) + q.uy[v] - q.uyp[v];
      dv += (q.uz[v] - q.uzp[v]);
    }
    put_inputs<SEL>(x0, o, v, plane, pd[v], q.ux[v], q.uy[v], q.uz[v], dv, f, sc);
  }
}

__global__ void __launch_bounds__(256) k_cnn_finish_fused4(const float* __restrict__ p_net, float* __restrict__ U,
                                                           const unsigned char* __restrict__ flags,
                                                           const float* __restrict__ scale, float* __restrict__ p_out,
                                                           BcPtrs bc, float lo, float hi, Geo gin) {
  const Geo g = static_geo<true>(gin);
  int b, k, j, i0;
  if (!thread_cell4(g, b, k, j, i0)) return;
  const int c0 = cell(g, k, j, i0);
  const int sy = g.nx, sz = g.nx * g.ny;
  const float sc = __ldg(scale + b);
  const float* pb = p_net + b * g.n;
  const long long ub = (long long)b * g.nc * g.n;
  const QuadFlags q = quad_flags(flags + b * g.n, g, c0, k, j, i0, true);
  float pc[4], py_[4], pz[4];
  ld4(pb + c0, pc);
  const float pl = i0 > 0 ? __ldg(pb + c0 - 1) : 0.0f;
  zero4(py_); zero4(pz);
  if (j > 0) ld4(pb + c0 - sy, py_);
  if (k > 0) ld4(pb + c0 - sz, pz);
  float u[3][4];
#pragma unroll
  for (int a = 0; a < 3; a++) {
    if (a < g.nc) {
      ld4_rw(U + ub + a * g.n + c0, u[a]);
#pragma unroll
      for (int v = 0; v < 4; v++) u[a][v] = u[a][v] / sc;
    }
  }
#pragma unroll
  for (int v = 0; v < 4; v++) {
    if (on_border(g, k, j, i0 + v)) continue;
    const int fc = q.c.c[v];
    const int fn[3] = {q.xm(v), q.ym.c[v], q.zm.c[v]};
    const float pn[3] = {v == 0 ? pl : pc[v - 1], py_[v], pz[v]};
    if (fc & kFluid) {
#pragma unroll
      for (int a = 0; a < 3; a++) {
        if (a < g.nc) {
          if (fn[a] & kFluid) u[a][v] -= (pc[v] - pn[a]);
          if (fn[a] & kEmpty) u[a][v] -= pc[v];
        }
      }
    } else if ((fc & kEmpty) && !(fc & kOutflow)) {
#pragma unroll
      for (int a = 0; a < 3; a++) {
        if (a < g.nc) {
          if (fn[a] & kFluid) u[a][v] += pn[a];
          else u[a][v] = 0.0f;
        }
      }
    }
  }
  bool z[4][3];
#pragma unroll
  for (int v = 0; v < 4; v++)
    wall_mask_from_flags(q.c.c[v], q.xm(v), q.xp(v), q.ym.c[v], q.yp.c[v], q.zm.c[v], q.zp.c[v], z[v]);
  const bool bc_identity_quad = bc.qmask && (__ldg(bc.qmask + ((b * g.n + c0) >> 2)) & 1);
#pragma unroll
  for (int a = 0; a < 3; a++) {
    if (a < g.nc) {
      float iv[4] = {1.0f, 1.0f, 1.0f, 1.0f}, bv[4] = {0.0f, 0.0f, 0.0f, 0.0f};
      if (bc.u_inv && !bc_identity_quad) {            // an identity quad keeps iv = 1, bv = +0: same operations below
        ld4(bc.u_inv + ub + a * g.n + c0, iv);
        ld4(bc.u_bc + ub + a * g.n + c0, bv);
      }
#pragma unroll
      for (int v = 0; v < 4; v++) {
        float w = u[a][v] * sc;
        if (z[v][a]) w = w * 0.0f;
        if (bc.u_inv) { const float t = w * iv[v]; w = t + bv[v]; }
        w = (w < lo) ? lo : ((w > hi) ? hi : w);
        u[a][v] = w;
      }
      st4(U + ub + a * g.n + c0, u[a]);
    }
  }
  float po[4];
#pragma unroll
  for (int v = 0; v < 4; v++) po[v] = pc[v] * sc;
  st4(p_out + b * g.n + c0, po);
}

// Six values of a row around a quad: x = i0 - 1 .. i0 + 4 (0 where the row or the cell is outside the grid).
__device__ __forceinline__ void row6(const float* __restrict__ p, bool row_ok, bool has_left, bool has_right,
                                     float (&o)[6]) {
  if (!row_ok) { o[0] = o[1] = o[2] = o[3] = o[4] = o[5] = 0.0f; return; }
  const float4 v = __ldg(reinterpret_cast<const float4*>(p));
  o[0] = has_left ? __ldg(p - 1) : 0.0f;
  o[1] = v.x; o[2] = v.y; o[3] = v.z; o[4] = v.w;
  o[5] = has_right ? __ldg(p + 4) : 0.0f;
}

// k_vort_curl for a quad: curl of the cell-centred velocity (GetCentered + GetCurl,
// third_party/tfluids.cc:1342-1409) with the centred velocity of border cells taken as zero.
template <bool IS3D>
__global__ void __launch_bounds__(256) k_vort_curl4(const float* __restrict__ U, float* __restrict__ curl,
                                                    float* __restrict__ cnorm, Geo gin) {
  const Geo g = static_geo<IS3D>(gin);
  int b, k, j, i0;
  if (!thread_cell4(g, b, k, j, i0)) return;
  const int c0 = cell(g, k, j, i0);
  const int sy = g.nx, sz = g.nx * g.ny;
  const float* ux = U + (long long)b * g.nc * g.n + c0;
  const float* uy = ux + g.n;
  const float* uz = ux + 2 * g.n;                       // only dereferenced in 3-D
  float wx[4], wy[4], wz[4], nr[4];
  zero4(wx); zero4(wy); zero4(wz); zero4(nr);
  const bool row_interior = j >= 1 && j <= g.ny - 2 && (!IS3D || (k >= 1 && k <= g.nz - 2));
  if (row_interior) {
    const bool hl = i0 > 0, hr = i0 + 4 < g.nx;
    // centred y (and z) velocity along this row, x = i0 - 1 .. i0 + 4
    float a[6], bb[6], cy[6], cz[6];
    row6(uy, true, hl, hr, a);
    row6(uy + sy, true, hl, hr, bb);
#pragma unroll
    for (int t = 0; t < 6; t++) cy[t] = 0.5f * (a[t] + bb[t]);
    if (IS3D) {
      row6(uz, true, hl, hr, a);
      row6(uz + sz, true, hl, hr, bb);
#pragma unroll
      for (int t = 0; t < 6; t++) cz[t] = 0.5f * (a[t] + bb[t]);
    }
    // centred x velocity on the rows j +- 1 (and k +- 1), x = i0 .. i0 + 3; zero if that row is a border row
    const bool yp_ok = j + 1 <= g.ny - 2, ym_ok = j - 1 >= 1;
    const bool zp_ok = IS3D && k + 1 <= g.nz - 2, zm_ok = IS3D && k - 1 >= 1;
    float cx_yp[4], cx_ym[4], cx_zp[4], cx_zm[4], cz_yp[4], cz_ym[4], cy_zp[4], cy_zm[4];
    auto centred_x = [&](const float* row, bool ok, float (&o)[4]) {
      float r6[6];
      row6(row, ok, false, hr, r6);                     // r6[1..5] = x = i0 .. i0 + 4
#pragma unroll
      for (int v = 0; v < 4; v++) o[v] = ok ? 0.5f * (r6[1 + v] + r6[2 + v]) : 0.0f;
    };
    auto centred_2rows = [&](const float* r0, const float* r1, bool ok, float (&o)[4]) {
      float p[4], q[4];
      if (ok) { ld4(r0, p); ld4(r1, q); } else { zero4(p); zero4(q); }
#pragma unroll
      for (int v = 0; v < 4; v++) o[v] = ok ? 0.5f * (p[v] + q[v]) : 0.0f;
    };
    centred_x(ux + sy, yp_ok, cx_yp);
    centred_x(ux - sy, ym_ok, cx_ym);
    if (IS3D) {
      centred_x(ux + sz, zp_ok, cx_zp);
      centred_x(ux - sz, zm_ok, cx_zm);
      centred_2rows(uz + sy, uz + sy + sz, yp_ok, cz_yp);
      centred_2rows(uz - sy, uz - sy + sz, ym_ok, cz_ym);
      centred_2rows(uy + sz, uy + sz + sy, zp_ok, cy_zp);
      centred_2rows(uy - sz, uy - sz + sy, zm_ok, cy_zm);
    }
#pragma unroll
    for (int v = 0; v < 4; v++) {
      const int i = i0 + v;
      if (i < 1 || i > g.nx - 2) continue;
      const bool xp_ok = i + 1 <= g.nx - 2, xm_ok = i - 1 >= 1;
      const float xp_y = xp_ok ? cy[v + 2] : 0.0f, xm_y = xm_ok ? cy[v] : 0.0f;
      V3 w = {0.0f, 0.0f, 0.0f};
      w.z = 0.5f * ((xp_y - xm_y) - (cx_yp[v] - cx_ym[v]));
      if (IS3D) {
        const float xp_z = xp_ok ? cz[v + 2] : 0.0f, xm_z = xm_ok ? cz[v] : 0.0f;
        w.x = 0.5f * ((cz_yp[v] - cz_ym[v]) - (cy_zp[v] - cy_zm[v]));
        w.y = 0.5f * ((cx_zp[v] - cx_zm[v]) - (xp_z - xm_z));
      }
      wx[v] = w.x; wy[v] = w.y; wz[v] = w.z;
      nr[v] = norm3(w);
    }
  }
  float* cb = curl + (long long)b * 3 * g.n + c0;
  st4(cb, wx); st4(cb + g.n, wy); st4(cb + 2 * g.n, wz);
  st4(cnorm + b * g.n + c0, nr);
}

// k_vort_force for a quad (conf_force of tfl_device.cuh, same arithmetic).
template <bool IS3D>
__global__ void __launch_bounds__(256) k_vort_force4(const float* __restrict__ curl, const float* __restrict__ cnorm,
                                                     float* __restrict__ force, float strength, Geo gin) {
  const Geo g = static_geo<IS3D>(gin);
  int b, k, j, i0;
  if (!thread_cell4(g, b, k, j, i0)) return;
  const int c0 = cell(g, k, j, i0);
  const int sy = g.nx, sz = g.nx * g.ny;
  const float* cn = cnorm + b * g.n + c0;
  const float* cb = curl + (long long)b * 3 * g.n + c0;
  float fx[4], fy[4], fz[4];
  zero4(fx); zero4(fy); zero4(fz);
  const bool row_interior = j >= 1 && j <= g.ny - 2 && (!IS3D || (k >= 1 && k <= g.nz - 2));
  if (row_interior) {
    float n6[6], nyp[4], nym[4], nzp[4], nzm[4], w0[4], w1[4], w2[4];
    row6(cn, true, i0 > 0, i0 + 4 < g.nx, n6);
    ld4(cn + sy, nyp); ld4(cn - sy, nym);
    zero4(nzp); zero4(nzm);
    if (IS3D) { ld4(cn + sz, nzp); ld4(cn - sz, nzm); }
    ld4(cb, w0); ld4(cb + g.n, w1); ld4(cb + 2 * g.n, w2);
#pragma unroll
    for (int v = 0; v < 4; v++) {
      const int i = i0 + v;
      if (i < 1 || i > g.nx - 2) continue;
      V3 gr = {0.0f, 0.0f, 0.0f};
      gr.x = 0.5f * (n6[v + 2] - n6[v]);
      gr.y = 0.5f * (nyp[v] - nym[v]);
      if (IS3D) gr.z = 0.5f * (nzp[v] - nzm[v]);
      const float gn = norm3(gr);
      if (gn > 1e-6f) { gr.x /= gn; gr.y /= gn; gr.z /= gn; } else { gr.x = gr.y = gr.z = 0.0f; }
      const V3 w = {w0[v], w1[v], w2[v]};
      fx[v] = ((gr.y * w.z) - (gr.z * w.y)) * strength;
      fy[v] = ((gr.z * w.x) - (gr.x * w.z)) * strength;
      fz[v] = ((gr.x * w.y) - (gr.y * w.x)) * strength;
    }
  }
  float* fb = force + (long long)b * 3 * g.n + c0;
  st4(fb, fx); st4(fb + g.n, fy); st4(fb + 2 * g.n, fz);
}

// One byte per quad: which BCs are the identity pair there (see BcPtrs::qmask).
__global__ void __launch_bounds__(256) k_bc_quad_mask(const float* __restrict__ u_inv, const float* __restrict__ u_bc,
                                                      const float* __restrict__ d_inv, const float* __restrict__ d_bc,
                                                      unsigned char* __restrict__ qmask, Geo gin) {
  const Geo g = static_geo<true>(gin);
  int b, k, j, i0;
  if (!thread_cell4(g, b, k, j, i0)) return;
  const long long o = b * g.n + cell(g, k, j, i0);
  const long long ub = (long long)b * g.nc * g.n + cell(g, k, j, i0);
  auto identity = [](const float* inv, const float* bcv) {
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(inv));
    const uint4 c = __ldg(reinterpret_cast<const uint4*>(bcv));
    const unsigned one = 0x3f800000u;
    return a.x == one && a.y == one && a.z == one && a.w == one && (c.x | c.y | c.z | c.w) == 0u;
  };
  int bits = 0;
  if (u_inv) {
    bool id = true;
#pragma unroll
    for (int a = 0; a < 3; a++) if (a < g.nc) id = id && identity(u_inv + ub + a * g.n, u_bc + ub + a * g.n);
    bits |= id ? 1 : 0;
  }
  if (d_inv && identity(d_inv + o, d_bc + o)) bits |= 2;
  qmask[o >> 2] = (unsigned char)bits;
}

// Rows the quad kernels cover: nx a multiple of 4 and a block shape that tiles 256 threads.
static inline bool quad_dims(const Geo& g, dim3& grid, dim3& block) {
  if (g.nx % 4 != 0 || g.zlo != 0 || g.zhi != g.nz) return false;
  const int quads = g.nx / 4;
  int bx;
  if (quads >= 32) bx = 32;
  else if ((quads & (quads - 1)) == 0) bx = quads;
  else return false;
  const int bz = g.nz > 1 ? 2 : 1;
  const int by = 256 / (bx * bz);
  block = dim3(bx, by, bz);
  grid = dim3((quads + bx - 1) / bx, (g.ny + by - 1) / by, ((long long)g.nb * g.nz + bz - 1) / bz);
  return true;
}
// The quad kernels use 16-byte accesses on caller-owned pointers: every one must be 16-byte aligned
// (null = absent), otherwise the scalar kernels run.
static inline bool aligned16(std::initializer_list<const void*> ptrs) {
  for (const void* p : ptrs)
    if (((uintptr_t)p & 15u) != 0) return false;
  return true;
}
// Quad versions of curl + force over the whole grid; false if the shape does not fit (caller falls back).
bool launch_vort_curl_quad(const float* U, float* curl, float* cnorm, float* force, float strength, const Geo& g,
                           cudaStream_t st) {
  dim3 qg, qb;
  if (!quad_dims(g, qg, qb) || !aligned16({U, curl, cnorm, force})) return false;
  if (g.is3d) {
    k_vort_curl4<true><<<qg, qb, 0, st>>>(U, curl, cnorm, g);
    k_vort_force4<true><<<qg, qb, 0, st>>>(curl, cnorm, force, strength, g);
  } else {
    k_vort_curl4<false><<<qg, qb, 0, st>>>(U, curl, cnorm, g);
    k_vort_force4<false><<<qg, qb, 0, st>>>(curl, cnorm, force, strength, g);
  }
  return true;
}

// false if the quad kernels do not cover this grid (the stages then run without the mask)
bool launch_bc_quad_mask(const float* u_inv, const float* u_bc, const float* d_inv, const float* d_bc,
                         unsigned char* qmask, const Geo& g, cudaStream_t st) {
  dim3 qg, qb;
  if (!quad_dims(g, qg, qb) || !aligned16({u_inv, u_bc, d_inv, d_bc}) || (!u_inv && !d_inv)) return false;
  k_bc_quad_mask<<<qg, qb, 0, st>>>(u_inv, u_bc, d_inv, d_bc, qmask, g);
  return true;
}

void launch_post_advect(const float* tmp_s, const float* tmp_u, const unsigned char* flags, float* density, float* U,
                        const float* u_inv, const float* u_bc, const float* d_inv, const float* d_bc,
                        const unsigned char* qmask, int do_buoy, const float s[3], const Geo& g, cudaStream_t st) {
  BcPtrs bc{u_inv, u_bc, d_inv, d_bc, qmask};
  dim3 grid, block;
  if (quad_dims(g, grid, block) && aligned16({tmp_s, tmp_u, flags, density, U, u_inv, u_bc, d_inv, d_bc})) {
    k_post_advect4<<<grid, block, 0, st>>>(tmp_s, tmp_u, flags, density, U, bc, do_buoy, s[0], s[1], s[2], g);
    return;
  }
  launch_dims(g, grid, block);
  k_post_advect<<<grid, block, 0, st>>>(tmp_s, tmp_u, flags, density, U, bc, do_buoy, s[0], s[1], s[2], g);
}
template <int STAT>
static void vort_bc_mask_stat(float* U, const unsigned char* flags, const float* force, int do_vort, const BcPtrs& bc,
                              int mask_mode, double* sums, const float* p_div, const Geo& g, cudaStream_t st) {
  dim3 grid, block;
  if (quad_dims(g, grid, block) &&
      aligned16({U, flags, force, bc.u_inv, bc.u_bc, STAT == kCnnStatPDiv ? p_div : nullptr})) {
    if (g.nb > 1)
      k_vort_bc_mask4<true, STAT><<<grid, block, 0, st>>>(U, flags, force, do_vort, bc, mask_mode, sums, g, p_div);
    else
      k_vort_bc_mask4<false, STAT><<<grid, block, 0, st>>>(U, flags, force, do_vort, bc, mask_mode, sums, g, p_div);
    return;
  }
  launch_dims(g, grid, block);
  if (g.nb > 1)
    k_vort_bc_mask<true, STAT><<<grid, block, 0, st>>>(U, flags, force, do_vort, bc, mask_mode, sums, g, p_div);
  else
    k_vort_bc_mask<false, STAT><<<grid, block, 0, st>>>(U, flags, force, do_vort, bc, mask_mode, sums, g, p_div);
}
void launch_vort_bc_mask(float* U, const unsigned char* flags, const float* force, int do_vort,
                         const float* u_inv, const float* u_bc, const unsigned char* qmask, int mask_mode, double* sums,
                         const Geo& g, cudaStream_t st, int stat, const float* p_div) {
  const BcPtrs bc{u_inv, u_bc, nullptr, nullptr, qmask};
  if (stat == kCnnStatU) vort_bc_mask_stat<kCnnStatU>(U, flags, force, do_vort, bc, mask_mode, sums, p_div, g, st);
  else if (stat == kCnnStatPDiv)
    vort_bc_mask_stat<kCnnStatPDiv>(U, flags, force, do_vort, bc, mask_mode, sums, p_div, g, st);
  else vort_bc_mask_stat<kCnnStatNone>(U, flags, force, do_vort, bc, mask_mode, sums, p_div, g, st);
}
void launch_cnn_div_stats_fused(const float* U1, const unsigned char* flags, double* sums, const Geo& g,
                                cudaStream_t st) {
  dim3 grid, block;
  if (quad_dims(g, grid, block) && aligned16({U1, flags})) {
    if (g.nb > 1) k_cnn_div_stats_fused4<true><<<grid, block, 0, st>>>(U1, flags, sums, g);
    else k_cnn_div_stats_fused4<false><<<grid, block, 0, st>>>(U1, flags, sums, g);
    return;
  }
  launch_dims(g, grid, block);
  if (g.nb > 1) k_cnn_div_stats_fused<true><<<grid, block, 0, st>>>(U1, flags, sums, g);
  else k_cnn_div_stats_fused<false><<<grid, block, 0, st>>>(U1, flags, sums, g);
}

// The arguments of one launch of the input kernels.
struct InputsArgs {
  const float *p_div, *U1;
  const unsigned char* flags;
  const double* sums;
  float threshold;
  float *scale_out, *x0;
  int px, py;
};
template <int SEL, int SCALE>
static void inputs_fused(const InputsArgs& a, const Geo& g, cudaStream_t st) {
  dim3 grid, block;
  if (quad_dims(g, grid, block) && aligned16({(SEL & kCnnInPDiv) ? a.p_div : nullptr, a.U1, a.flags, a.x0})) {
    k_cnn_inputs_fused4<SEL, SCALE><<<grid, block, 0, st>>>(a.p_div, a.U1, a.flags, a.sums, a.threshold, a.scale_out,
                                                            (float4*)a.x0, a.px, a.py, g);
    return;
  }
  launch_dims(g, grid, block);
  k_cnn_inputs_fused<SEL, SCALE><<<grid, block, 0, st>>>(a.p_div, a.U1, a.flags, a.sums, a.threshold, a.scale_out,
                                                         (float4*)a.x0, a.px, a.py, g);
}
template <int SEL>
static void inputs_fused_sel(int scale, const InputsArgs& a, const Geo& g, cudaStream_t st) {
  switch (scale) {
    case kFusedStdU: inputs_fused<SEL, kFusedStdU>(a, g, st); break;
    case kFusedStdN: inputs_fused<SEL, kFusedStdN>(a, g, st); break;
    case kFusedNorm: inputs_fused<SEL, kFusedNorm>(a, g, st); break;
    default: inputs_fused<SEL, kFusedOne>(a, g, st); break;
  }
}
bool launch_cnn_inputs_fused(const float* p_div, const float* U1, const unsigned char* flags, const double* sums,
                             float threshold, float* scale_out, float* x0, int px, int py, const Geo& g,
                             cudaStream_t st, int sel, int func, int chan) {
  const InputsArgs a{p_div, U1, flags, sums, threshold, scale_out, x0, px, py};
  const int scale = func == kCnnScaleOne    ? kFusedOne
                    : func == kCnnScaleNorm ? kFusedNorm
                    : chan == kCnnStatU     ? kFusedStdU
                                            : kFusedStdN;
  constexpr int P = kCnnInPDiv, U = kCnnInUDiv, D = kCnnInDiv;
  switch (sel) {     // the sets tfl_cnn_create accepts: UDiv or div, with or without pDiv
    case P | D: inputs_fused_sel<P | D>(scale, a, g, st); break;
    case P | U | D: inputs_fused_sel<P | U | D>(scale, a, g, st); break;
    case P | U: inputs_fused_sel<P | U>(scale, a, g, st); break;
    case U | D: inputs_fused_sel<U | D>(scale, a, g, st); break;
    case U: inputs_fused_sel<U>(scale, a, g, st); break;
    case D: inputs_fused_sel<D>(scale, a, g, st); break;
    default: return false;
  }
  return true;
}
void launch_cnn_finish_fused(const float* p_net, float* U, const unsigned char* flags, const float* scale, float* p_out,
                             const float* u_inv, const float* u_bc, const unsigned char* qmask, float lo, float hi,
                             const Geo& g, cudaStream_t st) {
  BcPtrs bc{u_inv, u_bc, nullptr, nullptr, qmask};
  dim3 grid, block;
  if (quad_dims(g, grid, block) && aligned16({p_net, U, flags, p_out, u_inv, u_bc})) {
    k_cnn_finish_fused4<<<grid, block, 0, st>>>(p_net, U, flags, scale, p_out, bc, lo, hi, g);
    return;
  }
  launch_dims(g, grid, block);
  k_cnn_finish_fused<<<grid, block, 0, st>>>(p_net, U, flags, scale, p_out, bc, lo, hi, g);
}

}  // namespace tfl
