// Non-convolutional nodes of the projection graph (torch/lib/model.lua:27-401), compiled
// with -fmad=false so they match the float arithmetic of the reference modules:
//   tfluids.SetWallBcs      tfluids/set_wall_bcs.lua:29-48   (U * {0,1} mask)
//   tfluids.VelocityDivergence, nn.StandardDeviation (lib/modules/variance.lua:44-76),
//   nn.Clamp, nn.ApplyScale (lib/modules/apply_scale.lua), tfluids.FlagsToOccupancy,
//   tfluids.VelocityUpdate  tfluids/velocity_update.lua:28-38
#include "tfl_device.cuh"
#include "tfl_kernels.h"

namespace tfl {

// U1 = U * wallmask; sums[b] += (sum f, sum f^2) over the owned planes (double), f = U1 (kCnnStatU) or pDiv
// (kCnnStatPDiv, normalizeInputChan 'pDiv'); kCnnStatDiv leaves the sums to k_cnn_div_stats.
template <bool IS3D>
__global__ void k_cnn_mask_stats(const float* __restrict__ U, const float* __restrict__ flags,
                                 float* __restrict__ U1, double* __restrict__ sums, int own_lo, int own_hi, int stat,
                                 const float* __restrict__ p_div, Geo gin) {
  const Geo g = static_geo<IS3D>(gin);
  int b, k, j, i;
  const bool live = thread_cell(g, b, k, j, i);
  double s = 0.0, ss = 0.0;
  if (live) {
    bool z[3];
    wall_bc_zero_mask(flags + b * g.n, g, k, j, i, z);
    const long long c = (long long)b * g.nc * g.n + cell(g, k, j, i);
    const bool owned = k >= own_lo && k < own_hi;     // the statistics cover owned planes only (z-slabs)
    for (int a = 0; a < g.nc; a++) {
      float u = U[c + a * g.n];
      if (z[a]) u = u * 0.0f;
      U1[c + a * g.n] = u;
      if (owned && stat == kCnnStatU) {
        const float sq = u * u;
        s += (double)u;
        ss += (double)sq;
      }
    }
    if (owned && stat == kCnnStatPDiv) {
      const float v = __ldg(p_div + b * g.n + cell(g, k, j, i));
      const float sq = v * v;
      s += (double)v;
      ss += (double)sq;
    }
  }
  add_entry_sums(s, ss, sums, live, b, g);
}

// tfluids.VelocityDivergence of the masked velocity at cell c (lib/model.lua:86-89).
__device__ __forceinline__ float cnn_div(const float* __restrict__ ub, const float* __restrict__ fb, const Geo& g, int k,
                                         int j, int i, int c, int* flag) {
  const int f = flag_i(fb, g, k, j, i);
  *flag = f;
  float dv = 0.0f;
  if (!on_border(g, k, j, i) && (f & kFluid)) {
    dv = __ldg(ub + c) - __ldg(ub + c + 1) + __ldg(ub + g.n + c) - __ldg(ub + g.n + c + g.nx);
    if (g.is3d) dv += (__ldg(ub + 2 * g.n + c) - __ldg(ub + 2 * g.n + c + (long long)g.nx * g.ny));
  }
  return dv;
}

// normalizeInputChan 'div': sums[b] += (sum div, sum div^2) over the owned planes, once U1 is complete.
template <bool IS3D>
__global__ void k_cnn_div_stats(const float* __restrict__ U1, const float* __restrict__ flags, double* __restrict__ sums,
                                int own_lo, int own_hi, Geo gin) {
  const Geo g = static_geo<IS3D>(gin);
  int b, k, j, i;
  const bool live = thread_cell(g, b, k, j, i);
  double s = 0.0, ss = 0.0;
  if (live && k >= own_lo && k < own_hi) {
    int f;
    const float dv = cnn_div(U1 + (long long)b * g.nc * g.n, flags + b * g.n, g, k, j, i, cell(g, k, j, i), &f);
    const float sq = dv * dv;
    s += (double)dv;
    ss += (double)sq;
  }
  add_entry_sums(s, ss, sums, live, b, g);
}

// nn.StandardDeviation (or nn.Power(2), nn.Sum, nn.Sqrt for 'norm') + nn.Clamp(threshold, inf): float tensor ops on
// the two sums; normalizeInput off: 1, with which every scaling below is exact.
__global__ void k_cnn_scale(const double* __restrict__ sums, float* __restrict__ scale, int nb,
                            long long n, float threshold, int func) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nb) return;
  if (func == kCnnScaleStd) {
    scale[b] = scale_from_sums(sums, b, n, threshold);
  } else if (func == kCnnScaleNorm) {
    const float out = sqrtf((float)sums[2 * b + 1]);
    scale[b] = (out < threshold) ? threshold : out;
  } else {
    scale[b] = 1.0f;
  }
}

// v[n++] = x with a register-resident v (the unrolled compare keeps the index static).
__device__ __forceinline__ void put_channel(float (&v)[8], int& n, float x) {
#pragma unroll
  for (int q = 0; q < 8; q++)
    if (q == n) v[q] = x;
  n++;
}

// The network input at one cell (nn.JoinTable(2), lib/model.lua:133-150): pDiv / s, U1 / s (nc), div / s,
// occupancy(flags), the channels of `sel` only, then zeros up to 8.  Returns the channel count.
__device__ __forceinline__ int cnn_input_channels(const float* __restrict__ p_div, const float* __restrict__ ub,
                                                  const float* __restrict__ fb, float sc, int sel, const Geo& g, int b,
                                                  int k, int j, int i, int c, float (&v)[8]) {
  int f;
  const float dv = cnn_div(ub, fb, g, k, j, i, c, &f);
  int n = 0;
#pragma unroll
  for (int q = 0; q < 8; q++) v[q] = 0.0f;
  if (sel & kCnnInPDiv) put_channel(v, n, __ldg(p_div + b * g.n + c) / sc);
  if (sel & kCnnInUDiv)
    for (int a = 0; a < g.nc; a++) put_channel(v, n, __ldg(ub + a * g.n + c) / sc);
  if (sel & kCnnInDiv) put_channel(v, n, dv / sc);
  put_channel(v, n, (f == kFluid) ? 0.0f : ((f == kObstacle) ? 1.0f : -1.0f));
  return n;
}

// x0 [b][cin][n] = the input channels of `sel` (default: pDiv / s, div(U1) / s, occupancy(flags)).
template <bool IS3D>
__global__ void k_cnn_inputs(const float* __restrict__ p_div, const float* __restrict__ U1,
                             const float* __restrict__ flags, const float* __restrict__ scale,
                             float* __restrict__ x0, int sel, int cin, Geo gin) {
  const Geo g = static_geo<IS3D>(gin);
  int b, k, j, i;
  if (!thread_cell(g, b, k, j, i)) return;
  const int c = cell(g, k, j, i);
  float v[8];
  const int n = cnn_input_channels(p_div, U1 + (long long)b * g.nc * g.n, flags + b * g.n, __ldg(scale + b), sel, g,
                                   b, k, j, i, c, v);
  float* xb = x0 + (long long)b * cin * g.n + c;
#pragma unroll
  for (int q = 0; q < 6; q++)
    if (q < n) xb[q * g.n] = v[q];
}

// Same input channels written channels-last into the padded activation layout the tensor-core convolution reads
// (tfl_cnn_tc.cu): the first float4 plane (planes = 1: up to 3 channels, zero fourth) or both planes (planes = 2:
// channels 0-3 and 4-7, zero-padded), e.g. the default set as (pDiv/s, div/s, occ, 0).
template <bool IS3D>
__global__ void k_cnn_inputs_padded(const float* __restrict__ p_div, const float* __restrict__ U1,
                                    const float* __restrict__ flags, const float* __restrict__ scale,
                                    float4* __restrict__ x0, int sel, int planes, int px, int py, Geo gin) {
  const Geo g = static_geo<IS3D>(gin);
  int b, k, j, i;
  if (!thread_cell(g, b, k, j, i)) return;
  const int c = cell(g, k, j, i);
  float v[8];
  cnn_input_channels(p_div, U1 + (long long)b * g.nc * g.n, flags + b * g.n, __ldg(scale + b), sel, g, b, k, j, i, c,
                     v);
  const long long plane = (long long)(g.nz + 2) * py * px;
  const long long o = (long long)b * 2 * plane + ((long long)(k + 1) * py + (j + 1)) * px + (i + 1);
  x0[o] = make_float4(v[0], v[1], v[2], v[3]);
  if (planes == 2) x0[o + plane] = make_float4(v[4], v[5], v[6], v[7]);
}

// addPressureSkip (lib/model.lua:357-361): the last convolution is 1x1, so its pDiv input channel adds
// w_skip * pDiv_scaled to p_net.  A pass of its own because the velocity update reads p at the neighbours while
// p_out, which may alias pDiv, is written.
template <bool IS3D>
__global__ void k_cnn_skip(float* __restrict__ p_net, const float* __restrict__ p_div, const float* __restrict__ scale,
                           float w_skip, Geo gin) {
  const Geo g = static_geo<IS3D>(gin);
  int b, k, j, i;
  if (!thread_cell(g, b, k, j, i)) return;
  const long long c = b * g.n + cell(g, k, j, i);
  p_net[c] = p_net[c] + w_skip * (__ldg(p_div + c) / __ldg(scale + b));
}

// U = setWallBcs(velocityUpdate(U1 / scale, p_net) * scale);  p = p_net * scale.
template <bool IS3D>
__global__ void k_cnn_finish(const float* __restrict__ p_net, const float* __restrict__ U1,
                             const float* __restrict__ flags, const float* __restrict__ scale,
                             float* __restrict__ p_out, float* __restrict__ U_out, Geo gin) {
  const Geo g = static_geo<IS3D>(gin);
  int b, k, j, i;
  if (!thread_cell(g, b, k, j, i)) return;
  const int c = cell(g, k, j, i);
  const float sc = __ldg(scale + b);
  const float* fl = flags + b * g.n;
  const float* pb = p_net + b * g.n;
  const float* ub = U1 + (long long)b * g.nc * g.n;
  const float pc = __ldg(pb + c);
  float u[3];
  for (int a = 0; a < g.nc; a++) u[a] = __ldg(ub + a * g.n + c) / sc;
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
  float* uo = U_out + (long long)b * g.nc * g.n + c;
  for (int a = 0; a < g.nc; a++) {
    float v = u[a] * sc;
    if (z[a]) v = v * 0.0f;
    uo[a * g.n] = v;
  }
  p_out[b * g.n + c] = pc * sc;
}

#define TFL_LAUNCH3B(kernel, g, st, ...)                                        \
  do {                                                                          \
    dim3 grid_, block_;                                                         \
    launch_dims(g, grid_, block_);                                              \
    if ((g).is3d) kernel<true><<<grid_, block_, 0, st>>>(__VA_ARGS__);          \
    else kernel<false><<<grid_, block_, 0, st>>>(__VA_ARGS__);                  \
  } while (0)

void launch_cnn_mask_stats(const float* U, const float* flags, float* U1, double* sums, int own_lo, int own_hi,
                           const Geo& g, cudaStream_t st, int stat, const float* p_div) {
  TFL_LAUNCH3B(k_cnn_mask_stats, g, st, U, flags, U1, sums, own_lo, own_hi, stat, p_div, g);
}
void launch_cnn_div_stats(const float* U1, const float* flags, double* sums, int own_lo, int own_hi, const Geo& g,
                          cudaStream_t st) {
  TFL_LAUNCH3B(k_cnn_div_stats, g, st, U1, flags, sums, own_lo, own_hi, g);
}
void launch_cnn_scale(const double* sums, float* scale, int nb, long long n_per_batch, float threshold,
                      cudaStream_t st, int func) {
  k_cnn_scale<<<(nb + 31) / 32, 32, 0, st>>>(sums, scale, nb, n_per_batch, threshold, func);
}
void launch_cnn_inputs(const float* p_div, const float* U1, const float* flags, const float* scale,
                       float* x0, const Geo& g, cudaStream_t st, int sel) {
  const int cin = ((sel & kCnnInPDiv) ? 1 : 0) + ((sel & kCnnInUDiv) ? g.nc : 0) + ((sel & kCnnInDiv) ? 1 : 0) + 1;
  TFL_LAUNCH3B(k_cnn_inputs, g, st, p_div, U1, flags, scale, x0, sel, cin, g);
}
void launch_cnn_inputs_padded(const float* p_div, const float* U1, const float* flags, const float* scale,
                              float* x0, int px, int py, const Geo& g, cudaStream_t st, int sel, int planes) {
  TFL_LAUNCH3B(k_cnn_inputs_padded, g, st, p_div, U1, flags, scale, (float4*)x0, sel, planes, px, py, g);
}
void launch_cnn_skip(float* p_net, const float* p_div, const float* scale, float w_skip, const Geo& g, cudaStream_t st) {
  TFL_LAUNCH3B(k_cnn_skip, g, st, p_net, p_div, scale, w_skip, g);
}
void launch_cnn_finish(const float* p_net, const float* U1, const float* flags, const float* scale,
                       float* p_out, float* U_out, const Geo& g, cudaStream_t st) {
  TFL_LAUNCH3B(k_cnn_finish, g, st, p_net, U1, flags, scale, p_out, U_out, g);
}

}  // namespace tfl
