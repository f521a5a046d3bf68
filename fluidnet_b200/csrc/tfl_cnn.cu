// Convolution stack of the pressure-projection network (torch/lib/model.lua:262-364:
// stride-1 zero-padded cross-correlation + bias (+ReLU), cudnn.Volumetric/Spatial
// Convolution in the reference, torch/lib/model_utils.lua:74-116).
//
// This file holds the fp32 FMA path: one thread per output voxel computing all output
// channels from shared-memory weights.  It is the numerically tight (1e-5 class)
// implementation and the parity anchor for the tensor-core path (tfl_cnn_tc.cu).
#include "tfl_device.cuh"
#include "tfl_kernels.h"
#include "tfl_cnn_tc.h"

namespace tfl {

// Non-linearity between layers (torch.addNonlinearity, lib/model_utils.lua): 0 none, 1 ReLU, 2 sigmoid, 3 ReLU6
// (nn.ReLU6, min(max(x, 0), 6)).
__device__ __forceinline__ float activate(float r, int act) {
  if (act == 1) return r < 0.0f ? 0.0f : r;
  if (act == 2) return 1.0f / (1.0f + expf(-r));
  if (act == 3) return r < 0.0f ? 0.0f : (r > 6.0f ? 6.0f : r);
  return r;
}

// weights in smem as [cin][tap][COUT]; taps ordered (dz, dy, dx).  DIL: tap t reads the input at offset
// (t - (k-1)/2) dil on every axis (nn.{Spatial,Volumetric}DilatedConvolution, stride 1, padding dil (k-1)/2); without
// it dil is not read and the kernel is the undilated one.
template <int COUT, int KS, bool IS3D, bool DIL>
__global__ void __launch_bounds__(256)
k_conv_direct(const float* __restrict__ in, float* __restrict__ out, const float* __restrict__ w,
              const float* __restrict__ bias, int cin, int act, Geo g, int dil) {
  extern __shared__ float sw[];
  constexpr int KZ = IS3D ? KS : 1;
  constexpr int TAPS = KZ * KS * KS;
  const int nthreads = blockDim.x * blockDim.y * blockDim.z;
  const int tid = (threadIdx.z * blockDim.y + threadIdx.y) * blockDim.x + threadIdx.x;
  for (int t = tid; t < cin * TAPS * COUT; t += nthreads) sw[t] = w[t];
  __syncthreads();

  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int j = blockIdx.y * blockDim.y + threadIdx.y;
  const int zz = blockIdx.z * blockDim.z + threadIdx.z;
  const int nzr = g.zhi - g.zlo;
  const int b = zz / nzr;
  const int k = g.zlo + (zz - b * nzr);
  if (i >= g.nx || j >= g.ny || b >= g.nb) return;

  float acc[COUT];
#pragma unroll
  for (int o = 0; o < COUT; o++) acc[o] = __ldg(bias + o);

  constexpr int P = (KS - 1) / 2;
  constexpr int PZ = (KZ - 1) / 2;
  const int d = DIL ? dil : 1;
  const int kg = k + g.zoff;
  for (int c = 0; c < cin; c++) {
    const float* ib = in + ((long long)b * cin + c) * g.n;
    const float* wc = sw + c * TAPS * COUT;
#pragma unroll
    for (int dz = 0; dz < KZ; dz++) {
      const int zg = DIL ? kg + (dz - PZ) * d : kg + dz - PZ;
      if (zg < 0 || zg >= g.gnz) continue;           // zero padding at the GLOBAL boundary
      const int zl = zg - g.zoff;
#pragma unroll
      for (int dy = 0; dy < KS; dy++) {
        const int yy = DIL ? j + (dy - P) * d : j + dy - P;
        if (yy < 0 || yy >= g.ny) continue;
#pragma unroll
        for (int dx = 0; dx < KS; dx++) {
          const int xx = DIL ? i + (dx - P) * d : i + dx - P;
          if (xx < 0 || xx >= g.nx) continue;
          const float v = __ldg(ib + ((long long)zl * g.ny + yy) * g.nx + xx);
          const float* wt = wc + ((dz * KS + dy) * KS + dx) * COUT;
#pragma unroll
          for (int o = 0; o < COUT; o++) acc[o] = fmaf(v, wt[o], acc[o]);
        }
      }
    }
  }
  const long long c0 = cell(g, k, j, i);
#pragma unroll
  for (int o = 0; o < COUT; o++) {
    out[((long long)b * COUT + o) * g.n + c0] = activate(acc[o], act);
  }
}


// Any (cout, k): one thread per output value, weights [cin][tap][cout] read through the cache.  The
// fallback for layer shapes outside the specialised table (e.g. the 256-channel 1x1x1 convolution
// inside a VolumetricConvolutionUpsample); same accumulation order as k_conv_direct, and the same DIL switch.
template <bool DIL>
__global__ void k_conv_any(const float* __restrict__ in, float* __restrict__ out, const float* __restrict__ w,
                           const float* __restrict__ bias, int cin, int cout, int ks, int act, Geo g, int dil) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)g.nb * cout * g.n;
  if (t >= total) return;
  const long long c0 = t % g.n;
  const int o = (int)((t / g.n) % cout);
  const int b = (int)(t / (g.n * cout));
  const int i = (int)(c0 % g.nx), j = (int)((c0 / g.nx) % g.ny), k = (int)(c0 / ((long long)g.nx * g.ny));
  const int kz = g.is3d ? ks : 1;
  const int P = (ks - 1) / 2, PZ = (kz - 1) / 2;
  const int taps = kz * ks * ks;
  const int d = DIL ? dil : 1;
  float acc = __ldg(bias + o);
  for (int c = 0; c < cin; c++) {
    const float* ib = in + ((long long)b * cin + c) * g.n;
    const float* wc = w + (long long)c * taps * cout;
    for (int dz = 0; dz < kz; dz++) {
      const int zz = DIL ? k + (dz - PZ) * d : k + dz - PZ;
      if (zz < 0 || zz >= g.nz) continue;
      for (int dy = 0; dy < ks; dy++) {
        const int yy = DIL ? j + (dy - P) * d : j + dy - P;
        if (yy < 0 || yy >= g.ny) continue;
        for (int dx = 0; dx < ks; dx++) {
          const int xx = DIL ? i + (dx - P) * d : i + dx - P;
          if (xx < 0 || xx >= g.nx) continue;
          acc = fmaf(__ldg(ib + ((long long)zz * g.ny + yy) * g.nx + xx), __ldg(wc + ((dz * ks + dy) * ks + dx) * cout + o), acc);
        }
      }
    }
  }
  out[t] = activate(acc, act);
}

// cudnn.{Spatial,Volumetric}{Average,Max}Pooling(p, p[, p], p, p[, p]) (lib/model_utils.lua:184-209):
// window p^d, stride p, no padding.  in [bc][nz][ny][nx] -> out [bc][nz/pz][ny/p][nx/p], pz = p in 3-D else 1.
__global__ void k_pool(const float* __restrict__ in, float* __restrict__ out, int nz, int ny, int nx, int p,
                       int is3d, int is_max, long long total) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int pz = is3d ? p : 1;
  const int ox = nx / p, oy = ny / p, oz = nz / pz;
  const int x = (int)(t % ox), y = (int)((t / ox) % oy), z = (int)((t / ((long long)ox * oy)) % oz);
  const long long bc = t / ((long long)ox * oy * oz);
  const float* ib = in + bc * (long long)nz * ny * nx;
  float acc = is_max ? -INFINITY : 0.0f;
  for (int dz = 0; dz < pz; dz++)
    for (int dy = 0; dy < p; dy++)
      for (int dx = 0; dx < p; dx++) {
        const float v = __ldg(ib + ((long long)(z * pz + dz) * ny + (y * p + dy)) * nx + (x * p + dx));
        acc = is_max ? fmaxf(acc, v) : acc + v;
      }
  out[t] = is_max ? acc : acc / (float)(pz * p * p);
}

// The view / permute / copy of nn.{Spatial,Volumetric}ConvolutionUpsample:updateOutput
// (lib/modules/*_convolution_upsample.lua): in [b][nO * sT * sH * sW][d][h][w] -> out [b][nO][d sT][h sH][w sW],
// out(b, o, z sT + st, y sH + sh, x sW + sw) = in(b, ((o sT + st) sH + sh) sW + sw, z, y, x); sT = 1 in 2-D.
__global__ void k_pixel_shuffle(const float* __restrict__ in, float* __restrict__ out, int n_out, int nz, int ny,
                                int nx, int s, int is3d, long long total) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int st_ = is3d ? s : 1;
  const int ox = nx * s, oy = ny * s, oz = nz * st_;
  const int X = (int)(t % ox), Y = (int)((t / ox) % oy), Z = (int)((t / ((long long)ox * oy)) % oz);
  const int o = (int)((t / ((long long)ox * oy * oz)) % n_out);
  const long long b = t / ((long long)ox * oy * oz * n_out);
  const int x = X / s, sw = X % s, y = Y / s, sh = Y % s, z = Z / st_, sz = Z % st_;
  const long long ch = ((long long)(o * st_ + sz) * s + sh) * s + sw;
  const long long cin_total = (long long)n_out * st_ * s * s;
  out[t] = __ldg(in + ((b * cin_total + ch) * nz + z) * (long long)ny * nx + (long long)y * nx + x);
}

// Join of the multi-resolution banks (lib/model.lua:297-318).  Bank i (1-based, i >= 2) is
// [nb][c][nz / rz][ny / r][nx / r] with r = 2^(i-1) (rz = r in 3-D, 1 in 2-D), upsampled nearest to the
// full grid on the fly.  concat: out is [nb][nbanks * c][nz][ny][nx] and bank i lands at channel offset
// (i-1) c (bank 1 is already in place); add: out is [nb][c][nz][ny][nx], holds bank 1 and gets banks 2..N
// added in bank order, as CAddTable does.  FULL: every bank is at the full resolution (banksType 'dilate', no
// upsampling, lib/model.lua:300-303); r = 1.
struct BankPtrs {
  const float* p[kMaxBankPtrs];
};
template <bool FULL>
__global__ void k_bank_join(BankPtrs banks, int nbanks, float* __restrict__ out, int c, int nz, int ny, int nx,
                            int is3d, int add, long long total) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const long long n = (long long)nz * ny * nx;
  const int x = (int)(t % nx), y = (int)((t / nx) % ny), z = (int)((t / ((long long)nx * ny)) % nz);
  const long long bc = t / n;                      // b * c + ch
  const long long b = bc / c, ch = bc % c;
  if (add) {
    float v = out[t];
    for (int i = 1; i < nbanks; i++) {
      const int s = FULL ? 0 : i;
      const int bx = nx >> s, by = ny >> s, bz = is3d ? nz >> s : nz;
      const int zi = is3d ? z >> s : z;
      v = v + __ldg(banks.p[i] + ((bc * bz + zi) * by + (y >> s)) * bx + (x >> s));
    }
    out[t] = v;
  } else {
    const long long cell = t % n;
    for (int i = 1; i < nbanks; i++) {
      const int s = FULL ? 0 : i;
      const int bx = nx >> s, by = ny >> s, bz = is3d ? nz >> s : nz;
      const int zi = is3d ? z >> s : z;
      out[((b * nbanks + i) * c + ch) * n + cell] = __ldg(banks.p[i] + ((bc * bz + zi) * by + (y >> s)) * bx + (x >> s));
    }
  }
}

// Batch normalization of x [nb][c][n] whose batch entries lie bstride floats apart (a stage's output written in
// place into its 'concat' slot has bstride > c n).  Batch statistics: block (blk, ch) of k_bn_stats owns the fixed
// contiguous range blk of channel ch's nb n values and writes its (sum d, sum d^2), d = x - K, in fp64 to slot
// ch (gridDim.x + 1) + blk; K, the channel's first value, goes to slot ch (gridDim.x + 1) + gridDim.x, so a constant
// channel has a variance of exactly 0.  k_bn_finalize sums a channel's slots in a fixed order.  No atomics: the
// result is the same bits on every run.
constexpr int kBnThreads = 256;

// (s, q) summed over the block in a fixed order; the total is valid in thread 0.
__device__ __forceinline__ void bn_block_sum(double& s, double& q, double* sh) {
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_down_sync(0xffffffffu, s, o);
    q += __shfl_down_sync(0xffffffffu, q, o);
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) {
    sh[2 * wid] = s;
    sh[2 * wid + 1] = q;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    s = 0.0;
    q = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) {
      s += sh[2 * w];
      q += sh[2 * w + 1];
    }
  }
}

__global__ void __launch_bounds__(kBnThreads)
k_bn_stats(const float* __restrict__ x, long long n, int nb, long long bstride, double* __restrict__ part) {
  __shared__ double sh[2 * kBnThreads / 32];
  const int ch = blockIdx.y;
  const long long total = (long long)nb * n, chunk = (total + gridDim.x - 1) / gridDim.x;
  const long long lo = (long long)blockIdx.x * chunk, hi = min(total, lo + chunk);
  const double K = __ldg(x + ch * n);
  double s = 0.0, q = 0.0;
  for (long long b = lo / n; b * n < hi; b++) {        // the block's range, one batch entry at a time
    const float* xb = x + b * bstride + ch * n;
    const long long i1 = min(hi, (b + 1) * n) - b * n;
    for (long long i = max(lo, b * n) - b * n + threadIdx.x; i < i1; i += blockDim.x) {
      const double d = (double)__ldg(xb + i) - K;
      s += d;
      q = fma(d, d, q);
    }
  }
  bn_block_sum(s, q, sh);
  if (threadIdx.x == 0) {
    double* slot = part + 2 * ((long long)ch * (gridDim.x + 1) + blockIdx.x);
    slot[0] = s;
    slot[1] = q;
    if (blockIdx.x == 0) {
      slot[2 * gridDim.x] = K;
      slot[2 * gridDim.x + 1] = 0.0;
    }
  }
}

// One block per channel: mean and biased variance over `count` values, invstd = 1 / sqrt(var + eps) (0 when
// var + eps == 0, as THNN), ac[ch] = a = w invstd, ac[c + ch] = b - mean a.  w / b may be null (1 / 0); stats (may be
// null) gets (mean, var) per channel.  part: [c][nslots + 1][2] as k_bn_stats writes it.
__global__ void __launch_bounds__(kBnThreads)
k_bn_finalize(const double* __restrict__ part, int nslots, int c, long long count, const float* __restrict__ w,
              const float* __restrict__ b, float eps, float* __restrict__ ac, double* __restrict__ stats) {
  __shared__ double sh[2 * kBnThreads / 32];
  const int ch = blockIdx.x;
  const double* pc = part + 2 * (long long)ch * (nslots + 1);
  double s = 0.0, q = 0.0;
  for (int i = threadIdx.x; i < nslots; i += blockDim.x) {
    s += pc[2 * i];
    q += pc[2 * i + 1];
  }
  bn_block_sum(s, q, sh);
  if (threadIdx.x != 0) return;
  const double md = s / (double)count;
  const double mean = pc[2 * nslots] + md;
  const double var = fmax(q / (double)count - md * md, 0.0);
  const double ve = var + (double)eps;
  const double invstd = ve == 0.0 ? 0.0 : 1.0 / sqrt(ve);
  const double a = (w ? (double)w[ch] : 1.0) * invstd;
  ac[ch] = (float)a;
  ac[c + ch] = (float)((b ? (double)b[ch] : 0.0) - mean * a);
  if (stats) {
    stats[2 * ch] = mean;
    stats[2 * ch + 1] = var;
  }
}

// y = a x + c in place, per channel.
__global__ void k_bn_apply(float* __restrict__ x, int c, long long n, long long bstride, const float* __restrict__ ac,
                           long long total) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const long long cn = (long long)c * n, b = t / cn, r = t - b * cn;
  const int ch = (int)(r / n);
  float* p = x + b * bstride + r;
  *p = fmaf(__ldg(ac + ch), *p, __ldg(ac + c + ch));
}


// ---- batch statistics on the tensor-core path's padded channels-last layout (tfl_cnn_tc.h) ----
// Block blk owns the fixed contiguous range blk of the nb nz ny interior rows and sums its 8 channels (two float4
// planes) in fp64, shifted by the values of the first interior voxel, as k_bn_stats does; the slots are those of
// k_bn_stats, so k_bn_finalize reads them.
struct TcRows {
  long long plane, batch;     // float4 per padded plane / batch entry
  long long rows;             // nb nz ny
};
__device__ __forceinline__ TcRows tc_rows(const ConvTcGeo& g) {
  TcRows r;
  r.plane = (long long)(g.nz + 2) * g.py * g.px;
  r.batch = 2 * r.plane;
  r.rows = (long long)g.nb * g.nz * g.ny;
  return r;
}
// float4 index of row `row`'s voxel x = 0 (first plane)
__device__ __forceinline__ long long tc_row_base(const ConvTcGeo& g, const TcRows& r, long long row) {
  const long long b = row / ((long long)g.nz * g.ny), zy = row - b * g.nz * g.ny;
  const int z = (int)(zy / g.ny), y = (int)(zy - (long long)z * g.ny);
  return b * r.batch + ((long long)(z + 1) * g.py + (y + 1)) * g.px + 1;
}
__device__ __forceinline__ void tc_load8(const float4* buf, const TcRows& r, long long i, float (&v)[8]) {
  const float4 a = __ldg(buf + i), b = __ldg(buf + i + r.plane);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
// The tail's hidden layer: h4 = act(w4 (a3 h3 + c3) + b4), sTail = w4[64] b4[8] w5[8] b5, ac3 [2][8].
__device__ __forceinline__ void tc_tail_h4(const float (&h3)[8], const float* sW, const float* sAc3, int relu6,
                                           float (&h4)[8]) {
  float x[8];
#pragma unroll
  for (int c = 0; c < 8; c++) x[c] = fmaf(sAc3[c], h3[c], sAc3[8 + c]);
#pragma unroll
  for (int o = 0; o < 8; o++) {
    float a = sW[64 + o];
#pragma unroll
    for (int c = 0; c < 8; c++) a = fmaf(x[c], sW[o * 8 + c], a);
    a = a > 0.0f ? a : 0.0f;
    h4[o] = relu6 && a > 6.0f ? 6.0f : a;
  }
}
// Fixed-order block sums of the 8 channels' (s, q) into part's slot blk, and the shift into the last slot.
__device__ __forceinline__ void tc_bn_write(double (&s)[8], double (&q)[8], const float (&K)[8], double* sh,
                                            double* part) {
#pragma unroll
  for (int ch = 0; ch < 8; ch++) {
    __syncthreads();
    bn_block_sum(s[ch], q[ch], sh);
    if (threadIdx.x == 0) {
      double* slot = part + 2 * ((long long)ch * (gridDim.x + 1) + blockIdx.x);
      slot[0] = s[ch];
      slot[1] = q[ch];
      if (blockIdx.x == 0) {
        slot[2 * gridDim.x] = K[ch];
        slot[2 * gridDim.x + 1] = 0.0;
      }
    }
  }
}

// TAIL = false: statistics of buf's 8 channels; TAIL = true: of the tail's h4 (pass A) or, with pass_b, p_net.
template <bool TAIL>
__global__ void __launch_bounds__(kBnThreads)
k_tc_bn_rows(const float4* __restrict__ buf, ConvTcGeo g, const float* __restrict__ ac3, const float* __restrict__ tail,
             int relu6, int pass_b, double* __restrict__ part, const float* __restrict__ ac4, float* __restrict__ p_net) {
  __shared__ double sh[2 * kBnThreads / 32];
  __shared__ float sW[64 + 8 + 8 + 1], sAc[32];
  if (TAIL) {
    for (int i = threadIdx.x; i < 81; i += blockDim.x) sW[i] = tail[i];
    for (int i = threadIdx.x; i < 16; i += blockDim.x) {
      sAc[i] = ac3[i];
      if (pass_b) sAc[16 + i] = ac4[i];
    }
    __syncthreads();
  }
  const TcRows r = tc_rows(g);
  const long long chunk = (r.rows + gridDim.x - 1) / gridDim.x;
  const long long lo = (long long)blockIdx.x * chunk, hi = min(r.rows, lo + chunk);
  float K[8];
  {
    float v[8];
    tc_load8(buf, r, tc_row_base(g, r, 0), v);
    if (TAIL) tc_tail_h4(v, sW, sAc, relu6, K);
    else
#pragma unroll
      for (int c = 0; c < 8; c++) K[c] = v[c];
  }
  double s[8] = {}, q[8] = {};
  for (long long row = lo; row < hi; row++) {
    const long long base = tc_row_base(g, r, row);
    for (int x = threadIdx.x; x < g.nx; x += blockDim.x) {
      float v[8], h[8];
      tc_load8(buf, r, base + x, v);
      if (TAIL) tc_tail_h4(v, sW, sAc, relu6, h);
      else
#pragma unroll
        for (int c = 0; c < 8; c++) h[c] = v[c];
      if (TAIL && pass_b) {
        float p = sW[80];
#pragma unroll
        for (int o = 0; o < 8; o++) p = fmaf(sW[72 + o], fmaf(sAc[16 + o], h[o], sAc[24 + o]), p);
        p_net[row * g.nx + x] = p;
        continue;
      }
#pragma unroll
      for (int c = 0; c < 8; c++) {
        const double d = (double)h[c] - (double)K[c];
        s[c] += d;
        q[c] = fma(d, d, q[c]);
      }
    }
  }
  if (TAIL && pass_b) return;       // uniform over the launch
  tc_bn_write(s, q, K, sh, part);
}

__global__ void k_tc_bn_apply(float4* __restrict__ buf, ConvTcGeo g, const float* __restrict__ ac, long long total) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const TcRows r = tc_rows(g);
  const long long row = t / g.nx;
  const long long i = tc_row_base(g, r, row) + (t - row * g.nx);
  float4 a = buf[i], b = buf[i + r.plane];
  a = make_float4(fmaf(__ldg(ac + 0), a.x, __ldg(ac + 8)), fmaf(__ldg(ac + 1), a.y, __ldg(ac + 9)),
                  fmaf(__ldg(ac + 2), a.z, __ldg(ac + 10)), fmaf(__ldg(ac + 3), a.w, __ldg(ac + 11)));
  b = make_float4(fmaf(__ldg(ac + 4), b.x, __ldg(ac + 12)), fmaf(__ldg(ac + 5), b.y, __ldg(ac + 13)),
                  fmaf(__ldg(ac + 6), b.z, __ldg(ac + 14)), fmaf(__ldg(ac + 7), b.w, __ldg(ac + 15)));
  buf[i] = a;
  buf[i + r.plane] = b;
}

template <int COUT, int KS, bool IS3D, bool DIL>
static bool conv_launch(const float* in, float* out, const float* w, const float* b, int cin, int act,
                        const Geo& g, int dil, cudaStream_t st) {
  const int nzr = g.zhi - g.zlo;
  dim3 block = IS3D ? dim3(32, 4, 2) : dim3(32, 8, 1);
  dim3 grid((g.nx + block.x - 1) / block.x, (g.ny + block.y - 1) / block.y,
            ((long long)g.nb * nzr + block.z - 1) / block.z);
  constexpr int KZ = IS3D ? KS : 1;
  const size_t smem = sizeof(float) * cin * KZ * KS * KS * COUT;
  if (smem > 200 * 1024) return false;             // weights do not fit shared memory: generic kernel
  if (smem > 48 * 1024) {
    static size_t allowed[64];                     // per instantiation and device (function attributes are per device)
    int dev = 0;
    cudaGetDevice(&dev);
    if (smem > allowed[dev & 63]) {
      if (cudaFuncSetAttribute(k_conv_direct<COUT, KS, IS3D, DIL>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               (int)smem) != cudaSuccess) {
        cudaGetLastError();
        return false;
      }
      allowed[dev & 63] = smem;
    }
  }
  k_conv_direct<COUT, KS, IS3D, DIL><<<grid, block, smem, st>>>(in, out, w, b, cin, act, g, dil);
  return true;
}

int launch_conv_direct(const float* in, float* out, const float* wdev, const float* bdev, int cin, int cout,
                       int ksize, int act, const Geo& g, cudaStream_t st, int dil) {
#define TFL_CONV_CASE(CO, KS_)                                                                          \
  if (cout == CO && ksize == KS_) {                                                                     \
    const bool ok_ = dil > 1 ? (g.is3d ? conv_launch<CO, KS_, true, true>(in, out, wdev, bdev, cin, act, g, dil, st)  \
                                       : conv_launch<CO, KS_, false, true>(in, out, wdev, bdev, cin, act, g, dil, st)) \
                             : (g.is3d ? conv_launch<CO, KS_, true, false>(in, out, wdev, bdev, cin, act, g, 1, st)    \
                                       : conv_launch<CO, KS_, false, false>(in, out, wdev, bdev, cin, act, g, 1, st)); \
    if (ok_) return kConvDirect;                                                                        \
  }
  TFL_CONV_CASE(8, 3) TFL_CONV_CASE(8, 1) TFL_CONV_CASE(1, 1) TFL_CONV_CASE(16, 3) TFL_CONV_CASE(16, 1)
  TFL_CONV_CASE(1, 3) TFL_CONV_CASE(6, 3) TFL_CONV_CASE(6, 1) TFL_CONV_CASE(32, 1) TFL_CONV_CASE(16, 5)
  TFL_CONV_CASE(32, 5) TFL_CONV_CASE(64, 5) TFL_CONV_CASE(64, 1)
#undef TFL_CONV_CASE
  return launch_conv_any(in, out, wdev, bdev, cin, cout, ksize, act, g, st, dil);
}

int launch_conv_any(const float* in, float* out, const float* wdev, const float* bdev, int cin, int cout, int ksize,
                    int act, const Geo& g, cudaStream_t st, int dil) {
  if (g.zlo != 0 || g.zhi != g.nz || g.zoff != 0) return -1;      // the generic kernel works on whole grids only
  const long long total = (long long)g.nb * cout * g.n;
  if (dil > 1)
    k_conv_any<true><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(in, out, wdev, bdev, cin, cout, ksize, act, g, dil);
  else
    k_conv_any<false><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(in, out, wdev, bdev, cin, cout, ksize, act, g, 1);
  return kConvGeneric;
}

void launch_pool(const float* in, float* out, int nbc, int nz, int ny, int nx, int p, int is3d, int is_max,
                 cudaStream_t st) {
  const int pz = is3d ? p : 1;
  const long long total = (long long)nbc * (nz / pz) * (ny / p) * (nx / p);
  k_pool<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(in, out, nz, ny, nx, p, is3d, is_max, total);
}
void launch_pixel_shuffle(const float* in, float* out, int nb, int n_out, int nz, int ny, int nx, int s, int is3d,
                          cudaStream_t st) {
  const long long total = (long long)nb * n_out * nz * (is3d ? s : 1) * ny * s * nx * s;
  k_pixel_shuffle<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(in, out, n_out, nz, ny, nx, s, is3d, total);
}
int launch_bank_join(const float* const* banks, int nbanks, float* out, int nb, int c, int nz, int ny, int nx,
                     int is3d, int add, cudaStream_t st, int full) {
  if (nbanks < 2 || nbanks > kMaxBankPtrs) return -1;
  BankPtrs bp = {};
  for (int i = 1; i < nbanks; i++) bp.p[i] = banks[i];
  const long long total = (long long)nb * c * nz * ny * nx;
  if (full)
    k_bank_join<true><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(bp, nbanks, out, c, nz, ny, nx, is3d, add, total);
  else
    k_bank_join<false><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(bp, nbanks, out, c, nz, ny, nx, is3d, add, total);
  return 1;
}

void launch_bn_stats(const float* x, int nb, int c, long long n, long long bstride, double* part, cudaStream_t st) {
  k_bn_stats<<<dim3(kBnBlocks, c), kBnThreads, 0, st>>>(x, n, nb, bstride, part);
}
void launch_bn_finalize(const double* part, int c, long long count, const float* w, const float* b, float eps,
                        float* ac, double* stats, cudaStream_t st) {
  k_bn_finalize<<<c, kBnThreads, 0, st>>>(part, kBnBlocks, c, count, w, b, eps, ac, stats);
}
void launch_tc_bn_stats(const float* buf, const ConvTcGeo& g, double* part, cudaStream_t st) {
  k_tc_bn_rows<false><<<kBnBlocks, kBnThreads, 0, st>>>((const float4*)buf, g, nullptr, nullptr, 0, 0, part, nullptr,
                                                         nullptr);
}
void launch_tc_bn_apply(float* buf, const ConvTcGeo& g, const float* ac, cudaStream_t st) {
  const long long total = (long long)g.nb * g.nz * g.ny * g.nx;
  k_tc_bn_apply<<<(unsigned)((total + 255) / 256), 256, 0, st>>>((float4*)buf, g, ac, total);
}
void launch_tc_bn_tail(const float* buf, const ConvTcGeo& g, const float* ac3, const float* tail, int relu6,
                       int pass_b, double* part, const float* ac4, float* p_net, cudaStream_t st) {
  k_tc_bn_rows<true><<<kBnBlocks, kBnThreads, 0, st>>>((const float4*)buf, g, ac3, tail, relu6, pass_b, part, ac4,
                                                        p_net);
}
void launch_bn_apply(float* x, int nb, int c, long long n, long long bstride, const float* ac, cudaStream_t st) {
  const long long total = (long long)nb * c * n;
  k_bn_apply<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(x, c, n, bstride, ac, total);
}

}  // namespace tfl
