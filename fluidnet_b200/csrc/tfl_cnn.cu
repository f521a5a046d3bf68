// Convolution stack of the pressure-projection network (torch/lib/model.lua:262-364:
// stride-1 zero-padded cross-correlation + bias (+ReLU), cudnn.Volumetric/Spatial
// Convolution in the reference, torch/lib/model_utils.lua:74-116).
//
// This file holds the fp32 FMA path: one thread per output voxel computing all output
// channels from shared-memory weights.  It is the numerically tight (1e-5 class)
// implementation and the parity anchor for the tensor-core path (tfl_cnn_tc.cu).
#include "tfl_device.cuh"
#include "tfl_kernels.h"

namespace tfl {

// Non-linearity between layers (torch.addNonlinearity, lib/model_utils.lua): 0 none, 1 ReLU, 2 sigmoid.
__device__ __forceinline__ float activate(float r, int act) {
  if (act == 1) return r < 0.0f ? 0.0f : r;
  if (act == 2) return 1.0f / (1.0f + expf(-r));
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

}  // namespace tfl
