// Tensor-core (Hopper wgmma) implementation of the 3x3x3 convolution layers of the 3-D
// pressure-projection network (torch/lib/model.lua:219-226: 3->8, 8->8, 8->8 with k=3, then
// 8->8 and 8->1 with k=1, ReLU between layers).  sm_90a only.
//
// Formulation (implicit GEMM, no im2col buffer):
//   * activations live in global memory channels-last in two float4 planes (channels 0-3 and
//     4-7) over a grid padded by one zero voxel on every side, so halo loads need no bounds
//     tests and the zero padding of the convolution is simply "there";
//   * a CTA stages a (32 x PY x PZ)-position box of both planes into shared memory
//     (cp.async, 16 B per position and plane).  In that box the positions are LINEAR
//     (x fastest, pitch 32), so ANY 64 consecutive positions form a valid K-major,
//     no-swizzle wgmma A operand: 8-row core matrices are 128 B apart (SBO), the two
//     4-channel K chunks are one plane apart (LBO), and shifting the operand by a filter
//     tap (dy, dz) is a pure start-address offset;
//   * the three x-taps of a (dy, dz) pair share ONE A operand: B holds their weights side by
//     side (N = 3 taps x 8 output channels = 24), so 9 wgmma (M=64, N=24, K=8, tf32 inputs,
//     fp32 accumulate in registers) cover the 27 taps, and the x shift is applied in the
//     epilogue: out[x] = D_{-1}[x-1] + D_0[x] + D_{+1}[x+1].  An M tile is 2 rows of 32
//     x-positions; the accumulators go through a small shared-memory buffer per warpgroup
//     so that every thread can read its x-1 / x+1 neighbours;
//   * 3xTF32 mode (SPLIT): A and B are split into tf32 "hi" and fp32-residual "lo" parts;
//     hi*hi, hi*lo (same wgmma, N = 48) and lo*hi (second wgmma, N = 24) are accumulated,
//     which restores ~fp32 accuracy at 2x the MMA count;
//   * the epilogue adds bias, applies ReLU and either writes the next layer's padded
//     channels-last planes or, for the last 3x3x3 layer, also runs the two 1x1x1 layers and
//     writes the pressure.
// Two warpgroups per CTA take alternate M tiles; two CTAs per SM overlap one CTA's loads with
// the other's math (the boxes are sized so that two fit the SM's 228 KB of shared memory).
#include <cuda_runtime.h>
#include <stdint.h>

#include "tfl_cnn_tc.h"

namespace tfl {

namespace {

constexpr int kTX = 32;                 // positions per row in the staged box (30 outputs + 2 halo)
constexpr int kGroups = 9;              // (dz, dy) pairs
constexpr int kThreads = 256;           // 2 warpgroups
constexpr int kDPitch = 24;             // floats per position in the accumulator staging buffer

// CTA box: 3xTF32 keeps 4 planes (hi/lo x 2 channel groups) in shared memory, so its box is
// smaller to still fit two CTAs per SM.
template <bool SPLIT> struct Tile {
  static constexpr int TY = SPLIT ? 4 : 8;      // output rows per CTA (multiple of 2)
  static constexpr int TZ = SPLIT ? 5 : 6;      // output planes per CTA
  static constexpr int PY = TY + 2, PZ = TZ + 2;
  static constexpr int RB = TY / 2;             // 2-row blocks (= M tiles) per plane
  static constexpr int POS = kTX * PY * PZ;
  static constexpr int PLANE_BYTES = POS * 16;
  static constexpr int MTILES = TZ * RB;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
// K-major, no-swizzle wgmma shared-memory matrix descriptor: start address, leading byte offset
// (between the two 16-byte K chunks) and stride byte offset (between 8-row core matrices), all
// in 16-byte units.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  return d;
}
// D[64 x 24] (+)= A[64 x 8] * B[8 x 24], tf32 inputs, fp32 accumulators in registers.
__device__ __forceinline__ void wgmma_n24(float (&d)[12], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %14, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n24k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11}, %12, %13, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11])
      : "l"(da), "l"(db), "r"(accumulate));
}
// D[64 x 48] (+)= A[64 x 8] * B[8 x 48].
__device__ __forceinline__ void wgmma_n48(float (&d)[24], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %26, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n48k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, "
      "%24, %25, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
      : "l"(da), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wg_barrier(int id) {
  asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory");
}
__device__ __forceinline__ float4 tf32_hi(float4 v) {
  float4 h;
  h.x = __uint_as_float(__float_as_uint(v.x) & 0xFFFFE000u);
  h.y = __uint_as_float(__float_as_uint(v.y) & 0xFFFFE000u);
  h.z = __uint_as_float(__float_as_uint(v.z) & 0xFFFFE000u);
  h.w = __uint_as_float(__float_as_uint(v.w) & 0xFFFFE000u);
  return h;
}

__device__ long long* g_tc_dbg = nullptr;   // optional phase timestamps (tests/dbg only)

template <int IN_PLANES, bool FINAL, bool SPLIT>
__global__ void __launch_bounds__(kThreads, 2)
k_conv3_tc(const float4* __restrict__ in, float4* __restrict__ out, float* __restrict__ p_net,
           const float* __restrict__ wB, const float* __restrict__ bias, const float* __restrict__ tail,
           ConvTcGeo g) {
  extern __shared__ __align__(1024) uint8_t smem[];
  using T = Tile<SPLIT>;
  constexpr int NB = SPLIT ? 48 : 32;
  constexpr int A_BYTES = (SPLIT ? 4 : 2) * T::PLANE_BYTES;
  constexpr int B_GROUP_BYTES = 2 * NB * 16;
  constexpr int B_BYTES = kGroups * B_GROUP_BYTES;
  uint8_t* sA = smem;
  uint8_t* sB = smem + A_BYTES;
  float* sD = (float*)(smem + A_BYTES + B_BYTES);            // [2 warpgroups][64][kDPitch]
  float* sTail = sD + 2 * 64 * kDPitch;                      // bias[8] (+ w4[64] b4[8] w5[8] b5[1] when FINAL)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tx = blockIdx.x, ty = blockIdx.y;
  long long* dbg = g_tc_dbg;
  const int cta_lin = (blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
  if (dbg && tid == 0) dbg[cta_lin * 8 + 0] = clock64();
  const int tzb = blockIdx.z % g.ntz, b = blockIdx.z / g.ntz;

  // ---- stage the input box ------------------------------------------------------------
  const long long plane_g = (long long)(g.nz + 2) * g.py * g.px;            // float4 per global plane
  const long long batch_g = plane_g * 2;
  const int x0 = tx * 30, y0 = ty * T::TY, z0 = g.z_lo + tzb * T::TZ;         // padded coords of box origin
  const float4* inb = in + b * batch_g;
  if (!SPLIT) {
    for (int idx = tid; idx < T::POS; idx += kThreads) {
      const int l = idx & 31, r = idx >> 5;
      const int yy = r % T::PY, zz = r / T::PY;
      int gx = x0 + l, gy = y0 + yy, gz = z0 + zz;
      const bool inside = gx < g.px && gy < g.py && gz < g.nz + 2;
      gx = inside ? gx : 0; gy = inside ? gy : 0; gz = inside ? gz : 0;      // (0,0,0) is a zero border voxel
      const long long go = ((long long)gz * g.py + gy) * g.px + gx;
#pragma unroll
      for (int h = 0; h < IN_PLANES; h++)
        cp_async16(smem_u32(sA + h * T::PLANE_BYTES + idx * 16), inb + h * plane_g + go);
      if (IN_PLANES == 1) *(float4*)(sA + T::PLANE_BYTES + idx * 16) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  } else {
    // 3xTF32: the hi/lo split happens in registers on the way in.  All loads are issued
    // before the first use so that one memory round trip covers the whole box.
    constexpr int PER = (T::POS + kThreads - 1) / kThreads;
    float4 v[PER][IN_PLANES];
#pragma unroll
    for (int it = 0; it < PER; it++) {
      const int idx = tid + it * kThreads;
      const int l = idx & 31, r = idx >> 5;
      const int yy = r % T::PY, zz = r / T::PY;
      int gx = x0 + l, gy = y0 + yy, gz = z0 + zz;
      const bool inside = idx < T::POS && gx < g.px && gy < g.py && gz < g.nz + 2;
      gx = inside ? gx : 0; gy = inside ? gy : 0; gz = inside ? gz : 0;
      const long long go = ((long long)gz * g.py + gy) * g.px + gx;
#pragma unroll
      for (int h = 0; h < IN_PLANES; h++) v[it][h] = __ldg(inb + h * plane_g + go);
    }
#pragma unroll
    for (int it = 0; it < PER; it++) {
      const int idx = tid + it * kThreads;
      if (idx < T::POS) {
#pragma unroll
        for (int h = 0; h < 2; h++) {
          float4 hi = make_float4(0.f, 0.f, 0.f, 0.f), lo = hi;
          if (h < IN_PLANES) {
            const float4 w = v[it][h < IN_PLANES ? h : 0];
            hi = tf32_hi(w);
            lo = make_float4(w.x - hi.x, w.y - hi.y, w.z - hi.z, w.w - hi.w);
          }
          *(float4*)(sA + h * T::PLANE_BYTES + idx * 16) = hi;
          *(float4*)(sA + (2 + h) * T::PLANE_BYTES + idx * 16) = lo;
        }
      }
    }
  }
  for (int i = tid; i < B_BYTES / 16; i += kThreads) cp_async16(smem_u32(sB + i * 16), (const float4*)wB + i);
  const int n_tail = FINAL ? (8 + 64 + 8 + 8 + 1) : 8;
  for (int i = tid; i < n_tail; i += kThreads) sTail[i] = (i < 8) ? bias[i] : tail[i - 8];
  asm volatile("cp.async.commit_group;" ::: "memory");
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  // generic-proxy writes (st.shared, cp.async) -> visible to the wgmma (async proxy) reads
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  if (dbg && tid == 0) { dbg[cta_lin * 8 + 1] = clock64(); unsigned smid; asm("mov.u32 %0, %%smid;" : "=r"(smid)); dbg[cta_lin * 8 + 7] = smid; }

  // ---- warpgroup wg takes M tiles t = wg, wg + 2, ... ------------------------------------
  const int wg = warp >> 2, wq = warp & 3;
  const uint32_t sA_u = smem_u32(sA), sB_u = smem_u32(sB);
  constexpr uint32_t LO_PLANES_16 = (uint32_t)(2 * T::PLANE_BYTES) >> 4;
  float* myD = sD + wg * 64 * kDPitch;
  const float* sBias = sTail;
  const int tw = tid & 127, p = tw >> 1, half = tw & 1;     // epilogue: position p, channels 4*half..+3
  const int xl = p & 31, ry = p >> 5;
  const int pm = xl > 0 ? p - 1 : p, pp = xl < 31 ? p + 1 : p;
  for (int t = wg; t < T::MTILES; t += 2) {
    // M tile t: padded plane 1 + t / RB, rows 1 + 2 * (t % RB) .. +1, positions 0..31.
    const uint32_t toff = (uint32_t)((((t / T::RB) * T::PY + 2 * (t % T::RB)) * kTX) * 16);
    float acc[SPLIT ? 24 : 12] = {}, acl[12] = {};
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
    for (int gi = 0; gi < kGroups; gi++) {
      const int dz = gi / 3 - 1, dy = gi % 3 - 1;
      const uint32_t a_addr = sA_u + toff + (uint32_t)((((1 + dz) * T::PY + (1 + dy)) * kTX) * 16);
      const uint64_t da = make_desc(a_addr, T::PLANE_BYTES, 128);
      const uint64_t db = make_desc(sB_u + gi * B_GROUP_BYTES, NB * 16, 128);
      if constexpr (SPLIT) {
        wgmma_n48(acc, da, db, gi > 0 ? 1u : 0u);
        wgmma_n24(acl, da + LO_PLANES_16, db, gi > 0 ? 1u : 0u);
      } else {
        wgmma_n24(acc, da, db, gi > 0 ? 1u : 0u);
      }
    }
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
    if (dbg && tid == 0 && t == 0) dbg[cta_lin * 8 + 2] = clock64();

    // accumulator fragment: element (row 16 wq + lane / 4 + 8 i, column 8 k + 2 (lane % 4) + j) is acc[4 k + 2 i + j]
#pragma unroll
    for (int k = 0; k < 3; k++)
#pragma unroll
      for (int i = 0; i < 2; i++) {
        const int row = 16 * wq + (lane >> 2) + 8 * i, col = 8 * k + 2 * (lane & 3);
        float2 v;
        if constexpr (SPLIT) {
          v.x = acc[4 * k + 2 * i] + (acc[12 + 4 * k + 2 * i] + acl[4 * k + 2 * i]);
          v.y = acc[4 * k + 2 * i + 1] + (acc[12 + 4 * k + 2 * i + 1] + acl[4 * k + 2 * i + 1]);
        } else {
          v.x = acc[4 * k + 2 * i];
          v.y = acc[4 * k + 2 * i + 1];
        }
        *(float2*)(myD + row * kDPitch + col) = v;
      }
    wg_barrier(1 + wg);

    const float4 dm = *(const float4*)(myD + pm * kDPitch + 4 * half);
    const float4 d0 = *(const float4*)(myD + p * kDPitch + 8 + 4 * half);
    const float4 dp = *(const float4*)(myD + pp * kDPitch + 16 + 4 * half);
    const float* bs = sBias + 4 * half;
    float h[4];
    h[0] = (dm.x + d0.x) + dp.x + bs[0];
    h[1] = (dm.y + d0.y) + dp.y + bs[1];
    h[2] = (dm.z + d0.z) + dp.z + bs[2];
    h[3] = (dm.w + d0.w) + dp.w + bs[3];
#pragma unroll
    for (int o = 0; o < 4; o++) h[o] = h[o] > 0.0f ? h[o] : 0.0f;
    const int xg = x0 + xl - 1;                         // unpadded coordinates of this position's voxel
    const int yg = y0 + 2 * (t % T::RB) + ry;
    const int zg = z0 + t / T::RB;
    const bool valid = xl >= 1 && xl <= 30 && xg < g.nx && yg < g.ny && zg < g.z_hi;
    if (!FINAL) {
      if (valid) {
        const long long o = b * batch_g + ((long long)(zg + 1) * g.py + (yg + 1)) * g.px + (xg + 1);
        out[o + half * plane_g] = make_float4(h[0], h[1], h[2], h[3]);
      }
    } else {
      float hh[8];
#pragma unroll
      for (int o = 0; o < 4; o++) {
        const float other = __shfl_xor_sync(0xffffffffu, h[o], 1);
        hh[o] = half ? other : h[o];
        hh[4 + o] = half ? h[o] : other;
      }
      const float* w4 = sTail + 8;      // [o][c]
      const float* b4 = w4 + 64;
      const float* w5 = b4 + 8;
      const float b5 = w5[8];
      float pacc = b5;
#pragma unroll
      for (int o = 0; o < 8; o++) {
        float a = b4[o];
#pragma unroll
        for (int c = 0; c < 8; c++) a = fmaf(hh[c], w4[o * 8 + c], a);
        a = a > 0.0f ? a : 0.0f;
        pacc = fmaf(a, w5[o], pacc);
      }
      if (valid && half == 0) p_net[(long long)b * g.nz * g.ny * g.nx + ((long long)zg * g.ny + yg) * g.nx + xg] = pacc;
    }
    wg_barrier(1 + wg);                                 // myD is rewritten by the next tile
  }
  if (dbg) {
    __syncthreads();
    if (tid == 0) dbg[cta_lin * 8 + 5] = clock64();
  }
}

template <int IN_PLANES, bool FINAL, bool SPLIT>
void launch_one(const float4* in, float4* out, float* p_net, const float* wB, const float* bias,
                const float* tail, const ConvTcGeo& g, cudaStream_t st) {
  using T = Tile<SPLIT>;
  constexpr int NB = SPLIT ? 48 : 32;
  const size_t smem = (size_t)(SPLIT ? 4 : 2) * T::PLANE_BYTES + kGroups * 2 * NB * 16 + 2 * 64 * kDPitch * 4 + 4 * 96;
  auto kern = k_conv3_tc<IN_PLANES, FINAL, SPLIT>;
  static unsigned long long configured = 0;       // per device (function attributes are)
  int dev = 0;
  cudaGetDevice(&dev);
  if (!((configured >> (dev & 63)) & 1ULL)) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    configured |= 1ULL << (dev & 63);
  }
  const int ntz = (g.z_hi - g.z_lo + T::TZ - 1) / T::TZ;       // output planes [z_lo, z_hi)
  ConvTcGeo gg = g;
  gg.ntz = ntz;
  gg.nty = (g.ny + T::TY - 1) / T::TY;
  dim3 grid(g.ntx, gg.nty, ntz * g.nb);
  kern<<<grid, kThreads, smem, st>>>(in, out, p_net, wB, bias, tail, gg);
}

}  // namespace

ConvTcGeo make_conv_tc_geo(int nb, int nz, int ny, int nx) {
  ConvTcGeo g;
  g.nb = nb; g.nx = nx; g.ny = ny; g.nz = nz;
  g.ntx = (nx + 29) / 30;
  g.nty = 0;
  g.ntz = 0;                         // depends on the arithmetic mode; set at launch
  g.z_lo = 0;
  g.z_hi = nz;
  g.px = (nx + 2 + 3) & ~3;
  g.py = ny + 2;
  return g;
}
size_t conv_tc_act_bytes(const ConvTcGeo& g) {
  return (size_t)g.nb * 2 * (g.nz + 2) * g.py * g.px * 16;
}
void conv_tc_set_debug(long long* dev_buf) { cudaMemcpyToSymbol(g_tc_dbg, &dev_buf, sizeof(dev_buf)); }

int conv_tc_b_floats(int split) { return kGroups * 2 * (split ? 48 : 32) * 4; }

// Host-side packing of one layer's weights [cout=8][cin][3][3][3] into the B operand blocks
// (tf32 "hi" truncation and fp32 residual "lo" when split).
void conv_tc_pack_weights(const float* w, int cin, int split, float* out) {
  const int NB = split ? 48 : 32;
  for (int i = 0; i < kGroups * 2 * NB * 4; i++) out[i] = 0.0f;
  for (int dz = 0; dz < 3; dz++)
    for (int dy = 0; dy < 3; dy++) {
      float* blk = out + (size_t)(dz * 3 + dy) * 2 * NB * 4;
      for (int kx = 0; kx < 3; kx++)
        for (int o = 0; o < 8; o++)
          for (int c = 0; c < cin; c++) {
            const float v = w[((((size_t)o * cin + c) * 3 + dz) * 3 + dy) * 3 + kx];
            union { float f; uint32_t u; } hi;
            hi.f = v;
            if (split) hi.u &= 0xFFFFE000u;
            const int n = kx * 8 + o;
            blk[((c >> 2) * NB + n) * 4 + (c & 3)] = hi.f;
            if (split) blk[((c >> 2) * NB + 24 + n) * 4 + (c & 3)] = v - hi.f;
          }
    }
}

int launch_conv3_tc(const float* in, float* out, float* p_net, const float* wB, const float* bias,
                    const float* tail, int in_planes, int final_layer, int split, const ConvTcGeo& g,
                    cudaStream_t st) {
  const float4* i4 = (const float4*)in;
  float4* o4 = (float4*)out;
#define TFL_TC_CASE(P, F, S)                                                   \
  if (in_planes == P && (final_layer != 0) == F && (split != 0) == S) {        \
    launch_one<P, F, S>(i4, o4, p_net, wB, bias, tail, g, st);                 \
    return 1;                                                                  \
  }
  TFL_TC_CASE(1, false, false) TFL_TC_CASE(2, false, false) TFL_TC_CASE(2, true, false)
  TFL_TC_CASE(1, false, true) TFL_TC_CASE(2, false, true) TFL_TC_CASE(2, true, true)
#undef TFL_TC_CASE
  return -1;
}

}  // namespace tfl
