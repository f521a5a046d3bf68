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
//     epilogue: out[x] = D_{-1}[x-1] + D_0[x] + D_{+1}[x+1].  Layer 1 (3 channels, one plane)
//     puts two (dy, dz) taps into the two K chunks instead, 5 wgmma (see Layout).  An M tile is 2 rows of 32
//     x-positions; the accumulators go through a small shared-memory buffer per warpgroup
//     so that every thread can read its x-1 / x+1 neighbours;
//   * 3xTF32 mode (SPLIT): A and B are split into tf32 "hi" and fp32-residual "lo" parts;
//     hi*hi, hi*lo (same wgmma, N = 48) and lo*hi (second wgmma, N = 24) are accumulated,
//     which restores ~fp32 accuracy at 2x the MMA count;
//   * the epilogue adds bias, applies ReLU and either writes the next layer's padded
//     channels-last planes or, for the last 3x3x3 layer, also runs the two 1x1x1 layers and
//     writes the pressure.
// Two warpgroups per CTA take alternate M tiles; two CTAs per SM overlap one CTA's loads with
// the other's math (the boxes are sized so that two fit the SM's 228 KB of shared memory).  The
// box kernel k_conv3_tc runs the join layer of banked models and layers 1-3 at nx > kWWMax.
//
// Layers 1-3 at nx <= kWWMax (k_conv3_tc_z): a persistent CTA (one per SM, four consumer warpgroups
// and one producer warpgroup) takes work items of TY output rows x the whole row x ZC output planes x
// one batch entry and streams along z through a ring of three staged planes.  A staged row is padded
// x = 1 .. ww (ww = 64 or kWWMax), so no x halo is staged or computed: D of the zero border voxels
// x = 0 and x = nx + 1 is zero and the epilogue uses 0 for it, and at nx = 128 a row is exactly two M
// tiles of 64.  The producer loads the next plane into registers, splits and stores it as soon as the
// consumers have released its slot (mbarrier `empty`) and hands it over (mbarrier `full`); the
// consumers release a slot as soon as their MMAs on it have completed, so that their epilogues overlap
// the producer's stores and the other warpgroups' MMAs.
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

// Shared-memory layout of one layer: the staged planes (hi, then lo when SPLIT), the B groups, the
// accumulator staging buffer and the bias / tail constants.
//   IN_PLANES == 2: planes [c0-3 | c4-7] (x hi/lo), 9 B groups, one (dz, dy) tap per group; K chunk 1
//                   is the second channel group, one plane further (LBO = PLANE_BYTES).
//   IN_PLANES == 1: (layer 1, 3 channels) every plane is followed by 64 zero positions and the two K
//                   chunks of a group are two taps of the same 4 channels (layer1_dz / _dy), so 5 B groups
//                   cover the 9 (dz, dy) taps.
template <int IN_PLANES, bool SPLIT> struct Layout {
  using T = Tile<SPLIT>;
  static constexpr int NB = SPLIT ? 48 : 32;
  static constexpr int GROUPS = IN_PLANES == 1 ? 5 : kGroups;
  static constexpr int ZERO_BYTES = IN_PLANES == 1 ? 64 * 16 : 0;
  static constexpr int PSTRIDE = T::PLANE_BYTES + ZERO_BYTES;     // bytes between staged planes
  static constexpr int LO_OFF = IN_PLANES * PSTRIDE;               // hi -> lo operand (SPLIT)
  static constexpr int A_BYTES = (SPLIT ? 2 : 1) * LO_OFF;
  static constexpr int B_GROUP_BYTES = 2 * NB * 16;
  static constexpr int B_BYTES = GROUPS * B_GROUP_BYTES;
  static constexpr int BYTES = A_BYTES + B_BYTES + 2 * 64 * kDPitch * 4 + 4 * 96;
};

// Layers 1-3 at nx <= kWWMax: four consumer warpgroups (the MMAs and the epilogues) and one producer warpgroup
// (loads, hi / lo split and stores of the staged planes); a staged row holds ww = 64 or kWWMax positions.
constexpr int kZWarpGroups = 4;                             // consumers
constexpr int kZThreads = 128 * (kZWarpGroups + 1);
constexpr int kWWMax = 128;
// Registers per thread: 640 threads launch with 96 (65536 / 640, rounded down to the allocation unit of 8), then
// setmaxnreg moves them between the warpgroups.  3xTF32: the producer holds one plane (6 positions x 2 float4 per
// thread) in 64, the consumers get 104 (128 x 64 + 512 x 104 = 640 x 96).  TF32 stages 10 rows per plane (10 positions
// x 2 float4 per producer thread), so there the producer takes 128 and the consumers, with one accumulator set of 12,
// keep 88.
constexpr int kZLaunchRegs = 96;
template <bool SPLIT> struct ZRegs {
  static constexpr int PRODUCER = SPLIT ? 64 : 128;
  static constexpr int CONSUMER = SPLIT ? 104 : 88;
  static_assert(128 * PRODUCER + 128 * kZWarpGroups * CONSUMER <= kZThreads * kZLaunchRegs, "register file");
};
// Bounded mbarrier waits: a wait that has not completed after this many clock cycles (about a second) records a fault
// in g_tc_z_fault, and every later wait of the CTA returns at once, so a pipeline bug ends the kernel with an error
// instead of hanging the device.
constexpr long long kZSpinCycles = 1ll << 31;

// Shared memory of k_conv3_tc_z for staged rows of ww positions:
//   ring   3 slots; a slot is one staged padded plane, PY rows x ww positions, as two 16-byte K chunks
//          [chunk 0 | chunk 1] of GB = PY * ww * 16 bytes each (hi, then lo when SPLIT, LO = 2 GB further);
//          IN_PLANES == 2: chunk c is channel group c of the plane (LBO = GB);
//          IN_PLANES == 1: (layer 1, 3 channels) chunk 0 is the plane and chunk 1 the NEXT plane, so the two
//          K chunks of a group are the taps (dz, dy) and (dz + 1, dy) (LBO = GB); every staged plane is
//          written twice, into its own slot's chunk 0 and the previous plane's chunk 1.  Group 3 pairs the
//          rows (dz, dy) = (1, -1) / (1, 0) of chunk 0 (LBO = one row), group 4 is the single tap (1, 1)
//          whose chunk 1 reads 64 zero positions (its B rows are zero too, but 0 * NaN would not be);
//   zeros  (layer 1) 64 positions;
//   B      the weight groups; D: one row buffer of ww x kDPitch floats per consumer warpgroup; then bias / tail;
//   bars   mbarriers full[3], empty[3] of the ring slots and the CTA's abort flag (64 bytes).
template <int IN_PLANES, bool SPLIT> struct ZLayout {
  static constexpr int TY = SPLIT ? 4 : 8;      // output rows of a work item
  static constexpr int PY = TY + 2;
  static constexpr int NB = SPLIT ? 48 : 32;
  static constexpr int GROUPS = IN_PLANES == 1 ? 5 : kGroups;
  static constexpr int ZERO_BYTES = IN_PLANES == 1 ? 64 * 16 : 0;
  static constexpr int B_GROUP_BYTES = 2 * NB * 16;
  static constexpr int B_BYTES = GROUPS * B_GROUP_BYTES;
  static constexpr int SLOT_CHUNKS = SPLIT ? 4 : 2;
  static constexpr size_t bytes(int ww) {
    return (size_t)3 * SLOT_CHUNKS * PY * ww * 16 + ZERO_BYTES + B_BYTES + (size_t)kZWarpGroups * ww * kDPitch * 4 +
           4 * 96 + 64;
  }
};

// Work decomposition of one k_conv3_tc_z launch: item = (b * nzc + zc) * nty + ty.
struct ZSched {
  int ww;        // staged positions per row: padded x = 1 .. ww (64 or kWWMax, >= nx)
  int nty;       // TY-row blocks
  int zc, nzc;   // output planes per item, z chunks
  int items;
};

// Layer 1 (one 4-channel plane): group gi's K chunk 0 is tap (layer1_dz(gi), layer1_dy(gi)); K chunk 1
// is the tap one z-plane further for gi < 3 (dz = -1 / 0 pairs), one row further for gi == 3
// ((dz, dy) = (1, -1) / (1, 0)), and zeros for gi == 4 (the single tap (1, 1)).
__host__ __device__ constexpr int layer1_dz(int gi) { return gi < 3 ? -1 : 1; }
__host__ __device__ constexpr int layer1_dy(int gi) { return gi < 3 ? gi - 1 : (gi == 3 ? -1 : 1); }

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
__device__ __forceinline__ void mbar_init(uint32_t bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(done)
      : "r"(bar), "r"(parity)
      : "memory");
  return done != 0;
}

__device__ unsigned int g_tc_z_fault = 0;   // k_conv3_tc_z: 1 once a wait of its pipeline ran out (kZSpinCycles)

// Waits for the completion of phase `parity` of the mbarrier at `bar`, for at most kZSpinCycles.  A wait that runs
// out records the fault and raises the CTA's abort flag; once it is raised, every wait returns at once.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, volatile int* abort) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (*abort) return;
    if (clock64() - t0 > kZSpinCycles) {
      *abort = 1;
      atomicOr(&g_tc_z_fault, 1u);
      return;
    }
  }
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

// The non-linearity of the epilogues: ReLU, or nn.ReLU6 (min(max(x, 0), 6)).
__device__ __forceinline__ float tc_act(float v, int relu6) {
  v = v > 0.0f ? v : 0.0f;
  return relu6 && v > 6.0f ? 6.0f : v;
}

// Bias, ReLU and (FINAL) the two 1x1x1 layers of one position's 4 channels (4 * half ..), as the two threads of a
// position share them; writes the next layer's padded plane or the pressure when `valid`.
template <bool FINAL>
__device__ __forceinline__ void conv_epilogue(float (&h)[4], bool valid, int half, const float* sTail, float4* out,
                                              float* p_net, long long out_idx, long long plane_g, long long p_idx,
                                              const TcEpi& ep) {
#pragma unroll
  for (int o = 0; o < 4; o++) h[o] = tc_act(h[o], ep.relu6);
  if constexpr (!FINAL) {
    if (ep.ac) {                                  // running-statistics BN after the activation (valid voxels only)
#pragma unroll
      for (int o = 0; o < 4; o++) h[o] = fmaf(sTail[8 + 4 * half + o], h[o], sTail[16 + 4 * half + o]);
    }
    if (valid) out[out_idx + half * plane_g] = make_float4(h[0], h[1], h[2], h[3]);
  } else {
    float hh[8];
#pragma unroll
    for (int o = 0; o < 4; o++) {
      const float other = __shfl_xor_sync(0xffffffffu, h[o], 1);
      hh[o] = half ? other : h[o];
      hh[4 + o] = half ? h[o] : other;
    }
    // The two threads of a position each take 4 of the 8 hidden channels of the 1x1x1 layers.
    const float* w4 = sTail + 8 + 32 * half;        // rows 4 half .. 4 half + 3 of w4[o][c]
    const float* b4 = sTail + 8 + 64 + 4 * half;
    const float* w5 = sTail + 8 + 64 + 8 + 4 * half;
    const float b5 = sTail[8 + 64 + 8 + 8];
    float part = 0.0f;
#pragma unroll
    for (int o = 0; o < 4; o++) {
      float a = b4[o];
#pragma unroll
      for (int c = 0; c < 8; c++) a = fmaf(hh[c], w4[o * 8 + c], a);
      a = tc_act(a, ep.relu6);
      part = fmaf(a, w5[o], part);
    }
    const float pacc = b5 + (part + __shfl_xor_sync(0xffffffffu, part, 1));
    if (valid && half == 0) p_net[p_idx] = pacc;
  }
}

// Layers 1-3 (see the file comment and ZLayout).
//
// Pipeline.  The CTA numbers the planes it stages across all of its work items, q = 0, 1, ...; plane q lives in
// ring slot q % 3.  full[s] completes (one arrival, the producer's) when the slot holds its plane; empty[s]
// completes (four arrivals, one per consumer warpgroup) when every consumer is done with it.  Both count their
// phases per slot, across planes and work items: use k = q / 3 of slot q % 3 waits for phase k & 1 of full and,
// before the producer overwrites the slot, for phase (k - 1) & 1 of empty.  An item with output planes [za, zb)
// stages the padded planes za .. zb + 1; output plane z reads planes z, z + 1, z + 2 and a consumer releases plane z
// when the MMAs of output plane z have completed (planes zb, zb + 1 after the item's last output plane), so every
// consumer warpgroup arrives on every staged plane exactly once and only after it has waited for that plane.
template <int IN_PLANES, bool FINAL, bool SPLIT>
__global__ void __launch_bounds__(kZThreads, 1)
k_conv3_tc_z(const float4* __restrict__ in, float4* __restrict__ out, float* __restrict__ p_net,
             const float* __restrict__ wB, const float* __restrict__ bias, const float* __restrict__ tail,
             ConvTcGeo g, ZSched s, TcEpi ep) {
  extern __shared__ __align__(1024) uint8_t smem[];
  using L = ZLayout<IN_PLANES, SPLIT>;
  using R = ZRegs<SPLIT>;
  constexpr int TY = L::TY, PY = L::PY;
  const int ww = s.ww, ntile = ww >> 6;
  const int gbytes = PY * ww * 16;                    // one K chunk of a slot
  const int lo_off = 2 * gbytes;                      // hi -> lo (SPLIT)
  const int slot_bytes = L::SLOT_CHUNKS * gbytes;
  uint8_t* sRing = smem;
  uint8_t* sZero = smem + 3 * slot_bytes;
  uint8_t* sB = sZero + L::ZERO_BYTES;
  float* sD = (float*)(sB + L::B_BYTES);              // [kZWarpGroups][ww][kDPitch]
  float* sTail = sD + kZWarpGroups * ww * kDPitch;    // bias[8] (+ w4[64] b4[8] w5[8] b5[1] when FINAL)
  uint64_t* sBar = (uint64_t*)(sTail + 96);           // full[3], empty[3]
  volatile int* sAbort = (volatile int*)(sBar + 6);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  const uint32_t bar_u = smem_u32(sBar);              // full[k] at bar_u + 8 k, empty[k] at bar_u + 24 + 8 k
  // Zeros, B, bias / tail and the mbarriers, by all threads.  Each role calls this after its setmaxnreg, so that
  // nothing is live across the register hand-over.
  auto setup = [&]() {
    for (int i = tid; i < L::ZERO_BYTES / 16; i += kZThreads) ((float4*)sZero)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
    for (int i = tid; i < L::B_BYTES / 16; i += kZThreads) ((float4*)sB)[i] = __ldg((const float4*)wB + i);
    const int n_tail = FINAL ? (8 + 64 + 8 + 8 + 1) : 8;
    for (int i = tid; i < n_tail; i += kZThreads) sTail[i] = (i < 8) ? bias[i] : tail[i - 8];
    if (!FINAL && ep.ac && tid < 16) sTail[8 + tid] = ep.ac[tid];
    if (tid == 0) {
      for (int k = 0; k < 3; k++) {
        mbar_init(bar_u + 8 * k, 1);
        mbar_init(bar_u + 24 + 8 * k, kZWarpGroups);
      }
      *sAbort = 0;
    }
    // generic-proxy writes (st.shared: zeros, B) -> visible to the wgmma (async proxy) reads
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
  };

  const long long plane_g = (long long)(g.nz + 2) * g.py * g.px;            // float4 per global plane
  const long long batch_g = plane_g * 2;
  const int npos = PY * ww;                                                 // staged positions of a plane
  const int wg = warp >> 2, wq = warp & 3;
  const int tw = tid & 127;
  // work item -> first padded row y0, output planes [za, zb), batch entry b
  auto item_geo = [&](int item, int& y0, int& za, int& zb, int& b) {
    const int ty = item % s.nty, zc = (item / s.nty) % s.nzc;
    b = item / s.nty / s.nzc;
    y0 = ty * TY;
    za = g.z_lo + zc * s.zc;
    zb = min(za + s.zc, g.z_hi);
  };

  if (wg == kZWarpGroups) {
    // ---- producer ------------------------------------------------------------------------------------------
    if constexpr (R::PRODUCER < kZLaunchRegs) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R::PRODUCER));
    if constexpr (R::PRODUCER > kZLaunchRegs) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R::PRODUCER));
    setup();
    constexpr int PER = (PY * kWWMax + 127) / 128;
    float4 v[PER][IN_PLANES];
    // padded plane pz of the item at (y0, b) -> registers (positions outside the buffer read the zero border voxel
    // (0, 0, 0))
    auto load = [&](int y0, int b, int pz) {
      const float4* inb = in + b * batch_g;
#pragma unroll
      for (int it = 0; it < PER; it++) {
        const int idx = tw + it * 128;
        const int row = idx / ww, gx = 1 + idx - row * ww, gy = y0 + row;
        const bool inside = idx < npos && gx < g.px && gy < g.py;
        const long long go = inside ? ((long long)pz * g.py + gy) * g.px + gx : 0;
#pragma unroll
        for (int h = 0; h < IN_PLANES; h++) v[it][h] = __ldg(inb + h * plane_g + go);
      }
    };
    int item = blockIdx.x, y0, za, zb, b;
    if (item < s.items) {
      item_geo(item, y0, za, zb, b);
      load(y0, b, za);
    }
    for (int q = 0, pz = za; item < s.items; q++) {
      const int slot = q % 3;
      // registers -> K chunk c of a slot, split into hi / lo when SPLIT
      auto put = [&](uint8_t* slot_p, int c) {
#pragma unroll
        for (int it = 0; it < PER; it++) {
          const int idx = tw + it * 128;
          if (idx < npos) {
            const float4 w = v[it][IN_PLANES == 2 ? c : 0];
            uint8_t* dst = slot_p + c * gbytes + idx * 16;
            if constexpr (SPLIT) {
              const float4 hi = tf32_hi(w);
              *(float4*)dst = hi;
              *(float4*)(dst + lo_off) = make_float4(w.x - hi.x, w.y - hi.y, w.z - hi.z, w.w - hi.w);
            } else {
              *(float4*)dst = w;
            }
          }
        }
      };
      // Layer 1 also writes the plane as K chunk 1 of the previous plane's slot (q - 1) % 3, before this plane's own
      // slot is free (not for an item's first plane: no output plane reads it with its predecessor).  Chunk 1 of
      // that slot was last read for output plane pz - 4, whose MMAs completed before the previous plane was stored;
      // it is read next for output plane pz - 1, after this plane's `full`.  Its chunk 0 (plane pz - 1) may still be
      // in use as base[2] of output plane pz - 3 while this runs, which is safe only because groups 3 and 4 never read
      // K chunk 1 of base[2]: group 3's second chunk is one row further inside chunk 0 and group 4's is the zero
      // block.  Keep it so.
      if (IN_PLANES == 1 && pz > za) put(sRing + ((q + 2) % 3) * slot_bytes, 1);
      if (q >= 3) mbar_wait(bar_u + 24 + 8 * slot, ((q / 3) - 1) & 1, sAbort);
      put(sRing + slot * slot_bytes, 0);
      if (IN_PLANES == 2) put(sRing + slot * slot_bytes, 1);
      // generic-proxy writes (st.shared) -> visible to the wgmma (async proxy) reads; then one arrival for all
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      wg_barrier(1 + kZWarpGroups);
      if (tw == 0) mbar_arrive(bar_u + 8 * slot);
      // the next plane (of this item, else of the next one) is in flight while the consumers work
      if (++pz > zb + 1) {
        item += gridDim.x;
        if (item >= s.items) break;
        item_geo(item, y0, za, zb, b);
        pz = za;
      }
      load(y0, b, pz);
    }
  } else {
    // ---- consumers ------------------------------------------------------------------------------------------
    if constexpr (R::CONSUMER > kZLaunchRegs) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R::CONSUMER));
    if constexpr (R::CONSUMER < kZLaunchRegs) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R::CONSUMER));
    long long* dbg = g_tc_dbg;
    if (dbg && tid == 0) dbg[blockIdx.x * 8 + 0] = clock64();
    setup();
    const uint32_t sRing_u = smem_u32(sRing), sB_u = smem_u32(sB), sZero_u = smem_u32(sZero);
    float* myD = sD + wg * ww * kDPitch;
    const int half = tw & 1;
    const float* bs = sTail + 4 * half;
    int qa = 0;                 // sequence number of the item's first staged plane
    int waited = 0;             // planes q < waited are known to be in their slots
    auto wait_plane = [&](int q) {
      for (; waited <= q; waited++) mbar_wait(bar_u + 8 * (waited % 3), (waited / 3) & 1, sAbort);
    };
    auto release_plane = [&](int q) {
      if (tw == 0) mbar_arrive(bar_u + 24 + 8 * (q % 3));
    };
    for (int item = blockIdx.x; item < s.items; item += gridDim.x) {
      int y0, za, zb, b;
      item_geo(item, y0, za, zb, b);
      const bool has_rows = y0 + wg < g.ny;   // warpgroup wg takes rows wg, wg + 4, ...

      for (int z = za; z < zb; z++) {
        const int qz = qa + (z - za);            // padded plane z; the output plane reads qz .. qz + 2
        uint32_t base[3];                        // slot of padded plane z + 1 + dz
#pragma unroll
        for (int d = 0; d < 3; d++) base[d] = sRing_u + (uint32_t)(((qz + d) % 3) * slot_bytes);
        wait_plane(qz + 1);
        if (dbg && tid == 0 && item == blockIdx.x && z == za) dbg[blockIdx.x * 8 + 1] = clock64();
        if (!has_rows) {
          wait_plane(qz + 2);
          release_plane(qz);
          continue;
        }

        // a row is ntile M tiles of 64 positions
        for (int r = wg; r < TY && y0 + r < g.ny; r += kZWarpGroups) {
          const bool last_row = r + kZWarpGroups >= TY || y0 + r + kZWarpGroups >= g.ny;
          for (int t = 0; t < ntile; t++) {
            const uint32_t row_off = (uint32_t)(((r + 1) * ww + 64 * t) * 16);
            float acc[SPLIT ? 24 : 12] = {}, acl[12] = {};
            asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
            for (int gi = 0; gi < L::GROUPS; gi++) {
              // The groups of padded plane z + 2 (dz = +1) wait until that plane is in its slot, so that the groups
              // of planes z and z + 1 run while the producer stores it.  The groups before are committed first:
              // ptxas serialises every wgmma of the sequence when uncommitted ones are in flight across the wait.
              if (gi == (IN_PLANES == 1 ? 3 : 6)) {
                asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
                wait_plane(qz + 2);
                asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
              }
              const int dz = IN_PLANES == 1 ? layer1_dz(gi) : gi / 3 - 1;
              const int dy = IN_PLANES == 1 ? layer1_dy(gi) : gi % 3 - 1;
              const uint32_t a = base[1 + dz] + row_off + (uint32_t)(dy * ww * 16);
              const bool zero_k1 = IN_PLANES == 1 && gi == 4;
              const uint32_t lbo = IN_PLANES == 1 && gi == 3 ? (uint32_t)(ww * 16) : zero_k1 ? sZero_u - a : (uint32_t)gbytes;
              const uint64_t da = make_desc(a, lbo, 128);
              const uint64_t db = make_desc(sB_u + gi * L::B_GROUP_BYTES, L::NB * 16, 128);
              if constexpr (SPLIT) {
                const uint32_t al = a + (uint32_t)lo_off;
                wgmma_n48(acc, da, db, gi > 0 ? 1u : 0u);
                wgmma_n24(acl, make_desc(al, zero_k1 ? sZero_u - al : lbo, 128), db, gi > 0 ? 1u : 0u);
              } else {
                wgmma_n24(acc, da, db, gi > 0 ? 1u : 0u);
              }
            }
            asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
            asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
            if (dbg && tid == 0 && item == blockIdx.x && z == za && t == 0) dbg[blockIdx.x * 8 + 2] = clock64();
            // this warpgroup's last MMAs on padded plane z: its slot may be refilled while D goes out
            if (last_row && t == ntile - 1) release_plane(qz);

            // accumulator fragment: element (row 16 wq + lane / 4 + 8 i, column 8 k + 2 (lane % 4) + j) is acc[4 k + 2 i + j]
            float* tD = myD + 64 * t * kDPitch;
#pragma unroll
            for (int k = 0; k < 3; k++)
#pragma unroll
              for (int i = 0; i < 2; i++) {
                const int row = 16 * wq + (lane >> 2) + 8 * i, col = 8 * k + 2 * (lane & 3);
                float2 d2;
                if constexpr (SPLIT) {
                  d2.x = acc[4 * k + 2 * i] + (acc[12 + 4 * k + 2 * i] + acl[4 * k + 2 * i]);
                  d2.y = acc[4 * k + 2 * i + 1] + (acc[12 + 4 * k + 2 * i + 1] + acl[4 * k + 2 * i + 1]);
                } else {
                  d2.x = acc[4 * k + 2 * i];
                  d2.y = acc[4 * k + 2 * i + 1];
                }
                *(float2*)(tD + row * kDPitch + col) = d2;
              }
          }
          wg_barrier(1 + wg);

          // epilogue: staged position i (padded x = i + 1), channels 4 half .. 4 half + 3; D of the zero border
          // voxels x = 0 and x = nx + 1 is 0
          const int yg = y0 + r;
          for (int j = 0; j < ntile; j++) {
            const int i = (tw >> 1) + 64 * j, xp = i + 1;
            const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
            const float4 dm = i >= 1 ? *(const float4*)(myD + (i - 1) * kDPitch + 4 * half) : zero4;
            const float4 d0 = *(const float4*)(myD + i * kDPitch + 8 + 4 * half);
            const float4 dp = xp < g.nx ? *(const float4*)(myD + (i + 1) * kDPitch + 16 + 4 * half) : zero4;
            float h[4];
            h[0] = (dm.x + d0.x) + dp.x + bs[0];
            h[1] = (dm.y + d0.y) + dp.y + bs[1];
            h[2] = (dm.z + d0.z) + dp.z + bs[2];
            h[3] = (dm.w + d0.w) + dp.w + bs[3];
            conv_epilogue<FINAL>(h, xp <= g.nx, half, sTail, out, p_net,
                                 b * batch_g + ((long long)(z + 1) * g.py + (yg + 1)) * g.px + xp, plane_g,
                                 (long long)b * g.nz * g.ny * g.nx + ((long long)z * g.ny + yg) * g.nx + (xp - 1), ep);
          }
          wg_barrier(1 + wg);                    // myD is rewritten by the next row
        }
      }
      // padded planes zb, zb + 1 are read by no later output plane of the item
      const int qb = qa + (zb - za);
      wait_plane(qb + 1);
      release_plane(qb);
      release_plane(qb + 1);
      qa = qb + 2;
    }
    if (dbg && tid == 0) {
      dbg[blockIdx.x * 8 + 5] = clock64();
      unsigned smid;
      asm("mov.u32 %0, %%smid;" : "=r"(smid));
      dbg[blockIdx.x * 8 + 7] = smid;
    }
  }
}

// JOIN (final layer only): the input box is the sum of the banks of `js`, each staged from its own resolution
// with nearest indexing (see TcJoinSrc), and the epilogue may write / add / read a partial sum (part_mode).
template <int IN_PLANES, bool FINAL, bool SPLIT, bool JOIN = false>
__global__ void __launch_bounds__(kThreads, 2)
k_conv3_tc(const float4* __restrict__ in, float4* __restrict__ out, float* __restrict__ p_net,
           const float* __restrict__ wB, const float* __restrict__ bias, const float* __restrict__ tail,
           ConvTcGeo g, TcJoinSrc js, TcEpi ep) {
  static_assert(!JOIN || (FINAL && IN_PLANES == 2), "the join is the last 3x3x3 layer");
  extern __shared__ __align__(1024) uint8_t smem[];
  using T = Tile<SPLIT>;
  using L = Layout<IN_PLANES, SPLIT>;
  uint8_t* sA = smem;
  uint8_t* sB = smem + L::A_BYTES;
  float* sD = (float*)(smem + L::A_BYTES + L::B_BYTES);      // [2 warpgroups][64][kDPitch]
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
  if constexpr (JOIN) {
    // Padded full-resolution coordinate g inside the grid -> bank coordinate ((g - 1) >> shift) + 1 (z: global
    // planes, ((g - 1 + zoff) >> shift) - org + 1); outside, the bank's (0, 0, 0) border voxel, which is zero.
    // Banks are summed in order (CAddTable).
    constexpr int PER = (T::POS + kThreads - 1) / kThreads;
    float4 v[PER][2];
#pragma unroll
    for (int it = 0; it < PER; it++) {
      const int idx = tid + it * kThreads;
      const int l = idx & 31, r = idx >> 5;
      const int yy = r % T::PY, zz = r / T::PY;
      const int gx = x0 + l, gy = y0 + yy, gz = z0 + zz;
      const bool interior = idx < T::POS && gx >= 1 && gx <= g.nx && gy >= 1 && gy <= g.ny && gz >= 1 && gz <= g.nz;
      v[it][0] = make_float4(0.f, 0.f, 0.f, 0.f);
      v[it][1] = v[it][0];
      for (int k = 0; k < js.n; k++) {
        const int sh = js.shift[k];
        const int bx = interior ? ((gx - 1) >> sh) + 1 : 0;
        const int by = interior ? ((gy - 1) >> sh) + 1 : 0;
        const int bz = interior ? ((gz - 1 + js.zoff) >> sh) - js.org[k] + 1 : 0;
        const long long plane_k = (long long)(js.nz[k] + 2) * js.py[k] * js.px[k];
        // phase sub-grids: batch entry of (b, the voxel's phase); outside the grid any entry's border voxel is zero
        const int pm = (1 << sh) - 1;
        const long long bk = js.phase[k] ? (((long long)b << (3 * sh)) | (((gz - 1) & pm) << (2 * sh)) |
                                            (((gy - 1) & pm) << sh) | ((gx - 1) & pm))
                                         : b;
        const float4* src = (const float4*)js.p[k] + bk * 2 * plane_k + ((long long)bz * js.py[k] + by) * js.px[k] + bx;
        const float4 a0 = __ldg(src), a1 = __ldg(src + plane_k);
        v[it][0] = make_float4(v[it][0].x + a0.x, v[it][0].y + a0.y, v[it][0].z + a0.z, v[it][0].w + a0.w);
        v[it][1] = make_float4(v[it][1].x + a1.x, v[it][1].y + a1.y, v[it][1].z + a1.z, v[it][1].w + a1.w);
      }
    }
#pragma unroll
    for (int it = 0; it < PER; it++) {
      const int idx = tid + it * kThreads;
      if (idx < T::POS) {
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const float4 w = v[it][h];
          if constexpr (SPLIT) {
            const float4 hi = tf32_hi(w);
            const float4 lo = make_float4(w.x - hi.x, w.y - hi.y, w.z - hi.z, w.w - hi.w);
            *(float4*)(sA + h * L::PSTRIDE + idx * 16) = hi;
            *(float4*)(sA + L::LO_OFF + h * L::PSTRIDE + idx * 16) = lo;
          } else {
            *(float4*)(sA + h * L::PSTRIDE + idx * 16) = w;
          }
        }
      }
    }
  } else if (!SPLIT) {
    for (int idx = tid; idx < T::POS; idx += kThreads) {
      const int l = idx & 31, r = idx >> 5;
      const int yy = r % T::PY, zz = r / T::PY;
      int gx = x0 + l, gy = y0 + yy, gz = z0 + zz;
      const bool inside = gx < g.px && gy < g.py && gz < g.nz + 2;
      gx = inside ? gx : 0; gy = inside ? gy : 0; gz = inside ? gz : 0;      // (0,0,0) is a zero border voxel
      const long long go = ((long long)gz * g.py + gy) * g.px + gx;
#pragma unroll
      for (int h = 0; h < IN_PLANES; h++)
        cp_async16(smem_u32(sA + h * L::PSTRIDE + idx * 16), inb + h * plane_g + go);
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
        for (int h = 0; h < IN_PLANES; h++) {
          const float4 w = v[it][h];
          const float4 hi = tf32_hi(w);
          const float4 lo = make_float4(w.x - hi.x, w.y - hi.y, w.z - hi.z, w.w - hi.w);
          *(float4*)(sA + h * L::PSTRIDE + idx * 16) = hi;
          *(float4*)(sA + L::LO_OFF + h * L::PSTRIDE + idx * 16) = lo;
        }
      }
    }
  }
  // Layer 1's single-tap group reads its K chunk 1 from these zeros (its B rows are zero too, but
  // 0 * NaN would not be).
  for (int i = tid; i < L::ZERO_BYTES / 16 * (SPLIT ? 2 : 1); i += kThreads)
    *(float4*)(sA + (i >> 6) * L::PSTRIDE + T::PLANE_BYTES + (i & 63) * 16) = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int i = tid; i < L::B_BYTES / 16; i += kThreads) cp_async16(smem_u32(sB + i * 16), (const float4*)wB + i);
  const int n_tail = FINAL ? (8 + 64 + 8 + 8 + 1) : 8;
  for (int i = tid; i < n_tail; i += kThreads) sTail[i] = (i < 8) ? bias[i] : tail[i - 8];
  if (!FINAL && ep.ac && tid < 16) sTail[8 + tid] = ep.ac[tid];
  asm volatile("cp.async.commit_group;" ::: "memory");
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  // generic-proxy writes (st.shared, cp.async) -> visible to the wgmma (async proxy) reads
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  if (dbg && tid == 0) { dbg[cta_lin * 8 + 1] = clock64(); unsigned smid; asm("mov.u32 %0, %%smid;" : "=r"(smid)); dbg[cta_lin * 8 + 7] = smid; }

  // ---- warpgroup wg takes M tiles t = wg, wg + 2, ... ------------------------------------
  const int wg = warp >> 2, wq = warp & 3;
  const uint32_t sA_u = smem_u32(sA), sB_u = smem_u32(sB);
  constexpr uint32_t LO_16 = (uint32_t)L::LO_OFF >> 4;
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
    for (int gi = 0; gi < L::GROUPS; gi++) {
      const int dz = IN_PLANES == 1 ? layer1_dz(gi) : gi / 3 - 1;
      const int dy = IN_PLANES == 1 ? layer1_dy(gi) : gi % 3 - 1;
      const uint32_t a_off = toff + (uint32_t)((((1 + dz) * T::PY + (1 + dy)) * kTX) * 16);
      // offset of K chunk 1 from chunk 0 (see Layout)
      const uint32_t lbo = IN_PLANES == 2 ? (uint32_t)T::PLANE_BYTES
                         : gi < 3         ? (uint32_t)(T::PY * kTX * 16)
                         : gi == 3        ? (uint32_t)(kTX * 16)
                                          : (uint32_t)T::PLANE_BYTES - a_off;
      const uint64_t da = make_desc(sA_u + a_off, lbo, 128);
      const uint64_t db = make_desc(sB_u + gi * L::B_GROUP_BYTES, L::NB * 16, 128);
      if constexpr (SPLIT) {
        wgmma_n48(acc, da, db, gi > 0 ? 1u : 0u);
        wgmma_n24(acl, da + LO_16, db, gi > 0 ? 1u : 0u);
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
    const int xg = x0 + xl - 1;                         // unpadded coordinates of this position's voxel
    const int yg = y0 + 2 * (t % T::RB) + ry;
    const int zg = z0 + t / T::RB;
    const bool valid = xl >= 1 && xl <= 30 && xg < g.nx && yg < g.ny && zg < g.z_hi;
    float h[4];
    bool tail_wanted = true;
    if constexpr (JOIN) {
      h[0] = (dm.x + d0.x) + dp.x;
      h[1] = (dm.y + d0.y) + dp.y;
      h[2] = (dm.z + d0.z) + dp.z;
      h[3] = (dm.w + d0.w) + dp.w;
      float4* part = (float4*)(js.partial + ((((long long)b * g.nz + zg) * g.ny + yg) * g.nx + xg) * 8 + 4 * half);
      if (js.part_mode == 1 || js.part_mode == 2) {
        tail_wanted = false;
        if (valid) {
          float4 o4 = make_float4(h[0], h[1], h[2], h[3]);
          if (js.part_mode == 2) {
            const float4 q = *part;
            o4 = make_float4(o4.x + q.x, o4.y + q.y, o4.z + q.z, o4.w + q.w);
          }
          *part = o4;
        }
      } else if (js.part_mode == 3 && valid) {
        const float4 q = *part;
        h[0] += q.x; h[1] += q.y; h[2] += q.z; h[3] += q.w;
      }
#pragma unroll
      for (int o = 0; o < 4; o++) h[o] += bs[o];
    } else {
      h[0] = (dm.x + d0.x) + dp.x + bs[0];
      h[1] = (dm.y + d0.y) + dp.y + bs[1];
      h[2] = (dm.z + d0.z) + dp.z + bs[2];
      h[3] = (dm.w + d0.w) + dp.w + bs[3];
    }
#pragma unroll
    for (int o = 0; o < 4; o++) h[o] = tc_act(h[o], ep.relu6);
    if (!FINAL) {
      if (ep.ac) {                                      // running-statistics BN after the activation
#pragma unroll
        for (int o = 0; o < 4; o++) h[o] = fmaf(sTail[8 + 4 * half + o], h[o], sTail[16 + 4 * half + o]);
      }
      if (valid) {
        const long long o = b * batch_g + ((long long)(zg + 1) * g.py + (yg + 1)) * g.px + (xg + 1);
        out[o + half * plane_g] = make_float4(h[0], h[1], h[2], h[3]);
      }
    } else if (tail_wanted) {          // uniform over the launch (part_mode)
      float hh[8];
#pragma unroll
      for (int o = 0; o < 4; o++) {
        const float other = __shfl_xor_sync(0xffffffffu, h[o], 1);
        hh[o] = half ? other : h[o];
        hh[4 + o] = half ? h[o] : other;
      }
      // The two threads of a position each take 4 of the 8 hidden channels of the 1x1x1 layers.
      const float* w4 = sTail + 8 + 32 * half;        // rows 4 half .. 4 half + 3 of w4[o][c]
      const float* b4 = sTail + 8 + 64 + 4 * half;
      const float* w5 = sTail + 8 + 64 + 8 + 4 * half;
      const float b5 = sTail[8 + 64 + 8 + 8];
      float part = 0.0f;
#pragma unroll
      for (int o = 0; o < 4; o++) {
        float a = b4[o];
#pragma unroll
        for (int c = 0; c < 8; c++) a = fmaf(hh[c], w4[o * 8 + c], a);
        a = tc_act(a, ep.relu6);
        part = fmaf(a, w5[o], part);
      }
      const float pacc = b5 + (part + __shfl_xor_sync(0xffffffffu, part, 1));
      if (valid && half == 0) p_net[(long long)b * g.nz * g.ny * g.nx + ((long long)zg * g.ny + yg) * g.nx + xg] = pacc;
    }
    wg_barrier(1 + wg);                                 // myD is rewritten by the next tile
  }
  if (dbg) {
    __syncthreads();
    if (tid == 0) dbg[cta_lin * 8 + 5] = clock64();
  }
}

template <int IN_PLANES, bool FINAL, bool SPLIT, bool JOIN = false>
void launch_one(const float4* in, float4* out, float* p_net, const float* wB, const float* bias,
                const float* tail, const ConvTcGeo& g, cudaStream_t st, const TcJoinSrc& js, const TcEpi& ep) {
  using T = Tile<SPLIT>;
  const size_t smem = Layout<IN_PLANES, SPLIT>::BYTES;
  auto kern = k_conv3_tc<IN_PLANES, FINAL, SPLIT, JOIN>;
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
  kern<<<grid, kThreads, smem, st>>>(in, out, p_net, wB, bias, tail, gg, js, ep);
}

// Work items of one k_conv3_tc_z launch on `nsm` SMs.  ZC (output planes per item) minimises the rounds of the
// persistent grid times the planes a round stages (ZC + 2); ties go to the larger ZC (fewer items, fewer halo
// planes).  128^3, 132 SMs: 3xTF32 32 row blocks x ZC 32 = 128 items, TF32 16 x 16 = 128 items, one round.
// Needs nx <= kWWMax and z_hi > z_lo.
ZSched z_schedule(const ConvTcGeo& g, int ty, int nsm) {
  ZSched s;
  s.zc = 1;
  s.ww = g.nx > 64 ? kWWMax : 64;
  s.nty = (g.ny + ty - 1) / ty;
  const long long cols = (long long)g.nb * s.nty;
  const int nzo = g.z_hi - g.z_lo;
  long long best = -1;
  for (int zc = 1; zc <= nzo; zc++) {
    const long long items = cols * ((nzo + zc - 1) / zc);
    const long long grid = items < nsm ? items : nsm;
    const long long cost = (items + grid - 1) / grid * (zc + 2);
    if (best < 0 || cost <= best) {
      best = cost;
      s.zc = zc;
    }
  }
  s.nzc = (nzo + s.zc - 1) / s.zc;
  s.items = (int)(cols * s.nzc);
  return s;
}

int g_z_grid_cap = 0;           // test hook: at most this many CTAs in a k_conv3_tc_z grid (0: one per SM)

template <int IN_PLANES, bool FINAL, bool SPLIT>
void launch_z(const float4* in, float4* out, float* p_net, const float* wB, const float* bias, const float* tail,
              const ConvTcGeo& g, cudaStream_t st, const TcEpi& ep) {
  using L = ZLayout<IN_PLANES, SPLIT>;
  if (g.z_hi <= g.z_lo || g.nb < 1 || g.ny < 1 || g.nx < 1) return;     // nothing to compute
  auto kern = k_conv3_tc_z<IN_PLANES, FINAL, SPLIT>;
  static unsigned long long configured = 0;       // per device (function attributes are)
  int dev = 0, nsm = 0;
  cudaGetDevice(&dev);
  if (!((configured >> (dev & 63)) & 1ULL)) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L::bytes(kWWMax));
    configured |= 1ULL << (dev & 63);
  }
  cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev);
  const ZSched s = z_schedule(g, L::TY, nsm);
  int grid = s.items < nsm ? s.items : nsm;
  if (g_z_grid_cap > 0 && grid > g_z_grid_cap) grid = g_z_grid_cap;
  kern<<<grid, kZThreads, L::bytes(s.ww), st>>>(in, out, p_net, wB, bias, tail, g, s, ep);
}

// 2x2x2 average of the first float4 plane (k_pool's summation order), zero fourth channel; output planes
// [go.z_lo, go.z_hi), input planes shifted by z_phase.  planes = 2: both float4 planes, all four channels each.
__global__ void k_tc_pyramid(const float4* __restrict__ in, ConvTcGeo gi, float4* __restrict__ out, ConvTcGeo go,
                             int z_phase, int planes, long long total) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int nzr = go.z_hi - go.z_lo;
  const int x = (int)(t % go.nx), y = (int)((t / go.nx) % go.ny);
  const int z = go.z_lo + (int)((t / ((long long)go.nx * go.ny)) % nzr);
  const long long b = t / ((long long)go.nx * go.ny * nzr);
  const long long iplane = (long long)(gi.nz + 2) * gi.py * gi.px, oplane = (long long)(go.nz + 2) * go.py * go.px;
  for (int q = 0; q < planes; q++) {
    const float4* ib = in + (b * 2 + q) * iplane;
    float sx = 0.0f, sy = 0.0f, sz = 0.0f, sw = 0.0f;
    for (int dz = 0; dz < 2; dz++)
      for (int dy = 0; dy < 2; dy++)
        for (int dx = 0; dx < 2; dx++) {
          const float4 v =
              __ldg(ib + ((long long)(2 * z + z_phase + dz + 1) * gi.py + (2 * y + dy + 1)) * gi.px + (2 * x + dx + 1));
          sx += v.x; sy += v.y; sz += v.z; sw += v.w;
        }
    out[(b * 2 + q) * oplane + ((long long)(z + 1) * go.py + (y + 1)) * go.px + (x + 1)] =
        make_float4(sx / 8.0f, sy / 8.0f, sz / 8.0f, planes == 2 ? sw / 8.0f : 0.0f);
  }
}

// Phase sub-grid voxel t (over gs.nb entries x gs.nz x gs.ny x gs.nx) -> its full-resolution voxel; false outside the
// full grid gf.
__device__ __forceinline__ bool phase_voxel(long long t, const ConvTcGeo& gs, int sh, const ConvTcGeo& gf, long long* e,
                                            int* sx, int* sy, int* sz, long long* b, int* x, int* y, int* z) {
  *sx = (int)(t % gs.nx);
  *sy = (int)((t / gs.nx) % gs.ny);
  *sz = (int)((t / ((long long)gs.nx * gs.ny)) % gs.nz);
  *e = t / ((long long)gs.nx * gs.ny * gs.nz);
  const int m = (1 << sh) - 1;
  const int r = (int)(*e & ((1LL << (3 * sh)) - 1));
  *b = *e >> (3 * sh);
  *x = (*sx << sh) | (r & m);
  *y = (*sy << sh) | ((r >> sh) & m);
  *z = (*sz << sh) | (r >> (2 * sh));
  return *x < gf.nx && *y < gf.ny && *z < gf.nz;
}

__global__ void k_tc_phase_copy(const float4* __restrict__ in, ConvTcGeo gf, float4* __restrict__ out, ConvTcGeo gs,
                                int sh, int planes, long long total) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  long long e, b;
  int sx, sy, sz, x, y, z;
  const bool valid = phase_voxel(t, gs, sh, gf, &e, &sx, &sy, &sz, &b, &x, &y, &z);
  const long long fplane = (long long)(gf.nz + 2) * gf.py * gf.px, splane = (long long)(gs.nz + 2) * gs.py * gs.px;
  for (int q = 0; q < planes; q++) {
    const float4 v = valid ? __ldg(in + (b * 2 + q) * fplane + ((long long)(z + 1) * gf.py + (y + 1)) * gf.px + (x + 1))
                           : make_float4(0.f, 0.f, 0.f, 0.f);
    out[(e * 2 + q) * splane + ((long long)(sz + 1) * gs.py + (sy + 1)) * gs.px + (sx + 1)] = v;
  }
}

__global__ void k_tc_phase_zero(float4* __restrict__ buf, ConvTcGeo gs, int sh, ConvTcGeo gf, long long total) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  long long e, b;
  int sx, sy, sz, x, y, z;
  if (phase_voxel(t, gs, sh, gf, &e, &sx, &sy, &sz, &b, &x, &y, &z)) return;
  const long long splane = (long long)(gs.nz + 2) * gs.py * gs.px;
  for (int q = 0; q < 2; q++)
    buf[(e * 2 + q) * splane + ((long long)(sz + 1) * gs.py + (sy + 1)) * gs.px + (sx + 1)] = make_float4(0.f, 0.f, 0.f, 0.f);
}

__global__ void k_tc_phase_gather(const float4* __restrict__ in, ConvTcGeo gs, float4* __restrict__ out, ConvTcGeo gf,
                                  int sh, long long total) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  long long e, b;
  int sx, sy, sz, x, y, z;
  if (!phase_voxel(t, gs, sh, gf, &e, &sx, &sy, &sz, &b, &x, &y, &z)) return;
  const long long fplane = (long long)(gf.nz + 2) * gf.py * gf.px, splane = (long long)(gs.nz + 2) * gs.py * gs.px;
  for (int q = 0; q < 2; q++)
    out[(b * 2 + q) * fplane + ((long long)(z + 1) * gf.py + (y + 1)) * gf.px + (x + 1)] =
        __ldg(in + (e * 2 + q) * splane + ((long long)(sz + 1) * gs.py + (sy + 1)) * gs.px + (sx + 1));
}

}  // namespace

ConvTcGeo make_conv_tc_phase_geo(int nb, int nz, int ny, int nx, int sh) {
  const int d = 1 << sh;
  return make_conv_tc_geo(nb << (3 * sh), (nz + d - 1) >> sh, (ny + d - 1) >> sh, (nx + d - 1) >> sh);
}
static long long phase_cells(const ConvTcGeo& gs) { return (long long)gs.nb * gs.nz * gs.ny * gs.nx; }
void launch_tc_phase_copy(const float* in, const ConvTcGeo& gfull, float* out, const ConvTcGeo& gsub, int sh,
                          int planes, cudaStream_t st) {
  const long long total = phase_cells(gsub);
  k_tc_phase_copy<<<(unsigned)((total + 255) / 256), 256, 0, st>>>((const float4*)in, gfull, (float4*)out, gsub, sh,
                                                                    planes, total);
}
void launch_tc_phase_zero(float* buf, const ConvTcGeo& gsub, int sh, const ConvTcGeo& gfull, cudaStream_t st) {
  const long long total = phase_cells(gsub);
  k_tc_phase_zero<<<(unsigned)((total + 255) / 256), 256, 0, st>>>((float4*)buf, gsub, sh, gfull, total);
}
void launch_tc_phase_gather(const float* in, const ConvTcGeo& gsub, float* out, const ConvTcGeo& gfull, int sh,
                            cudaStream_t st) {
  const long long total = phase_cells(gsub);
  k_tc_phase_gather<<<(unsigned)((total + 255) / 256), 256, 0, st>>>((const float4*)in, gsub, (float4*)out, gfull, sh,
                                                                      total);
}

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
void conv_tc_set_z_grid(int ctas) { g_z_grid_cap = ctas > 0 ? ctas : 0; }
int conv_tc_take_z_fault(cudaStream_t st) {
  unsigned int v = 0;
  if (cudaMemcpyFromSymbolAsync(&v, g_tc_z_fault, sizeof(v), 0, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
      cudaStreamSynchronize(st) != cudaSuccess)
    return 0;                        // a CUDA error is reported by the caller's own checks
  if (v) {
    const unsigned int zero = 0;
    cudaMemcpyToSymbolAsync(g_tc_z_fault, &zero, sizeof(zero), 0, cudaMemcpyHostToDevice, st);
    cudaStreamSynchronize(st);
  }
  return v ? 1 : 0;
}

int conv_tc_b_floats(int split) { return kGroups * 2 * (split ? 48 : 32) * 4; }

// Host-side packing of one layer's weights [cout=8][cin][3][3][3] into the B operand blocks
// (tf32 "hi" truncation and fp32 residual "lo" when split).  A block is [K chunk][NB][4 channels].
// cin > 4: block dz * 3 + dy holds tap (dz, dy), channels 4 kc .. 4 kc + 3 in K chunk kc.
// cin <= 4 (layer 1): blocks 0-4 hold the tap pairs of layer1_dz / layer1_dy, channels 0-3 in both
// K chunks; block 4's K chunk 1 stays zero.
void conv_tc_pack_weights(const float* w, int cin, int split, float* out) {
  const int NB = split ? 48 : 32;
  for (int i = 0; i < kGroups * 2 * NB * 4; i++) out[i] = 0.0f;
  for (int dz = 0; dz < 3; dz++)
    for (int dy = 0; dy < 3; dy++) {
      int blk_i = dz * 3 + dy, kc0 = 0;
      if (cin <= 4) {
        if (dz < 2) {
          blk_i = dy; kc0 = dz;                 // (dz, dy) = (-1, dy) / (0, dy)
        } else {
          blk_i = dy < 2 ? 3 : 4; kc0 = dy < 2 ? dy : 0;   // (1, -1) / (1, 0), then (1, 1) alone
        }
      }
      float* blk = out + (size_t)blk_i * 2 * NB * 4;
      for (int kx = 0; kx < 3; kx++)
        for (int o = 0; o < 8; o++)
          for (int c = 0; c < cin; c++) {
            const float v = w[((((size_t)o * cin + c) * 3 + dz) * 3 + dy) * 3 + kx];
            union { float f; uint32_t u; } hi;
            hi.f = v;
            if (split) hi.u &= 0xFFFFE000u;
            const int n = kx * 8 + o, kc = kc0 + (c >> 2);
            blk[(kc * NB + n) * 4 + (c & 3)] = hi.f;
            if (split) blk[(kc * NB + 24 + n) * 4 + (c & 3)] = v - hi.f;
          }
    }
}

int launch_conv3_tc_join(const TcJoinSrc& src, float* p_net, const float* wB, const float* bias, const float* tail,
                         int split, const ConvTcGeo& g, cudaStream_t st, const TcEpi& ep) {
  if (src.n < 1 || src.n > kTcMaxBanks) return -1;
  if (split) launch_one<2, true, true, true>(nullptr, nullptr, p_net, wB, bias, tail, g, st, src, ep);
  else launch_one<2, true, false, true>(nullptr, nullptr, p_net, wB, bias, tail, g, st, src, ep);
  return 1;
}

void launch_tc_pyramid(const float* in, const ConvTcGeo& gin, float* out, const ConvTcGeo& gout, int z_phase,
                       cudaStream_t st, int planes) {
  const long long total = (long long)gout.nb * (gout.z_hi - gout.z_lo) * gout.ny * gout.nx;
  if (total <= 0) return;
  k_tc_pyramid<<<(unsigned)((total + 255) / 256), 256, 0, st>>>((const float4*)in, gin, (float4*)out, gout, z_phase,
                                                                 planes, total);
}

int launch_conv3_tc(const float* in, float* out, float* p_net, const float* wB, const float* bias,
                    const float* tail, int in_planes, int final_layer, int split, const ConvTcGeo& g,
                    cudaStream_t st, const TcEpi& ep) {
  const float4* i4 = (const float4*)in;
  float4* o4 = (float4*)out;
  // Rows up to kWWMax positions stream along z without an x halo; wider rows would need overlapping row windows
  // whose 64-position M tiles compute more positions per kept voxel than the box's 32-wide rows (256^3: 320 or 384
  // per row against 288), so they keep the one-shot box.
#define TFL_TC_CASE(P, F, S)                                                   \
  if (in_planes == P && (final_layer != 0) == F && (split != 0) == S) {        \
    if (g.nx <= kWWMax) launch_z<P, F, S>(i4, o4, p_net, wB, bias, tail, g, st, ep); \
    else launch_one<P, F, S>(i4, o4, p_net, wB, bias, tail, g, st, TcJoinSrc{}, ep); \
    return 1;                                                                  \
  }
  TFL_TC_CASE(1, false, false) TFL_TC_CASE(2, false, false) TFL_TC_CASE(2, true, false)
  TFL_TC_CASE(1, false, true) TFL_TC_CASE(2, false, true) TFL_TC_CASE(2, true, true)
#undef TFL_TC_CASE
  return -1;
}

}  // namespace tfl
