// Preconditioned conjugate gradient pressure solve, entirely on the device and matrix-free
// (tfluids.solveLinearSystemPCG, torch/tfluids/init.lua:645-676; reference implementation
// torch/tfluids/generic/tfluids.cu:864-1759: connected components + CSR assembly on the CPU,
// cuSPARSE csric0/csrilu0 + csrsv + csrmv and cuBLAS dots per component).
//
// Same algorithm, different machine mapping:
//   * connected components of fluid cells: union-find on the device (the reference flood-fills on
//     the host, find_connected_fluid_components.cc:17-82);
//   * ALL components of ALL batch elements are iterated together: a component is closed under the
//     7-point adjacency, so one sweep over the grid applies every component's operator, and the CG
//     scalars (alpha, beta, residual, iteration count, convergence) are kept PER COMPONENT in device
//     memory -- each component sees exactly the reference's sequence `while (r.r > tol^2 && iter <=
//     maxIter)` (generic/tfluids.cu:1588) and freezes when it terminates;
//   * no matrix: a 16-bit code per cell (in-system, 6 links, diagonal count, preconditioner on);
//   * IC(0) / ILU(0) (one operator for a symmetric matrix) in the system's lexicographic order, like
//     csric0 + two csrsv.  The triangular solves are wavefront-sequential; they run as a pipeline of
//     persistent CTAs over a SKEWED layout: cell (i, j) of plane k is stored at row (i + j) mod
//     max(nx, ny), column j -- a bijection onto a compact array in which a 2-D wavefront i + j = s is
//     (part of) one contiguous row, a thread owns grid row j and carries its x-neighbour in a
//     register, the y-neighbour comes from the adjacent thread through shared memory and the
//     z-neighbour from the thread group one plane below, which runs one step ahead in the same CTA
//     (shared memory) or in the previous CTA (global memory + a progress word).  Every vector of the
//     solver lives in that layout, so nothing is permuted per iteration.
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include <algorithm>
#include <vector>

#include "tfl_kernels.h"

namespace tfl {

namespace {

constexpr unsigned kInSys = 1u;
constexpr unsigned kXM = 2u, kXP = 4u, kYM = 8u, kYP = 16u, kZM = 32u, kZP = 64u;
constexpr unsigned kDiagShift = 7;      // 3 bits
constexpr unsigned kPreOn = 1u << 10;
constexpr long long kSpinLimit = 1ll << 22;

struct PcgGeo {
  int nx, ny, nz, nb, is3d;
  int S, NYP, P;           // wavefronts per plane (nx + ny - 1), padded row length, planes (nb * nz)
  int R;                   // rows stored per plane: wavefront s lives in row s mod R, R = max(nx, ny)
  long long n;             // cells per batch element
  long long plane;         // R * NYP
  long long slots;         // P * plane
  int GP, chunks;          // planes per CTA, plane chunks
};

__device__ __forceinline__ long long skew_index(const PcgGeo& g, int pl, int j, int i) {
  const int s = i + j;
  return ((long long)pl * g.R + (s >= g.R ? s - g.R : s)) * g.NYP + j;
}

// ---- connected components (union-find, lock-free) ----------------------------------------
__device__ __forceinline__ int find_root(volatile int* parent, int a) {
  for (;;) {
    const int p = parent[a];
    if (p == a) return a;
    a = p;
  }
}
__device__ __forceinline__ void unite(int* parent, int a, int b) {
  for (;;) {
    a = find_root(parent, a);
    b = find_root(parent, b);
    if (a == b) return;
    if (a < b) { const int t = a; a = b; b = t; }
    const int old = atomicMin(parent + a, b);     // hang the larger root under the smaller
    if (old == a) return;
    a = old;
  }
}

__global__ void k_label_init(const float* __restrict__ flags, int* __restrict__ parent, PcgGeo g,
                             int* __restrict__ status) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= g.n * g.nb) return;
  const int fluid = ((int)flags[c]) & 1;
  parent[c] = fluid ? (int)c : -1;
  if (fluid) {
    const long long cc = c % g.n;
    const int i = (int)(cc % g.nx), j = (int)((cc / g.nx) % g.ny), k = (int)(cc / ((long long)g.nx * g.ny));
    const bool border = i < 1 || i > g.nx - 2 || j < 1 || j > g.ny - 2 || (g.is3d && (k < 1 || k > g.nz - 2));
    if (border) atomicOr(status, 1);          // generic/tfluids.cu:1083-1090 raises
  }
}
// SAFE: fluid cells may sit on the domain border (normalizePressureMean accepts any flag grid), so the
// backward neighbours are bounds-checked; the PCG path has already rejected such grids.
template <bool SAFE>
__global__ void k_label_union(int* __restrict__ parent, PcgGeo g, const int* __restrict__ status) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= g.n * g.nb || (!SAFE && *status)) return;
  if (parent[c] < 0) return;
  bool xm = true, ym = true, zm = g.is3d != 0;
  if (SAFE) {
    const long long cc = c % g.n;
    const int i = (int)(cc % g.nx), j = (int)((cc / g.nx) % g.ny), k = (int)(cc / ((long long)g.nx * g.ny));
    xm = i > 0; ym = j > 0; zm = zm && k > 0;
  }
  if (xm && parent[c - 1] >= 0) unite(parent, (int)c, (int)c - 1);
  if (ym && parent[c - g.nx] >= 0) unite(parent, (int)c, (int)c - g.nx);
  if (zm && parent[c - (long long)g.nx * g.ny] >= 0) unite(parent, (int)c, (int)(c - (long long)g.nx * g.ny));
}
__global__ void k_label_flatten(int* __restrict__ parent, int* __restrict__ csize, PcgGeo g) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= g.n * g.nb) return;
  if (parent[c] < 0) return;
  const int r = find_root(parent, (int)c);
  parent[c] = r;
  atomicAdd(csize + r, 1);
}
// Dense ids for components of at least two cells (size 1 is skipped, generic/tfluids.cu:1386-1392).
__global__ void k_label_assign(const int* __restrict__ parent, const int* __restrict__ csize, int* __restrict__ cid,
                               PcgGeo g, int* __restrict__ ncomp) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= g.n * g.nb) return;
  if (parent[c] == (int)c && csize[c] >= 2) cid[c] = atomicAdd(ncomp, 1);
}

// Natural layout -> skewed system arrays.
__global__ void k_build(const float* __restrict__ flags, const float* __restrict__ div, const int* __restrict__ parent,
                        const int* __restrict__ csize, const int* __restrict__ cid, unsigned short* __restrict__ cf,
                        int* __restrict__ comp, float* __restrict__ r, int* __restrict__ cnt, PcgGeo g, int precond) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= g.n * g.nb) return;
  const int root = parent[c];
  if (root < 0) return;
  const int sz = csize[root];
  if (sz < 2) return;
  const int id = cid[root];
  const int b = (int)(c / g.n);
  const long long cc = c % g.n;
  const int i = (int)(cc % g.nx), j = (int)((cc / g.nx) % g.ny), k = (int)(cc / ((long long)g.nx * g.ny));
  const long long sy = g.nx, szs = (long long)g.nx * g.ny;
  unsigned code = kInSys;
  unsigned diag = 0;
  auto look = [&](long long off, unsigned bit) {
    const int f = (int)flags[c + off];
    if (!(f & 2)) diag++;                      // not an obstacle: contributes to the diagonal (:962-979)
    if (f & 1) code |= bit;                    // fluid: off-diagonal -1 (:982-1004)
  };
  look(-1, kXM); look(1, kXP); look(-sy, kYM); look(sy, kYP);
  if (g.is3d) { look(-szs, kZM); look(szs, kZP); }
  code |= diag << kDiagShift;
  if (precond != 0 && sz >= 5) code |= kPreOn;   // fewer than 5 cells: no preconditioner (:1399-1401)
  const long long q = skew_index(g, b * g.nz + k, j, i);
  cf[q] = (unsigned short)code;
  comp[q] = id;
  r[q] = div[c];                               // copyDivergenceToSystem (:1190-1209)
  if (root == (int)c) cnt[id] = sz;
}

// ---- per-component reductions --------------------------------------------------------------
// Every lane of the warp calls.  comp < 0 = nothing to add.
__device__ __forceinline__ void warp_comp_add(double* __restrict__ acc, int comp, double v) {
  const unsigned full = 0xffffffffu;
  const unsigned has = __ballot_sync(full, comp >= 0);
  if (!has) return;
  const int c0 = __shfl_sync(full, comp, __ffs(has) - 1);
  const bool uniform = __all_sync(full, comp < 0 || comp == c0);
  if (uniform) {
    double s = comp >= 0 ? v : 0.0;
    for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(full, s, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(acc + c0, s);
  } else if (comp >= 0) {
    atomicAdd(acc + comp, v);
  }
}
// Running (component, sum) of a thread that walks over cells.
struct CompAcc {
  int comp = -1;
  double v = 0.0;
  __device__ __forceinline__ void add(double* __restrict__ acc, int c, double x) {
    if (c != comp) {
      if (comp >= 0) atomicAdd(acc + comp, v);
      comp = c;
      v = 0.0;
    }
    v += x;
  }
};

__device__ __forceinline__ double clamp_eps(double v) {     // clampToEpsilon, generic/tfluids.cu:1153-1163
  const double eps = 1.17549435e-38;
  if (fabs(v) < eps) return v < 0 ? -eps : eps;
  return v;
}

struct CompScalars {
  double* rz_new; double* rz_old; double* pw; double* rr_new; double* rr_cur; double* xsum;
  int* cnt; int* done; int* iters;
  int* header;       // [0] active components, [1] nan seen, [2] pipeline faults
};

__global__ void k_rr_init(const unsigned short* __restrict__ cf, const int* __restrict__ comp,
                          const float* __restrict__ r, CompScalars sc, long long slots) {
  CompAcc a;
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < slots; q += (long long)gridDim.x * blockDim.x) {
    if (!(cf[q] & kInSys)) continue;
    const float v = r[q];
    a.add(sc.rr_cur, comp[q], (double)v * (double)v);
  }
  warp_comp_add(sc.rr_cur, a.comp, a.v);
}

// p_new = z + beta p_old (beta = r.z / r_old.z_old per component; 0 on the first iteration),
// w = A p_new, pw += p_new . w.  Neighbours' p_new are recomputed instead of a second pass.
__global__ void k_direction_spmv(const unsigned short* __restrict__ cf, const int* __restrict__ comp,
                                 const float* __restrict__ z, const float* __restrict__ p_old,
                                 float* __restrict__ p_new, float* __restrict__ w, CompScalars sc, PcgGeo g,
                                 int no_precond) {
  CompAcc a;
  const long long pl = g.plane;
  const int j = threadIdx.x;                      // blockDim.x == NYP: one stored row per block iteration
  for (long long row = blockIdx.x; row < (long long)g.P * g.R; row += gridDim.x) {
    const int r = (int)(row % g.R);
    // rows of the -x / +x neighbours (the wavefront index wraps around the R stored rows)
    const long long dm = r > 0 ? -(long long)g.NYP : (long long)(g.R - 1) * g.NYP;
    const long long dp = r < g.R - 1 ? (long long)g.NYP : -(long long)(g.R - 1) * g.NYP;
    const long long q = row * g.NYP + j;
    const unsigned c = cf[q];
    if (!(c & kInSys)) continue;
    const int id = comp[q];
    if (sc.done[id]) continue;
    float beta = 0.0f;
    if (sc.iters[id] > 0) {
      const double num = no_precond ? sc.rr_cur[id] : sc.rz_new[id];
      beta = (float)(num / clamp_eps(sc.rz_old[id]));
    }
    const float ps = z[q] + beta * p_old[q];
    float acc = (float)((c >> kDiagShift) & 7u) * ps;
    if (c & kXM) acc -= z[q + dm] + beta * p_old[q + dm];
    if (c & kXP) acc -= z[q + dp] + beta * p_old[q + dp];
    if (c & kYM) acc -= z[q + dm - 1] + beta * p_old[q + dm - 1];
    if (c & kYP) acc -= z[q + dp + 1] + beta * p_old[q + dp + 1];
    if (c & kZM) acc -= z[q - pl] + beta * p_old[q - pl];
    if (c & kZP) acc -= z[q + pl] + beta * p_old[q + pl];
    p_new[q] = ps;
    w[q] = acc;
    a.add(sc.pw, id, (double)ps * (double)acc);
  }
  warp_comp_add(sc.pw, a.comp, a.v);
}

// x += alpha p, r -= alpha w, rr_new += r.r
__global__ void k_update(const unsigned short* __restrict__ cf, const int* __restrict__ comp,
                         const float* __restrict__ p, const float* __restrict__ w, float* __restrict__ x,
                         float* __restrict__ r, CompScalars sc, long long slots, int no_precond) {
  CompAcc a;
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < slots; q += (long long)gridDim.x * blockDim.x) {
    if (!(cf[q] & kInSys)) continue;
    const int id = comp[q];
    if (sc.done[id]) continue;
    const double num = no_precond ? sc.rr_cur[id] : sc.rz_new[id];
    const float alpha = (float)(num / clamp_eps(sc.pw[id]));
    x[q] = x[q] + alpha * p[q];
    const float rv = r[q] - alpha * w[q];
    r[q] = rv;
    a.add(sc.rr_new, id, (double)rv * (double)rv);
  }
  warp_comp_add(sc.rr_new, a.comp, a.v);
}

// End of an iteration (or, with `start`, before the first): termination test per component.  The component count
// is `ncomp`, or *ncomp_dev when that is given (captured solves, which never read it back to the host).
__global__ void k_scalars(CompScalars sc, const int* __restrict__ ncomp_dev, int ncomp, double tol2, int max_iter,
                          int start, int no_precond) {
  const int n = ncomp_dev ? *ncomp_dev : ncomp;
  for (int id = blockIdx.x * blockDim.x + threadIdx.x; id < n; id += gridDim.x * blockDim.x) {
    if (!sc.done[id]) {
      if (!start) {
        sc.rz_old[id] = no_precond ? sc.rr_cur[id] : sc.rz_new[id];
        sc.rr_cur[id] = sc.rr_new[id];
        sc.iters[id] += 1;
      }
      const double rr = sc.rr_cur[id];
      if (rr != rr) atomicOr(sc.header + 1, 1);
      if (!(rr > tol2) || sc.iters[id] > max_iter) sc.done[id] = 1;     // while (rr > tol^2 && iter <= maxIter)
      else atomicAdd(sc.header, 1);
    }
    sc.rz_new[id] = 0.0;
    sc.pw[id] = 0.0;
    sc.rr_new[id] = 0.0;
  }
}

// ---- the captured solve's own kernels ---------------------------------------------------------
// Zeroes the scalars of the header[3] components labelling found (a direct solve memsets them, knowing the count).
__global__ void k_comp_clear(CompScalars sc) {
  const int n = sc.header[3];
  for (int id = blockIdx.x * blockDim.x + threadIdx.x; id < n; id += gridDim.x * blockDim.x) {
    sc.rz_new[id] = 0.0; sc.rz_old[id] = 0.0; sc.pw[id] = 0.0; sc.rr_new[id] = 0.0; sc.rr_cur[id] = 0.0;
    sc.xsum[id] = 0.0;
    sc.cnt[id] = 0; sc.done[id] = 0; sc.iters[id] = 0;
  }
}

// Sets the WHILE node's condition: another pass while a component is active and no NaN, sweep fault or border cell
// was seen (what pcg_solve's host loop tests).  `passes` (or null) counts the passes of the body.
__global__ void k_pcg_continue(const int* __restrict__ header, cudaGraphConditionalHandle loop,
                               unsigned long long* __restrict__ passes) {
  const bool more = header[0] > 0 && !header[1] && !header[2] && !header[4];
  cudaGraphSetConditional(loop, more ? 1u : 0u);
  if (passes) *passes += 1;
}

// What pcg_solve reports, into the graph's words: the status (border, then sweep fault, then NaN, as pcg_solve tests
// them) is kept if no earlier solve's is pending; residual = max over components of (float)sqrt(r.r), -inf without
// components; iterations = the longest component's.  One block.
__global__ void k_pcg_finish(CompScalars sc, int* __restrict__ words) {
  __shared__ float s_res[32];
  __shared__ int s_it[32];
  const int n = sc.header[3];
  float worst = -INFINITY;
  int worst_it = 0;
  for (int id = threadIdx.x; id < n; id += blockDim.x) {
    worst = fmaxf(worst, (float)sqrt(sc.rr_cur[id]));
    worst_it = max(worst_it, sc.iters[id]);
  }
  for (int o = 16; o > 0; o >>= 1) {
    worst = fmaxf(worst, __shfl_down_sync(0xffffffffu, worst, o));
    worst_it = max(worst_it, __shfl_down_sync(0xffffffffu, worst_it, o));
  }
  if ((threadIdx.x & 31) == 0) { s_res[threadIdx.x >> 5] = worst; s_it[threadIdx.x >> 5] = worst_it; }
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int w = 1; w < (int)(blockDim.x >> 5); w++) { worst = fmaxf(worst, s_res[w]); worst_it = max(worst_it, s_it[w]); }
  const int status = sc.header[4] ? 1 : sc.header[2] ? 5 : sc.header[1] ? 2 : 0;
  if (status && words[0] == 0) words[0] = status;
  words[1] = worst_it;
  words[2] = __float_as_int(worst);
}

__global__ void k_xsum(const unsigned short* __restrict__ cf, const int* __restrict__ comp,
                       const float* __restrict__ x, CompScalars sc, long long slots) {
  CompAcc a;
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < slots; q += (long long)gridDim.x * blockDim.x) {
    if (!(cf[q] & kInSys)) continue;
    a.add(sc.xsum, comp[q], (double)x[q]);
  }
  warp_comp_add(sc.xsum, a.comp, a.v);
}

// copyPressureFromSystem (:1165-1188): p = x - mean(x of the component); cells outside any solved
// system keep the 0 of THCudaTensor_zero (:1337).  remove_mean = 0: x as it is (the preconditioner hook).
__global__ void k_writeback(float* __restrict__ p, const int* __restrict__ parent, const int* __restrict__ csize,
                            const int* __restrict__ cid, const float* __restrict__ x, CompScalars sc, PcgGeo g,
                            int remove_mean) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= g.n * g.nb) return;
  float out = 0.0f;
  const int root = parent[c];
  if (root >= 0 && csize[root] >= 2) {
    const int id = cid[root];
    const int b = (int)(c / g.n);
    const long long cc = c % g.n;
    const int i = (int)(cc % g.nx), j = (int)((cc / g.nx) % g.ny), k = (int)(cc / ((long long)g.nx * g.ny));
    const float mean = remove_mean ? (float)(sc.xsum[id] / (double)sc.cnt[id]) : 0.0f;
    out = x[skew_index(g, b * g.nz + k, j, i)] - mean;
  }
  p[c] = out;
}

// ---- the triangular sweeps -------------------------------------------------------------------
__device__ __forceinline__ unsigned long long ld_acquire(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ int ld_acquire_cta(const int* p) {
  int v;
  asm volatile("ld.acquire.cta.shared.s32 %0, [%1];" : "=r"(v) : "r"((unsigned)__cvta_generic_to_shared(p)) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_cta(int* p, int v) {
  asm volatile("st.release.cta.shared.s32 [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(p)), "r"(v) : "memory");
}
// Per-tick barrier of the compute warps and the gate warp (the talk warp never joins it).
__device__ __forceinline__ void compute_barrier(int n_threads) {
  asm volatile("bar.sync 1, %0;" ::"r"(n_threads) : "memory");
}

// Bounded wait: a stalled pipeline records a fault instead of hanging the device.
__device__ __forceinline__ bool spin_expired(long long spins, int* faults) {
  if (spins > kSpinLimit) { atomicAdd(faults, 1); return true; }
  if ((spins & 1023) == 0 && *(volatile int*)faults != 0) return true;
  return false;
}

struct SweepArgs {
  const unsigned short* cf;
  const int* comp;
  const float* r;
  float* z;
  float* pre;
  unsigned long long* prog_f;     // [chunks] steps of the chunk's TOP plane completed, forward
  unsigned long long* prog_b;     // [chunks] steps of the chunk's BOTTOM plane completed, backward
  unsigned long long base;        // epoch offset of this launch
  double* rz;                     // per-component r.z accumulators
  int* faults;
  unsigned long long* timing;     // debug: [chunk][4] globaltimer at fwd start / end, bwd start / end (or null)
};

// One CTA = GP thread groups of NYP threads; group gq works on plane chunk * GP + gq and runs one
// wavefront step behind the group below it (forward) / above it (backward).
// FACTOR: forward only, computes pre = 1 / R_ii of the IC(0) factor.
template <bool FACTOR>
__global__ void __launch_bounds__(1024, 1) k_sweep(SweepArgs a, PcgGeo g) {
  extern __shared__ float sh[];                 // [GP][2][W], W = NYP + 2, slot j + 1 = grid row j
  __shared__ int sm_done;                       // ticks the compute warps have completed in this chunk
  __shared__ int sm_avail;                      // steps of the neighbour chunk known to be complete
  const int W = g.NYP + 2;
  const int T = g.NYP;                          // threads per group
  const int n_compute = g.GP * T;
  // Two service warps behind the compute warps.  The GATE warp joins the per-tick barrier and then
  // publishes the tick count to shared memory: it has no loads in flight, so its release store costs
  // nothing (a compute thread's release would first wait for its own prefetches, one memory latency per
  // tick).  The TALK warp (one lane) moves progress between shared memory and the global progress words.
  const bool is_aux = (int)threadIdx.x >= n_compute;
  const bool is_gate = is_aux && (int)threadIdx.x < n_compute + 32;
  const int n_barrier = n_compute + 32;
  const int gq = is_aux ? 0 : threadIdx.x / T;  // group within the CTA
  const int j = threadIdx.x - gq * T;           // grid row owned by this thread
  for (int q = threadIdx.x; q < g.GP * 2 * W; q += blockDim.x) sh[q] = 0.0f;
  const int ticks = g.S + g.GP - 1;
  constexpr int kDepth = 3;                     // loads run kDepth ticks ahead of their use (ring of 4)
  struct Slot { unsigned c; float r, pre, z, nb, nb2; };   // nb, nb2: values of the neighbour chunk's plane
  Slot ring[4];

  // Aux lane: forwards the neighbour chunk's progress word into sm_avail and this chunk's progress
  // (sm_done, minus the lag of the plane the neighbour reads) into its own progress word.
  const int ticks4_ = (ticks + 3) & ~3;
  auto aux_loop = [&](const unsigned long long* their_word, unsigned long long* my_word) {
    int published = 0, avail = 0;
    long long spins = 0;
    for (;;) {
      const int d = ld_acquire_cta(&sm_done);
      if (their_word && avail < g.S) {
        const unsigned long long v = ld_acquire(their_word);
        const int steps = v > a.base ? (int)min(v - a.base, (unsigned long long)g.S) : 0;
        if (steps > avail) { avail = steps; st_release_cta(&sm_avail, avail); }
      }
      const int lead = min(d - (g.GP - 1), g.S);         // steps completed by the slowest group
      if (lead > published) { st_release(my_word, a.base + (unsigned long long)lead); published = lead; }
      if (d >= ticks4_) break;
      if (spin_expired(++spins, a.faults)) break;
    }
  };
  // Group that reads the neighbour chunk: block until `steps` of it are known complete.
  auto need_steps = [&](int steps) {
    steps = min(steps, g.S);
    long long spins = 0;
    while (ld_acquire_cta(&sm_avail) < steps) if (spin_expired(++spins, a.faults)) break;
  };

  // Arithmetic notes for both sweeps.  A neighbour that is in the system is always linked (fluid
  // neighbours belong to the same component) and one that is not contributes an exchanged value of 0,
  // so no link bits are tested: the exchanged values are simply added.  Cells of un-preconditioned
  // components (pre = 1) exchange 0 so that they reduce to z = r, and cells outside the system have
  // pre = 0, which makes their results 0.  In 2-D the planes of a CTA are different batch elements and
  // the z term is switched off.
  const int ticks4 = (ticks + 3) & ~3;          // the tick loops are unrolled by 4; surplus ticks do nothing
  auto row_of = [&](int s) { return s >= g.R ? s - g.R : s; };   // stored row of wavefront s
  const float use_z = g.is3d ? 1.0f : 0.0f;

  // ---------------- forward: R^T y = r (or the factor) ----------------
  for (int chunk = blockIdx.x; chunk < g.chunks; chunk += gridDim.x) {
    const bool wait_below = g.is3d && chunk > 0;
    if (threadIdx.x == 0) { sm_done = 0; sm_avail = 0; }
    __syncthreads();
    if (a.timing && threadIdx.x == 0) a.timing[chunk * 4 + 0] = global_ns();
    if (is_aux) {
      if (is_gate) {
        for (int tick = 0; tick < ticks4; tick++) {
          compute_barrier(n_barrier);
          if (threadIdx.x == n_compute) st_release_cta(&sm_done, tick + 1);
        }
      } else if (threadIdx.x == n_compute + 32) {
        aux_loop(wait_below ? a.prog_f + chunk - 1 : nullptr, a.prog_f + chunk);
      }
    } else {
      const int pl = chunk * g.GP + gq;
      const bool plane_ok = pl < g.P && j < g.ny;
      const bool from_global = wait_below && gq == 0;
      const long long plane0 = (long long)pl * g.plane + j;
      const unsigned short* p_cf = a.cf + plane0;
      const float* p_r = a.r + plane0;
      float* p_pre = a.pre + plane0;
      float* p_z = a.z + plane0;
      float* sm = sh + gq * 2 * W + j;           // sm[1 + parity * W] = this row's exchange slot
      const int below_off = gq > 0 ? 1 - 2 * W : 0;   // same slot of the group one plane below (previous parity)
      // Everything step s of this thread needs from global memory.
      auto fetch = [&](int tick) {
        Slot f;
        f.c = 0; f.r = 0.0f; f.pre = 0.0f; f.z = 0.0f; f.nb = 0.0f; f.nb2 = 0.0f;
        const int s = tick - gq;
        if (plane_ok && (unsigned)(s - j) < (unsigned)g.nx) {        // cell (s - j, j) exists
          const int off = (s >= g.R ? s - g.R : s) * g.NYP;
          f.c = p_cf[off];
          if (!FACTOR) { f.r = p_r[off]; f.pre = p_pre[off]; }
          if (from_global) {                   // no arithmetic here: a use would wait for the loads
            f.nb = __ldcg(p_pre + off - g.plane);
            f.nb2 = FACTOR ? 1.0f : __ldcg(p_z + off - g.plane);
          }
        }
        return f;
      };
      float carry = 0.0f;                        // this row's previous cell
      if (from_global) need_steps(kDepth);
#pragma unroll
      for (int u = 0; u < kDepth; u++) ring[u] = fetch(u);
      for (int tick0 = 0; tick0 < ticks4; tick0 += 4) {
#pragma unroll
        for (int u = 0; u < 4; u++) {
          const int tick = tick0 + u;
          if (from_global) need_steps(tick + kDepth + 1);
          ring[(u + kDepth) & 3] = fetch(tick + kDepth);
          const Slot f = ring[u];
          const int prv = (u & 1) ^ 1;            // tick0 is a multiple of 4: parities are compile-time
          const float ym = sm[prv * W];
          // The plane below passes on * pre * y of its cell through shared memory; global memory holds
          // only pre and y, so that term is masked with THIS cell's bit (a fluid z-neighbour belongs to
          // the same component, and an un-preconditioned cell must reduce to z = r).
          const float zm = (gq > 0 ? sm[prv * W + below_off] : ((f.c & kPreOn) ? f.nb * f.nb2 : 0.0f)) * use_z;
          const float on = (f.c & kPreOn) ? 1.0f : 0.0f;
          float out;
          if (FACTOR) {
            const float dg = (float)((f.c >> kDiagShift) & 7u);
            float e = dg - carry * carry - ym * ym - zm * zm;
            if (!(e > 1e-6f * dg)) e = dg;                     // vanishing pivot guard
            const float pv = on != 0.0f ? 1.0f / sqrtf(e) : 1.0f;
            if (f.c & kInSys) __stcg(p_pre + row_of(tick - gq) * g.NYP, pv);
            out = on * pv;
          } else {
            const float y = (f.r + carry + ym + zm) * f.pre;
            if (f.c & kInSys) __stcg(p_z + row_of(tick - gq) * g.NYP, y);
            out = on * f.pre * y;
          }
          carry = out;
          sm[1 + (u & 1) * W] = out;
          compute_barrier(n_barrier);
        }
      }
    }
    __syncthreads();
    if (a.timing && threadIdx.x == 0) a.timing[chunk * 4 + 1] = global_ns();
  }
  if (FACTOR) return;

  // ---------------- backward: R z = y, and r.z per component ----------------
  CompAcc racc;
  const int my_last = blockIdx.x + ((g.chunks - 1 - blockIdx.x) / gridDim.x) * gridDim.x;   // highest chunk of this CTA
  for (int chunk = my_last; chunk >= 0; chunk -= gridDim.x) {
    const bool wait_above = g.is3d && chunk < g.chunks - 1;
    if (threadIdx.x == 0) { sm_done = 0; sm_avail = 0; }
    for (int q = threadIdx.x; q < g.GP * 2 * W; q += blockDim.x) sh[q] = 0.0f;
    __syncthreads();
    if (a.timing && threadIdx.x == 0) a.timing[chunk * 4 + 2] = global_ns();
    if (is_aux) {
      if (is_gate) {
        for (int tick = 0; tick < ticks4; tick++) {
          compute_barrier(n_barrier);
          if (threadIdx.x == n_compute) st_release_cta(&sm_done, tick + 1);
        }
      } else if (threadIdx.x == n_compute + 32) {
        aux_loop(wait_above ? a.prog_b + chunk + 1 : nullptr, a.prog_b + chunk);
      }
    } else {
      const int pl = chunk * g.GP + gq;
      const bool plane_ok = pl < g.P && j < g.ny;
      const bool from_global = wait_above && gq == g.GP - 1;
      const int lag = g.GP - 1 - gq;            // the top group leads
      const long long plane0 = (long long)pl * g.plane + j;
      const unsigned short* p_cf = a.cf + plane0;
      const float* p_r = a.r + plane0;
      const float* p_pre = a.pre + plane0;
      float* p_z = a.z + plane0;
      const int* p_comp = a.comp + plane0;
      float* sm = sh + gq * 2 * W + j;
      const int above_off = gq < g.GP - 1 ? 1 + 2 * W : 0;
      auto fetch = [&](int tick) {
        Slot f;
        f.c = 0; f.r = 0.0f; f.pre = 0.0f; f.z = 0.0f; f.nb = 0.0f; f.nb2 = 0.0f;
        const int st = tick - lag;
        const int s = g.S - 1 - st;
        if (plane_ok && (unsigned)(s - j) < (unsigned)g.nx) {
          const int off = row_of(s) * g.NYP;
          f.c = p_cf[off];
          f.r = p_r[off];
          f.pre = p_pre[off];
          f.z = __ldcg(p_z + off);              // y of the forward sweep (written by this thread)
          if (from_global) f.nb = __ldcg(p_z + off + g.plane);
        }
        return f;
      };
      float carry = 0.0f;
      if (from_global) need_steps(kDepth);
#pragma unroll
      for (int u = 0; u < kDepth; u++) ring[u] = fetch(u);
      for (int tick0 = 0; tick0 < ticks4; tick0 += 4) {
#pragma unroll
        for (int u = 0; u < 4; u++) {
          const int tick = tick0 + u;
          if (from_global) need_steps(tick + kDepth + 1);
          ring[(u + kDepth) & 3] = fetch(tick + kDepth);
          const Slot f = ring[u];
          const int prv = (u & 1) ^ 1;
          const float yp = sm[prv * W + 2];
          const float zp = (gq < g.GP - 1 ? sm[prv * W + above_off] : f.nb) * use_z;
          const float on = (f.c & kPreOn) ? 1.0f : 0.0f;
          const float out = (f.z + f.pre * on * (carry + yp + zp)) * f.pre;
          if (f.c & kInSys) {
            const int off = row_of(g.S - 1 - (tick - lag)) * g.NYP;
            __stcg(p_z + off, out);
            racc.add(a.rz, p_comp[off], (double)f.r * (double)out);
          }
          carry = out;
          sm[1 + (u & 1) * W] = out;
          compute_barrier(n_barrier);
        }
      }
    }
    __syncthreads();
    if (a.timing && threadIdx.x == 0) a.timing[chunk * 4 + 3] = global_ns();
  }
  if (!is_aux) warp_comp_add(a.rz, racc.comp, racc.v);
}

// ---- normalizePressureMean (generic/tfluids.cc:845-921) -----------------------------------------
__global__ void k_npm_sum(const float* __restrict__ p, const int* __restrict__ parent, double* __restrict__ sums,
                          long long cells) {
  CompAcc a;
  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < cells; c += (long long)gridDim.x * blockDim.x) {
    const int root = parent[c];
    if (root >= 0) a.add(sums, root, (double)p[c]);
  }
  warp_comp_add(sums, a.comp, a.v);
}
__global__ void k_npm_subtract(float* __restrict__ p, const int* __restrict__ parent, const int* __restrict__ csize,
                               const double* __restrict__ sums, long long cells) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cells) return;
  const int root = parent[c];
  if (root < 0) return;
  const float mean = (float)sums[root] / (float)csize[root];
  p[c] = p[c] - mean;
}

inline unsigned blocks_for(long long n) { return (unsigned)((n + 255) / 256); }

}  // namespace

// ------------------------------------------------------------------------------------------------
size_t pcg_workspace_bytes(int nb, int nz, int ny, int nx) {
  const long long cells = (long long)nb * nz * ny * nx;
  const long long NYP = (ny + 31) / 32 * 32;
  const long long slots = (long long)nb * nz * (nx > ny ? nx : ny) * NYP;
  return (size_t)(cells * 12 + slots * (2 + 4 + 7 * 4) + 16 * 256 + 1024);
}

const char* pcg_status_string(int rc) {
  switch (rc) {
    case 0: return "ok";
    case 1: return "Non fluid cell found in a connected component or fluid cell found on the domain border";
    case 2: return "PCG Error: residual is nan!";
    case 3: return "PCG: CUDA error";
    case 4: return "PCG: grid too large for the sweep kernel (ny > 960)";
    case 5: return "PCG: internal error, sweep pipeline stalled";
    default: return "PCG: unknown error";
  }
}

namespace {

// What the solve and the preconditioner hook share: geometry, components, the system arrays in the
// skewed layout, the per-component scalars and the launch shape of the sweeps.
struct PcgSystem {
  PcgGeo g;
  int *parent, *csize, *cid;
  unsigned short* cf;
  int* comp;
  float *r, *z, *pre, *p0, *p1, *w, *x;
  int* header;                 // [0] active, [1] nan, [2] faults, [3] ncomp, [4] border status
  int ncomp;
  CompScalars cs;
  SweepArgs sa;
  int sweep_threads, sweep_grid;
  size_t sweep_smem;
  unsigned ew_blocks;
};

#define PCG_CUDA(call) do { if ((call) != cudaSuccess) return 3; } while (0)

// Geometry of the skewed layout and the sweeps' plane chunks.  Returns 0 or 4 (rows too long for a CTA).
int pcg_geometry(const PcgScratch& sc, int nb, int nz, int ny, int nx, int is3d, PcgGeo& g) {
  g.nx = nx; g.ny = ny; g.nz = nz; g.nb = nb; g.is3d = is3d ? 1 : 0;
  g.S = nx + ny - 1;
  g.NYP = (ny + 31) / 32 * 32;
  g.P = nb * nz;
  g.n = (long long)nz * ny * nx;
  g.R = nx > ny ? nx : ny;
  g.plane = (long long)g.R * g.NYP;
  g.slots = (long long)g.P * g.plane;
  if (g.NYP > 960) return 4;
  g.GP = (1024 - 64) / g.NYP;      // two service warps per CTA (gate, talk)
  if (sc.groups_override > 0 && sc.groups_override < g.GP) g.GP = sc.groups_override;
  if (g.GP > g.P) g.GP = g.P;
  g.chunks = (g.P + g.GP - 1) / g.GP;
  return 0;
}

// One-time setup of the scratch: host words, the sweeps' shared-memory limit, the SM count.
int pcg_init_once(PcgScratch& sc) {
  if (sc.sm_count) return 0;
  int dev = 0, sms = 0;
  PCG_CUDA(cudaGetDevice(&dev));
  PCG_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  if (!(sc.host = pinned_alloc<int>(16))) return 3;
  PCG_CUDA(cudaFuncSetAttribute(k_sweep<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
  PCG_CUDA(cudaFuncSetAttribute(k_sweep<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
  sc.sm_count = sms;
  return 0;
}

// What both drivers do first: geometry and launch shape of the sweeps, the workspace carved, and the labelling
// enqueued (header[3] = components of two or more cells, header[4] = a fluid cell on the border; with one, the union
// pass does nothing, so every component has one cell and no system is built).
int pcg_label(PcgScratch& sc, void* workspace, const float* flags, int nb, int nz, int ny, int nx, int is3d,
              long long* launches, cudaStream_t st, PcgSystem& s) {
  PcgGeo& g = s.g;
  if (pcg_geometry(sc, nb, nz, ny, nx, is3d, g)) return 4;
  const long long cells = g.n * nb;
  if (pcg_init_once(sc)) return 3;
  s.sweep_threads = g.GP * g.NYP + 64;
  s.sweep_smem = (size_t)g.GP * 2 * (g.NYP + 2) * sizeof(float);
  int occ = 0;
  PCG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_sweep<false>, s.sweep_threads, s.sweep_smem));
  if (occ < 1) return 3;
  s.sweep_grid = std::min(g.chunks, occ * sc.sm_count);
  s.ew_blocks = (unsigned)std::min<long long>((g.slots + 255) / 256, (long long)sc.sm_count * 8);
  // carve the workspace
  char* base = (char*)workspace;
  size_t off = 0;
  auto take = [&](size_t bytes) { off = (off + 255) & ~(size_t)255; char* r_ = base + off; off += bytes; return r_; };
  s.parent = (int*)take(cells * 4);
  s.csize = (int*)take(cells * 4);
  s.cid = (int*)take(cells * 4);
  s.cf = (unsigned short*)take(g.slots * 2);
  s.comp = (int*)take(g.slots * 4);
  s.r = (float*)take(g.slots * 4);
  s.z = (float*)take(g.slots * 4);
  s.pre = (float*)take(g.slots * 4);
  s.p0 = (float*)take(g.slots * 4);
  s.p1 = (float*)take(g.slots * 4);
  s.w = (float*)take(g.slots * 4);
  s.x = (float*)take(g.slots * 4);
  s.header = (int*)take(64);

  PCG_CUDA(cudaMemsetAsync(s.header, 0, 64, st));
  PCG_CUDA(cudaMemsetAsync(s.csize, 0, cells * 4, st));
  k_label_init<<<blocks_for(cells), 256, 0, st>>>(flags, s.parent, g, s.header + 4);
  k_label_union<false><<<blocks_for(cells), 256, 0, st>>>(s.parent, g, s.header + 4);
  k_label_flatten<<<blocks_for(cells), 256, 0, st>>>(s.parent, s.csize, g);
  k_label_assign<<<blocks_for(cells), 256, 0, st>>>(s.parent, s.csize, s.cid, g, s.header + 3);
  *launches += 4;
  return 0;
}

// The per-component scalars in `buf`, `stride` entries per array.
CompScalars comp_scalars(char* buf, size_t stride, int* header) {
  CompScalars cs;
  double* d = (double*)buf;
  cs.rz_new = d; cs.rz_old = d + stride; cs.pw = d + 2 * stride; cs.rr_new = d + 3 * stride;
  cs.rr_cur = d + 4 * stride; cs.xsum = d + 5 * stride;
  int* q = (int*)(d + 6 * stride);
  cs.cnt = q; cs.done = q + stride; cs.iters = q + 2 * stride;
  cs.header = header;
  return cs;
}
constexpr size_t kCompBytes = 6 * 8 + 3 * 4;     // scalars of one component

// The system arrays (cleared, then k_build) and the sweeps' arguments over the progress words `prog` ([2][chunks]);
// s.cs must be set.
int pcg_build(PcgScratch& sc, PcgSystem& s, const float* flags, const float* div, int precond,
              unsigned long long* prog, long long* launches, cudaStream_t st) {
  const PcgGeo& g = s.g;
  PCG_CUDA(cudaMemsetAsync(s.cf, 0, g.slots * 2, st));
  PCG_CUDA(cudaMemsetAsync(s.comp, 0xff, g.slots * 4, st));
  for (float* v : {s.r, s.z, s.pre, s.p0, s.p1, s.w, s.x}) PCG_CUDA(cudaMemsetAsync(v, 0, g.slots * 4, st));
  k_build<<<blocks_for(g.n * g.nb), 256, 0, st>>>(flags, div, s.parent, s.csize, s.cid, s.cf, s.comp, s.r, s.cs.cnt,
                                                  g, precond);
  *launches += 1;

  SweepArgs& sa = s.sa;
  sa.cf = s.cf; sa.comp = s.comp; sa.r = s.r; sa.z = s.z; sa.pre = s.pre;
  sa.prog_f = prog; sa.prog_b = prog + g.chunks;
  sa.base = 0;
  sa.rz = s.cs.rz_new; sa.faults = s.header + 2;
  sa.timing = (unsigned long long*)sc.debug_timing;
  return 0;
}

// Labelling, and (when there is a system of two or more cells, s.ncomp > 0) the per-component scalars, the progress
// words and the system arrays.  `out` is zeroed: cells outside every system keep that 0.  Returns 0 or a status for
// pcg_status_string.
int pcg_setup(PcgScratch& sc, void* workspace, float* out, const float* flags, const float* div, int nb, int nz,
              int ny, int nx, int is3d, int precond, long long* launches, cudaStream_t st, PcgSystem& s) {
  const int rc = pcg_label(sc, workspace, flags, nb, nz, ny, nx, is3d, launches, st, s);
  if (rc) return rc;
  const PcgGeo& g = s.g;
  const long long cells = g.n * nb;
  PCG_CUDA(cudaMemcpyAsync(sc.host.get(), s.header, 32, cudaMemcpyDeviceToHost, st));
  PCG_CUDA(cudaStreamSynchronize(st));
  if (sc.host.get()[4]) return 1;
  const int ncomp = s.ncomp = sc.host.get()[3];
  PCG_CUDA(cudaMemsetAsync(out, 0, cells * 4, st));                     // :1337
  if (ncomp == 0) return 0;
  // per-component scalars; a capacity is recorded once its buffer exists
  if ((size_t)ncomp * kCompBytes + 256 > sc.comp_cap) {
    const size_t cap = (size_t)ncomp * kCompBytes * 2 + 4096;
    sc.comp_buf = dev_alloc<char>(cap);
    sc.comp_cap = sc.comp_buf ? cap : 0;
    if (!sc.comp_buf) return 3;
  }
  PCG_CUDA(cudaMemsetAsync(sc.comp_buf.get(), 0, (size_t)ncomp * kCompBytes + 256, st));
  s.cs = comp_scalars(sc.comp_buf.get(), (size_t)ncomp, s.header);
  if ((size_t)g.chunks * 2 > sc.prog_cap) {
    const size_t cap = (size_t)g.chunks * 2 + 64;
    sc.prog = dev_alloc<unsigned long long>(cap);
    sc.prog_cap = 0;
    if (!sc.prog) return 3;
    PCG_CUDA(cudaMemsetAsync(sc.prog.get(), 0, cap * 8, st));
    sc.prog_cap = cap;
    sc.epoch = 0;
  }
  return pcg_build(sc, s, flags, div, precond, sc.prog.get(), launches, st);
}

// One cooperative launch of the sweep pipeline: the IC(0) factor (pre) or one solve z = M^-1 r, with s.sa.base set.
cudaError_t launch_sweep_at(PcgSystem& s, bool factor, long long* launches, cudaStream_t st) {
  void* args[] = {(void*)&s.sa, (void*)&s.g};
  *launches += 1;
  return cudaLaunchCooperativeKernel(factor ? (void*)k_sweep<true> : (void*)k_sweep<false>, dim3(s.sweep_grid),
                                     dim3(s.sweep_threads), args, s.sweep_smem, st);
}
// Direct solves: every launch gets the next epoch of the scratch's progress words, so no wait is satisfied by
// progress an earlier launch left there.
cudaError_t launch_sweep(PcgScratch& sc, PcgSystem& s, bool factor, long long* launches, cudaStream_t st) {
  s.sa.base = sc.epoch;
  sc.epoch += (unsigned long long)s.g.S + 1;
  return launch_sweep_at(s, factor, launches, st);
}

}  // namespace

int pcg_solve(PcgScratch& sc, void* workspace, float* p, const float* flags, const float* div, int nb, int nz, int ny,
              int nx, int is3d, int precond, float tol, int max_iter, float* residual, int* iterations,
              long long* launches, cudaStream_t st) {
  PcgSystem s;
  const int rc = pcg_setup(sc, workspace, p, flags, div, nb, nz, ny, nx, is3d, precond, launches, st, s);
  if (rc) return rc;
  if (s.ncomp == 0) {
    if (residual) *residual = -INFINITY;                               // :1343
    if (iterations) *iterations = 0;
    return 0;
  }
  const PcgGeo& g = s.g;
  const long long cells = g.n * nb;
  const int ncomp = s.ncomp;
  const CompScalars& cs = s.cs;
  int* header = s.header;
  int* const host = sc.host.get();
  const unsigned ew_blocks = s.ew_blocks;
  const int no_precond = precond == 0;
  if (!no_precond) PCG_CUDA(launch_sweep(sc, s, true, launches, st));
  k_rr_init<<<ew_blocks, 256, 0, st>>>(s.cf, s.comp, s.r, cs, g.slots);
  const double tol2 = (double)tol * (double)tol;
  k_scalars<<<(ncomp + 255) / 256, 256, 0, st>>>(cs, nullptr, ncomp, tol2, max_iter, 1, no_precond);
  *launches += 2;
  PCG_CUDA(cudaMemcpyAsync(host, header, 16, cudaMemcpyDeviceToHost, st));
  PCG_CUDA(cudaStreamSynchronize(st));
  float* p_old = s.p0;
  float* p_new = s.p1;
  // The host only needs to learn when every component has terminated; termination itself (tolerance or
  // iteration cap) is decided per component on the device, so reading back every 4th iteration changes
  // nothing in the result -- iterations past a component's end are no-ops for it.
  while (host[0] > 0 && !host[1] && !host[2]) {
    for (int rep = 0; rep < 4; rep++) {
      PCG_CUDA(cudaMemsetAsync(header, 0, 4, st));
      if (!no_precond) PCG_CUDA(launch_sweep(sc, s, false, launches, st));
      k_direction_spmv<<<ew_blocks, g.NYP, 0, st>>>(s.cf, s.comp, no_precond ? s.r : s.z, p_old, p_new, s.w, cs, g,
                                                    no_precond);
      k_update<<<ew_blocks, 256, 0, st>>>(s.cf, s.comp, p_new, s.w, s.x, s.r, cs, g.slots, no_precond);
      k_scalars<<<(ncomp + 255) / 256, 256, 0, st>>>(cs, nullptr, ncomp, tol2, max_iter, 0, no_precond);
      *launches += 3;
      float* tswap = p_old; p_old = p_new; p_new = tswap;
    }
    PCG_CUDA(cudaMemcpyAsync(host, header, 16, cudaMemcpyDeviceToHost, st));
    PCG_CUDA(cudaStreamSynchronize(st));
  }
  if (host[2]) return 5;
  if (host[1]) return 2;
  k_xsum<<<ew_blocks, 256, 0, st>>>(s.cf, s.comp, s.x, cs, g.slots);
  k_writeback<<<blocks_for(cells), 256, 0, st>>>(p, s.parent, s.csize, s.cid, s.x, cs, g, 1);
  *launches += 2;
  // residual = max over components of sqrt(r.r) (:1728), iterations = the longest component
  std::vector<double> rr(ncomp);
  std::vector<int> it(ncomp);
  PCG_CUDA(cudaMemcpyAsync(rr.data(), cs.rr_cur, sizeof(double) * ncomp, cudaMemcpyDeviceToHost, st));
  PCG_CUDA(cudaMemcpyAsync(it.data(), cs.iters, sizeof(int) * ncomp, cudaMemcpyDeviceToHost, st));
  PCG_CUDA(cudaStreamSynchronize(st));
  if (cudaPeekAtLastError() != cudaSuccess) return 3;         // the caller reads (and clears) the error
  float worst = -INFINITY;
  int worst_it = 0;
  for (int c = 0; c < ncomp; c++) {
    const float v = (float)sqrt(rr[c]);
    if (v > worst) worst = v;
    if (it[c] > worst_it) worst_it = it[c];
  }
  if (residual) *residual = worst;
  if (iterations) *iterations = worst_it;
  return 0;
}

cudaError_t capture_while_handle(cudaStream_t st, unsigned initial, cudaGraphConditionalHandle* loop) {
  cudaStreamCaptureStatus cap_status;
  cudaGraph_t graph = nullptr;
  cudaError_t e = cudaStreamGetCaptureInfo(st, &cap_status, nullptr, &graph, nullptr, nullptr);
  if (e != cudaSuccess) return e;
  if (cap_status != cudaStreamCaptureStatusActive) return cudaErrorStreamCaptureInvalidated;
  return cudaGraphConditionalHandleCreate(loop, graph, initial, cudaGraphCondAssignDefault);
}

int pcg_graph_alloc(PcgGraphScratch& gs, PcgScratch& sc, int nb, int nz, int ny, int nx, int is3d) {
  PcgGeo g;
  if (pcg_geometry(sc, nb, nz, ny, nx, is3d, g)) return 4;
  if (pcg_init_once(sc)) return 3;
  // A component in the system has at least two cells, so there are at most cells / 2 of them, whatever the flags
  // hold at a replay.
  const long long cap = std::max(1ll, g.n * nb / 2);
  if (!(gs.comp_buf = dev_alloc<char>((size_t)cap * kCompBytes))) return 3;
  gs.comp_cap = cap;
  gs.prog_words = 2ll * g.chunks;
  if (!(gs.prog = dev_zeros<unsigned long long>((size_t)gs.prog_words))) return 3;
  if (!(gs.words = dev_zeros<int>(8))) return 3;
  return 0;
}

// The loop runs two iterations per pass, so p_old / p_new swap as pointers (the body's launches are fixed) and a
// replay runs at most one iteration more than the longest component needs, where pcg_solve's reads every 4th
// iteration allow up to three; the extra ones are no-ops for finished components, so the results are pcg_solve's.
//
// Progress words: k_sweep's cross-CTA waits accept a progress value above the launch's base.  A base taken from a
// host counter would be frozen by the capture, and the second sweep of a replay would find the words already past it
// and read z values not yet written.  So each captured sweep is preceded by a memset node that zeroes the graph's own
// words, and runs with base 0: the nodes of one replay run in stream order, a replay of an executable graph never
// overlaps another of the same graph, and no other solve writes these words, so every value a sweep reads was
// published by that sweep.
int pcg_solve_graph(PcgGraphScratch& gs, PcgScratch& sc, void* workspace, float* p, const float* flags,
                    const float* div, int nb, int nz, int ny, int nx, int is3d, int precond, float tol, int max_iter,
                    long long* launches, cudaStream_t st, cudaStream_t loop_body) {
  PcgSystem s;
  int rc = pcg_label(sc, workspace, flags, nb, nz, ny, nx, is3d, launches, st, s);
  if (rc) return rc;
  const PcgGeo& g = s.g;
  if (!gs.comp_buf || gs.comp_cap < std::max(1ll, g.n * nb / 2) || gs.prog_words < 2ll * g.chunks) return 3;
  s.cs = comp_scalars(gs.comp_buf.get(), (size_t)gs.comp_cap, s.header);
  const CompScalars& cs = s.cs;
  const unsigned comp_blocks = (unsigned)sc.sm_count;     // loops over the device's component count
  k_comp_clear<<<comp_blocks, 256, 0, st>>>(cs);
  *launches += 1;
  if ((rc = pcg_build(sc, s, flags, div, precond, gs.prog.get(), launches, st))) return rc;
  const int no_precond = precond == 0;
  const double tol2 = (double)tol * (double)tol;
  const unsigned ew_blocks = s.ew_blocks;
  auto sweep = [&](bool factor, long long* n, cudaStream_t q) {
    const cudaError_t e = cudaMemsetAsync(gs.prog.get(), 0, (size_t)gs.prog_words * 8, q);
    return e != cudaSuccess ? e : launch_sweep_at(s, factor, n, q);
  };
  if (!no_precond) PCG_CUDA(sweep(true, launches, st));
  k_rr_init<<<ew_blocks, 256, 0, st>>>(s.cf, s.comp, s.r, cs, g.slots);
  k_scalars<<<comp_blocks, 256, 0, st>>>(cs, s.header + 3, 0, tol2, max_iter, 1, no_precond);
  *launches += 2;

  // the WHILE node after what is captured so far; the first test arms it
  cudaGraphConditionalHandle loop;
  PCG_CUDA(capture_while_handle(st, 0, &loop));
  k_pcg_continue<<<1, 1, 0, st>>>(s.header, loop, nullptr);
  *launches += 1;

  // the body, captured on loop_body into the node's body graph
  long long body = 0;
  const cudaError_t be = capture_while(st, loop, loop_body, [&](cudaStream_t bs) {
    float* p_old = s.p0;
    float* p_new = s.p1;
    for (int rep = 0; rep < 2; rep++) {
      cudaError_t e = cudaMemsetAsync(s.header, 0, 4, bs);
      if (e == cudaSuccess && !no_precond) e = sweep(false, &body, bs);
      if (e != cudaSuccess) return e;
      k_direction_spmv<<<ew_blocks, g.NYP, 0, bs>>>(s.cf, s.comp, no_precond ? s.r : s.z, p_old, p_new, s.w, cs, g,
                                                    no_precond);
      k_update<<<ew_blocks, 256, 0, bs>>>(s.cf, s.comp, p_new, s.w, s.x, s.r, cs, g.slots, no_precond);
      k_scalars<<<comp_blocks, 256, 0, bs>>>(cs, s.header + 3, 0, tol2, max_iter, 0, no_precond);
      body += 3;
      float* tswap = p_old; p_old = p_new; p_new = tswap;
    }
    k_pcg_continue<<<1, 1, 0, bs>>>(s.header, loop, (unsigned long long*)(gs.words.get() + 4));
    body += 1;
    return cudaSuccess;
  });
  if (be != cudaSuccess) return 3;
  gs.body_launches = body;

  k_xsum<<<ew_blocks, 256, 0, st>>>(s.cf, s.comp, s.x, cs, g.slots);
  k_writeback<<<blocks_for(g.n * nb), 256, 0, st>>>(p, s.parent, s.csize, s.cid, s.x, cs, g, 1);
  k_pcg_finish<<<1, 256, 0, st>>>(cs, gs.words.get());
  *launches += 3;
  gs.captured = true;
  return cudaPeekAtLastError() == cudaSuccess ? 0 : 3;
}

int pcg_precond(PcgScratch& sc, void* workspace, float* z, const float* flags, const float* r, int nb, int nz, int ny,
                int nx, int is3d, int precond, int* geometry, long long* launches, cudaStream_t st) {
  PcgSystem s;
  const int rc = pcg_setup(sc, workspace, z, flags, r, nb, nz, ny, nx, is3d, precond, launches, st, s);
  if (rc) return rc;
  if (geometry) {
    geometry[0] = s.g.NYP; geometry[1] = s.g.GP; geometry[2] = s.g.chunks; geometry[3] = s.sweep_grid;
  }
  if (s.ncomp == 0) return 0;
  PCG_CUDA(launch_sweep(sc, s, true, launches, st));
  PCG_CUDA(launch_sweep(sc, s, false, launches, st));
  PCG_CUDA(cudaMemcpyAsync(sc.host.get(), s.header, 16, cudaMemcpyDeviceToHost, st));
  PCG_CUDA(cudaStreamSynchronize(st));
  if (sc.host.get()[2]) return 5;
  k_writeback<<<blocks_for(s.g.n * nb), 256, 0, st>>>(z, s.parent, s.csize, s.cid, s.z, s.cs, s.g, 0);
  *launches += 1;
  return cudaPeekAtLastError() == cudaSuccess ? 0 : 3;
#undef PCG_CUDA
}

// p -= mean of p over the cell's connected fluid component, every component of every batch element.
// The reference copies p and flags to the host, flood-fills there and copies back (init.lua:747-765).
int normalize_pressure_mean(void* workspace, float* p, const float* flags, int nb, int nz, int ny, int nx, int is3d,
                            long long* launches, cudaStream_t st) {
  PcgGeo g;
  g.nx = nx; g.ny = ny; g.nz = nz; g.nb = nb; g.is3d = is3d ? 1 : 0;
  g.n = (long long)nz * ny * nx;
  g.S = 0; g.NYP = 0; g.R = 0; g.P = nb * nz; g.plane = 0; g.slots = 0; g.GP = 1; g.chunks = 0;
  const long long cells = g.n * nb;
  char* base = (char*)workspace;
  size_t off = 0;
  auto take = [&](size_t bytes) { off = (off + 255) & ~(size_t)255; char* r_ = base + off; off += bytes; return r_; };
  int* parent = (int*)take(cells * 4);
  int* csize = (int*)take(cells * 4);
  double* sums = (double*)take(cells * 8);
  int* status = (int*)take(64);
  if (cudaMemsetAsync(csize, 0, cells * 4, st) != cudaSuccess) return 3;
  if (cudaMemsetAsync(sums, 0, cells * 8, st) != cudaSuccess) return 3;
  if (cudaMemsetAsync(status, 0, 64, st) != cudaSuccess) return 3;
  k_label_init<<<blocks_for(cells), 256, 0, st>>>(flags, parent, g, status);
  k_label_union<true><<<blocks_for(cells), 256, 0, st>>>(parent, g, status);
  k_label_flatten<<<blocks_for(cells), 256, 0, st>>>(parent, csize, g);
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const unsigned blocks = (unsigned)std::min<long long>((cells + 255) / 256, (long long)sms * 8);
  k_npm_sum<<<blocks, 256, 0, st>>>(p, parent, sums, cells);
  k_npm_subtract<<<blocks_for(cells), 256, 0, st>>>(p, parent, csize, sums, cells);
  *launches += 5;
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

}  // namespace tfl
