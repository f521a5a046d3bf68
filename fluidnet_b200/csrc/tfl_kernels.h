// Host-callable launchers of the CUDA kernels (internal to libtfl; the public surface is
// include/tfl.h).
#pragma once
#include <cuda_runtime.h>
#include "../../include/tfl.h"
#include "tfl_device.cuh"
#include "tfl_holders.h"

namespace tfl {

// ---- tfl_stencils.cu (-fmad=false) ----
void launch_empty_domain(float* flags, const Geo& g, int bnd, cudaStream_t st);
void launch_flags_to_occupancy(const float* flags, float* occ, long long n, unsigned long long* bad,
                               cudaStream_t st);
void launch_set_wall_bcs(float* U, const float* flags, const Geo& g, int as_mask, cudaStream_t st);
void launch_divergence(const float* U, const float* flags, float* div, const Geo& g, cudaStream_t st);
void launch_velocity_update(float* U, const float* flags, const float* p, const Geo& g, cudaStream_t st);
void launch_add_buoyancy(float* U, const float* flags, const float* rho, const float s[3], const Geo& g,
                         cudaStream_t st);
int launch_vorticity(float* U, const float* flags, float strength, float* curl, float* cnorm, float* force,
                     const Geo& g, cudaStream_t st);
// Gravity and advection take the operators' float flags or the fused step's byte flags (FT float or unsigned char).
template <typename FT>
void launch_add_gravity(float* U, const FT* flags, const float f[3], const Geo& g, cudaStream_t st);
// g: range of the result; g_fwd: (wider, in slab mode) range of the forward pass.
// clear: clearance field of the same grid (launch_clearance) or nullptr (general code everywhere).
template <typename FT>
int launch_advect_scalar(float dt, const float* s, const float* U, const FT* flags, const unsigned char* clear,
                         int method, int outside, float strength, float* dst, float* fwd, float* fwd_pos,
                         const Geo& g, const Geo& g_fwd, cudaStream_t st);
template <typename FT>
int launch_advect_vel(float dt, const float* U, const FT* flags, const unsigned char* clear, int method,
                      float strength, float* dst, float* fwd, const Geo& g, const Geo& g_fwd, cudaStream_t st);
// ---- tfl_advect_tile.cu (-fmad=false): maccormackOurs advectVel as one kernel over shared-memory tiles ----
// hf: halo of the forward field in cells (1: traces < ~0.5 cell are served from the tile, 2: < ~1.5; longer ones
// take the general code).  longest: optional device word, atomicMax of the longest trace (float bits).
// One launch covers every batch entry.  Returns false when the grid does not qualify (2-D, nx % 4 != 0, nz < 3,
// unaligned U): run launch_advect_vel then.
bool launch_advect_vel_tile(float dt, const float* U, const unsigned char* flags, const unsigned char* clear,
                            float strength, float* dst, const Geo& g, int hf, unsigned int* longest, cudaStream_t st);
// advectScalar('maccormackOurs') on the same tiles.
bool launch_advect_scalar_tile(float dt, const float* src, const float* U, const unsigned char* flags,
                               const unsigned char* clear, int outside, float strength, float* dst, const Geo& g, int hf,
                               cudaStream_t st);
// Clearance of every cell of the local storage (advection fast path, tfl_device.cuh) from the byte flags; tmp:
// scratch of the same size; gate: optional device word, the kernels do nothing when it is 0.  Returns the launch count.
int launch_clearance(const unsigned char* flags, unsigned char* clear, unsigned char* tmp, const Geo& g, const int* gate,
                     cudaStream_t st);
void launch_jacobi_mask(const float* flags, unsigned char* mask, const Geo& g, cudaStream_t st);
// done: optional device word (JacobiState::done); the sweep does nothing once it is set.
void launch_jacobi_iter(const unsigned char* mask, const float* div, const float* prev, float* cur,
                        const Geo& g, cudaStream_t st, const int* done = nullptr);
// One block of `sweeps` sweeps on local planes [z_lo, z_hi) that shrink by shr_lo / shr_hi planes per sweep
// (sweep s reads pa and writes pb for even s, the reverse for odd s).  launch_jacobi_block runs them in one
// cooperative launch and returns its block depth in planes (4, or 6 with `deep`), or 0 when the shape / device does
// not qualify or the range does not fit co-resident; it serves the z-slab blocks and, with [0, nz) and no shrink,
// the whole-grid solve.  launch_jacobi_range_sweeps launches one kernel per sweep.
int launch_jacobi_block(const unsigned char* mask, const float* div, float* pa, float* pb, const Geo& g, int z_lo,
                        int z_hi, int shr_lo, int shr_hi, int sweeps, bool deep, cudaStream_t st);
void launch_jacobi_range_sweeps(const unsigned char* mask, const float* div, float* pa, float* pb, const Geo& g,
                                int z_lo, int z_hi, int shr_lo, int shr_hi, int sweeps, cudaStream_t st);
void launch_sqdiff(const float* a, const float* b, long long n, int nb, double* out, cudaStream_t st);
// The Jacobi solve run to a tolerance on the device (tfl_solve_linear_system_jacobi_dev): the host loop's state.
struct JacobiState {
  int done;            // set once the solve has stopped
  int iter;            // the host loop's iteration counter
  unsigned arrived;    // CTAs of the current residual launch that have written their slot
  int last;            // index of the last sweep run: it wrote p when even, pPrev when odd
  float res;           // residual of the last sweep
};
// The host loop's test after sweep s (0-based) with residual res: stop when res < tol, before the counter counts the
// sweep, or once the counter reaches max_iter.  *iter receives the counter.
__device__ __forceinline__ bool jacobi_stops(float res, float tol, int s, int max_iter, int* iter) {
  if (res < tol) {
    *iter = s;
    return true;
  }
  *iter = s + 1;
  return s + 1 >= max_iter;
}
struct JacobiTolArgs {
  double* slots = nullptr;          // per-CTA partial sums of (p - pPrev)^2 per batch entry (jacobi_tol_slots doubles)
  JacobiState* state = nullptr;     // zeroed before the first sweep
  float* res_out = nullptr;         // optional device copies of the final residual and iteration count
  int* iter_out = nullptr;
  float tol = 0.0f;
  int max_iter = 0;
  cudaGraphConditionalHandle loop = 0;   // the WHILE node of a captured solve (has_loop): cleared when it stops
  int has_loop = 0;
  // launch_jacobi_block_planes (the z-slab tolerance solve): slots receive the per-plane residuals, save the block's
  // start; nothing runs while *gate is set
  const int* gate = nullptr;
  float* save = nullptr;
  int own_lo = 0, own_hi = 0;
};
// Doubles of JacobiTolArgs::slots either path below needs on grid g.
long long jacobi_tol_slots(const Geo& g);
// The whole solve in one cooperative launch (k_jacobi_resident<4, true>): sweep 0 reads p_prev and writes p, p gets
// the result, state and the outputs are written.  false (nothing launched) when the grid does not qualify (3-D,
// nz >= 4, up to 3 x 2^20 cells, nx % 128, ny % 8, aligned, co-resident).
bool launch_jacobi_tol_resident(const unsigned char* mask, const float* div, float* p_prev, float* p, const Geo& g,
                                int max_iter, const JacobiTolArgs& t, cudaStream_t st);
// The device-driven loop on every other grid: after each launch_jacobi_iter with done = &state->done, one residual
// launch; once the loop has stopped, the copy back moves the result into p when it ended in p_prev.
void launch_jacobi_residual(const float* p, const float* p_prev, const Geo& g, const JacobiTolArgs& t, cudaStream_t st);
void launch_jacobi_copy_back(float* p, const float* p_prev, long long cells, const JacobiState* state, cudaStream_t st);
// One block of the z-slab tolerance solve in one cooperative launch (k_jacobi_resident_planes<4>): the sweeps of
// launch_jacobi_block with 4-plane blocks, plus t.save <- pa on [z_lo, z_hi) first and, per sweep, the owned planes'
// residuals in t.slots[sweep][plane][tile] with launch_jacobi_plane_residual's bits.  Returns 4, or 0 (nothing
// launched) where launch_jacobi_block would return 0 without `deep`.
int launch_jacobi_block_planes(const unsigned char* mask, const float* div, float* pa, float* pb, const Geo& g, int z_lo,
                               int z_hi, int shr_lo, int shr_hi, int sweeps, const JacobiTolArgs& t, cudaStream_t st);
// The z-slab tolerance solve's per-plane residual of one sweep (one batch entry): slots[plane][tile] receives the sum
// of (cur - prev)^2 over each 128 x 8 tile of local planes [z_lo, z_lo + planes), jacobi_plane_tiles(nx, ny) tiles per
// plane, in an order fixed by nx and ny alone.  Does nothing once *done is set.
int jacobi_plane_tiles(int nx, int ny);
void launch_jacobi_plane_residual(const float* cur, const float* prev, int nx, int ny, int z_lo, int planes,
                                  double* slots, const int* done, cudaStream_t st);
// changed: optional device word that is OR-ed with 1 when a byte differs from what `o` held before.
void launch_flags_to_u8(const float* f, unsigned char* o, long long n, int* changed, cudaStream_t st);
void launch_apply_bc(float* x, const float* inv, const float* bc, long long n, cudaStream_t st);
void launch_clamp(float* x, float lo, float hi, long long n, cudaStream_t st);

// CNN pre/post stages (exact float semantics of lib/model.lua's non-conv nodes).
// The input block (tfl_cnn_inputs): channel set bits, the field the scale is computed from, the scale function.
enum : int { kCnnInPDiv = 1, kCnnInUDiv = 2, kCnnInDiv = 4 };
// kCnnStatNone: the fused step's point-wise stage sums nothing (normalizeInput off, or 'div', summed after it).
enum : int { kCnnStatU = 0, kCnnStatPDiv = 1, kCnnStatDiv = 2, kCnnStatNone = 3 };
enum : int { kCnnScaleStd = 0, kCnnScaleNorm = 1, kCnnScaleOne = 2 };
// U1 = wall mask * U; sums[b] += (sum f, sum f^2) over the planes [own_lo, own_hi) of f = U1 (stat kCnnStatU) or
// p_div (kCnnStatPDiv); kCnnStatDiv accumulates nothing here (launch_cnn_div_stats, once U1 is complete).
void launch_cnn_mask_stats(const float* U, const float* flags, float* U1, double* sums, int own_lo, int own_hi,
                           const Geo& g, cudaStream_t st, int stat = kCnnStatU, const float* p_div = nullptr);
void launch_cnn_div_stats(const float* U1, const float* flags, double* sums, int own_lo, int own_hi, const Geo& g,
                          cudaStream_t st);
// n_per_batch: the sample count of the field (std only).
void launch_cnn_scale(const double* sums, float* scale, int nb, long long n_per_batch, float threshold,
                      cudaStream_t st, int func = kCnnScaleStd);
// x0 [nb][cin][n]: the channels of `sel` in the order pDiv, UDiv, div, occupancy, scaled.
void launch_cnn_inputs(const float* p_div, const float* U1, const float* flags, const float* scale,
                       float* x0, const Geo& g, cudaStream_t st, int sel = kCnnInPDiv | kCnnInDiv);
// The same channels in the padded channels-last layout of tfl_cnn_tc.cu, on the first float4 plane (planes = 1,
// up to 3 channels and a zero fourth) or on both (planes = 2, zero-padded to 8 channels).
void launch_cnn_inputs_padded(const float* p_div, const float* U1, const float* flags, const float* scale,
                              float* x0, int px, int py, const Geo& g, cudaStream_t st,
                              int sel = kCnnInPDiv | kCnnInDiv, int planes = 1);
// addPressureSkip with a 1x1 last convolution: p_net += w_skip * (p_div / scale).
void launch_cnn_skip(float* p_net, const float* p_div, const float* scale, float w_skip, const Geo& g, cudaStream_t st);
void launch_cnn_finish(const float* p_net, const float* U1, const float* flags, const float* scale,
                       float* p_out, float* U_out, const Geo& g, cudaStream_t st);

// ---- tfl_fused.cu (-fmad=false): fused point-wise stages of the convnet step ----
// The stages other than launch_vort_curl(_quad), which the 2-D vorticity confinement shares, run on 3-D grids with
// byte flags only: the fused step requires them (fused_step_applies, tfl_api.cu).
// qmask (may be null): BcPtrs::qmask of tfl_fused.cu, filled by launch_bc_quad_mask for the same step.
bool launch_bc_quad_mask(const float* u_inv, const float* u_bc, const float* d_inv, const float* d_bc,
                         unsigned char* qmask, const Geo& g, cudaStream_t st);
void launch_post_advect(const float* tmp_s, const float* tmp_u, const unsigned char* flags, float* density, float* U,
                        const float* u_inv, const float* u_bc, const float* d_inv, const float* d_bc,
                        const unsigned char* qmask, int do_buoy, const float s[3], const Geo& g, cudaStream_t st);
void launch_vort_curl(const float* U, float* curl, float* cnorm, float* force, float strength, const Geo& g,
                      cudaStream_t st);
bool launch_vort_curl_quad(const float* U, float* curl, float* cnorm, float* force, float strength, const Geo& g,
                           cudaStream_t st);
// sums[b] += (sum f, sum f^2) of f = the masked U (stat kCnnStatU) or p_div (kCnnStatPDiv); any other stat: no sums.
void launch_vort_bc_mask(float* U, const unsigned char* flags, const float* force, int do_vort, const float* u_inv,
                         const float* u_bc, const unsigned char* qmask, int mask_mode, double* sums, const Geo& g,
                         cudaStream_t st, int stat, const float* p_div);
// normalizeInputChan 'div': sums[b] += (sum div, sum div^2) of U1 (launch_cnn_div_stats on byte flags).
void launch_cnn_div_stats_fused(const float* U1, const unsigned char* flags, double* sums, const Geo& g,
                                cudaStream_t st);
// The conv input of the channel set `sel` (kCnnIn* bits) with the scale of `func` (kCnnScale*) computed from the sums
// of the field `chan` (kCnnStat*), in the layout of launch_cnn_inputs_padded with planes = 2 when sel has UDiv;
// scale_out[b] receives the scale.  false (nothing launched) for a set no model has.
bool launch_cnn_inputs_fused(const float* p_div, const float* U1, const unsigned char* flags, const double* sums,
                             float threshold, float* scale_out, float* x0, int px, int py, const Geo& g,
                             cudaStream_t st, int sel, int func, int chan);
void launch_cnn_finish_fused(const float* p_net, float* U, const unsigned char* flags, const float* scale, float* p_out,
                             const float* u_inv, const float* u_bc, const unsigned char* qmask, float lo, float hi,
                             const Geo& g, cudaStream_t st);

// ---- tfl_cnn.cu ----
// Generic direct convolution (fp32 FMA): in [b][cin][z][y][x] -> out [b][cout][z][y][x].
// wdev: device weights re-laid out as [cin][tap][cout_pad], bias [cout].
// act: 0 none, 1 ReLU, 2 sigmoid, 3 ReLU6.
// dil > 1: dilated convolution (nn.{Spatial,Volumetric}DilatedConvolution with dilation dil on every axis, stride 1,
// padding dil (k-1)/2: same grid out as in); dil = 1 runs the undilated kernels.
// Returns the kernel that ran: kConvDirect (k_conv_direct, a specialised (cout, k) whose weights fit shared
// memory) or kConvGeneric (k_conv_any, every other shape, whole grids only); -1 if none can run.
enum : int { kConvDirect = 1, kConvGeneric = 2 };
int launch_conv_direct(const float* in, float* out, const float* wdev, const float* bdev, int cin, int cout,
                       int ksize, int act, const Geo& g, cudaStream_t st, int dil = 1);
// The generic kernel alone (launch_conv_direct's fallback): same operands, same accumulation order.
int launch_conv_any(const float* in, float* out, const float* wdev, const float* bdev, int cin, int cout, int ksize,
                    int act, const Geo& g, cudaStream_t st, int dil = 1);
void launch_pool(const float* in, float* out, int nbc, int nz, int ny, int nx, int p, int is3d, int is_max,
                 cudaStream_t st);
void launch_pixel_shuffle(const float* in, float* out, int nb, int n_out, int nz, int ny, int nx, int s, int is3d,
                          cudaStream_t st);
// Join of multi-resolution banks: banks[i] (i = 1 .. nbanks-1; banks[0] unused) is bank i+1 at 2^-i the
// resolution of the full [nz][ny][nx] grid (z kept in 2-D), c channels; upsampled nearest and written at
// channel offset i c of out [nb][nbanks c][n] (add == 0) or added in bank order to out [nb][c][n] (add == 1).
// full = 1: every bank is at the full resolution (dilated banks), no upsampling.
constexpr int kMaxBankPtrs = 8;
int launch_bank_join(const float* const* banks, int nbanks, float* out, int nb, int c, int nz, int ny, int nx,
                     int is3d, int add, cudaStream_t st, int full = 0);
// Batch normalization of x [nb][c][n] with batch entries bstride floats apart (>= c n).  launch_bn_stats: per-channel
// fp64 partials of (sum d, sum d^2), d = x - K with K the channel's first value, into part [c][kBnBlocks + 1][2] (the
// last slot holds K), one slot per block of a fixed range, no atomics.  launch_bn_finalize: mean and biased variance
// over count = nb n values per channel, ac [2][c] = (w invstd, b - mean w invstd) with invstd = 1 / sqrt(var + eps), 0
// when var + eps == 0 (a constant channel has var exactly 0) (w / b null: 1 / 0); stats (may be null) [c][2] gets
// (mean, var).  launch_bn_apply: x = a x + c in place.
constexpr int kBnBlocks = 128;
void launch_bn_stats(const float* x, int nb, int c, long long n, long long bstride, double* part, cudaStream_t st);
void launch_bn_finalize(const double* part, int c, long long count, const float* w, const float* b, float eps,
                        float* ac, double* stats, cudaStream_t st);
void launch_bn_apply(float* x, int nb, int c, long long n, long long bstride, const float* ac, cudaStream_t st);

// ---- tfl_pcg.cu: matrix-free PCG pressure solve ----
struct PcgScratch {            // owned by the context, grow-only
  DevPtr<char> comp_buf;       // per-component CG scalars
  size_t comp_cap = 0;
  DevPtr<unsigned long long> prog;   // progress words of the triangular-sweep pipeline
  size_t prog_cap = 0;
  unsigned long long epoch = 0;
  PinnedPtr<int> host;         // pinned read-back words
  int sm_count = 0;            // set once the one-time setup (host words, kernel attributes) has succeeded
  void* debug_timing = nullptr;   // debug: device buffer [chunks][4] of sweep timestamps
  int groups_override = 0;     // debug: planes per CTA of the sweep kernel (0 = as many as fit)
};
// What a PCG solve captured into a step graph uses besides the arena (pcg_solve_graph): owned by the graph and sized
// for the worst case before the capture, so replays never allocate and share no per-component scalars or progress
// words with direct solves or with other graphs.
struct PcgGraphScratch {
  DevPtr<char> comp_buf;       // per-component CG scalars of up to comp_cap components
  long long comp_cap = 0;      // floor(cells / 2): every component of the system has at least two cells
  DevPtr<unsigned long long> prog;   // progress words of the captured sweeps, [2][chunks]
  long long prog_words = 0;
  // [0] status of the first failed solve since the last read (pcg_status_string, sticky), [1] iterations and [2]
  // residual (float bits) of the last solve, [4..5] passes of the loop body since the last read (u64)
  DevPtr<int> words;
  long long body_launches = 0; // kernels in one pass of the loop body
  bool captured = false;       // a solve was captured
};
// A conditional WHILE node in a stream capture (the PCG solve of a step graph, the Jacobi tolerance solves).
// capture_while_handle: a handle on the graph st is capturing, reset to `initial` at every launch of the graph.
// capture_while: the node, after what st has captured so far, with what enqueue(bs) enqueues on stream bs as its body
// graph.  It ends that capture on every path and returns the first failure of: enqueue (cudaSuccess or the error it
// met), a launch, ending the capture.  A body kernel re-arms or clears the handle.
cudaError_t capture_while_handle(cudaStream_t st, unsigned initial, cudaGraphConditionalHandle* loop);
template <typename Enqueue>
cudaError_t capture_while(cudaStream_t st, cudaGraphConditionalHandle loop, cudaStream_t bs, Enqueue&& enqueue) {
  cudaStreamCaptureStatus cap_status;
  cudaGraph_t graph = nullptr;
  const cudaGraphNode_t* deps = nullptr;
  size_t ndeps = 0;
  cudaError_t e = cudaStreamGetCaptureInfo(st, &cap_status, nullptr, &graph, &deps, &ndeps);
  if (e != cudaSuccess) return e;
  cudaGraphNodeParams np = {};
  np.type = cudaGraphNodeTypeConditional;
  np.conditional.handle = loop;
  np.conditional.type = cudaGraphCondTypeWhile;
  np.conditional.size = 1;
  cudaGraphNode_t node;
  if ((e = cudaGraphAddNode(&node, graph, deps, ndeps, &np)) != cudaSuccess) return e;
  if ((e = cudaStreamUpdateCaptureDependencies(st, &node, 1, cudaStreamSetCaptureDependencies)) != cudaSuccess) return e;
  if ((e = cudaStreamBeginCaptureToGraph(bs, np.conditional.phGraph_out[0], nullptr, nullptr, 0,
                                         cudaStreamCaptureModeRelaxed)) != cudaSuccess)
    return e;
  e = enqueue(bs);
  if (e == cudaSuccess) e = cudaGetLastError();
  cudaGraph_t body = nullptr;
  const cudaError_t ee = cudaStreamEndCapture(bs, &body);
  return e != cudaSuccess ? e : ee;
}
size_t pcg_workspace_bytes(int nb, int nz, int ny, int nx);
const char* pcg_status_string(int rc);
// precond: 0 none, 1 ilu0, 2 ic0.  Returns 0 or a status for pcg_status_string.  Synchronises `st`.
int pcg_solve(PcgScratch& sc, void* workspace, float* p, const float* flags, const float* div, int nb, int nz, int ny,
              int nx, int is3d, int precond, float tol, int max_iter, float* residual, int* iterations,
              long long* launches, cudaStream_t st);
// Allocates gs for solves on this grid (before a capture: status 4 for ny > 960, 3 for a CUDA failure).
int pcg_graph_alloc(PcgGraphScratch& gs, PcgScratch& sc, int nb, int nz, int ny, int nx, int is3d);
// pcg_solve for a stream being captured: the same kernels per iteration, no host read.  The iteration loop is a
// conditional WHILE node whose body the device re-arms, captured on loop_body; the result goes to gs.words.
// `launches` gets the kernels outside the loop, gs.body_launches those of one pass of the body.
int pcg_solve_graph(PcgGraphScratch& gs, PcgScratch& sc, void* workspace, float* p, const float* flags,
                    const float* div, int nb, int nz, int ny, int nx, int is3d, int precond, float tol, int max_iter,
                    long long* launches, cudaStream_t st, cudaStream_t loop_body);
// Debug: the preconditioner alone.  Same labelling, system and sweeps as pcg_solve; z = M^-1 r in the
// natural layout (0 outside every system of two or more cells); geometry = NYP, planes per CTA,
// chunks, cooperative grid of the sweeps.  Synchronises `st`.
int pcg_precond(PcgScratch& sc, void* workspace, float* z, const float* flags, const float* r, int nb, int nz, int ny,
                int nx, int is3d, int precond, int* geometry, long long* launches, cudaStream_t st);
int normalize_pressure_mean(void* workspace, float* p, const float* flags, int nb, int nz, int ny, int nx, int is3d,
                            long long* launches, cudaStream_t st);

// ---- tfl_aux_ops.cu (-fmad=false): operators of tfluids/init.lua around the step ----
void launch_upsample_nearest(const float* in, float* out, int nbf, int nz, int ny, int nx, int ratio, cudaStream_t st);
// axis: 0 = x, 1 = y, 2 = z of a [nbf][nz][ny][nx] array.
void launch_blur_axis(const float* src, float* dst, int nbf, int nz, int ny, int nx, int axis, int rad, cudaStream_t st);
void launch_signed_distance_field(const float* flags, float* dst, int nb, int nz, int ny, int nx, int rad,
                                  cudaStream_t st);
void launch_velocity_divergence_backward(const float* flags, const float* go, float* grad_u, int nb, int nz, int ny,
                                         int nx, int is3d, cudaStream_t st);
void launch_velocity_update_backward(const float* flags, const float* go, float* grad_p, int nb, int nz, int ny, int nx,
                                     int is3d, cudaStream_t st);
void launch_upsample_nearest_backward(const float* go, float* gi, int nbf, int nz, int ny, int nx, int ratio,
                                      cudaStream_t st);

}  // namespace tfl
