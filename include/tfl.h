/*
 * libtfl -- C ABI of the H100-native Eulerian fluid step (drop-in for the tfluids
 * operators that FluidNet's `tfluids.simulate` calls).
 *
 * Every entry point replaces one reference `lua_CFunction` (registered in
 * torch/tfluids/generic/tfluids.cu:1932-1953, wrapped by torch/tfluids/init.lua) or one
 * cutorch tensor call that torch/lib/simulate.lua makes on the step.  Paths below are
 * relative to /root/reference/torch/.
 *
 * Conventions
 *  - All grids are float32, contiguous, 5-D [b][c][z][y][x] (x fastest), exactly the
 *    layout the reference's Grid classes view (tfluids/third_party/grid.h:26-262):
 *    flags / p / density / div have c == 1, U has c == 3 (3-D) or c == 2 (2-D, nz == 1).
 *    `tfl_grid.data` is a DEVICE pointer owned by the caller (e.g. a LuaJIT cdata, a
 *    torch tensor's data_ptr, or memory from tfl_alloc).  Nothing is retained across
 *    calls except the context.
 *  - Flags are float-encoded bit codes (tfluids/third_party/cell_type.h:22-33).
 *  - Every function returns 0 on success, non-zero on error; tfl_last_error() gives the
 *    message (the reference raises luaL_error / THError instead).
 *  - A context is single-threaded; all work is enqueued on the context's stream and is
 *    asynchronous unless stated.  Temporaries come from a context-owned arena (the
 *    reference's Lua-side getTempStorage, tfluids/init.lua:35-64).
 *  - There is no CPU fallback: without a CUDA device tfl_create fails.
 *
 * Slab decomposition (multi-GPU, no reference counterpart): a grid may be a z-slab of a
 * larger global domain.  tfl_set_slab() tells the context where the local array sits in
 * the global grid; border tests, getDx and line traces then use GLOBAL coordinates, as
 * the single-GPU run would.
 */
#ifndef TFL_H_
#define TFL_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct tfl_ctx tfl_ctx;
typedef struct tfl_cnn tfl_cnn;

typedef struct tfl_grid {
  float* data;                    /* device pointer */
  int32_t nb, nc, nz, ny, nx;     /* sizes of the 5 dims */
} tfl_grid;

/* tfluids.CellType (tfluids/init.cu:108-124, third_party/cell_type.h:22-33). */
enum {
  TFL_CELL_NONE = 0, TFL_CELL_FLUID = 1, TFL_CELL_OBSTACLE = 2, TFL_CELL_EMPTY = 4,
  TFL_CELL_INFLOW = 8, TFL_CELL_OUTFLOW = 16, TFL_CELL_OPEN = 32, TFL_CELL_STICK = 128
};

/* Advection methods, same order as AdvectMethod (tfluids/generic/advect_type.h:21-28);
 * strings: "euler", "maccormack", "eulerOurs", "rk2Ours", "rk3Ours", "maccormackOurs"
 * (advect_type.cc:19-38). */
enum {
  TFL_ADVECT_EULER = 0, TFL_ADVECT_MACCORMACK = 1, TFL_ADVECT_EULER_OURS = 2,
  TFL_ADVECT_RK2_OURS = 3, TFL_ADVECT_RK3_OURS = 4, TFL_ADVECT_MACCORMACK_OURS = 5
};
int tfl_advect_method_from_string(const char* name);   /* -1 if unknown */

/* ---- context ------------------------------------------------------------------------ */
int tfl_create(tfl_ctx** out, int device);              /* fails without a CUDA device */
void tfl_destroy(tfl_ctx* ctx);
const char* tfl_last_error(const tfl_ctx* ctx);
const char* tfl_version(void);
/* Adopt an external cudaStream_t (e.g. torch's current stream); NULL = own stream.
 * Replaces THCState_getCurrentStream (tfluids/generic/tfluids.cu:106,127). */
int tfl_set_stream(tfl_ctx* ctx, void* cuda_stream);
void* tfl_get_stream(tfl_ctx* ctx);
int tfl_sync(tfl_ctx* ctx);
/* Number of line traces since the last reset that hit a condition the reference CPU code
 * treats as a hard error (generic/calc_line_trace.cc THError sites) or that left the
 * local z-slab (halo too small).  Synchronises. */
int tfl_trace_faults(tfl_ctx* ctx, int64_t* count, int reset);
/* Kernels launched by this context since creation (bench.py's gpu_launches).  A step graph's replay adds the kernels
 * it runs outside a PCG solve's iteration loop; the loop's kernels, whose number only the device knows, are added by
 * the next tfl_step_graph_pcg_status of that graph (loop passes counted on the device times the body's kernels). */
int64_t tfl_launch_count(const tfl_ctx* ctx);

/* z-slab placement of subsequent grids: local plane 0 is global plane `z_offset` of a
 * domain with `global_nz` planes; operators compute local planes [z_lo, z_hi).
 * tfl_set_slab(ctx, 0, 0, 0, 0) restores single-domain behaviour. */
int tfl_set_slab(tfl_ctx* ctx, int32_t z_offset, int32_t global_nz, int32_t z_lo, int32_t z_hi);
/* Planes beyond [z_lo, z_hi) on which the MacCormack forward passes are also evaluated (they feed
 * the backward traces of the owned planes); default 2 = traces shorter than one cell. */
int tfl_set_slab_margin(tfl_ctx* ctx, int32_t planes);

/* ---- memory helpers (optional; callers may bring their own device pointers) ----------- */
int tfl_alloc(tfl_ctx* ctx, size_t bytes, void** dev_ptr);
int tfl_free(tfl_ctx* ctx, void* dev_ptr);
int tfl_alloc_host(tfl_ctx* ctx, size_t bytes, void** pinned_host_ptr);
int tfl_free_host(tfl_ctx* ctx, void* pinned_host_ptr);
int tfl_memcpy_h2d(tfl_ctx* ctx, void* dev_dst, const void* host_src, size_t bytes);  /* async */
int tfl_memcpy_d2h(tfl_ctx* ctx, void* host_dst, const void* dev_src, size_t bytes);  /* async */
int tfl_memcpy_d2d(tfl_ctx* ctx, void* dev_dst, const void* dev_src, size_t bytes);   /* async */

/* ---- operators (one per reference lua_CFunction) --------------------------------------- */
/* tfluids.advectScalar (init.lua:89-149; CudaMain_advectScalar third_party/tfluids.cu:524-633;
 * CPU third_party/tfluids.cc:415-588).  s_dst == NULL advects in place (init.lua:145-148).
 * boundaryWidth is fixed to 1 as in the reference (third_party/tfluids.cc:436,467). */
int tfl_advect_scalar(tfl_ctx* ctx, float dt, const tfl_grid* s, const tfl_grid* U,
                      const tfl_grid* flags, int method, int sample_outside_fluid,
                      float maccormack_strength, const tfl_grid* s_dst);
/* tfluids.advectVel (init.lua:170-219; third_party/tfluids.cu:876-963; .cc:776-920). */
int tfl_advect_vel(tfl_ctx* ctx, float dt, const tfl_grid* U, const tfl_grid* flags, int method,
                   float maccormack_strength, const tfl_grid* U_dst);
/* tfluids.setWallBcsForward (init.lua:228-247; third_party/tfluids.cu:969-1046). In place. */
int tfl_set_wall_bcs_forward(tfl_ctx* ctx, const tfl_grid* U, const tfl_grid* flags);
/* tfluids.velocityDivergenceForward (init.lua:256-279; third_party/tfluids.cu:1052-1105). */
int tfl_velocity_divergence_forward(tfl_ctx* ctx, const tfl_grid* U, const tfl_grid* flags,
                                    const tfl_grid* div);
/* tfluids.velocityUpdateForward (init.lua:324-349; third_party/tfluids.cu:1111-1195). In place. */
int tfl_velocity_update_forward(tfl_ctx* ctx, const tfl_grid* U, const tfl_grid* flags,
                                const tfl_grid* p);
/* tfluids.addBuoyancy (init.lua:442-471; third_party/tfluids.cu:1201-1273). gravity: 3 host floats. */
int tfl_add_buoyancy(tfl_ctx* ctx, const tfl_grid* U, const tfl_grid* flags,
                     const tfl_grid* density, const float gravity[3], float dt);
/* tfluids.addGravity (init.lua:481-507; third_party/tfluids.cu:1279-1349). */
int tfl_add_gravity(tfl_ctx* ctx, const tfl_grid* U, const tfl_grid* flags,
                    const float gravity[3], float dt);
/* tfluids.vorticityConfinement (init.lua:394-431; third_party/tfluids.cu:1355-1497). In place. */
int tfl_vorticity_confinement(tfl_ctx* ctx, const tfl_grid* U, const tfl_grid* flags,
                              float strength);
/* tfluids.solveLinearSystemJacobi (init.lua:693-734; generic/tfluids.cu:1765-1927).
 * p_tol > 0 runs tfl_solve_linear_system_jacobi_dev, then synchronises once, at the end, when residual or
 * iterations is non-NULL (the reference syncs every iteration, generic/tfluids.cu:1886).  p_tol <= 0 runs max_iter
 * sweeps and synchronises only when residual or iterations is non-NULL.  A call that reads its result on the host
 * (p_tol > 0, or a non-NULL residual or iterations) refuses inside a stream capture: capture the _dev entry point. */
int tfl_solve_linear_system_jacobi(tfl_ctx* ctx, const tfl_grid* p, const tfl_grid* flags,
                                   const tfl_grid* div, int is_3d, float p_tol, int max_iter,
                                   float* residual, int* iterations);
/* The same solve with its results left on the device: p, and the float residual and iteration count of the host loop
 * (dev_residual / dev_iterations, device pointers, each may be NULL), bit for bit those of
 * tfl_solve_linear_system_jacobi.  The residual's per-entry sums are added in a fixed order, so identical solves give
 * identical bits.  L2-resident 3-D grids (nx % 128 == 0, ny % 8 == 0, nz >= 4, up to 3 x 2^20 cells) run the whole
 * solve in one cooperative launch and never wait.  Other grids run a device-driven loop: inside a stream capture it
 * is one conditional WHILE node and never waits; otherwise the host enqueues chunks of 8, 16, ... 256 sweeps and reads
 * a device word after each, about log2(iterations / 8) + iterations / 256 waits.  Capturable on a non-default
 * stream once the solve has run outside the capture on the same grid (the context's scratch arena must not grow in
 * the capture); the graph then holds pointers into that arena, so replay it only while no larger call on the context
 * has regrown it.  tfl_launch_count counts a captured solve's loop body once.  Refuses, before enqueueing anything,
 * on a z-slab context, for max_iter < 1 and for a capture on the default stream. */
int tfl_solve_linear_system_jacobi_dev(tfl_ctx* ctx, const tfl_grid* p, const tfl_grid* flags, const tfl_grid* div,
                                       int is_3d, float p_tol, int max_iter, float* dev_residual,
                                       int32_t* dev_iterations);

/* tfluids.solveLinearSystemPCG (init.lua:645-676; generic/tfluids.cu:1245-1759, CUDA only in the
 * reference: host flood fill + CSR assembly, cuSPARSE ic0/ilu0 + csrsv + csrmv, cuBLAS dots).
 * Here matrix-free and device-resident: p <- 0, then per connected component of fluid cells
 * (components of one cell skipped, fewer than 5 cells un-preconditioned) Golub & Van Loan PCG with
 * x0 = 0 until ||r||^2 <= tol^2 or iter > max_iter, the component's mean removed from the result.
 * precond: TFL_PRECOND_NONE / ILU0 / IC0 (for the symmetric 7-point matrix ILU0 and IC0 are the
 * same operator and share one factor).  *residual = max over components of ||r||_2 (-inf when no
 * component was solved, as the reference), *iterations = the longest component's count.
 * Errors like the reference: a fluid cell on the domain border, a NaN residual. */
enum { TFL_PRECOND_NONE = 0, TFL_PRECOND_ILU0 = 1, TFL_PRECOND_IC0 = 2 };
int tfl_precond_from_string(const char* name);   /* "none" | "ilu0" | "ic0"; -1 if unknown */
int tfl_solve_linear_system_pcg(tfl_ctx* ctx, const tfl_grid* p, const tfl_grid* flags,
                                const tfl_grid* div, int is_3d, int precond, float tol, int max_iter,
                                float* residual, int* iterations);

/* ---- operators of tfluids/init.lua around the step --------------------------------------- */
/* tfluids.normalizePressureMean (init.lua:747-765; generic/tfluids.cc:845-921): subtract from every
 * fluid cell the mean of p over its connected fluid component.  The reference round-trips through the
 * host for the flood fill; here the labelling runs on the device. */
int tfl_normalize_pressure_mean(tfl_ctx* ctx, const tfl_grid* p, const tfl_grid* flags, int is_3d);
/* tfluids.volumetricUpSamplingNearestForward (init.lua:618-622; generic/tfluids.cc:509-557):
 * output [b][f][z*r][y*r][x*r] = input [b][f][z][y][x] replicated. */
int tfl_volumetric_up_sampling_nearest_forward(tfl_ctx* ctx, int ratio, const tfl_grid* input,
                                               const tfl_grid* output);
/* tfluids.rectangularBlur (init.lua:583-596; generic/tfluids.cc:641-760): separable box blur of
 * radius blur_rad with clamped edges, z (3-D only) then y then x; dst may not alias src. */
int tfl_rectangular_blur(tfl_ctx* ctx, const tfl_grid* src, int blur_rad, int is_3d, const tfl_grid* dst);
/* tfluids.signedDistanceField (init.lua:604-614; generic/tfluids.cc:766-822): 0 in obstacle cells,
 * else the distance to the nearest obstacle cell within search_rad, capped at search_rad. */
int tfl_signed_distance_field(tfl_ctx* ctx, const tfl_grid* flags, int search_rad, int is_3d,
                              const tfl_grid* dst);

/* ---- backward passes (training side; forward operators above are what the simulation loop uses) ---- */
/* tfluids.velocityDivergenceBackward (init.lua:288-314; generic/tfluids.cc:49-134): gradient of
 * velocityDivergenceForward w.r.t. U.  U only supplies the shape, as in the reference. */
int tfl_velocity_divergence_backward(tfl_ctx* ctx, const tfl_grid* U, const tfl_grid* flags,
                                     const tfl_grid* grad_output, const tfl_grid* grad_U);
/* tfluids.velocityUpdateBackward (init.lua:358-384; generic/tfluids.cc:216-345): gradient of
 * velocityUpdateForward w.r.t. p. */
int tfl_velocity_update_backward(tfl_ctx* ctx, const tfl_grid* U, const tfl_grid* flags, const tfl_grid* p,
                                 const tfl_grid* grad_output, const tfl_grid* grad_p);
/* tfluids.volumetricUpSamplingNearestBackward (init.lua:623-627; generic/tfluids.cc:563-635). */
int tfl_volumetric_up_sampling_nearest_backward(tfl_ctx* ctx, int ratio, const tfl_grid* input,
                                                const tfl_grid* grad_output, const tfl_grid* grad_input);
/* tfluids.emptyDomain (init.lua:545-555; generic/tfluids.cu:314-353). */
int tfl_empty_domain(tfl_ctx* ctx, const tfl_grid* flags, int is_3d, int bnd);
/* tfluids.flagsToOccupancy (init.lua:571-576; generic/tfluids.cu:355-401).  Cells that are
 * neither Fluid nor Obstacle get -1 as in the CUDA reference; *bad_cells (may be NULL,
 * synchronises if not) counts them so the host can raise like the CPU reference does. */
int tfl_flags_to_occupancy(tfl_ctx* ctx, const tfl_grid* flags, const tfl_grid* occupancy,
                           int64_t* bad_cells);

/* ---- cutorch tensor calls made by lib/simulate.lua on the step ------------------------ */
/* x:cmul(inv_mask); x:add(bc)  (setConstVals, lib/simulate.lua:136-158). */
int tfl_apply_bc(tfl_ctx* ctx, const tfl_grid* x, const tfl_grid* inv_mask, const tfl_grid* bc);
/* U:clamp(lo, hi)  (lib/simulate.lua:326). */
int tfl_clamp(tfl_ctx* ctx, const tfl_grid* x, float lo, float hi);

/* ---- CNN pressure projection (lib/model.lua:27-401, forward only) ---------------------- */
/* Layer l is a stride-1, zero-padded ((k-1)/2) cross-correlation cin[l] -> cout[l] with a
 * cubic (3-D) or square (2-D) kernel of edge ksize[l], bias, and ReLU after every layer
 * but the last.  weights[l] is a HOST pointer to [cout][cin][kz][ky][kx] floats (Torch
 * layout, kz == 1 in 2-D); biases[l] to [cout].  cin[0] must be 3 (pDiv, div, occupancy:
 * the 'default' input set, lib/default_conf.lua:76-81; other sets: tfl_cnn_create_model) and cout[last]
 * must be 1. */
int tfl_cnn_create(tfl_ctx* ctx, int is_3d, int n_layers, const int32_t* cin, const int32_t* cout,
                   const int32_t* ksize, const float* const* weights, const float* const* biases,
                   tfl_cnn** out);
/* The other single-bank graphs of lib/model.lua:164-239 ('tog', 'yang'): layer l is
 *   convolution cin[l] -> cout[l] * up[l]^d channels (kernel ksize[l], zero padding), the pixel shuffle of
 *   nn.{Spatial,Volumetric}ConvolutionUpsample when up[l] > 1, the non-linearity (all layers but the
 *   last; ReLU, or sigmoid when nonlin_sigmoid), then cudnn average / max pooling of size pool[l].
 * weights[l]: [cout[l] * up[l]^d][cin[l]][kz][ky][kx].  pool / up may be NULL (all 1: tfl_cnn_create).
 * These graphs run on the fp32 path; the tensor-core kernels cover the 3-D 'default' graph. */
int tfl_cnn_create_graph(tfl_ctx* ctx, int is_3d, int n_layers, const int32_t* cin, const int32_t* cout,
                         const int32_t* ksize, const int32_t* pool, const int32_t* up, int pool_is_max,
                         int nonlin_sigmoid, const float* const* weights, const float* const* biases,
                         tfl_cnn** out);
/* Multi-resolution banks (lib/model.lua:252-361, banksType 'mres'): num = banksNum, split_stage =
 * banksSplitStage, join_stage = banksJoinStage (stages numbered 1..n_layers, 1 <= split < join < n_layers),
 * aggregate_add = 0 for banksAggregateMethod 'concat', 1 for 'add'. */
typedef struct tfl_cnn_banks {
  int32_t num, split_stage, join_stage, aggregate_add;
} tfl_cnn_banks;
/* tfl_cnn_create_graph with banks.  Before stage split, bank 1 is the hidden layer and bank i a 2x average
 * pool of bank i-1; stages split .. join-1 run one convolution (+ shuffle, non-linearity, pooling) per bank;
 * before stage join, bank i is upsampled (nearest) by 2^(i-1) and the banks are concatenated along the
 * channels in bank order (cin[join-1] = num * cout[join-2]) or summed left to right.  cin, cout, ksize, pool
 * and up are per stage; weights / biases list the convolutions stage by stage, bank 1 .. num for a banked
 * stage.  banks == NULL or num == 1: exactly tfl_cnn_create_graph.  The grid at the split resolution must be
 * divisible by 2^(num-1).  The 3-D 'default' graph with split_stage 1 and join_stage 3 (num <= 8) runs on the
 * tensor cores (3xTF32 by default), also on z-slabs (tfl_slab_sim_step with margin >= tfl_slab_cnn_margin(num));
 * every other banked graph runs on the fp32 path, on whole grids only. */
int tfl_cnn_create_banked(tfl_ctx* ctx, int is_3d, int n_layers, const int32_t* cin, const int32_t* cout,
                          const int32_t* ksize, const int32_t* pool, const int32_t* up, int pool_is_max,
                          int nonlin_sigmoid, const tfl_cnn_banks* banks, const float* const* weights,
                          const float* const* biases, tfl_cnn** out);
/* The network's input block (lib/model.lua:27-150, :357-387; defaults lib/default_conf.lua:45-47, 76-81, 103-106).
 * p_div, u_div, div: inputChannels.{pDiv, UDiv, div}; the network input joins, in this order, pDiv, UDiv (2 or 3
 * channels, after the wall mask), div and the occupancy of the flags, which are always an input.  normalize:
 * normalizeInput; norm_func: normalizeInputFunc 0 'std' (unbiased) or 1 'norm' (L2); norm_chan: normalizeInputChan
 * 0 'UDiv', 1 'pDiv' or 2 'div', the field the per-entry scale max(f(field), threshold) is computed from.
 * pressure_skip: addPressureSkip, the last (1x1) convolution also takes the scaled pDiv (cin[last] = cout[last-1]
 * + 1, pDiv its last input channel).  Defaults: {1, 0, 1, 1, 0, 0, 0}. */
typedef struct tfl_cnn_inputs {
  int32_t p_div, u_div, div;
  int32_t normalize;
  int32_t norm_func;              /* 0 std, 1 norm */
  int32_t norm_chan;              /* 0 UDiv, 1 pDiv, 2 div */
  int32_t pressure_skip;
} tfl_cnn_inputs;
/* tfl_cnn_create_banked with the input block `inputs` (NULL: the defaults, exactly tfl_cnn_create_banked).
 * cin[0] must be the channel count of the set.  Combinations the reference cannot build are refused: no pDiv,
 * UDiv or div; neither UDiv nor div (the velocity update needs UDiv); normalizeInputChan 'div' without the div
 * input; 'yang' with another set than pDiv, div; the skip on a graph whose last convolution is not 1x1 ('tog').
 * Any set runs on the fp32 path and, for the 3-D 'default' graph (single-bank or banks split 1 / join 3), on the
 * tensor cores; models with a non-default block run whole grids only (no z-slabs) and step through the
 * per-operator path of tfl_simulate_step. */
int tfl_cnn_create_model(tfl_ctx* ctx, int is_3d, int n_layers, const int32_t* cin, const int32_t* cout,
                         const int32_t* ksize, const int32_t* pool, const int32_t* up, int pool_is_max,
                         int nonlin_sigmoid, const tfl_cnn_banks* banks, const tfl_cnn_inputs* inputs,
                         const float* const* weights, const float* const* biases, tfl_cnn** out);
/* Banks of either type: tfl_cnn_banks plus dilate = 0 for banksType 'mres', 1 for 'dilate' (lib/model.lua:279-285,
 * :300-303, :319-322; lib/model_utils.lua:122-146).  Dilated banks build no pyramid: every bank takes the hidden layer
 * of the split stage as it is, bank i's convolutions in stages split .. join-1 are dilated by 2^(i-1) on every axis
 * (stride 1, padding 2^(i-1) (k-1)/2, so each bank stays at bank 1's resolution), each followed by its non-linearity
 * and pooling, and the join concatenates or sums the banks without upsampling.  The weights are laid out as for
 * 'mres'.  The grid needs no divisibility beyond what pooling asks; up[l] > 1 in a banked stage is refused
 * ("upsampling not supported for dilated convolutions.").  num == 1 is the single-bank graph. */
typedef struct tfl_cnn_banks_ex {
  int32_t num, split_stage, join_stage, aggregate_add;
  int32_t dilate;
} tfl_cnn_banks_ex;
/* tfl_cnn_create_model with tfl_cnn_banks_ex (dilate = 0: exactly tfl_cnn_create_model).  Dilated banks run on whole
 * grids (tfl_cnn_project, tfl_simulate_step, step graphs, tfl_host_sim_step): on the fp32 path for every graph, and
 * for the 3-D 'default' graph with split_stage 1 and join_stage 3 (num <= 8) on the tensor cores (3xTF32 by default,
 * TF32), each dilated bank as 8^(i-1) ordinary convolutions on its phase sub-grids.  The z-slab entry points refuse
 * them. */
int tfl_cnn_create_model_ex(tfl_ctx* ctx, int is_3d, int n_layers, const int32_t* cin, const int32_t* cout,
                            const int32_t* ksize, const int32_t* pool, const int32_t* up, int pool_is_max,
                            int nonlin_sigmoid, const tfl_cnn_banks_ex* banks, const tfl_cnn_inputs* inputs,
                            const float* const* weights, const float* const* biases, tfl_cnn** out);
/* The non-linearity 'relu6' and batch normalization (lib/model.lua:316-350, lib/model_utils.lua:22-62).
 * relu6: nonlinType 'relu6', nn.ReLU6 = min(max(x, 0), 6) after every convolution but the last (nonlin_sigmoid must
 * be 0).  batch_norm: addBatchNorm; every stage but the last, and every bank of a banked stage, ends with
 * {Spatial,Volumetric}BatchNormalization over its osize channels: convolution -> non-linearity -> pooling -> BN, after
 * the pixel shuffle of an upsampling stage, at the stage's output resolution (a multi-resolution bank at its own
 * resolution, before the join).  bn[i] (HOST) belongs to convolution i in the order of `weights`, every one but the
 * last: [4][c] floats = weight, bias (1 and 0 for a module built without batchNormAffine), running_mean, running_var;
 * eps[i] its eps (batchNormEps, default 1e-4).
 * batch_stats = 1 for modules saved with train = true, the nn.Module default: the reference's simulators never call
 * evaluate(), so such a module normalises with the statistics of the batch it is given -- per channel, the mean and
 * the biased variance over all batch entries and voxels, y = (x - mean) / sqrt(var + eps) w + b, with 1 / sqrt taken
 * as 0 where var + eps == 0.  The entries of a batch are then coupled: entry 0's output depends on entry 1's input.
 * Batch statistics are summed in fp64 in a fixed order, so a result is the same bits on every run.  A training-mode
 * forward of the reference also updates the running averages; no output reads them, and the library does not update
 * them.  batch_stats = 0 (train = false): y = (x - running_mean) / sqrt(running_var + eps) w + b.
 * These models run on whole grids (tfl_cnn_project, tfl_simulate_step, step graphs, tfl_host_sim_step): on the fp32
 * path for every graph and, for the 3-D 'default' graph, on the tensor cores (3xTF32 by default, TF32; relu6 also with
 * banks split 1 / join 3, batch normalization single-bank only), where running statistics apply in the layers'
 * epilogues and fold into the 1x1x1 tail, and batch statistics take passes of their own over each layer's output
 * (also inside the fused step).  tfl_cnn_set_mode refuses the tensor-core modes for banked models with batch
 * normalization, and the z-slab entry points refuse every model with batch normalization.  norm == NULL, or all its fields 0: exactly tfl_cnn_create_model_ex.  Refused by name:
 * relu6 with nonlin_sigmoid, a missing bn / eps array or entry where batch_norm is set, a negative eps. */
typedef struct tfl_cnn_norm {
  int32_t relu6;
  int32_t batch_norm;
  int32_t batch_stats;            /* 1: batch statistics (train = true); 0: running statistics */
  const float* const* bn;         /* one per convolution but the last: [4][c] weight, bias, running_mean, running_var */
  const float* eps;               /* one per BN module */
} tfl_cnn_norm;
int tfl_cnn_create_model_norm(tfl_ctx* ctx, int is_3d, int n_layers, const int32_t* cin, const int32_t* cout,
                              const int32_t* ksize, const int32_t* pool, const int32_t* up, int pool_is_max,
                              int nonlin_sigmoid, const tfl_cnn_banks_ex* banks, const tfl_cnn_inputs* inputs,
                              const tfl_cnn_norm* norm, const float* const* weights, const float* const* biases,
                              tfl_cnn** out);
void tfl_cnn_destroy(tfl_ctx* ctx, tfl_cnn* cnn);
/* Arithmetic of the convolution stack: 0 = fp32 FMA on the CUDA cores; 1 = TF32 tensor cores
 * (wgmma, fp32 accumulate); 2 = 3xTF32 tensor cores (error-compensated split, fp32-class
 * accuracy; the default where available).  Modes 1 and 2 cover the 3-D 'default' architecture, single-bank
 * or with banks split at stage 1 and joined at stage 3 (with batch normalization: single-bank only). */
int tfl_cnn_set_mode(tfl_ctx* ctx, tfl_cnn* cnn, int mode);
int tfl_cnn_get_mode(const tfl_cnn* cnn);
/* model:forward({pDiv, UDiv, flags}) -> {p, U} (lib/model.lua:421-450).  threshold is
 * mconf.normalizeInputThreshold (lib/default_conf.lua:106).  p_out / U_out may alias
 * p_div / U_div.  scale_out (nb floats, HOST, may be NULL) synchronises if given. */
int tfl_cnn_project(tfl_ctx* ctx, tfl_cnn* cnn, const tfl_grid* p_div, const tfl_grid* U_div,
                    const tfl_grid* flags, const tfl_grid* p_out, const tfl_grid* U_out,
                    float threshold, float* scale_out);

/* z-slab variant of model:forward, split around its one global reduction (the input scale):
 * tfl_cnn_stats writes U1 = wall-mask * U and the (sum, sum of squares) of U1 over the OWNED planes
 * into dev_sums[2 * nb] (device doubles, to be all-reduced by the caller, e.g. NCCL);
 * tfl_cnn_project_from_sums does the rest, on the tensor-core path only: it computes p on the owned planes and the
 * one below them and U on the owned planes, which needs the inputs on 4 planes beyond each owned end that is not a
 * global end (3 * 2^(banksNum-1) + 1 for a banked model, whose margin set by tfl_set_slab_margin must then be at
 * least tfl_slab_cnn_margin(banksNum) and whose global grid must be divisible by 2^(banksNum-1)). */
int tfl_cnn_stats(tfl_ctx* ctx, const tfl_grid* U_div, const tfl_grid* flags, const tfl_grid* U1,
                  double* dev_sums);
int tfl_cnn_project_from_sums(tfl_ctx* ctx, tfl_cnn* cnn, const tfl_grid* p_div, const tfl_grid* U1,
                              const tfl_grid* flags, const double* dev_sums, const tfl_grid* p_out,
                              const tfl_grid* U_out, float threshold);

/* ---- the whole step: tfluids.simulate (lib/simulate.lua:175-327) ----------------------- */
typedef struct tfl_mconf {        /* keys the loop reads (lib/simulate.lua:188-291) */
  float dt;
  int32_t advection_method;       /* TFL_ADVECT_* */
  float maccormack_strength;
  double buoyancy_scale;          /* Lua numbers: the loop scales them in double */
  double gravity_scale;
  float gravity[3];               /* default (0, 1, 0), lib/simulate.lua:204-213 */
  double vorticity_confinement_amp;
  int32_t sim_method;             /* 0 convnet, 1 jacobi, 2 pcg */
  int32_t max_iter;               /* <= 0: reference default (100) */
  float normalize_input_threshold;
} tfl_mconf;
enum { TFL_SIM_CONVNET = 0, TFL_SIM_JACOBI = 1, TFL_SIM_PCG = 2 };

typedef struct tfl_state {        /* the `batch` table; any BC pointer may be NULL */
  tfl_grid p, U, flags, density;  /* density.data may be NULL */
  tfl_grid U_bc, U_bc_inv_mask, density_bc, density_bc_inv_mask, p_bc, p_bc_inv_mask;
  tfl_grid div;                   /* scratch for the non-convnet paths (batch.div) */
} tfl_state;

/* One call == one tfluids.simulate(conf, mconf, batch, model, false). Asynchronous.
 * The operator sequence is fused into fewer kernels than the per-operator entry points
 * use; results are identical to calling the operators one by one. */
int tfl_simulate_step(tfl_ctx* ctx, const tfl_state* state, const tfl_mconf* mconf, tfl_cnn* cnn);

/* Same step through HOST buffers (what a host application holding CPU tensors calls):
 * copies p, U, density in (pinned staging inside the context), runs the step, copies
 * p, U, density back, and synchronises.  flags / BC arrays are uploaded by
 * tfl_host_state_create once.  Used for the end-to-end number in bench.py.  tfl_host_sim_create refuses, before
 * it allocates and with *out left NULL, a grid with an extent < 1, is_3d = 0 with nz != 1, and a grid too large for
 * the operators. */
typedef struct tfl_host_sim tfl_host_sim;
int tfl_host_sim_create(tfl_ctx* ctx, int32_t nb, int32_t nz, int32_t ny, int32_t nx, int is_3d,
                        const float* flags, const float* U_bc, const float* U_bc_inv_mask,
                        const float* density_bc, const float* density_bc_inv_mask,
                        tfl_host_sim** out);
void tfl_host_sim_destroy(tfl_ctx* ctx, tfl_host_sim* hs);
int tfl_host_sim_step(tfl_ctx* ctx, tfl_host_sim* hs, float* p, float* U, float* density,
                      const tfl_mconf* mconf, tfl_cnn* cnn);

/* The step as a CUDA graph: tfl_simulate_step captured once (kernels of both internal streams, memsets, the
 * telemetry copy) and replayed with one launch per step.  The context must run on a non-default stream and one
 * tfl_simulate_step with the same state must have run before (capturing cannot allocate).  State pointers,
 * mconf and every host-side choice of the captured call are frozen into the graph.
 * The graph also holds pointers into buffers the library owns, and these calls free and reallocate them:
 *   - any call on the context that needs more scratch than it has (an operator or step on a larger grid);
 *   - tfl_advect_scalar / tfl_advect_vel with a traced method, tfl_simulate_step or another step on a grid of
 *     another shape, smaller ones included (the context's flag cache);
 *   - tfl_cnn_project or a step with the captured model on another grid (the model's activation buffers).
 * After any of them tfl_step_graph_launch fails, naming the buffer, and replays nothing: capture again (after one
 * tfl_simulate_step).  Destroying the model or the context while a graph that uses them exists is a caller error.
 * Every simMethod is captured.  With 'pcg' the solve's iteration loop is a conditional node: the device decides after
 * every second iteration whether any component still runs, so a replay never waits for the host, follows flags
 * changed in place (the graph owns per-component scalars for cells / 2 components, about 30 bytes per cell) and runs
 * at most one iteration past the longest component.  The direct solve's limits are refused at creation by name
 * (ny > 960, z-slabs).  A replay cannot fail on the device: tfl_step_graph_pcg_status synchronises the context's
 * stream and gives the last replay's residual and iterations as tfl_solve_linear_system_pcg returns them (-inf and
 * 0 when no component was solved), or fails with the direct call's message for the first replay since the previous
 * call whose solve failed (a fluid cell on the border, a NaN residual, a stalled sweep pipeline); that error stays
 * until this call reads it.  *iterations = -1 for a graph without a PCG solve. */
typedef struct tfl_step_graph tfl_step_graph;
int tfl_step_graph_create(tfl_ctx* ctx, const tfl_state* state, const tfl_mconf* mconf, tfl_cnn* cnn,
                          tfl_step_graph** out);
int tfl_step_graph_launch(tfl_ctx* ctx, tfl_step_graph* graph);
int tfl_step_graph_pcg_status(tfl_ctx* ctx, tfl_step_graph* graph, float* residual, int32_t* iterations);
void tfl_step_graph_destroy(tfl_ctx* ctx, tfl_step_graph* graph);
/* ---- one domain in z-slabs over the GPUs of a node (no counterpart in the reference, which is single-GPU;
 * SURVEY.md section 8e).  One process and one context per GPU.  The context owns the NCCL communicator
 * (libnccl.so.2 is loaded on demand); rank 0 makes an id, the host application distributes its
 * TFL_COMM_ID_BYTES bytes to every rank by its own means, every rank calls tfl_comm_init.
 * world 1: no NCCL.  A NULL id_bytes with world > 1 sets the context's rank and world without a communicator: the
 * slab step then exchanges halos and reduces its sums only over peer memory (tfl_slab_sim_ipc_connect on every
 * rank before any rank steps; ranks may also be processes sharing one GPU).  Unconnected, its exchanges move
 * nothing and the all-reduce is skipped -- one rank's workload alone, for profiling. */
#define TFL_COMM_ID_BYTES 128
int tfl_comm_unique_id(tfl_ctx* ctx, char* id_out /* TFL_COMM_ID_BYTES */);
int tfl_comm_init(tfl_ctx* ctx, const char* id_bytes, int32_t rank, int32_t world);
int tfl_comm_destroy(tfl_ctx* ctx);
/* Rank r keeps planes [z0, z1) of a [gnz][ny][nx] domain plus 2 * margin + 2 ghost planes per interior side
 * (margin = planes a backward trace may reach = ceil(max|u| dt) + 1, >= 2).  The host arrays are GLOBAL
 * [c][gnz][ny][nx] fields, identical on every rank; the BC pointers may be NULL. */
typedef struct tfl_slab_sim tfl_slab_sim;
int tfl_slab_sim_create(tfl_ctx* ctx, int32_t gnz, int32_t ny, int32_t nx, int32_t margin, const float* flags,
                        const float* U_bc, const float* U_bc_inv_mask, const float* density_bc,
                        const float* density_bc_inv_mask, tfl_slab_sim** out);
void tfl_slab_sim_destroy(tfl_ctx* ctx, tfl_slab_sim* sim);
/* Device views of the local slab and info = {z offset of local plane 0, local planes, first / past-last owned
 * local plane, z0, z1}. */
int tfl_slab_sim_layout(const tfl_slab_sim* sim, tfl_state* state_out, int32_t info[6]);
int tfl_slab_sim_upload(tfl_ctx* ctx, tfl_slab_sim* sim, const float* p, const float* U, const float* density);
int tfl_slab_sim_download(tfl_ctx* ctx, tfl_slab_sim* sim, float* p, float* U, float* density);
/* One tfluids.simulate on this rank's slab.  Asynchronous.  A trace that leaves the local slab (margin too small)
 * raises tfl_trace_faults.
 * simMethod 'convnet': three neighbour halo exchanges (one packed ncclSend / ncclRecv per neighbour and direction,
 * one NCCL group per phase) and one 2-double all-reduce.
 * simMethod 'jacobi' (cnn may be NULL): the two exchanges before the forces, then setWallBcsForward, one exchange
 * of U, the divergence, mconf->max_iter sweeps (0: 100) from p = 0 with pTol = 0 in the blocks of
 * tfl_slab_jacobi_schedule (one p exchange before every block but the first), the velocity update.  No global
 * reduction: p, U and density are bit-identical to tfl_simulate_step's.
 * simMethod 'pcg' is refused (its IC(0) triangular solves do not shard over z).  The model runs on the tensor cores
 * (mode 1 or 2): the 3-D 'default' graph, single-bank or with banks split at stage 1 and joined at stage 3, for which
 * the slab's margin must be at least tfl_slab_cnn_margin(banksNum) and the global grid divisible by
 * 2^(banksNum-1); the U / p exchange before the projection is then 2 * tfl_slab_cnn_margin(banksNum) + 1 planes wide
 * (5 for a single bank).  Other models are refused before anything is launched. */
int tfl_slab_sim_step(tfl_ctx* ctx, tfl_slab_sim* sim, const tfl_mconf* mconf, tfl_cnn* cnn);
/* Device time (ms) of the last step's three halo exchanges and of its all-reduce (0 on the Jacobi path), and the
 * bytes this rank sent in each exchange.  Synchronises. */
int tfl_slab_sim_exchange_stats(tfl_ctx* ctx, tfl_slab_sim* sim, float ms[4], int64_t bytes[3]);
/* The last step's p exchanges of the Jacobi path: count, summed device time (ms), bytes sent.  Synchronises.  After a
 * step that solved to a tolerance (direct or replayed) the count and bytes are those of the exchanges that ran, read
 * from the device, and ms is -1: those exchanges run inside the device-driven loop and are not timed. */
int tfl_slab_sim_jacobi_stats(tfl_ctx* ctx, tfl_slab_sim* sim, int32_t* exchanges, float* ms, int64_t* bytes);
/* Jacobi to a tolerance on z-slabs: the pTol of later 'jacobi' steps of this sim (convnet steps ignore it).  0, the
 * default, is the fixed count of mconf->max_iter sweeps described at tfl_slab_sim_step, with the same launches and
 * bits.  With p_tol > 0 the solve is the whole-grid loop of tfl_solve_linear_system_jacobi_dev over the global domain:
 * p = pPrev = 0; after each sweep res = (float) sqrt(sum over the global grid of (p - pPrev)^2); stop when res < p_tol
 * before the counter counts the sweep, or when it reaches max_iter; p is that loop's last iterate.  Owned p, U and
 * density equal the whole-grid operator sequence with tfl_solve_linear_system_jacobi_dev as its solve bit for bit, and
 * the iteration count equals its count.  The residual adds per-plane sums in ascending global z, each over fixed
 * 128 x 8 tiles, so its bits are the same at every world size; they differ from the whole-grid residual's in the last
 * bits.  The solve runs in blocks of 2 * margin + 2 sweeps, each followed by one gather of the per-plane residuals
 * and one stop decision that every rank makes alike; a direct step waits for the device once per chunk of 1, 2, 4 ..
 * 32 blocks (once per block over NCCL), a captured one (tfl_slab_graph_create) is one conditional WHILE node and does
 * not wait.  A graph keeps the tolerance it was captured with.  Refuses negative and NaN values by name; the first
 * p_tol > 0 allocates the solve's buffers (a stream being captured is refused then). */
int tfl_slab_sim_set_jacobi_tolerance(tfl_ctx* ctx, tfl_slab_sim* sim, float p_tol);
/* The last 'jacobi' step's residual and iteration count, direct or replayed, when that step solved to a tolerance.
 * Synchronises once.  Refused, by name, before any step with a tolerance, after a fixed-count (pTol 0) 'jacobi' step,
 * and while the context's stream is being captured.  tfl_slab_sim_step with a tolerance is refused on a stream that is
 * being captured (it waits for its stop decision on the host): capture it with tfl_slab_graph_create. */
int tfl_slab_sim_jacobi_status(tfl_ctx* ctx, tfl_slab_sim* sim, float* residual, int32_t* iterations);
/* The Jacobi sweep schedule of rank `rank` (pure function; the step, and any host that emulates it, use it).  With
 * halo = 2 * margin + 2, a block of k sweeps after a p exchange of width w computes owned +- (w - 1 - s) planes in its
 * sweep s (0-based) on each side with a neighbour, and the whole local slab up to the global ends on the others.
 * Writes min(count, cap) blocks of TFL_JACOBI_BLOCK_INTS int32, in the rank's LOCAL plane indices:
 *   {sweeps (0 .. halo), width of the p exchange before the block (0: none), first plane, past-last plane of
 *    sweep 0, 1 if the range loses a plane per sweep at the bottom, ... at the top},
 * and planes = {first, past-last local plane on which the divergence and the mask must be valid, width of the U
 * exchange that makes them so}.  Returns the block count: 1 for one rank, ceil((max_iter + 1) / halo) otherwise;
 * -1 for bad arguments (max_iter < 1, margin < 2, slabs thinner than the halo). */
#define TFL_JACOBI_BLOCK_INTS 6
int tfl_slab_jacobi_schedule(int32_t gnz, int32_t world, int32_t rank, int32_t margin, int32_t max_iter,
                             int32_t planes[3], int32_t* blocks, int32_t cap);
/* The smallest slab margin (tfl_slab_sim_create) a projection network with banks_num banks runs with (pure
 * function): 2 for banks_num <= 1, ceil(3 * 2^(banks_num-1) / 2) for 2 .. 8 banks (3, 6, 12, ...), -1 above.  The
 * coarsest bank's stencil reaches 3 * 2^(banks_num-1) + 2 planes across a rank boundary, which the halo of
 * 2 * margin + 2 planes must hold.  Use max(this, the advection's margin). */
int tfl_slab_cnn_margin(int32_t banks_num);
/* One block of Jacobi sweeps under the context's slab placement (tfl_set_slab: offset and global extent; the
 * placement's plane range is not used): sweep s = 0 .. sweeps-1 computes local planes
 * [z_lo + s * shrink_lo, z_hi - s * shrink_hi) of p from the other buffer -- even sweeps read pa and write pb, odd
 * sweeps the reverse -- with the mask of the solve computed from flags on [z_lo, z_hi).  Planes outside a sweep's
 * range are not written.  path: 0 one launch per sweep, 1 the whole block in one cooperative launch (3-D,
 * nx % 128 == 0, ny % 8 == 0 and the range co-resident on the device: 3.24M cells on an H100; refused otherwise),
 * -1 automatic (the one launch for ranges of up to 2.16M cells, where it measured faster); path_out (may be
 * NULL) receives the path taken.  The result equals `sweeps` tfl_solve_linear_system_jacobi sweeps bit for bit on
 * every plane the last sweep computes. */
int tfl_jacobi_slab_block(tfl_ctx* ctx, const tfl_grid* pa, const tfl_grid* pb, const tfl_grid* flags,
                          const tfl_grid* div, int is_3d, int32_t z_lo, int32_t z_hi, int32_t shrink_lo,
                          int32_t shrink_hi, int32_t sweeps, int32_t path, int32_t* path_out);
/* The exchanges over peer memory instead of NCCL: every rank exports its inbox as a CUDA IPC handle, the host
 * application gives every rank the handles of ALL ranks (world x TFL_IPC_HANDLE_BYTES, rank order), and after
 * tfl_slab_sim_ipc_connect on EVERY rank (host-side barrier before the first step) a halo exchange is one kernel
 * that writes the boundary planes straight into the neighbours' memory over NVLink and raises their step counters,
 * and one kernel that waits for this rank's counters and scatters its inbox into the ghost planes; the two sums are
 * reduced the same way (every rank stores its pair into every inbox and adds the pairs in rank order).  Optional:
 * without it -- or after tfl_slab_sim_ipc_connect(ctx, sim, NULL) -- the exchanges use NCCL. */
#define TFL_IPC_HANDLE_BYTES 64
int tfl_slab_sim_ipc_export(tfl_ctx* ctx, tfl_slab_sim* sim, char* handle_out /* TFL_IPC_HANDLE_BYTES */);
int tfl_slab_sim_ipc_connect(tfl_ctx* ctx, tfl_slab_sim* sim, const char* handles);
/* The slab step as a CUDA graph: one tfl_slab_sim_step captured on the context's stream (convnet, single-bank or
 * banked, or Jacobi with its cooperative block kernel; the exchange-statistics events become event-record nodes) and
 * replayed with one launch per step.  The exchanges' sequence numbers live on the device, so replays and direct steps
 * may be interleaved freely, on one rank and across ranks; every rank creates its own graph (capture involves no peer)
 * and the ranks still take the same steps, as with direct steps alone.  Pointers, mconf and the captured step's
 * host-side choices (advection tile halo, Jacobi path and block schedule) are frozen into the graph.
 * tfl_slab_graph_create refuses, by name and before anything is captured: whatever tfl_slab_sim_step refuses (same
 * messages), the default stream, no earlier tfl_slab_sim_step with this sim, model and simMethod (or a buffer below
 * reallocated since), and world > 1 without peer memory (NCCL is not captured).
 * tfl_slab_graph_launch refuses a stale graph, naming the buffer, like tfl_step_graph_launch (the context's scratch
 * arena and flag cache, the model's activation buffers; also the peers' inboxes mapped again); it adds the captured
 * step's kernels to tfl_launch_count, and tfl_slab_sim_exchange_stats / _jacobi_stats then report the replayed step.
 * Destroying the sim, the model or the context while a graph that uses them exists is a caller error. */
typedef struct tfl_slab_graph tfl_slab_graph;
int tfl_slab_graph_create(tfl_ctx* ctx, tfl_slab_sim* sim, const tfl_mconf* mconf, tfl_cnn* cnn, tfl_slab_graph** out);
int tfl_slab_graph_launch(tfl_ctx* ctx, tfl_slab_graph* graph);
void tfl_slab_graph_destroy(tfl_ctx* ctx, tfl_slab_graph* graph);

/* ---- frame output behind the running step (the save branch of fluid_net_3d_sim.lua:266-291) ------------------------
 * A recorder moves a scalar grid [1][1][nz][ny][nx] to the host in `.vbox` order -- the value at (x, y, z) at index
 * (x * ny + y) * nz + z, the demo's permute(3, 2, 1) -- without stalling the context's stream.
 * tfl_recorder_create: one device staging frame, `slots` >= 1 pinned host frames, a copy stream and its events; on
 *   failure *out stays NULL and nothing is kept.
 * tfl_recorder_capture: enqueues the pack (k_pack_vbox, a bit copy) on the context's current stream, so it sees `field`
 *   as the stream leaves it; the copy stream then moves the staging frame into the next free slot.  The next pack waits
 *   on the device for that copy out of the staging frame.  Never synchronises.  *frame_out = the frame's index (0, 1,
 *   ... per recorder).  Refused before anything is enqueued: every slot holds a frame not yet released, a field that is
 *   not [1][1][nz][ny][nx] of the recorder (nb > 1, nc > 1 by name), a stream being captured into a graph.
 * tfl_recorder_take: the oldest captured frame not yet taken.  wait = 1 blocks on that frame's copy only; wait = 0 sets
 *   *frame_out = -1 and *host_out = NULL if the copy has not landed.  Fails at once, without waiting, when no captured
 *   frame is left.  *host_out (pinned, nx * ny * nz floats) stays valid until the frame is released.
 * tfl_recorder_release: gives back the oldest taken frame's slot (strictly first in, first out); fails if none is taken.
 * tfl_recorder_destroy: waits for the copies in flight, then frees everything.
 * Cost: k_pack_vbox moves 8 bytes per cell; the copy runs beside the following steps (DESIGN.md section 6a).
 *
 * Z-slab runs (one frame gathered from every rank of a decomposed domain, DESIGN.md section 6a):
 * tfl_recorder_create_slab: the recorder of rank `rank` of `world` (1 .. 64) for a [gnz][ny][nx] domain.  The rank
 *   owns global planes [z0, z1) by the slab simulator's rule (gnz / world planes each, one more for the first
 *   gnz % world ranks).  Rank 0 is the writer: its recorder is the one above with nz = gnz and `slots` host frames;
 *   `slots` is ignored on the other ranks.  Refused before anything is allocated when a slab would be empty.
 *   With world = 1 it is a whole-grid recorder that captures with tfl_recorder_capture_slab.
 * tfl_recorder_ipc_export (rank 0): TFL_RECORDER_HANDLE_BYTES naming rank 0's staging frame and counters (a CUDA IPC
 *   handle) and the recorder's gnz, ny, nx and world.  The host application hands these bytes to every other rank.
 * tfl_recorder_ipc_connect (every other rank): maps rank 0's frame; refuses a handle of another shape or world, and
 *   fails by name where the mapping is refused (there is no NCCL path for frames).  Every rank must export or
 *   connect before any rank captures (a host-side barrier).
 * tfl_recorder_capture_slab: collective -- every rank calls it the same number of times, in step order.  `field`
 *   holds this rank's planes, its local plane 0 being global plane z_offset (tfl_slab_sim_layout's info[0]).  Rank
 *   r > 0 waits on the device (bounded, ~2 s) until rank 0's copy of its previous frame is done, then packs its planes
 *   into rank 0's staging frame with remote stores and raises its arrival counter.  Rank 0 packs its own planes like
 *   tfl_recorder_capture; its copy stream, not the context's stream, waits (bounded) for every rank's arrival before
 *   the copy to the host.  A wait that times out writes nothing and raises tfl_trace_faults.  Refused with nothing
 *   enqueued: a field that does not hold the rank's planes, wrong ny / nx, nb or nc != 1, a stream being captured, a
 *   world > 1 recorder not exported / connected, and on rank 0 a full ring (retry after a release: the frame index
 *   does not advance).  *frame_out counts the captures on every rank.
 * tfl_recorder_take / tfl_recorder_release: rank 0 only (refused by name elsewhere).  A frame whose ranks did not all
 *   arrive within the wait bound is not handed out: take fails naming the frame and the missing ranks, sets
 *   *frame_out to the frame (host_out stays NULL) and counts it as taken, so release it to go on.
 * tfl_recorder_destroy: on a rank r > 0 it drains the context's stream and unmaps rank 0's frame.  Caller contract, as
 *   for the slab simulator: rank 0 destroys its recorder only after every other rank has destroyed its own (a
 *   host-side barrier), since their packs write into rank 0's memory.
 * tfl_recorder_capture refuses a recorder of world > 1. */
typedef struct tfl_recorder tfl_recorder;
int tfl_recorder_create(tfl_ctx* ctx, int32_t nz, int32_t ny, int32_t nx, int32_t slots, tfl_recorder** out);
void tfl_recorder_destroy(tfl_ctx* ctx, tfl_recorder* rec);
int tfl_recorder_capture(tfl_ctx* ctx, tfl_recorder* rec, const tfl_grid* field, int64_t* frame_out);
int tfl_recorder_take(tfl_ctx* ctx, tfl_recorder* rec, int wait, const float** host_out, int64_t* frame_out);
int tfl_recorder_release(tfl_ctx* ctx, tfl_recorder* rec);
#define TFL_RECORDER_HANDLE_BYTES 128
int tfl_recorder_create_slab(tfl_ctx* ctx, int32_t gnz, int32_t ny, int32_t nx, int32_t rank, int32_t world,
                             int32_t slots, tfl_recorder** out);
int tfl_recorder_ipc_export(tfl_ctx* ctx, tfl_recorder* rec, char* handle_out /* TFL_RECORDER_HANDLE_BYTES */);
int tfl_recorder_ipc_connect(tfl_ctx* ctx, tfl_recorder* rec, const char* handle);
int tfl_recorder_capture_slab(tfl_ctx* ctx, tfl_recorder* rec, const tfl_grid* field, int32_t z_offset,
                              int64_t* frame_out);

/* ---- step monitor: the divergence statistics of torch/lib/calc_stats.lua:81-123 behind the running step ------------
 * One record per call, per batch entry: div_norm = sqrt(sum d^2) over all cells, div_max = max |d|, u_max = max |U| over
 * every face and component, where d is what tfl_velocity_divergence_forward writes (u(i) - u(i+1) + ..., 0 outside
 * interior fluid cells).  Summed in fp64 in an order fixed by the field alone: one partial per (batch entry, global
 * plane) from a fixed split of the plane into rows, then the planes in ascending global z, then the square root
 * (DESIGN.md section 6b).  The same fields give the same bits on every run, whole grid or z-slabs.  The maxima
 * propagate NaN: a NaN anywhere in U makes u_max NaN, one in d makes div_max (and div_norm) NaN.
 * tfl_monitor_create: `capacity` >= 1 record slots in pinned, mapped host memory for grids of nb batch entries and gnz
 *   global planes; on failure *out stays NULL.
 * tfl_monitor_record: enqueues two kernels on the context's current stream, which read U and flags as the stream leaves
 *   them; the second stores the record straight into its host slot and then, with release semantics, its sequence
 *   number.  Never synchronises.  *index_out (may be NULL) = the record's index (0, 1, ... per monitor).  The first
 *   record fixes the monitor's nc, ny and nx.  On a context with a slab placement (tfl_set_slab) it reduces the
 *   placement's planes [z_lo, z_hi) only, and the record keeps their per-plane partials (sum d^2, max |d|, max |U|)
 *   with the global index of the first; d on the placement's last plane reads U_z on the plane above it, which the
 *   caller keeps current (tfl_slab_sim_monitor_record does).  Refused with nothing enqueued: a stream being captured
 *   into a graph (record after tfl_step_graph_launch instead), a ring whose slots all hold records not yet taken, and a
 *   grid whose nb, gnz or shape differs from the monitor's (the message names it).
 * tfl_monitor_take: the oldest record not yet taken, first in, first out.  values_out receives nb x 3 doubles {div_norm,
 *   div_max, u_max} and *planes_out = 0 for a whole-grid record, or nb x planes x 3 doubles {sum d^2, max |d|, max |U|}
 *   for global planes [*z0_out, *z0_out + *planes_out) of a z-slab record (size it nb x gnz x 3).  wait = 0 returns at
 *   once with *index_out = -1 if the record has not landed; wait = 1 polls its sequence word.  Fails at once when no
 *   record is left.
 * tfl_monitor_destroy: waits for the records in flight, then frees everything.
 * tfl_slab_sim_monitor_record: collective over the ranks of a slab simulator, like a step: refreshes the ghost plane
 *   of U_z above each rank's owned planes from its neighbour (the step leaves it stale), then tfl_monitor_record of the
 *   owned planes.  Adding every rank's plane partials in ascending global z gives the whole grid's record bit for bit. */
typedef struct tfl_monitor tfl_monitor;
int tfl_monitor_create(tfl_ctx* ctx, int32_t nb, int32_t gnz, int32_t capacity, tfl_monitor** out);
void tfl_monitor_destroy(tfl_ctx* ctx, tfl_monitor* mon);
int tfl_monitor_record(tfl_ctx* ctx, tfl_monitor* mon, const tfl_grid* U, const tfl_grid* flags, int64_t* index_out);
int tfl_monitor_take(tfl_ctx* ctx, tfl_monitor* mon, int wait, int64_t* index_out, double* values_out, int32_t* z0_out,
                     int32_t* planes_out);
int tfl_slab_sim_monitor_record(tfl_ctx* ctx, tfl_slab_sim* sim, tfl_monitor* mon, int64_t* index_out);
#ifdef __cplusplus
}
#endif
#endif /* TFL_H_ */
