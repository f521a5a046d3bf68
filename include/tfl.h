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
/* Kernels launched by this context since creation (bench.py's gpu_launches). */
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
 * Synchronises once at the end to return the residual (the reference syncs every
 * iteration, generic/tfluids.cu:1886). residual may be NULL (no sync then, if p_tol <= 0). */
int tfl_solve_linear_system_jacobi(tfl_ctx* ctx, const tfl_grid* p, const tfl_grid* flags,
                                   const tfl_grid* div, int is_3d, float p_tol, int max_iter,
                                   float* residual, int* iterations);

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
 * the 'default' input set, lib/default_conf.lua:76-81) and cout[last] must be 1. */
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
void tfl_cnn_destroy(tfl_ctx* ctx, tfl_cnn* cnn);
/* Arithmetic of the convolution stack: 0 = fp32 FMA on the CUDA cores; 1 = TF32 tensor cores
 * (wgmma, fp32 accumulate); 2 = 3xTF32 tensor cores (error-compensated split, fp32-class
 * accuracy; the default where available).  Modes 1 and 2 cover the 3-D 'default' architecture. */
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
 * tfl_cnn_project_from_sums does the rest.  The conv stack runs on the whole local slab, so results
 * are exact on planes >= 4 planes away from a local end that is not a global end. */
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
 * tfl_host_state_create once.  Used for the end-to-end number in bench.py. */
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
 * mconf and every host-side choice of the captured call are frozen into the graph. */
typedef struct tfl_step_graph tfl_step_graph;
int tfl_step_graph_create(tfl_ctx* ctx, const tfl_state* state, const tfl_mconf* mconf, tfl_cnn* cnn,
                          tfl_step_graph** out);
int tfl_step_graph_launch(tfl_ctx* ctx, tfl_step_graph* graph);
void tfl_step_graph_destroy(tfl_ctx* ctx, tfl_step_graph* graph);
/* ---- one domain in z-slabs over the GPUs of a node (no counterpart in the reference, which is single-GPU;
 * SURVEY.md section 8e).  One process and one context per GPU.  The context owns the NCCL communicator
 * (libnccl.so.2 is loaded on demand); rank 0 makes an id, the host application distributes its
 * TFL_COMM_ID_BYTES bytes to every rank by its own means, every rank calls tfl_comm_init. */
#define TFL_COMM_ID_BYTES 128
int tfl_comm_unique_id(tfl_ctx* ctx, char* id_out /* TFL_COMM_ID_BYTES */);
int tfl_comm_init(tfl_ctx* ctx, const char* id_bytes, int32_t rank, int32_t world);   /* world 1: no NCCL */
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
/* One tfluids.simulate (convnet path) on this rank's slab: three neighbour halo exchanges (one packed ncclSend /
 * ncclRecv per neighbour and direction, one NCCL group per phase) and one 2-double all-reduce.  Asynchronous.
 * A trace that leaves the local slab (margin too small) raises tfl_trace_faults. */
int tfl_slab_sim_step(tfl_ctx* ctx, tfl_slab_sim* sim, const tfl_mconf* mconf, tfl_cnn* cnn);
int tfl_slab_sim_exchange_stats(tfl_ctx* ctx, tfl_slab_sim* sim, float ms[4], int64_t bytes[3]);
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
#ifdef __cplusplus
}
#endif
#endif /* TFL_H_ */
