-- tfluids_ffi.lua -- LuaJIT FFI shim that re-creates the reference's `tfluids.*` operator
-- surface (torch/tfluids/init.lua) on top of libtfl.so (include/tfl.h).  No Torch7 / cutorch
-- on the hot path: tensors are plain device pointers wrapped in a small `Grid` object.
--
-- NOTE: there is no LuaJIT in the build image, so this file is delivered unexecuted; it is
-- kept deliberately thin -- every behaviour it relies on is exercised through the same C ABI
-- by the Python mirror (fluidnet_b200/tfluids.py) and its GPU tests.
--
-- Usage (drop-in for `local tfluids = require('tfluids')` in torch/lib/simulate.lua):
--   local tfluids = require('tfluids_ffi')
--   local flags   = tfluids.Grid(1, 1, 128, 128, 128)       -- device memory via tfl_alloc
--   tfluids.emptyDomain(flags, true)
--   tfluids.advectScalar(dt, density, U, flags, 'maccormackOurs', nil, false, 0.6)

local ffi = require('ffi')

ffi.cdef[[
typedef struct tfl_ctx tfl_ctx;
typedef struct tfl_cnn tfl_cnn;
typedef struct tfl_grid { float* data; int32_t nb, nc, nz, ny, nx; } tfl_grid;
typedef struct tfl_mconf {
  float dt; int32_t advection_method; float maccormack_strength;
  double buoyancy_scale; double gravity_scale; float gravity[3];
  double vorticity_confinement_amp; int32_t sim_method; int32_t max_iter;
  float normalize_input_threshold;
} tfl_mconf;
typedef struct tfl_state {
  tfl_grid p, U, flags, density;
  tfl_grid U_bc, U_bc_inv_mask, density_bc, density_bc_inv_mask, p_bc, p_bc_inv_mask;
  tfl_grid div;
} tfl_state;
int tfl_create(tfl_ctx** out, int device);
void tfl_destroy(tfl_ctx* ctx);
const char* tfl_last_error(const tfl_ctx* ctx);
int tfl_sync(tfl_ctx* ctx);
int tfl_alloc(tfl_ctx* ctx, size_t bytes, void** dev_ptr);
int tfl_free(tfl_ctx* ctx, void* dev_ptr);
int tfl_memcpy_h2d(tfl_ctx* ctx, void* dev_dst, const void* host_src, size_t bytes);
int tfl_memcpy_d2h(tfl_ctx* ctx, void* host_dst, const void* dev_src, size_t bytes);
int tfl_advect_method_from_string(const char* name);
int tfl_advect_scalar(tfl_ctx*, float dt, const tfl_grid* s, const tfl_grid* U, const tfl_grid* flags,
                      int method, int sample_outside_fluid, float maccormack_strength, const tfl_grid* s_dst);
int tfl_advect_vel(tfl_ctx*, float dt, const tfl_grid* U, const tfl_grid* flags, int method,
                   float maccormack_strength, const tfl_grid* U_dst);
int tfl_set_wall_bcs_forward(tfl_ctx*, const tfl_grid* U, const tfl_grid* flags);
int tfl_velocity_divergence_forward(tfl_ctx*, const tfl_grid* U, const tfl_grid* flags, const tfl_grid* div);
int tfl_velocity_update_forward(tfl_ctx*, const tfl_grid* U, const tfl_grid* flags, const tfl_grid* p);
int tfl_add_buoyancy(tfl_ctx*, const tfl_grid* U, const tfl_grid* flags, const tfl_grid* density,
                     const float gravity[3], float dt);
int tfl_add_gravity(tfl_ctx*, const tfl_grid* U, const tfl_grid* flags, const float gravity[3], float dt);
int tfl_vorticity_confinement(tfl_ctx*, const tfl_grid* U, const tfl_grid* flags, float strength);
int tfl_solve_linear_system_jacobi(tfl_ctx*, const tfl_grid* p, const tfl_grid* flags, const tfl_grid* div,
                                   int is_3d, float p_tol, int max_iter, float* residual, int* iterations);
int tfl_solve_linear_system_jacobi_dev(tfl_ctx*, const tfl_grid* p, const tfl_grid* flags, const tfl_grid* div,
                                       int is_3d, float p_tol, int max_iter, float* dev_residual,
                                       int32_t* dev_iterations);
int tfl_precond_from_string(const char* name);
int tfl_solve_linear_system_pcg(tfl_ctx*, const tfl_grid* p, const tfl_grid* flags, const tfl_grid* div,
                                int is_3d, int precond, float tol, int max_iter, float* residual, int* iterations);
int tfl_normalize_pressure_mean(tfl_ctx*, const tfl_grid* p, const tfl_grid* flags, int is_3d);
int tfl_volumetric_up_sampling_nearest_forward(tfl_ctx*, int ratio, const tfl_grid* input, const tfl_grid* output);
int tfl_rectangular_blur(tfl_ctx*, const tfl_grid* src, int blur_rad, int is_3d, const tfl_grid* dst);
int tfl_signed_distance_field(tfl_ctx*, const tfl_grid* flags, int search_rad, int is_3d, const tfl_grid* dst);
int tfl_velocity_divergence_backward(tfl_ctx*, const tfl_grid* U, const tfl_grid* flags, const tfl_grid* grad_output, const tfl_grid* grad_U);
int tfl_velocity_update_backward(tfl_ctx*, const tfl_grid* U, const tfl_grid* flags, const tfl_grid* p, const tfl_grid* grad_output, const tfl_grid* grad_p);
int tfl_volumetric_up_sampling_nearest_backward(tfl_ctx*, int ratio, const tfl_grid* input, const tfl_grid* grad_output, const tfl_grid* grad_input);
int tfl_empty_domain(tfl_ctx*, const tfl_grid* flags, int is_3d, int bnd);
int tfl_flags_to_occupancy(tfl_ctx*, const tfl_grid* flags, const tfl_grid* occupancy, int64_t* bad_cells);
int tfl_apply_bc(tfl_ctx*, const tfl_grid* x, const tfl_grid* inv_mask, const tfl_grid* bc);
int tfl_clamp(tfl_ctx*, const tfl_grid* x, float lo, float hi);
int tfl_cnn_create(tfl_ctx*, int is_3d, int n_layers, const int32_t* cin, const int32_t* cout,
                   const int32_t* ksize, const float* const* weights, const float* const* biases, tfl_cnn** out);
void tfl_cnn_destroy(tfl_ctx*, tfl_cnn*);
int tfl_cnn_project(tfl_ctx*, tfl_cnn*, const tfl_grid* p_div, const tfl_grid* U_div, const tfl_grid* flags,
                    const tfl_grid* p_out, const tfl_grid* U_out, float threshold, float* scale_out);
int tfl_cnn_create_graph(tfl_ctx*, int is_3d, int n_layers, const int32_t* cin, const int32_t* cout, const int32_t* ksize,
                         const int32_t* pool, const int32_t* up, int pool_is_max, int nonlin_sigmoid,
                         const float* const* weights, const float* const* biases, tfl_cnn** out);
typedef struct tfl_cnn_banks { int32_t num, split_stage, join_stage, aggregate_add; } tfl_cnn_banks;
int tfl_cnn_create_banked(tfl_ctx*, int is_3d, int n_layers, const int32_t* cin, const int32_t* cout, const int32_t* ksize,
                          const int32_t* pool, const int32_t* up, int pool_is_max, int nonlin_sigmoid,
                          const tfl_cnn_banks* banks, const float* const* weights, const float* const* biases,
                          tfl_cnn** out);
typedef struct tfl_cnn_inputs { int32_t p_div, u_div, div, normalize, norm_func, norm_chan, pressure_skip; } tfl_cnn_inputs;
int tfl_cnn_create_model(tfl_ctx*, int is_3d, int n_layers, const int32_t* cin, const int32_t* cout, const int32_t* ksize,
                         const int32_t* pool, const int32_t* up, int pool_is_max, int nonlin_sigmoid,
                         const tfl_cnn_banks* banks, const tfl_cnn_inputs* inputs, const float* const* weights,
                         const float* const* biases, tfl_cnn** out);
typedef struct tfl_cnn_banks_ex { int32_t num, split_stage, join_stage, aggregate_add, dilate; } tfl_cnn_banks_ex;
int tfl_cnn_create_model_ex(tfl_ctx*, int is_3d, int n_layers, const int32_t* cin, const int32_t* cout,
                            const int32_t* ksize, const int32_t* pool, const int32_t* up, int pool_is_max,
                            int nonlin_sigmoid, const tfl_cnn_banks_ex* banks, const tfl_cnn_inputs* inputs,
                            const float* const* weights, const float* const* biases, tfl_cnn** out);
int tfl_simulate_step(tfl_ctx*, const tfl_state*, const tfl_mconf*, tfl_cnn*);
typedef struct tfl_step_graph tfl_step_graph;
typedef struct tfl_slab_sim tfl_slab_sim;
int tfl_set_stream(tfl_ctx* ctx, void* cuda_stream);
int tfl_step_graph_create(tfl_ctx*, const tfl_state* state, const tfl_mconf* mconf, tfl_cnn* cnn, tfl_step_graph** out);
int tfl_step_graph_launch(tfl_ctx*, tfl_step_graph* graph);
int tfl_step_graph_pcg_status(tfl_ctx*, tfl_step_graph* graph, float* residual, int32_t* iterations);
void tfl_step_graph_destroy(tfl_ctx*, tfl_step_graph* graph);
typedef struct tfl_slab_graph tfl_slab_graph;
int tfl_slab_graph_create(tfl_ctx*, tfl_slab_sim* sim, const tfl_mconf* mconf, tfl_cnn* cnn, tfl_slab_graph** out);
int tfl_slab_graph_launch(tfl_ctx*, tfl_slab_graph* graph);
void tfl_slab_graph_destroy(tfl_ctx*, tfl_slab_graph* graph);
int tfl_comm_unique_id(tfl_ctx*, char* id_out);
int tfl_comm_init(tfl_ctx*, const char* id_bytes, int32_t rank, int32_t world);
int tfl_comm_destroy(tfl_ctx*);
int tfl_slab_sim_create(tfl_ctx*, int32_t gnz, int32_t ny, int32_t nx, int32_t margin, const float* flags,
                        const float* U_bc, const float* U_bc_inv_mask, const float* density_bc,
                        const float* density_bc_inv_mask, tfl_slab_sim** out);
void tfl_slab_sim_destroy(tfl_ctx*, tfl_slab_sim* sim);
int tfl_slab_sim_upload(tfl_ctx*, tfl_slab_sim* sim, const float* p, const float* U, const float* density);
int tfl_slab_sim_download(tfl_ctx*, tfl_slab_sim* sim, float* p, float* U, float* density);
int tfl_slab_sim_step(tfl_ctx*, tfl_slab_sim* sim, const tfl_mconf* mconf, tfl_cnn* cnn);
int tfl_slab_sim_ipc_export(tfl_ctx*, tfl_slab_sim* sim, char* handle_out);
int tfl_slab_sim_ipc_connect(tfl_ctx*, tfl_slab_sim* sim, const char* handles);
int tfl_slab_sim_jacobi_stats(tfl_ctx*, tfl_slab_sim* sim, int32_t* exchanges, float* ms, int64_t* bytes);
int tfl_slab_sim_set_jacobi_tolerance(tfl_ctx*, tfl_slab_sim* sim, float p_tol);
int tfl_slab_sim_jacobi_status(tfl_ctx*, tfl_slab_sim* sim, float* residual, int32_t* iterations);
int tfl_slab_jacobi_schedule(int32_t gnz, int32_t world, int32_t rank, int32_t margin, int32_t max_iter,
                             int32_t planes[3], int32_t* blocks, int32_t cap);
int tfl_slab_cnn_margin(int32_t banks_num);
int tfl_jacobi_slab_block(tfl_ctx*, const tfl_grid* pa, const tfl_grid* pb, const tfl_grid* flags,
                          const tfl_grid* div, int is_3d, int32_t z_lo, int32_t z_hi, int32_t shrink_lo,
                          int32_t shrink_hi, int32_t sweeps, int32_t path, int32_t* path_out);
typedef struct tfl_recorder tfl_recorder;
int tfl_recorder_create(tfl_ctx*, int32_t nz, int32_t ny, int32_t nx, int32_t slots, tfl_recorder** out);
void tfl_recorder_destroy(tfl_ctx*, tfl_recorder* rec);
int tfl_recorder_capture(tfl_ctx*, tfl_recorder* rec, const tfl_grid* field, int64_t* frame_out);
int tfl_recorder_take(tfl_ctx*, tfl_recorder* rec, int wait, const float** host_out, int64_t* frame_out);
int tfl_recorder_release(tfl_ctx*, tfl_recorder* rec);
int tfl_recorder_create_slab(tfl_ctx*, int32_t gnz, int32_t ny, int32_t nx, int32_t rank, int32_t world, int32_t slots,
                             tfl_recorder** out);
int tfl_recorder_ipc_export(tfl_ctx*, tfl_recorder* rec, char* handle_out);
int tfl_recorder_ipc_connect(tfl_ctx*, tfl_recorder* rec, const char* handle);
int tfl_recorder_capture_slab(tfl_ctx*, tfl_recorder* rec, const tfl_grid* field, int32_t z_offset, int64_t* frame_out);
typedef struct tfl_monitor tfl_monitor;
int tfl_monitor_create(tfl_ctx*, int32_t nb, int32_t gnz, int32_t capacity, tfl_monitor** out);
void tfl_monitor_destroy(tfl_ctx*, tfl_monitor* mon);
int tfl_monitor_record(tfl_ctx*, tfl_monitor* mon, const tfl_grid* U, const tfl_grid* flags, int64_t* index_out);
int tfl_monitor_take(tfl_ctx*, tfl_monitor* mon, int wait, int64_t* index_out, double* values_out, int32_t* z0_out,
                     int32_t* planes_out);
]]

local lib = ffi.load('tfl')          -- libtfl.so on the library path
local tfluids = {}

-- tfluids.CellType (torch/tfluids/init.cu:108-124)
tfluids.CellType = {TypeNone = 0, TypeFluid = 1, TypeObstacle = 2, TypeEmpty = 4, TypeInflow = 8,
                    TypeOutflow = 16, TypeOpen = 32, TypeStick = 128, TypeReserved = 256,
                    TypeZeroPressure = 32768}
tfluids.withCUDA = true

local ctxp = ffi.new('tfl_ctx*[1]')
assert(lib.tfl_create(ctxp, 0) == 0, 'libtfl: no CUDA device (there is no CPU fallback)')
local ctx = ctxp[0]
tfluids._ctx = ctx

local function check(rc)
  if rc ~= 0 then error(ffi.string(lib.tfl_last_error(ctx)), 3) end
end

-- Minimal 5-D tensor: device storage + sizes (the only tensor API the wrappers below use).
local Grid = {}
Grid.__index = Grid
function tfluids.Grid(nb, nc, nz, ny, nx)
  local p = ffi.new('void*[1]')
  check(lib.tfl_alloc(ctx, nb * nc * nz * ny * nx * 4, p))
  local g = ffi.new('tfl_grid', {ffi.cast('float*', p[0]), nb, nc, nz, ny, nx})
  return setmetatable({c = g}, Grid)
end
function Grid:dim() return 5 end
function Grid:size(d) local s = {self.c.nb, self.c.nc, self.c.nz, self.c.ny, self.c.nx}; return s[d] end
function Grid:isSameSizeAs(o)
  for d = 1, 5 do if self:size(d) ~= o:size(d) then return false end end
  return true
end
function Grid:isContiguous() return true end
function Grid:numel() return self.c.nb * self.c.nc * self.c.nz * self.c.ny * self.c.nx end
function Grid:copyFromHost(ptr) check(lib.tfl_memcpy_h2d(ctx, self.c.data, ptr, self:numel() * 4)) end
function Grid:copyToHost(ptr) check(lib.tfl_memcpy_d2h(ctx, ptr, self.c.data, self:numel() * 4)); lib.tfl_sync(ctx) end

local function checkUFlags(U, flags)               -- init.lua:177-191
  assert(U:dim() == 5 and flags:dim() == 5, 'Dimension mismatch')
  assert(flags:size(2) == 1, 'flags is not scalar')
  local is3D = U:size(2) == 3
  if not is3D then
    assert(flags:size(3) == 1, '2D velocity field but zdepth > 1')
    assert(U:size(2) == 2, '2D velocity field must have only 2 channels')
  end
  assert(U:size(1) == flags:size(1) and U:size(3) == flags:size(3) and U:size(4) == flags:size(4) and
         U:size(5) == flags:size(5), 'Size mismatch')
  return is3D
end

local function method(m)
  local id = lib.tfl_advect_method_from_string(m or 'maccormackOurs')
  if id < 0 then error('advection method (' .. tostring(m) .. ') not supported') end
  return id
end

function tfluids.advectScalar(dt, s, U, flags, meth, sDst, sampleOutsideFluid, maccormackStrength, boundaryWidth)
  if sampleOutsideFluid == nil then sampleOutsideFluid = false end        -- init.lua:92-97
  maccormackStrength = maccormackStrength or 0.75
  checkUFlags(U, flags)
  assert(s:isSameSizeAs(flags), 'Size mismatch')
  check(lib.tfl_advect_scalar(ctx, dt, s.c, U.c, flags.c, method(meth), sampleOutsideFluid and 1 or 0,
                              maccormackStrength, sDst and sDst.c or nil))
end

function tfluids.advectVel(dt, U, flags, meth, UDst, maccormackStrength, boundaryWidth)
  maccormackStrength = maccormackStrength or 0.75                          -- init.lua:172-174
  checkUFlags(U, flags)
  check(lib.tfl_advect_vel(ctx, dt, U.c, flags.c, method(meth), maccormackStrength, UDst and UDst.c or nil))
end

function tfluids.setWallBcsForward(U, flags)
  checkUFlags(U, flags)
  check(lib.tfl_set_wall_bcs_forward(ctx, U.c, flags.c))
end

function tfluids.velocityDivergenceForward(U, flags, UDiv)
  checkUFlags(U, flags)
  assert(flags:isSameSizeAs(UDiv), 'Size mismatch')
  check(lib.tfl_velocity_divergence_forward(ctx, U.c, flags.c, UDiv.c))
end

function tfluids.velocityUpdateForward(U, flags, p)
  checkUFlags(U, flags)
  assert(p:isSameSizeAs(flags), 'Size mismatch')
  check(lib.tfl_velocity_update_forward(ctx, U.c, flags.c, p.c))
end

local function vec3(g) return ffi.new('float[3]', {g[1], g[2], g[3]}) end

function tfluids.addBuoyancy(U, flags, density, gravity, dt)
  checkUFlags(U, flags)
  assert(density:isSameSizeAs(flags), 'Size mismatch')
  check(lib.tfl_add_buoyancy(ctx, U.c, flags.c, density.c, vec3(gravity), dt))
end

function tfluids.addGravity(U, flags, gravity, dt)
  checkUFlags(U, flags)
  check(lib.tfl_add_gravity(ctx, U.c, flags.c, vec3(gravity), dt))
end

function tfluids.vorticityConfinement(U, flags, strength)
  checkUFlags(U, flags)
  assert(type(strength) == 'number')
  check(lib.tfl_vorticity_confinement(ctx, U.c, flags.c, strength))
end

function tfluids.emptyDomain(flags, is3D, bnd)
  bnd = bnd or 1
  assert(flags:size(2) == 1, 'Flags should be a scalar')
  check(lib.tfl_empty_domain(ctx, flags.c, is3D and 1 or 0, bnd))
  return flags
end

function tfluids.getDx(flags)                                             -- init.lua:560-565
  return 1.0 / math.max(math.max(flags:size(3), flags:size(4)), flags:size(5))
end

function tfluids.flagsToOccupancy(flags, occupancy)
  local bad = ffi.new('int64_t[1]')
  check(lib.tfl_flags_to_occupancy(ctx, flags.c, occupancy.c, bad))
  if bad[0] ~= 0 then error('ERROR: unsupported flag cell found!') end
end

function tfluids.solveLinearSystemJacobi(p, flags, div, is3D, pTol, maxIter, verbose)
  pTol = pTol or 1e-5                                                      -- init.lua:709-713
  maxIter = maxIter or 1000
  local res = ffi.new('float[1]')
  check(lib.tfl_solve_linear_system_jacobi(ctx, p.c, flags.c, div.c, is3D and 1 or 0, pTol, maxIter, res, nil))
  return res[0]
end

-- The same solve with no host wait: the residual (float) and the iteration count (int32) go to the device pointers
-- residual and iterations (each may be nil, e.g. from tfl_alloc).
function tfluids.solveLinearSystemJacobiDevice(p, flags, div, is3D, pTol, maxIter, residual, iterations)
  check(lib.tfl_solve_linear_system_jacobi_dev(ctx, p.c, flags.c, div.c, is3D and 1 or 0, pTol, maxIter,
                                               ffi.cast('float*', residual), ffi.cast('int32_t*', iterations)))
end

function tfluids.solveLinearSystemPCG(p, flags, div, is3D, tol, maxIter, precondType, verbose)
  precondType = precondType or 'ic0'                                       -- init.lua:661-666
  tol = tol or 1e-6
  maxIter = maxIter or 1000
  local kind = lib.tfl_precond_from_string(precondType)
  if kind < 0 then error("Incorrect preconType ('none', 'ic0', 'ilu0')") end
  local res = ffi.new('float[1]')
  check(lib.tfl_solve_linear_system_pcg(ctx, p.c, flags.c, div.c, is3D and 1 or 0, kind, tol, maxIter, res, nil))
  return res[0]
end

function tfluids.normalizePressureMean(p, flags, is3D)                      -- init.lua:747-765 (no host round trip)
  check(lib.tfl_normalize_pressure_mean(ctx, p.c, flags.c, is3D and 1 or 0))
end
function tfluids.volumetricUpSamplingNearestForward(ratio, input, output)  -- init.lua:618-622
  check(lib.tfl_volumetric_up_sampling_nearest_forward(ctx, ratio, input.c, output.c))
end
function tfluids.rectangularBlur(src, blurRad, is3D, dst)                  -- init.lua:583-596
  assert(blurRad > 0 and math.floor(blurRad) == blurRad, 'blurRad must be a positive, non-zero integer')
  check(lib.tfl_rectangular_blur(ctx, src.c, blurRad, is3D and 1 or 0, dst.c))
end
function tfluids.signedDistanceField(flags, searchRad, is3D, dst)          -- init.lua:604-614
  assert(searchRad > 0 and math.floor(searchRad) == searchRad, 'searchRad must be a positive, non-zero integer')
  check(lib.tfl_signed_distance_field(ctx, flags.c, searchRad, is3D and 1 or 0, dst.c))
end

function tfluids.velocityDivergenceBackward(U, flags, gradOutput, gradU)      -- init.lua:288-314
  check(lib.tfl_velocity_divergence_backward(ctx, U.c, flags.c, gradOutput.c, gradU.c))
end
function tfluids.velocityUpdateBackward(U, flags, p, gradOutput, gradP)      -- init.lua:358-384
  check(lib.tfl_velocity_update_backward(ctx, U.c, flags.c, p.c, gradOutput.c, gradP.c))
end
function tfluids.volumetricUpSamplingNearestBackward(ratio, input, gOut, gIn)   -- init.lua:623-627
  check(lib.tfl_volumetric_up_sampling_nearest_backward(ctx, ratio, input.c, gOut.c, gIn.c))
end

-- The cutorch pair inside setConstVals (lib/simulate.lua:136-158) and U:clamp (:326).
function tfluids.applyBC(x, invMask, bc) check(lib.tfl_apply_bc(ctx, x.c, invMask.c, bc.c)) end
function tfluids.clamp(x, lo, hi) check(lib.tfl_clamp(ctx, x.c, lo, hi)) end

-- model:forward replacement (lib/model.lua:421-450): `model` is a tfl_cnn* from tfl_cnn_create.
function tfluids.modelForward(model, pDiv, UDiv, flags, pOut, UOut, threshold)
  check(lib.tfl_cnn_project(ctx, model, pDiv.c, UDiv.c, flags.c, (pOut or pDiv).c, (UOut or UDiv).c,
                            threshold or 1e-5, nil))
end

-- One tfluids.simulate(conf, mconf, batch, model) (lib/simulate.lua:175-327) in one call.
local simMethods = {convnet = 0, jacobi = 1, pcg = 2}
function tfluids.simulateStep(mconf, batch, model)
  local st = ffi.new('tfl_state')
  local function set(field, t) if t ~= nil then st[field] = t.c end end
  set('p', batch.pDiv); set('U', batch.UDiv); set('flags', batch.flags); set('density', batch.density)
  set('U_bc', batch.UBC); set('U_bc_inv_mask', batch.UBCInvMask)
  set('density_bc', batch.densityBC); set('density_bc_inv_mask', batch.densityBCInvMask)
  set('p_bc', batch.pBC); set('p_bc_inv_mask', batch.pBCInvMask); set('div', batch.div)
  local g = mconf.gravity or {0, 1, 0}
  local mc = ffi.new('tfl_mconf', {mconf.dt, method(mconf.advectionMethod), mconf.maccormackStrength or 0.75,
                                   mconf.buoyancyScale or 0, mconf.gravityScale or 0, {g[1], g[2], g[3]},
                                   mconf.vorticityConfinementAmp or 0, simMethods[mconf.simMethod or 'convnet'],
                                   mconf.maxIter or 0, mconf.normalizeInputThreshold or 1e-5})
  check(lib.tfl_simulate_step(ctx, st, mc, model))
end

-- ---- beyond the reference: the step as a CUDA graph, and one domain in z-slabs over the GPUs of a node --------
-- (one LuaJIT process per GPU; `id` is the 128-byte NCCL id of rank 0, moved between the processes by the host
-- application: a file, a socket, MPI ...)
function tfluids.captureStep(cstate, cmconf, model)          -- after one tfluids.simulateStep on a non-default stream
  local g = ffi.new('tfl_step_graph*[1]')
  check(lib.tfl_step_graph_create(ctx, cstate, cmconf, model, g))
  return g[0]
end
function tfluids.launchStep(graph) check(lib.tfl_step_graph_launch(ctx, graph)) end
-- residual, iterations of the last replay's PCG solve (iterations -1 without one); raises the reference's error
-- string for the first failed solve since the previous call.  Synchronises.
function tfluids.stepPcgStatus(graph)
  local res, it = ffi.new('float[1]'), ffi.new('int32_t[1]')
  check(lib.tfl_step_graph_pcg_status(ctx, graph, res, it))
  return res[0], it[0]
end
function tfluids.commUniqueId()
  local id = ffi.new('char[128]')
  check(lib.tfl_comm_unique_id(ctx, id))
  return ffi.string(id, 128)
end
function tfluids.commInit(id, rank, world) check(lib.tfl_comm_init(ctx, id, rank, world)) end
function tfluids.slabCreate(gnz, ny, nx, margin, flagsHost, UBC, UBCInvMask, densityBC, densityBCInvMask)
  local sim = ffi.new('tfl_slab_sim*[1]')
  check(lib.tfl_slab_sim_create(ctx, gnz, ny, nx, margin or 2, flagsHost, UBC, UBCInvMask, densityBC, densityBCInvMask, sim))
  return sim[0]
end
function tfluids.slabIpcHandle(sim)                 -- 64 bytes for the neighbours (peer-memory halos, optional)
  local h = ffi.new('char[64]')
  check(lib.tfl_slab_sim_ipc_export(ctx, sim, h))
  return ffi.string(h, 64)
end
function tfluids.slabIpcConnect(sim, allHandles)     -- the 64-byte handles of every rank, concatenated in rank order
  check(lib.tfl_slab_sim_ipc_connect(ctx, sim, allHandles))
end
function tfluids.slabUpload(sim, p, U, density) check(lib.tfl_slab_sim_upload(ctx, sim, p, U, density)) end
function tfluids.slabStep(sim, cmconf, model) check(lib.tfl_slab_sim_step(ctx, sim, cmconf, model)) end
function tfluids.slabCaptureStep(sim, cmconf, model)  -- after one tfluids.slabStep on a non-default stream
  local g = ffi.new('tfl_slab_graph*[1]')
  check(lib.tfl_slab_graph_create(ctx, sim, cmconf, model, g))
  return g[0]
end
function tfluids.slabLaunchStep(graph) check(lib.tfl_slab_graph_launch(ctx, graph)) end
function tfluids.slabDownload(sim, p, U, density) check(lib.tfl_slab_sim_download(ctx, sim, p, U, density)) end
function tfluids.slabJacobiStats(sim)                -- p exchanges of the last 'jacobi' step: count, ms, bytes
  local n, ms, by = ffi.new('int32_t[1]'), ffi.new('float[1]'), ffi.new('int64_t[1]')
  check(lib.tfl_slab_sim_jacobi_stats(ctx, sim, n, ms, by))
  return n[0], ms[0], tonumber(by[0])
end
-- pTol of later 'jacobi' steps of a slab sim (0: the fixed count of maxIter sweeps)
function tfluids.slabSetJacobiTolerance(sim, pTol) check(lib.tfl_slab_sim_set_jacobi_tolerance(ctx, sim, pTol)) end
function tfluids.slabJacobiStatus(sim)               -- residual, iterations of the last tolerance step (waits once)
  local res, it = ffi.new('float[1]'), ffi.new('int32_t[1]')
  check(lib.tfl_slab_sim_jacobi_status(ctx, sim, res, it))
  return res[0], it[0]
end
function tfluids.slabJacobiSchedule(gnz, world, rank, margin, maxIter)   -- {planes = {lo, hi, uWidth}, blocks = {...}}
  local planes = ffi.new('int32_t[3]')
  local n = lib.tfl_slab_jacobi_schedule(gnz, world, rank, margin, maxIter, planes, nil, 0)
  assert(n > 0, 'slabJacobiSchedule: bad arguments')
  local raw = ffi.new('int32_t[?]', 6 * n)
  lib.tfl_slab_jacobi_schedule(gnz, world, rank, margin, maxIter, planes, raw, n)
  local blocks = {}
  for b = 0, n - 1 do
    local o = 6 * b
    blocks[b + 1] = {sweeps = raw[o], exchange = raw[o + 1], zLo = raw[o + 2], zHi = raw[o + 3],
                     shrinkLo = raw[o + 4], shrinkHi = raw[o + 5]}
  end
  return {planes = {planes[0], planes[1], planes[2]}, blocks = blocks}
end
function tfluids.slabCnnMargin(banksNum)             -- smallest slab margin of a model with banksNum banks
  local m = lib.tfl_slab_cnn_margin(banksNum)
  assert(m > 0, 'slabCnnMargin: banksNum above 8')
  return m
end

-- ---- density frames to the host behind the running step (the demo's save branch, fluid_net_3d_sim.lua:266-291) ----
-- A frame is nx * ny * nz floats in .vbox order (x slowest); the pointer stays valid until recorderRelease.
function tfluids.recorderCreate(nz, ny, nx, slots)
  local r = ffi.new('tfl_recorder*[1]')
  check(lib.tfl_recorder_create(ctx, nz, ny, nx, slots or 3, r))
  return r[0]
end
function tfluids.recorderCapture(rec, field)       -- enqueued on the context's stream; never waits
  local idx = ffi.new('int64_t[1]')
  check(lib.tfl_recorder_capture(ctx, rec, field.c, idx))
  return tonumber(idx[0])
end
function tfluids.recorderTake(rec, wait)           -- -> frame index, const float* (nil, nil: not landed yet)
  local ptr, idx = ffi.new('const float*[1]'), ffi.new('int64_t[1]')
  check(lib.tfl_recorder_take(ctx, rec, (wait == nil or wait) and 1 or 0, ptr, idx))
  if idx[0] < 0 then return nil, nil end
  return tonumber(idx[0]), ptr[0]
end
function tfluids.recorderRelease(rec) check(lib.tfl_recorder_release(ctx, rec)) end
function tfluids.recorderDestroy(rec) lib.tfl_recorder_destroy(ctx, rec) end
-- z-slab runs: one frame gathered on rank 0 from every rank's owned planes (collective captures, rank 0 takes).
-- Rank 0 passes recorderIpcHandle's 128 bytes to the other ranks, which recorderIpcConnect; then a barrier, then
-- captures.  Destroy on the other ranks first, then a barrier, then on rank 0.
function tfluids.recorderCreateSlab(gnz, ny, nx, rank, world, slots)
  local r = ffi.new('tfl_recorder*[1]')
  check(lib.tfl_recorder_create_slab(ctx, gnz, ny, nx, rank, world, slots or 3, r))
  return r[0]
end
function tfluids.recorderIpcHandle(rec)
  local h = ffi.new('char[128]')
  check(lib.tfl_recorder_ipc_export(ctx, rec, h))
  return ffi.string(h, 128)
end
function tfluids.recorderIpcConnect(rec, handle) check(lib.tfl_recorder_ipc_connect(ctx, rec, handle)) end
function tfluids.recorderCaptureSlab(rec, field, zOffset)   -- field: the rank's local slab, plane 0 = global zOffset
  local idx = ffi.new('int64_t[1]')
  check(lib.tfl_recorder_capture_slab(ctx, rec, field.c, zOffset, idx))
  return tonumber(idx[0])
end

-- ---- divergence statistics after every step (lib/calc_stats.lua:81-123), behind the running step ----
-- monitorTake -> record index and a table of nb entries {divNorm, divMax, uMax} (nil, nil: not landed yet).
function tfluids.monitorCreate(nb, gnz, capacity)
  local m = ffi.new('tfl_monitor*[1]')
  check(lib.tfl_monitor_create(ctx, nb, gnz, capacity or 64, m))
  return {c = m[0], nb = nb, buf = ffi.new('double[?]', nb * gnz * 3)}
end
function tfluids.monitorRecord(mon, U, flags)        -- enqueued on the context's stream; never waits
  local idx = ffi.new('int64_t[1]')
  check(lib.tfl_monitor_record(ctx, mon.c, U.c, flags.c, idx))
  return tonumber(idx[0])
end
function tfluids.monitorTake(mon, wait)
  local idx, z0, planes = ffi.new('int64_t[1]'), ffi.new('int32_t[1]'), ffi.new('int32_t[1]')
  check(lib.tfl_monitor_take(ctx, mon.c, (wait == nil or wait) and 1 or 0, idx, mon.buf, z0, planes))
  if idx[0] < 0 then return nil, nil end
  assert(planes[0] == 0, 'monitorTake: a z-slab record holds plane partials')
  local out = {}
  for b = 0, mon.nb - 1 do
    out[b + 1] = {divNorm = mon.buf[3 * b], divMax = mon.buf[3 * b + 1], uMax = mon.buf[3 * b + 2]}
  end
  return tonumber(idx[0]), out
end
function tfluids.monitorDestroy(mon) lib.tfl_monitor_destroy(ctx, mon.c) end

function tfluids.synchronize() check(lib.tfl_sync(ctx)) end

return tfluids
