"""ctypes binding of libtfl.so (include/tfl.h).  Fails loudly when the library is absent."""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
# TFL_LIB_PATH: a differently-tuned build of the same library (kernel experiments); still no fallback.
LIB_PATH = os.environ.get("TFL_LIB_PATH") or os.path.join(HERE, "libtfl.so")


class TflError(RuntimeError):
    pass


class Grid(C.Structure):
    _fields_ = [("data", C.c_void_p), ("nb", C.c_int32), ("nc", C.c_int32), ("nz", C.c_int32),
                ("ny", C.c_int32), ("nx", C.c_int32)]


class MConf(C.Structure):
    _fields_ = [("dt", C.c_float), ("advection_method", C.c_int32),
                ("maccormack_strength", C.c_float), ("buoyancy_scale", C.c_double),
                ("gravity_scale", C.c_double), ("gravity", C.c_float * 3),
                ("vorticity_confinement_amp", C.c_double), ("sim_method", C.c_int32),
                ("max_iter", C.c_int32), ("normalize_input_threshold", C.c_float)]


class CnnBanks(C.Structure):
    _fields_ = [("num", C.c_int32), ("split_stage", C.c_int32), ("join_stage", C.c_int32),
                ("aggregate_add", C.c_int32)]


class CnnBanksEx(C.Structure):
    _fields_ = [("num", C.c_int32), ("split_stage", C.c_int32), ("join_stage", C.c_int32),
                ("aggregate_add", C.c_int32), ("dilate", C.c_int32)]


class CnnInputs(C.Structure):
    _fields_ = [("p_div", C.c_int32), ("u_div", C.c_int32), ("div", C.c_int32), ("normalize", C.c_int32),
                ("norm_func", C.c_int32), ("norm_chan", C.c_int32), ("pressure_skip", C.c_int32)]


class CnnNorm(C.Structure):
    _fields_ = [("relu6", C.c_int32), ("batch_norm", C.c_int32), ("batch_stats", C.c_int32),
                ("bn", C.POINTER(C.POINTER(C.c_float))), ("eps", C.POINTER(C.c_float))]


class State(C.Structure):
    _fields_ = [(n, Grid) for n in ("p", "U", "flags", "density", "U_bc", "U_bc_inv_mask",
                                    "density_bc", "density_bc_inv_mask", "p_bc", "p_bc_inv_mask",
                                    "div")]


# Every symbol include/tfl.h declares (tests check that the library exports all of them).
SYMBOLS = [
    "tfl_advect_method_from_string", "tfl_create", "tfl_destroy", "tfl_last_error", "tfl_version",
    "tfl_set_stream", "tfl_get_stream", "tfl_sync", "tfl_trace_faults", "tfl_launch_count",
    "tfl_set_slab", "tfl_set_slab_margin", "tfl_cnn_stats", "tfl_cnn_project_from_sums", "tfl_alloc", "tfl_free", "tfl_alloc_host", "tfl_free_host", "tfl_memcpy_h2d",
    "tfl_memcpy_d2h", "tfl_memcpy_d2d", "tfl_advect_scalar", "tfl_advect_vel",
    "tfl_set_wall_bcs_forward", "tfl_velocity_divergence_forward", "tfl_velocity_update_forward",
    "tfl_add_buoyancy", "tfl_add_gravity", "tfl_vorticity_confinement",
    "tfl_solve_linear_system_jacobi", "tfl_solve_linear_system_pcg", "tfl_precond_from_string", "tfl_normalize_pressure_mean",
    "tfl_volumetric_up_sampling_nearest_forward", "tfl_rectangular_blur", "tfl_signed_distance_field", "tfl_velocity_divergence_backward",
    "tfl_velocity_update_backward", "tfl_volumetric_up_sampling_nearest_backward", "tfl_empty_domain", "tfl_flags_to_occupancy", "tfl_apply_bc",
    "tfl_clamp", "tfl_cnn_create", "tfl_cnn_create_graph", "tfl_cnn_create_banked", "tfl_cnn_create_model", "tfl_cnn_create_model_ex", "tfl_cnn_create_model_norm", "tfl_cnn_destroy", "tfl_cnn_set_mode", "tfl_cnn_get_mode", "tfl_cnn_project", "tfl_simulate_step",
    "tfl_host_sim_create", "tfl_host_sim_destroy", "tfl_host_sim_step",
    "tfl_step_graph_create", "tfl_step_graph_launch", "tfl_step_graph_pcg_status", "tfl_step_graph_destroy",
    "tfl_comm_unique_id", "tfl_comm_init", "tfl_comm_destroy", "tfl_slab_sim_create", "tfl_slab_sim_destroy",
    "tfl_slab_sim_layout", "tfl_slab_sim_upload", "tfl_slab_sim_download", "tfl_slab_sim_step",
    "tfl_slab_sim_exchange_stats", "tfl_slab_sim_ipc_export", "tfl_slab_sim_ipc_connect",
    "tfl_slab_sim_jacobi_stats", "tfl_slab_jacobi_schedule", "tfl_jacobi_slab_block", "tfl_slab_cnn_margin",
    "tfl_recorder_create", "tfl_recorder_destroy", "tfl_recorder_capture", "tfl_recorder_take", "tfl_recorder_release",
    "tfl_recorder_create_slab", "tfl_recorder_ipc_export", "tfl_recorder_ipc_connect", "tfl_recorder_capture_slab",
]
JACOBI_BLOCK_INTS = 6
COMM_ID_BYTES = 128
IPC_HANDLE_BYTES = 64
RECORDER_HANDLE_BYTES = 128

_lib = None


def load():
    """Load libtfl.so; raises TflError (never falls back to anything else)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise TflError("libtfl.so is not built (%s). Run `python -c 'import __graft_entry__ as g; "
                       "g.build()'` or `make -C fluidnet_b200/csrc`. There is no CPU fallback."
                       % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    lib.tfl_last_error.restype = C.c_char_p
    lib.tfl_version.restype = C.c_char_p
    lib.tfl_get_stream.restype = C.c_void_p
    lib.tfl_launch_count.restype = C.c_int64
    lib.tfl_create.argtypes = [C.POINTER(C.c_void_p), C.c_int]
    lib.tfl_destroy.argtypes = [C.c_void_p]
    lib.tfl_last_error.argtypes = [C.c_void_p]
    lib.tfl_set_stream.argtypes = [C.c_void_p, C.c_void_p]
    lib.tfl_get_stream.argtypes = [C.c_void_p]
    lib.tfl_sync.argtypes = [C.c_void_p]
    lib.tfl_launch_count.argtypes = [C.c_void_p]
    lib.tfl_trace_faults.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.c_int]
    lib.tfl_set_slab.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32]
    lib.tfl_set_slab_margin.argtypes = [C.c_void_p, C.c_int32]
    G = C.POINTER(Grid)
    lib.tfl_advect_scalar.argtypes = [C.c_void_p, C.c_float, G, G, G, C.c_int, C.c_int, C.c_float, G]
    lib.tfl_advect_vel.argtypes = [C.c_void_p, C.c_float, G, G, C.c_int, C.c_float, G]
    lib.tfl_set_wall_bcs_forward.argtypes = [C.c_void_p, G, G]
    lib.tfl_velocity_divergence_forward.argtypes = [C.c_void_p, G, G, G]
    lib.tfl_velocity_update_forward.argtypes = [C.c_void_p, G, G, G]
    lib.tfl_add_buoyancy.argtypes = [C.c_void_p, G, G, G, C.POINTER(C.c_float), C.c_float]
    lib.tfl_add_gravity.argtypes = [C.c_void_p, G, G, C.POINTER(C.c_float), C.c_float]
    lib.tfl_vorticity_confinement.argtypes = [C.c_void_p, G, G, C.c_float]
    lib.tfl_solve_linear_system_jacobi.argtypes = [C.c_void_p, G, G, G, C.c_int, C.c_float, C.c_int,
                                                   C.POINTER(C.c_float), C.POINTER(C.c_int)]
    lib.tfl_solve_linear_system_pcg.argtypes = [C.c_void_p, G, G, G, C.c_int, C.c_int, C.c_float, C.c_int,
                                                C.POINTER(C.c_float), C.POINTER(C.c_int)]
    lib.tfl_precond_from_string.argtypes = [C.c_char_p]
    lib.tfl_normalize_pressure_mean.argtypes = [C.c_void_p, G, G, C.c_int]
    lib.tfl_volumetric_up_sampling_nearest_forward.argtypes = [C.c_void_p, C.c_int, G, G]
    lib.tfl_rectangular_blur.argtypes = [C.c_void_p, G, C.c_int, C.c_int, G]
    lib.tfl_signed_distance_field.argtypes = [C.c_void_p, G, C.c_int, C.c_int, G]
    lib.tfl_velocity_divergence_backward.argtypes = [C.c_void_p, G, G, G, G]
    lib.tfl_velocity_update_backward.argtypes = [C.c_void_p, G, G, G, G, G]
    lib.tfl_volumetric_up_sampling_nearest_backward.argtypes = [C.c_void_p, C.c_int, G, G, G]
    lib.tfl_empty_domain.argtypes = [C.c_void_p, G, C.c_int, C.c_int]
    lib.tfl_flags_to_occupancy.argtypes = [C.c_void_p, G, G, C.POINTER(C.c_int64)]
    lib.tfl_apply_bc.argtypes = [C.c_void_p, G, G, G]
    lib.tfl_clamp.argtypes = [C.c_void_p, G, C.c_float, C.c_float]
    lib.tfl_cnn_create_graph.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                         C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int,
                                         C.c_int, C.POINTER(C.POINTER(C.c_float)), C.POINTER(C.POINTER(C.c_float)),
                                         C.POINTER(C.c_void_p)]
    lib.tfl_cnn_create_banked.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                          C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int,
                                          C.c_int, C.POINTER(CnnBanks), C.POINTER(C.POINTER(C.c_float)),
                                          C.POINTER(C.POINTER(C.c_float)), C.POINTER(C.c_void_p)]
    lib.tfl_cnn_create_model.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                         C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int,
                                         C.c_int, C.POINTER(CnnBanks), C.POINTER(CnnInputs),
                                         C.POINTER(C.POINTER(C.c_float)), C.POINTER(C.POINTER(C.c_float)),
                                         C.POINTER(C.c_void_p)]
    lib.tfl_cnn_create_model_ex.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                            C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int,
                                            C.c_int, C.POINTER(CnnBanksEx), C.POINTER(CnnInputs),
                                            C.POINTER(C.POINTER(C.c_float)), C.POINTER(C.POINTER(C.c_float)),
                                            C.POINTER(C.c_void_p)]
    lib.tfl_cnn_create_model_norm.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                              C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int,
                                              C.c_int, C.POINTER(CnnBanksEx), C.POINTER(CnnInputs), C.POINTER(CnnNorm),
                                              C.POINTER(C.POINTER(C.c_float)), C.POINTER(C.POINTER(C.c_float)),
                                              C.POINTER(C.c_void_p)]
    lib.tfl_cnn_create.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int32),
                                   C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                   C.POINTER(C.POINTER(C.c_float)), C.POINTER(C.POINTER(C.c_float)),
                                   C.POINTER(C.c_void_p)]
    lib.tfl_cnn_destroy.argtypes = [C.c_void_p, C.c_void_p]
    lib.tfl_cnn_set_mode.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    lib.tfl_cnn_get_mode.argtypes = [C.c_void_p]
    lib.tfl_cnn_project.argtypes = [C.c_void_p, C.c_void_p, G, G, G, G, G, C.c_float,
                                    C.POINTER(C.c_float)]
    lib.tfl_cnn_stats.argtypes = [C.c_void_p, G, G, G, C.c_void_p]
    lib.tfl_cnn_project_from_sums.argtypes = [C.c_void_p, C.c_void_p, G, G, G, C.c_void_p, G, G, C.c_float]
    lib.tfl_simulate_step.argtypes = [C.c_void_p, C.POINTER(State), C.POINTER(MConf), C.c_void_p]
    lib.tfl_host_sim_create.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.POINTER(C.c_void_p)]
    lib.tfl_host_sim_destroy.argtypes = [C.c_void_p, C.c_void_p]
    lib.tfl_host_sim_step.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.POINTER(MConf), C.c_void_p]
    lib.tfl_step_graph_create.argtypes = [C.c_void_p, C.POINTER(State), C.POINTER(MConf), C.c_void_p, C.POINTER(C.c_void_p)]
    lib.tfl_step_graph_launch.argtypes = [C.c_void_p, C.c_void_p]
    lib.tfl_step_graph_pcg_status.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_int32)]
    lib.tfl_step_graph_destroy.argtypes = [C.c_void_p, C.c_void_p]
    lib.tfl_comm_unique_id.argtypes = [C.c_void_p, C.c_char_p]
    lib.tfl_comm_init.argtypes = [C.c_void_p, C.c_char_p, C.c_int32, C.c_int32]
    lib.tfl_comm_destroy.argtypes = [C.c_void_p]
    lib.tfl_slab_sim_create.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]
    lib.tfl_slab_sim_destroy.argtypes = [C.c_void_p, C.c_void_p]
    lib.tfl_slab_sim_layout.argtypes = [C.c_void_p, C.POINTER(State), C.POINTER(C.c_int32)]
    lib.tfl_slab_sim_upload.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.tfl_slab_sim_download.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.tfl_slab_sim_step.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(MConf), C.c_void_p]
    lib.tfl_slab_sim_ipc_export.argtypes = [C.c_void_p, C.c_void_p, C.c_char_p]
    lib.tfl_slab_sim_ipc_connect.argtypes = [C.c_void_p, C.c_void_p, C.c_char_p]
    lib.tfl_slab_sim_exchange_stats.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_int64)]
    lib.tfl_slab_sim_jacobi_stats.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_float),
                                              C.POINTER(C.c_int64)]
    lib.tfl_slab_jacobi_schedule.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                             C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int32]
    lib.tfl_slab_cnn_margin.argtypes = [C.c_int32]
    lib.tfl_jacobi_slab_block.argtypes = [C.c_void_p, G, G, G, G, C.c_int, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                          C.c_int32, C.c_int32, C.POINTER(C.c_int32)]
    lib.tfl_alloc_host.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p)]
    lib.tfl_free_host.argtypes = [C.c_void_p, C.c_void_p]
    lib.tfl_recorder_create.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]
    lib.tfl_recorder_destroy.argtypes = [C.c_void_p, C.c_void_p]
    lib.tfl_recorder_capture.argtypes = [C.c_void_p, C.c_void_p, G, C.POINTER(C.c_int64)]
    lib.tfl_recorder_take.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.POINTER(C.c_float)),
                                      C.POINTER(C.c_int64)]
    lib.tfl_recorder_release.argtypes = [C.c_void_p, C.c_void_p]
    lib.tfl_recorder_create_slab.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                             C.POINTER(C.c_void_p)]
    lib.tfl_recorder_ipc_export.argtypes = [C.c_void_p, C.c_void_p, C.c_char_p]
    lib.tfl_recorder_ipc_connect.argtypes = [C.c_void_p, C.c_void_p, C.c_char_p]
    lib.tfl_recorder_capture_slab.argtypes = [C.c_void_p, C.c_void_p, G, C.c_int32, C.POINTER(C.c_int64)]
    _lib = lib
    return lib
