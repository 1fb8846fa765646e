"""ctypes binding of libbjx.so (include/bjx.h).  The product path has NO CPU fallback: if the
CUDA library is missing this module raises at import of the first op."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libbjx.so")

TARGET_DIAG_GAUSSIAN, TARGET_FUNNEL, TARGET_DENSE_GAUSSIAN, TARGET_BANANA, TARGET_HIER_LOGIT, TARGET_USER = 0, 1, 2, 3, 4, 5
METRIC_DIAG, METRIC_DENSE, METRIC_DIAG_PER_CHAIN, METRIC_LOW_RANK, METRIC_DENSE_PER_CHAIN = 0, 1, 2, 3, 4
CHEES_WHITEN, CHEES_LENGTH_FLOOR = 1, 2
AMCLMC_STEPS_FIXED, AMCLMC_STEPS_RANDINT, AMCLMC_STEPS_UNIFORM = 0, 1, 2
GIST_TRAJECTORY_LENGTH, GIST_STEP_SIZE = 0, 1
GIST_SYMMETRIC, GIST_ASYMMETRIC = 0, 1
SLICE_DOUBLING, SLICE_STEPPING_OUT = 0, 1
RW_ADDITIVE, RW_INDEPENDENT = 0, 1

_f32p = C.c_void_p  # device pointers travel as integers


class TargetDesc(C.Structure):
    _fields_ = [("kind", C.c_int32), ("dim", C.c_int32), ("inv_var", C.c_void_p), ("mean", C.c_void_p),
                ("precision", C.c_void_p), ("logp_offset", C.c_float), ("data_x", C.c_void_p), ("data_y", C.c_void_p),
                ("n_groups", C.c_int32), ("n_user_params", C.c_int32), ("user_params", C.c_void_p),
                ("user_plugin", C.c_void_p)]


class Config(C.Structure):
    _fields_ = [("device", C.c_int32), ("n_chains", C.c_int32), ("dim", C.c_int32),
                ("max_tree_depth", C.c_int32), ("divergence_threshold", C.c_float), ("stream", C.c_void_p),
                ("target", TargetDesc)]


class Info(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "acceptance_rate", "is_accepted", "is_divergent", "is_turning", "energy", "num_integration_steps",
        "num_trajectory_expansions", "momentum", "proposal_position", "proposal_momentum", "left_position",
        "left_momentum", "right_position", "right_momentum")]


class MclmcInfo(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("kinetic_change", "energy_change", "nonans")]


class GistParams(C.Structure):
    _fields_ = [("instance", C.c_int32), ("path_fraction", C.c_float), ("max_num_steps", C.c_int32),
                ("num_integration_steps", C.c_int32), ("max_search_steps", C.c_int32), ("criterion", C.c_int32)]


class GistInfo(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "acceptance_rate", "is_accepted", "is_divergent", "energy", "momentum", "num_integration_steps", "forward",
        "reverse", "rejected", "a", "b", "step_size")]


class LangevinInfo(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("acceptance_rate", "is_accepted", "proposal_position", "proposal_logdensity",
                                          "proposal_grad")]


class EllipticalSliceInfo(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("momentum", "theta", "subiter", "exhausted")]


class SliceInfo(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("is_accepted", "num_expansions", "num_shrink", "bracket_left",
                                          "bracket_right")]


class RwInfo(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("acceptance_rate", "is_accepted")]


class LapsBurnInConfig(C.Structure):
    _fields_ = [("save_num", C.c_int32), ("alpha", C.c_float), ("C", C.c_float), ("r_end", C.c_float),
                ("bias_type", C.c_int32), ("early_stop", C.c_int32), ("equi_full", C.c_int32)]


class BjxError(RuntimeError):
    pass


_lib = None

_SIGNATURES = {
    "bjx_version": (C.c_int, []),
    "bjx_create": (C.c_int, [C.POINTER(Config), C.POINTER(C.c_void_p)]),
    "bjx_destroy": (C.c_int, [C.c_void_p]),
    "bjx_last_error": (C.c_char_p, [C.c_void_p]),
    "bjx_set_target": (C.c_int, [C.c_void_p, C.POINTER(TargetDesc)]),
    "bjx_plugin_load": (C.c_int, [C.c_char_p, C.POINTER(C.c_void_p)]),
    "bjx_plugin_abi": (C.c_int, []),
    "bjx_set_integrator": (C.c_int, [C.c_void_p, C.POINTER(C.c_float), C.c_int32]),
    "bjx_set_key_mode": (C.c_int, [C.c_void_p, C.c_int32, C.c_uint32]),
    "bjx_set_ghmc_noise": (C.c_int, [C.c_void_p, _f32p]),
    "bjx_set_integration_steps": (C.c_int, [C.c_void_p, C.c_void_p]),
    "bjx_synchronize": (C.c_int, [C.c_void_p]),
    "bjx_set_metric": (C.c_int, [C.c_void_p, C.c_int32, _f32p]),
    "bjx_set_metric_low_rank": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, C.c_int32]),
    "bjx_get_mass_matrix_sqrt": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "bjx_init_state": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p]),
    "bjx_sample_momentum": (C.c_int, [C.c_void_p, _f32p, _f32p]),
    "bjx_leapfrog": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, C.c_float, _f32p, C.c_int32]),
    "bjx_metric_velocity": (C.c_int, [C.c_void_p, _f32p, _f32p]),
    "bjx_energy": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p]),
    "bjx_is_turning": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p]),
    "bjx_hmc_step": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, C.c_float, _f32p,
                               C.c_int32, C.POINTER(Info)]),
    "bjx_mhmc_step": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, C.c_float, _f32p,
                                C.c_int32, C.POINTER(Info)]),
    "bjx_hmc_sample": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, C.c_float, _f32p, C.c_int32, C.c_int32, C.c_int32,
                                 _f32p, C.c_int32, _f32p]),
    "bjx_mclmc_init": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, _f32p]),
    "bjx_mclmc_step": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, _f32p, C.c_float, _f32p, C.c_float, _f32p,
                                 C.c_float, C.POINTER(MclmcInfo)]),
    "bjx_mclmc_sample": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, _f32p, C.c_float, _f32p, C.c_float, _f32p,
                                   C.c_float, C.c_int32, _f32p, C.c_int32, _f32p]),
    "bjx_mclmc_tune_step": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, C.c_float, _f32p, C.c_float,
                                      _f32p, _f32p, _f32p, _f32p, _f32p, C.c_int32, C.c_double, C.c_double, C.c_double,
                                      C.c_void_p]),
    "bjx_mclmc_ess_per_chain": (C.c_int, [C.c_void_p, _f32p, C.c_int32, _f32p, C.c_void_p]),
    "bjx_mclmc_find_l_and_step_size": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p,
                                                 C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float,
                                                 C.c_double, C.c_double, C.c_double, C.c_double, C.c_int64, C.c_void_p]),
    "bjx_adjusted_mclmc_step": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, C.c_float, _f32p,
                                          C.c_int32, C.c_float, C.POINTER(Info)]),
    "bjx_adjusted_mclmc_sample": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, C.c_float, _f32p, C.c_float, C.c_int32,
                                            C.c_int32, C.c_float, C.c_int32, C.c_void_p, C.c_int32, _f32p, C.c_int32, _f32p,
                                            C.c_void_p]),
    "bjx_set_integration_steps_avg": (C.c_int, [C.c_void_p, _f32p]),
    "bjx_adjusted_mclmc_num_steps": (C.c_int, [C.c_void_p, C.c_int32, _f32p, C.c_int32, C.c_void_p, C.c_void_p]),
    "bjx_adjusted_mclmc_tune_step": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, C.c_void_p, C.c_int32, C.c_int32,
                                               _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, C.c_int32, C.c_int32, C.c_float,
                                               C.c_void_p, C.c_void_p]),
    "bjx_adjusted_mclmc_find_l_and_step_size": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, C.c_void_p, C.c_int32,
                                                          C.c_int32, _f32p, _f32p, _f32p, C.c_int32, C.c_int32, C.c_int32,
                                                          C.c_int32, C.c_float, C.c_int32, C.c_int32, C.c_float, C.c_float,
                                                          C.c_double, C.c_int64, _f32p]),
    "bjx_gist_step": (C.c_int, [C.c_void_p, C.POINTER(GistParams), _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p,
                                C.c_float, _f32p, C.POINTER(GistInfo)]),
    "bjx_gist_sample": (C.c_int, [C.c_void_p, C.POINTER(GistParams), _f32p, _f32p, _f32p, _f32p, C.c_float, _f32p,
                                  C.c_int32, _f32p, C.c_int32, _f32p, C.c_void_p]),
    "bjx_mala_step": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, C.c_float, _f32p,
                                C.POINTER(LangevinInfo)]),
    "bjx_barker_step": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, C.c_float, _f32p,
                                  C.POINTER(LangevinInfo)]),
    "bjx_mala_sample": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, C.c_float, _f32p, C.c_int32, _f32p, C.c_int32,
                                  _f32p]),
    "bjx_barker_sample": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, C.c_float, _f32p, C.c_int32, _f32p,
                                    C.c_int32, _f32p]),
    "bjx_set_elliptical_prior": (C.c_int, [C.c_void_p, C.c_int32, _f32p, _f32p]),
    "bjx_elliptical_slice_step": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, _f32p, C.c_int32,
                                            C.POINTER(EllipticalSliceInfo)]),
    "bjx_elliptical_slice_sample": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, C.c_int32, C.c_int32, _f32p, C.c_int32,
                                              C.c_void_p]),
    "bjx_set_slice_direction_scale": (C.c_int, [C.c_void_p, C.c_int32, _f32p]),
    "bjx_slice_step": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, _f32p, C.c_float, _f32p, C.c_int32, C.c_int32,
                                 C.c_int32, C.POINTER(SliceInfo)]),
    "bjx_slice_sample": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, C.c_int32, C.c_float, _f32p, C.c_int32, C.c_int32,
                                   C.c_int32, _f32p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "bjx_set_rw_proposal": (C.c_int, [C.c_void_p, C.c_int32, _f32p, C.c_int32, _f32p]),
    "bjx_rw_step": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, _f32p, C.c_int32, C.POINTER(RwInfo)]),
    "bjx_rw_sample": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, C.c_int32, C.c_int32, _f32p, C.c_int32, _f32p]),
    "bjx_laps_state_floats": (C.c_int64, [C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "bjx_laps_init": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, _f32p, C.c_int32]),
    "bjx_laps_burn_in_step": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint32), C.c_int32, C.c_int32, _f32p, _f32p, _f32p,
                                        _f32p, _f32p, C.POINTER(LapsBurnInConfig), _f32p]),
    "bjx_laps_burn_in_run": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint32), C.c_int32, _f32p, _f32p, _f32p, _f32p, _f32p,
                                       C.POINTER(LapsBurnInConfig), _f32p, C.c_int32, C.POINTER(C.c_int32)]),
    "bjx_laps_switch": (C.c_int, [C.c_void_p, _f32p, C.c_int32]),
    "bjx_laps_adjusted_step": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint32), C.c_int32, C.c_int32, _f32p, _f32p, _f32p,
                                         _f32p, C.c_int32, C.c_int32, C.c_float, C.c_int32, _f32p]),
    "bjx_laps_adjusted_run": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint32), C.c_int32, _f32p, _f32p, _f32p, _f32p,
                                        C.c_int32, C.c_int32, C.c_float, C.c_int32, _f32p]),
    "bjx_nuts_step": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, C.c_float, _f32p,
                                C.c_int32, C.POINTER(Info), _f32p, _f32p]),
    "bjx_nuts_sample": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, C.c_float, _f32p, C.c_int32, C.c_int32, _f32p,
                                  C.c_int32, _f32p, C.c_void_p]),
    "bjx_adapt_shared_run": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, _f32p, C.c_char_p, C.c_int32, _f32p, _f32p, _f32p,
                                       _f32p, _f32p, _f32p, C.c_float, C.c_int32, C.c_int32, _f32p, _f32p, C.c_void_p,
                                       C.c_void_p]),
    "bjx_nuts_last_stats": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "bjx_prng_split": (C.c_int, [C.c_void_p, _f32p, C.c_int64, C.c_int32, _f32p]),
    "bjx_prng_fold_in": (C.c_int, [C.c_void_p, _f32p, C.c_int64, C.c_uint32, _f32p]),
    "bjx_prng_random_bits": (C.c_int, [C.c_void_p, _f32p, C.c_int64, C.c_int64, _f32p]),
    "bjx_prng_uniform": (C.c_int, [C.c_void_p, _f32p, C.c_int64, C.c_int64, _f32p]),
    "bjx_prng_normal": (C.c_int, [C.c_void_p, _f32p, C.c_int64, C.c_int64, _f32p]),
    "bjx_prng_randint": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_void_p]),
    "bjx_da_init": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p]),
    "bjx_da_update": (C.c_int, [C.c_void_p, _f32p, _f32p, C.c_float, _f32p]),
    "bjx_da_reset": (C.c_int, [C.c_void_p, _f32p, _f32p]),
    "bjx_da_final": (C.c_int, [C.c_void_p, _f32p, _f32p]),
    "bjx_welford_update": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, C.c_int32]),
    "bjx_welford_final": (C.c_int, [C.c_void_p, _f32p, _f32p, C.c_int32, _f32p]),
    "bjx_welford_dense_update": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, C.c_int32]),
    "bjx_welford_dense_final": (C.c_int, [C.c_void_p, _f32p, _f32p, C.c_int32, _f32p]),
    "bjx_pooled_stats": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p]),
    "bjx_pooled_stats_dense": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p]),
    "bjx_nccl_unique_id": (C.c_int, [C.c_void_p]),
    "bjx_nccl_comm_init_rank": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]),
    "bjx_nccl_comm_destroy": (C.c_int, [C.c_void_p]),
    "bjx_allgather_stats": (C.c_int, [C.c_void_p, C.c_void_p, _f32p, C.c_int64, _f32p]),
    "bjx_adapt_shared_state_floats": (C.c_int64, [C.c_int32, C.c_int32, C.c_int32]),
    "bjx_adapt_shared_init": (C.c_int, [C.c_void_p, _f32p, C.c_float, _f32p, _f32p]),
    "bjx_adapt_shared_update": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, _f32p, _f32p, _f32p, C.c_int32, C.c_int32,
                                          C.c_float, _f32p, _f32p, _f32p]),
    "bjx_adapt_shared_final": (C.c_int, [C.c_void_p, _f32p, _f32p]),
    "bjx_set_default_stream": (C.c_int, [C.c_void_p]),
    "bjx_chees_state_floats": (C.c_int64, [C.c_int32, C.c_int32, C.c_int32]),
    "bjx_chees_init": (C.c_int, [C.c_void_p, _f32p, C.c_float, C.c_int32, C.c_float, _f32p, C.c_void_p]),
    "bjx_chees_update": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, _f32p, _f32p, _f32p, _f32p, _f32p, C.c_void_p,
                                   C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int32, _f32p, C.c_void_p, _f32p]),
    "bjx_chees_final": (C.c_int, [C.c_void_p, _f32p, C.POINTER(C.c_float)]),
    "bjx_chees_metric_state_floats": (C.c_int64, [C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "bjx_chees_metric_init": (C.c_int, [C.c_void_p, _f32p, C.c_int32, C.c_int32, _f32p]),
    "bjx_chees_update_metric": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, _f32p, _f32p, _f32p, _f32p, _f32p,
                                          _f32p, _f32p, C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float,
                                          C.c_int32, C.c_int32, C.c_int32, _f32p, C.c_void_p, _f32p, _f32p, _f32p, _f32p]),
    "bjx_chees_final_metric": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, _f32p, _f32p, C.c_int32, _f32p,
                                         C.POINTER(C.c_float)]),
    "bjx_chees_metric_fold_covariance": (C.c_int, [C.c_void_p, C.c_int32, _f32p, _f32p]),
    "bjx_chees_metric_covariance": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, _f32p, _f32p]),
    "bjx_ghmc_step": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, C.c_float, _f32p, C.c_float, _f32p,
                                C.c_float, _f32p, _f32p, _f32p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(Info)]),
    "bjx_meads_state_floats": (C.c_size_t, [C.c_int32, C.c_int32]),
    "bjx_meads_scratch_floats": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32]),
    "bjx_meads_update": (C.c_int, [C.c_void_p, _f32p, _f32p, C.c_int32, C.c_int32, C.c_float, C.c_float, _f32p, _f32p]),
    "bjx_meads_lrd_state_floats": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32]),
    "bjx_meads_lrd_scratch_floats": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32]),
    "bjx_meads_lrd_update": (C.c_int, [C.c_void_p, _f32p, _f32p, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_float,
                                       _f32p, _f32p, _f32p]),
    "bjx_meads_lrd_metric": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, _f32p]),
    "bjx_lowrank_window_state_floats": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32]),
    "bjx_lowrank_window_init": (C.c_int, [C.c_void_p, _f32p, C.c_float, _f32p]),
    "bjx_lowrank_window_update": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, C.c_int32, C.c_float, C.c_float,
                                            C.c_float, _f32p, _f32p]),
    "bjx_lowrank_window_run": (C.c_int, [C.c_void_p, _f32p, C.c_char_p, C.c_int32, _f32p, _f32p, _f32p, _f32p, _f32p,
                                         C.c_float, C.c_float, C.c_float, C.c_int32, C.c_int32, _f32p, _f32p, C.c_void_p,
                                         C.c_void_p]),
    "bjx_lowrank_window_final": (C.c_int, [C.c_void_p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p]),
    "bjx_maximum_eigenvalue_scratch_floats":(C.c_size_t, [C.c_int64, C.c_int32]),
    "bjx_maximum_eigenvalue": (C.c_int, [C.c_void_p, _f32p, C.c_int64, C.c_int32, _f32p, _f32p]),
    "bjx_permutation_scratch_bytes": (C.c_size_t, [C.c_int64]),
    "bjx_permutation": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]),
    "bjx_gather_rows": (C.c_int, [C.c_void_p, C.c_void_p, _f32p, _f32p, C.c_int64, C.c_int32]),
    "bjx_potential_scale_reduction": (C.c_int, [C.c_void_p, _f32p, C.c_int32, _f32p, _f32p]),
    "bjx_ess_scratch_floats": (C.c_int64, [C.c_int32, C.c_int32, C.c_int32]),
    "bjx_effective_sample_size": (C.c_int, [C.c_void_p, _f32p, C.c_int32, _f32p, _f32p]),
    "bjx_rank_diagnostics_scratch_bytes": (C.c_int64, [C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "bjx_rank_normalize": (C.c_int, [C.c_void_p, _f32p, C.c_int32, C.c_int32, _f32p, C.c_void_p, C.c_size_t]),
    "bjx_rank_diagnostics": (C.c_int, [C.c_void_p, _f32p, C.c_int32, C.c_double, _f32p, _f32p, _f32p, C.c_void_p,
                                       C.c_size_t]),
}
EXPORTED_SYMBOLS = tuple(_SIGNATURES)


def lib():
    """Load libbjx.so once; fail loudly if it has not been built (no fallback path exists)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise BjxError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(or `make -C blackjax_b200/csrc`).  blackjax_b200 has no CPU or PyTorch fallback.")
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def check(rc, handle=None):
    if rc != 0:
        msg = lib().bjx_last_error(handle)
        raise BjxError(f"libbjx error {rc}: {msg.decode() if msg else '?'}")


def ptr(t):
    """Device pointer of a torch tensor (or None)."""
    return None if t is None else t.data_ptr()
