"""ctypes declarations for include/heyoka_b200.h. Loading fails loudly if the native library is missing."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libheyoka_b200.so")


class HyError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(msg)
        self.code = code


HY_OK = 0
HY_ERR_INVALID_ARG = -1
HY_ERR_NOT_IMPLEMENTED = -2
HY_ERR_CUDA = -3
HY_ERR_OVERFLOW = -4
HY_ERR_CALLBACK = -5

# taylor_outcome (include/heyoka/taylor.hpp): values below -2^32 so that they never collide with event indices.
HY_OUTCOME_SUCCESS = -4294967297
HY_OUTCOME_STEP_LIMIT = -4294967298
HY_OUTCOME_TIME_LIMIT = -4294967299
HY_OUTCOME_ERR_NF_STATE = -4294967300
HY_OUTCOME_CB_STOP = -4294967301

if not os.path.exists(LIB_PATH):
    raise ImportError(
        "heyoka_b200: native library %s not found. Build it with `python -m heyoka_b200.build` (needs nvcc); "
        "there is no Python/CPU fallback for the compute path." % LIB_PATH)

lib = C.CDLL(LIB_PATH)


class hy_program_desc(C.Structure):
    _fields_ = [
        ("n_eq", C.c_uint32), ("n_uvars", C.c_uint32), ("n_pars", C.c_uint32), ("order", C.c_uint32),
        ("n_args", C.c_uint32), ("n_consts", C.c_uint32), ("high_accuracy", C.c_int32), ("n_ev", C.c_uint32),
        ("ops", C.c_void_p), ("args", C.c_void_p), ("consts", C.c_void_p), ("sv_defs", C.c_void_p),
        ("ev_defs", C.c_void_p),
    ]


class hy_event_rec(C.Structure):
    _fields_ = [("lane", C.c_uint32), ("idx", C.c_uint32), ("terminal", C.c_int32), ("d_sgn", C.c_int32),
                ("t", C.c_double), ("abs_der", C.c_double)]


class hy_batch_ptrs(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("state", "pars", "t_hi", "t_lo", "last_h", "tc", "d_out", "step_outcome",
                                          "prop_outcome", "prop_min_h", "prop_max_h", "prop_n_steps")]


class hy_kernel_info(C.Structure):
    _fields_ = [("tape_mode", C.c_int32), ("lanes_per_warp", C.c_uint32), ("lanes_per_thread", C.c_uint32),
                ("block_threads", C.c_uint32), ("blocks_per_sm", C.c_uint32), ("grid", C.c_uint32),
                ("smem_bytes", C.c_uint64), ("tape_slots_per_lane", C.c_uint32), ("n_segments", C.c_uint32),
                ("n_fused", C.c_uint32), ("n_sms", C.c_uint32), ("tmem_cols_per_warp", C.c_uint32),
                ("reserved", C.c_uint32)]


_dp = C.POINTER(C.c_double)
_vp = C.c_void_p
_vpp = C.POINTER(C.c_void_p)

# name -> (restype, argtypes); mirrors include/heyoka_b200.h one to one.
SIGNATURES = {
    "hy_last_error": (C.c_char_p, []),
    "hy_version": (C.c_char_p, []),
    "hy_ex_num": (_vp, [C.c_double]),
    "hy_ex_var": (_vp, [C.c_char_p]),
    "hy_ex_par": (_vp, [C.c_uint32]),
    "hy_ex_time": (_vp, []),
    "hy_ex_binary": (_vp, [C.c_char, _vp, _vp]),
    "hy_ex_func": (_vp, [C.c_char_p, _vpp, C.c_uint32]),
    "hy_ex_copy": (_vp, [_vp]),
    "hy_ex_free": (None, [_vp]),
    "hy_ex_str": (C.c_size_t, [_vp, C.c_char_p, C.c_size_t]),
    "hy_ex_diff": (_vp, [_vp, _vp]),
    "hy_var_ode_sys": (C.c_int, [_vpp, _vpp, C.c_uint32, C.c_uint32, _vpp, C.c_uint32, C.c_uint32,
                                 C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), _vpp, _vpp, _vpp]),
    "hy_model_nbody": (C.c_int, [C.c_uint32, _dp, C.c_uint32, C.c_double, _vpp, _vpp]),
    "hy_model_pendulum": (C.c_int, [C.c_double, C.c_double, _vpp, _vpp]),
    "hy_model_ffnn": (C.c_int, [_vpp, C.c_uint32, C.POINTER(C.c_uint32), C.c_uint32, C.c_uint32, C.POINTER(C.c_int), _dp,
                                C.c_uint32, _vpp]),
    "hy_order_from_tol": (C.c_int, [C.c_double, C.POINTER(C.c_uint32)]),
    "hy_program_from_sys": (C.c_int, [_vpp, _vpp, C.c_uint32, C.c_double, C.c_int, _vpp]),
    "hy_program_from_sys_ev": (C.c_int, [_vpp, _vpp, C.c_uint32, _vpp, C.c_uint32, C.c_double, C.c_int, _vpp]),
    "hy_program_create": (C.c_int, [C.POINTER(hy_program_desc), _vpp]),
    "hy_program_get_desc": (C.c_int, [_vp, C.POINTER(hy_program_desc)]),
    "hy_program_dc_size": (C.c_uint32, [_vp]),
    "hy_program_dc_str": (C.c_size_t, [_vp, C.c_char_p, C.c_size_t]),
    "hy_program_costs": (C.c_int, [_vp, _dp, _dp, _dp]),
    "hy_program_destroy": (None, [_vp]),
    "hy_batch_create": (C.c_int, [_vp, C.c_uint32, C.c_int, _vpp]),
    "hy_batch_destroy": (None, [_vp]),
    "hy_selftest_div": (C.c_int, [C.c_uint64, C.c_uint64, C.POINTER(C.c_uint64)]),
    "hy_host_pin": (C.c_int, [_vp, C.c_size_t]),
    "hy_host_unpin": (C.c_int, [_vp]),
    "hy_batch_set_stream": (C.c_int, [_vp, _vp]),
    "hy_batch_sync": (C.c_int, [_vp]),
    "hy_batch_upload": (C.c_int, [_vp, _dp, _dp, _dp, _dp]),
    "hy_batch_download": (C.c_int, [_vp, _dp, _dp, _dp, _dp]),
    "hy_batch_download_step_res": (C.c_int, [_vp, C.POINTER(C.c_int64), _dp]),
    "hy_batch_download_prop_res": (C.c_int, [_vp, C.POINTER(C.c_int64), _dp, _dp, C.POINTER(C.c_uint64)]),
    "hy_batch_download_tc": (C.c_int, [_vp, _dp]),
    "hy_batch_upload_tc": (C.c_int, [_vp, _dp]),
    "hy_batch_create_multi": (C.c_int, [_vp, C.c_uint32, C.POINTER(C.c_int), C.c_uint32, C.POINTER(_vp)]),
    "hy_batch_n_shards": (C.c_uint32, [_vp]),
    "hy_device_count": (C.c_int, []),
    "hy_batch_get_ptrs": (C.c_int, [_vp, C.POINTER(hy_batch_ptrs)]),
    "hy_batch_step": (C.c_int, [_vp, _dp, C.c_int, C.c_int, C.c_int]),
    "hy_batch_propagate_until": (C.c_int, [_vp, _dp, _dp, _dp, C.c_uint64, C.c_int]),
    "hy_batch_propagate_until_host": (C.c_int, [_vp, _dp, _dp, _dp, _dp, _dp, _dp, _dp, C.c_uint64, _dp, _dp, _dp, _dp,
                                                C.POINTER(C.c_int64), _dp, _dp, C.POINTER(C.c_uint64)]),
    "hy_batch_propagate_until_dev": (C.c_int, [_vp, _dp, _dp, _dp, C.c_uint64, C.c_int, C.POINTER(C.c_int)]),
    "hy_batch_propagate_grid": (C.c_int, [_vp, _dp, C.c_uint64, _dp, C.c_uint64, _dp]),
    "hy_batch_check_grid": (C.c_int, [_vp, _dp, C.c_uint64, _dp]),
    "hy_batch_propagate_until_cout": (C.c_int, [_vp, _dp, _dp, _dp, C.c_uint64, _vpp]),
    "hy_cout_rec_begin": (C.c_int, [_vp, _vpp]),
    "hy_cout_rec_append": (C.c_int, [_vp, _vp]),
    "hy_cout_rec_finish": (C.c_int, [_vp, _vp, C.POINTER(C.c_uint8), _vpp]),
    "hy_cout_rec_destroy": (None, [_vp]),
    "hy_batch_propagate_until_cout_cb": (C.c_int, [_vp, _dp, _dp, _dp, C.c_uint64, C.c_void_p, C.c_void_p, _vpp]),
    "hy_cout_eval": (C.c_int, [_vp, _dp, _dp]),
    "hy_cout_get_bounds": (C.c_int, [_vp, _dp, _dp]),
    "hy_cout_n_steps": (C.c_uint64, [_vp]),
    "hy_cout_download": (C.c_int, [_vp, _dp, _dp, _dp]),
    "hy_cout_destroy": (None, [_vp]),
    "hy_batch_d_output": (C.c_int, [_vp, _dp, _dp]),
    "hy_batch_eval_taylor_map": (C.c_int, [_vp, C.c_uint32, C.c_uint32, _dp, _dp, C.c_int]),
    "hy_batch_set_events": (C.c_int, [_vp, C.c_uint32, C.POINTER(C.c_int32), _dp, C.c_double]),
    "hy_batch_n_events": (C.c_uint32, [_vp]),
    "hy_batch_get_events": (C.c_int, [_vp, C.POINTER(hy_event_rec), C.c_uint32]),
    "hy_batch_download_tc_events": (C.c_int, [_vp, _dp]),
    "hy_batch_reset_cooldowns": (C.c_int, [_vp, C.c_int64]),
    "hy_batch_get_cooldowns": (C.c_int, [_vp, C.POINTER(C.c_uint8), _dp, _dp]),
    "hy_batch_set_cooldowns": (C.c_int, [_vp, C.POINTER(C.c_uint8), _dp, _dp]),
    "hy_batch_launch_count": (C.c_int, [_vp, C.POINTER(C.c_uint64)]),
    "hy_batch_set_launch_config": (C.c_int, [_vp, C.c_uint32, C.c_uint32]),
    "hy_batch_set_kernel": (C.c_int, [_vp, C.c_int, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32]),
    "hy_batch_get_kernel": (C.c_int, [_vp, C.POINTER(hy_kernel_info)]),
}

for _name, (_res, _args) in SIGNATURES.items():
    _f = getattr(lib, _name)  # AttributeError here = the library does not export a declared symbol
    _f.restype = _res
    _f.argtypes = _args


def last_error():
    return lib.hy_last_error().decode(errors="replace")


_EXC = {HY_ERR_INVALID_ARG: ValueError, HY_ERR_NOT_IMPLEMENTED: NotImplementedError, HY_ERR_OVERFLOW: OverflowError}


def check(code):
    """Translate a status code into the exception the reference would throw."""
    if code == HY_OK:
        return
    msg = last_error()
    exc = _EXC.get(code)
    if exc is not None:
        raise exc(msg)
    raise HyError(code, msg)


def ex_checked(handle):
    if not handle:
        msg = last_error()
        if "not implemented" in msg:
            raise NotImplementedError(msg)
        raise ValueError(msg)
    return int(handle)
