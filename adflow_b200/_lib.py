"""ctypes loader for libadflow_b200.so (the C ABI of include/adflow_b200.h).

The product has no CPU path: loading fails loudly when the shared library has not
been built, and every compute entry point returns an error when no CUDA device
is available (``AdflowB200Error``).
"""
import ctypes as C
import os

from .params import AdfbParams

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("ADFLOW_B200_LIB", os.path.join(_HERE, "libadflow_b200.so"))  # override: tuning experiments only

# every symbol include/adflow_b200.h declares (checked by tests/test_abi.py)
ABI_SYMBOLS = [
    "adfb_init", "adfb_finalize", "adfb_get_unique_id", "adfb_last_error", "adfb_device_count",
    "adfb_block_create", "adfb_block_destroy", "adfb_block_set_geometry", "adfb_block_set_bc",
    "adfb_set_params", "adfb_upload_state", "adfb_download_state", "adfb_upload_visc",
    "adfb_download_residual", "adfb_download_intermed", "adfb_residual", "adfb_norms", "adfb_synchronize", "adfb_forces",
    "adfb_get_states", "adfb_set_states", "adfb_get_res", "adfb_state_size",
    "adfb_comm_set_pattern", "adfb_comm_set_overset", "adfb_block_set_orphans", "adfb_halo_exchange",
    "adfb_reference_shock_sensor", "adfb_form_function", "adfb_mffd_set_base", "adfb_mffd_apply", "adfb_mffd_apply_device", "adfb_mffd_last_h",
    "adfb_apply_bcs", "adfb_timestep", "adfb_smoother_residual", "adfb_rk_stage", "adfb_rk_cycle", "adfb_dadi_step", "adfb_dadi_cycle", "adfb_sa_ddadi",
    "adfb_block_set_mg", "adfb_mg_restrict", "adfb_mg_prolong", "adfb_mg_cycle",
    "adfb_set_ground_level", "adfb_get_ground_level", "adfb_mg_prolong_solution",
    "adfb_ank_set_params", "adfb_ank_time_step_mat", "adfb_ank_form_function", "adfb_ank_mffd_set_base", "adfb_ank_mffd_apply", "adfb_ank_mffd_apply_device",
    "adfb_ank_physicality_check", "adfb_ank_form_function_turb", "adfb_ank_mffd_turb_set_base", "adfb_ank_mffd_turb_apply",
    "adfb_ank_physicality_check_turb", "adfb_gmres_solve",
]


class AdflowB200Error(RuntimeError):
    pass


class AdfbSubface(C.Structure):
    _fields_ = [
        ("bcType", C.c_int32), ("faceId", C.c_int32),
        ("icBeg", C.c_int32), ("icEnd", C.c_int32), ("jcBeg", C.c_int32), ("jcEnd", C.c_int32),
        ("norm", C.c_void_p), ("rface", C.c_void_p), ("uSlip", C.c_void_p), ("TNSWall", C.c_void_p),
        ("ps", C.c_void_p), ("rho", C.c_void_p), ("velx", C.c_void_p), ("vely", C.c_void_p), ("velz", C.c_void_p),
        ("ptInlet", C.c_void_p), ("ttInlet", C.c_void_p), ("htInlet", C.c_void_p), ("flowXdirInlet", C.c_void_p),
        ("flowYdirInlet", C.c_void_p), ("flowZdirInlet", C.c_void_p), ("turbInlet", C.c_void_p),
        ("subsonicInletTreatment", C.c_int32), ("pad_", C.c_int32),
    ]


_lib = None


def load():
    """Return the loaded library; raises if it was never built (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise AdflowB200Error(
            "%s not found: build it with `python -m adflow_b200.build` (nvcc, sm_90a). "
            "There is no CPU fallback." % LIB_PATH
        )
    L = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
    vp, ci, cu = C.c_void_p, C.c_int, C.c_uint
    L.adfb_init.argtypes = [ci, vp, ci, ci]
    L.adfb_get_unique_id.argtypes = [vp]
    L.adfb_last_error.argtypes = [C.c_char_p, ci]
    L.adfb_block_create.argtypes = [ci] * 7
    L.adfb_block_destroy.argtypes = [ci]
    L.adfb_block_set_geometry.argtypes = [ci] + [vp] * 11
    L.adfb_block_set_bc.argtypes = [ci, ci, vp]
    L.adfb_set_params.argtypes = [C.POINTER(AdfbParams)]
    L.adfb_upload_state.argtypes = [ci, vp, vp]
    L.adfb_download_state.argtypes = [ci, vp, vp, vp, vp]
    L.adfb_upload_visc.argtypes = [ci, vp, vp]
    L.adfb_download_residual.argtypes = [ci, vp]
    L.adfb_download_intermed.argtypes = [ci, vp, vp, vp, vp]
    L.adfb_download_array.argtypes = [ci, C.c_char_p, vp]
    L.adfb_residual.argtypes = [ci, cu]
    L.adfb_norms.argtypes = [C.POINTER(C.c_double)]
    L.adfb_forces.argtypes = [ci, C.POINTER(C.c_double), C.c_double, C.POINTER(C.c_double)]
    for fn in (L.adfb_get_states, L.adfb_set_states, L.adfb_get_res):
        fn.argtypes = [vp, C.c_longlong]
    L.adfb_state_size.restype = C.c_longlong
    L.adfb_reference_shock_sensor.argtypes = [ci]
    L.adfb_form_function.argtypes = [vp, vp, C.c_longlong]
    L.adfb_mffd_set_base.argtypes = [vp, C.c_longlong]
    L.adfb_mffd_apply.argtypes = [vp, vp, C.c_longlong, C.c_double]
    L.adfb_mffd_apply_device.argtypes = [vp, vp, C.c_longlong, C.c_double]
    L.adfb_mffd_last_h.restype = C.c_double
    L.adfb_comm_set_pattern.argtypes = [ci, ci, vp, vp, vp, vp, vp, ci, vp, vp]
    L.adfb_comm_set_overset.argtypes = [ci, ci, vp, vp, vp, vp, vp, vp, ci, vp, vp, vp]
    L.adfb_block_set_orphans.argtypes = [ci, ci, vp, C.c_double, C.c_double]
    L.adfb_ank_form_function_turb.argtypes = [vp, vp, C.c_longlong]
    L.adfb_ank_mffd_turb_set_base.argtypes = [vp, C.c_longlong]
    L.adfb_ank_mffd_turb_apply.argtypes = [vp, vp, C.c_longlong, C.c_double]
    L.adfb_ank_physicality_check_turb.argtypes = [vp, vp, C.c_longlong, vp]
    L.adfb_halo_exchange.argtypes = [ci] * 6
    L.adfb_apply_bcs.argtypes = [ci, ci, ci]
    L.adfb_timestep.argtypes = [ci, ci]
    L.adfb_smoother_residual.argtypes = [ci, ci]
    L.adfb_rk_stage.argtypes = [ci, ci]
    L.adfb_rk_cycle.argtypes = [ci]
    L.adfb_dadi_step.argtypes = [ci]
    L.adfb_dadi_cycle.argtypes = [ci, ci]
    L.adfb_sa_ddadi.argtypes = [ci, ci]
    L.adfb_block_set_mg.argtypes = [ci, ci] + [vp] * 9
    L.adfb_mg_restrict.argtypes = [ci]
    L.adfb_mg_prolong.argtypes = [ci]
    L.adfb_set_ground_level.argtypes = [ci]
    L.adfb_get_ground_level.argtypes = []
    L.adfb_mg_prolong_solution.argtypes = [ci]
    L.adfb_mg_cycle.argtypes = [ci, vp, ci]
    L.adfb_ank_set_params.argtypes = [vp]
    L.adfb_ank_form_function.argtypes = [vp, vp, C.c_longlong]
    L.adfb_ank_mffd_set_base.argtypes = [vp, C.c_longlong]
    L.adfb_ank_mffd_apply.argtypes = [vp, vp, C.c_longlong, C.c_double]
    L.adfb_ank_mffd_apply_device.argtypes = [vp, vp, C.c_longlong, C.c_double]
    L.adfb_ank_physicality_check.argtypes = [vp, vp, C.c_longlong, C.POINTER(C.c_double)]
    L.adfb_gmres_solve.argtypes = [ci, vp, vp, C.c_longlong, ci, ci, C.c_double, C.c_double, vp, vp, C.POINTER(ci), C.POINTER(C.c_double)]
    L.adfb_launch_count.restype = C.c_longlong
    L.adfb_stream.restype = C.c_void_p
    _lib = L
    return L


def check(rc, what=""):
    if rc != 0:
        buf = C.create_string_buffer(1024)
        load().adfb_last_error(buf, 1024)
        raise AdflowB200Error("%s failed: %s" % (what or "adflow_b200 call", buf.value.decode(errors="replace")))


def ptr(a):
    """Raw pointer of a Fortran-contiguous numpy array (None -> NULL)."""
    if a is None:
        return None
    assert a.flags.f_contiguous, "host arrays must be Fortran contiguous (reference layout)"
    return a.ctypes.data
