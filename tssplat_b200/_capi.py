"""ctypes binding of the C ABI declared in ``include/tssplat_b200.h``.

There is no CPU fallback: if ``libtssplat_b200.so`` is missing or does not load, importing the
product modules raises.  Build it with ``python -m tssplat_b200.build`` (needs nvcc, no GPU).
"""
from __future__ import annotations

import ctypes as C
import os

from . import build as _build

# TSSPLAT_B200_LIB: developer override (e.g. the -DTSB_TRACE profiling build of tools/trace_phases.py)
LIB_PATH = os.environ.get("TSSPLAT_B200_LIB") or _build.LIB_PATH

TSB_OK, TSB_E_INVALID, TSB_E_MESH, TSB_E_CUDA, TSB_E_NOMEM = 0, -1, -2, -3, -4
TSB_LINE_MAX_ALPHA = 8
TSB_LBFGS_MAX_M = 16
TSB_PCG_MAXITER, TSB_PCG_CONVERGED, TSB_PCG_NEGCURV, TSB_PCG_NEGCURV_FIRST, TSB_PCG_ZERO_RHS = 0, 1, 2, 3, 4
TSB_PCG_BOUNDARY, TSB_PCG_NEGCURV_BOUNDARY = 5, 6
TSB_NEWTON_ACTIVE, TSB_NEWTON_CONVERGED, TSB_NEWTON_STALLED = 0, 1, 2

# every symbol include/tssplat_b200.h declares (tests check the library exports each one)
EXPORTED_SYMBOLS = (
    "tsb_create", "tsb_destroy", "tsb_last_error", "tsb_get_info", "tsb_energy_grad", "tsb_energy_grad_ex", "tsb_energy_grad_spheres", "tsb_hvp", "tsb_hvp_ex",
    "tsb_line_search", "tsb_hess_diag", "tsb_pcg_create", "tsb_pcg_destroy", "tsb_pcg_last_error", "tsb_pcg_device_bytes",
    "tsb_pcg_set_blocks", "tsb_pcg_solve", "tsb_sphere_axpy", "tsb_pcg_set_blocks_ex", "tsb_pcg_solve_ex",
    "tsb_pcg_enable_psd", "tsb_pcg_hvp_psd", "tsb_pcg_solve_tr",
    "tsb_hessian_create", "tsb_hessian_destroy", "tsb_hessian_last_error", "tsb_hessian_device_bytes", "tsb_hessian_pattern",
    "tsb_hessian_assemble", "tsb_pcg_enable_sgs", "tsb_pcg_set_matrix", "tsb_pcg_apply_precond", "tsb_pcg_sgs_colors",
    "tsb_pcg_enable_coarse", "tsb_pcg_set_coarse", "tsb_pcg_coarse_matrix",
    "tsb_newton_create", "tsb_newton_destroy", "tsb_newton_last_error", "tsb_newton_device_bytes", "tsb_newton_reset",
    "tsb_newton_step", "tsb_newton_prox_step", "tsb_newton_tr_step", "tsb_newton_tr_step_ex", "tsb_newton_lbfgs_step",
    "tsb_energy_grad_host", "tsb_scale",
    "tsb_grad_limit", "tsb_adam_uniform_step",
    "tsb_surface_create", "tsb_surface_destroy", "tsb_surface_last_error", "tsb_surface_forward", "tsb_surface_backward",
    "tsb_surface_extract", "tsb_free_host", "tsb_setup_last_error",
)


class tsb_options_t(C.Structure):
    _fields_ = [("warps_per_cta", C.c_int32), ("laplacian_scale", C.c_int32), ("ring_slots", C.c_int32),
                ("force_global", C.c_int32), ("tet_cost_x100", C.c_int32), ("enable_amips", C.c_int32),
                ("deterministic", C.c_int32), ("reserved", C.c_int32 * 1)]


class tsb_terms_t(C.Structure):
    _fields_ = [("c1", C.c_float), ("c2", C.c_float), ("order", C.c_int32), ("c3", C.c_float), ("reserved", C.c_int32 * 4)]


class tsb_sphere_stats_t(C.Structure):
    _fields_ = [("smooth", C.c_double), ("barrier", C.c_double), ("amips", C.c_double), ("min_J", C.c_float),
                ("n_inverted", C.c_int32), ("n_tets", C.c_int32), ("first_vertex", C.c_int32)]


class tsb_pcg_options_t(C.Structure):
    _fields_ = [("max_iter", C.c_int32), ("rtol", C.c_float), ("check_every", C.c_int32), ("reserved", C.c_int32 * 5)]


class tsb_pcg_sphere_t(C.Structure):
    _fields_ = [("rel_residual", C.c_float), ("b_dot_d", C.c_float), ("d_H_d", C.c_float), ("n_hvp", C.c_int32),
                ("status", C.c_int32), ("first_vertex", C.c_int32), ("n_vertices", C.c_int32), ("reserved", C.c_int32)]


class tsb_newton_options_t(C.Structure):
    _fields_ = [("max_iter", C.c_int32), ("rtol", C.c_float), ("rel_floor", C.c_float), ("tau", C.c_float),
                ("mu_min", C.c_float), ("mu_max", C.c_float), ("gtol", C.c_float), ("sigma", C.c_float), ("eta", C.c_float),
                ("n_alpha", C.c_int32), ("reserved", C.c_int32 * 6)]


class tsb_newton_sphere_t(C.Structure):
    _fields_ = [("mu", C.c_double), ("rho", C.c_double), ("grad_norm", C.c_float), ("alpha", C.c_float), ("delta", C.c_float),
                ("b_dot_d", C.c_float), ("k", C.c_int32), ("pcg_status", C.c_int32), ("n_hvp", C.c_int32),
                ("status", C.c_int32), ("first_vertex", C.c_int32), ("reserved", C.c_int32 * 3)]


class tsb_newton_tr_options_t(C.Structure):
    _fields_ = [("max_iter", C.c_int32), ("rtol", C.c_float), ("rel_floor", C.c_float), ("gtol", C.c_float),
                ("radius_init", C.c_float), ("radius_min", C.c_float), ("radius_max", C.c_float), ("accept", C.c_float),
                ("eta", C.c_float), ("reserved", C.c_int32 * 7)]


class tsb_newton_tr_sphere_t(C.Structure):
    _fields_ = [("radius", C.c_double), ("rho", C.c_double), ("grad_norm", C.c_float), ("alpha", C.c_float),
                ("delta", C.c_float), ("b_dot_d", C.c_float), ("pred", C.c_float), ("d_norm", C.c_float),
                ("pcg_status", C.c_int32), ("n_hvp", C.c_int32), ("status", C.c_int32), ("first_vertex", C.c_int32),
                ("reserved", C.c_int32 * 2)]


class tsb_newton_backtrack_t(C.Structure):
    _fields_ = [("n_alpha", C.c_int32), ("sigma", C.c_float), ("reserved", C.c_int32 * 6)]


class tsb_newton_lbfgs_options_t(C.Structure):
    _fields_ = [("m", C.c_int32), ("gtol", C.c_float), ("sigma", C.c_float), ("eta", C.c_float), ("n_alpha", C.c_int32),
                ("rel_floor", C.c_float), ("curv_eps", C.c_float), ("reserved", C.c_int32 * 9)]


class tsb_newton_lbfgs_sphere_t(C.Structure):
    _fields_ = [("grad_norm", C.c_float), ("alpha", C.c_float), ("delta", C.c_float), ("b_dot_d", C.c_float),
                ("d_norm", C.c_float), ("k", C.c_int32), ("status", C.c_int32), ("n_pairs", C.c_int32),
                ("pair_kept", C.c_int32), ("history_cleared", C.c_int32), ("first_vertex", C.c_int32),
                ("reserved", C.c_int32 * 5)]


class tsb_info_t(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("nele", C.c_int32), ("n_components", C.c_int32), ("grid", C.c_int32),
        ("warps_per_cta", C.c_int32), ("ctas_per_sm", C.c_int32), ("mode_global", C.c_int32),
        ("smem_bytes", C.c_int32), ("ring_slots", C.c_int32), ("n_segments", C.c_int32),
        ("n_boundary_faces", C.c_int32), ("max_component_vertices", C.c_int32),
        ("nnz", C.c_int64), ("nnz_padded", C.c_int64), ("device_bytes", C.c_int64), ("stream_bytes", C.c_int64),
    ]


_RECORD_DTYPES = {C.c_float: "float32", C.c_double: "float64", C.c_int32: "int32"}


def record_fields(raw, struct) -> dict:
    """Views of the scalar fields of ``struct`` (a ctypes Structure above) in ``raw``, a [S, sizeof(struct)] uint8 tensor
    of S such records: field name -> [S] tensor of the field's type (array fields such as ``reserved`` are left out)."""
    import torch
    out = {}
    for name, ctype in struct._fields_:
        if ctype in _RECORD_DTYPES:
            off = getattr(struct, name).offset
            out[name] = raw[:, off:off + C.sizeof(ctype)].view(getattr(torch, _RECORD_DTYPES[ctype]))[:, 0]
    return out


def _load() -> C.CDLL:
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: the CUDA library has not been built "
            "(run `python -m tssplat_b200.build`); tssplat_b200 has no CPU fallback")
    try:
        lib = C.CDLL(LIB_PATH)
    except OSError as e:  # pragma: no cover
        raise ImportError(f"cannot load {LIB_PATH}: {e}; tssplat_b200 has no CPU fallback") from e
    vp, f32, i32, i64 = C.c_void_p, C.c_float, C.c_int32, C.c_int64
    lib.tsb_create.restype = C.c_int
    lib.tsb_create.argtypes = [vp, vp, i32, i32, C.POINTER(tsb_options_t), C.c_int, C.POINTER(vp)]
    lib.tsb_destroy.restype = None
    lib.tsb_destroy.argtypes = [vp]
    lib.tsb_last_error.restype = C.c_char_p
    lib.tsb_last_error.argtypes = [vp]
    lib.tsb_get_info.restype = C.c_int
    lib.tsb_get_info.argtypes = [vp, C.POINTER(tsb_info_t)]
    lib.tsb_energy_grad.restype = C.c_int
    lib.tsb_energy_grad.argtypes = [vp, vp, f32, f32, i32, f32, vp, vp, vp, vp]
    lib.tsb_energy_grad_ex.restype = C.c_int
    lib.tsb_energy_grad_ex.argtypes = [vp, vp, C.POINTER(tsb_terms_t), f32, vp, vp, vp, vp]
    lib.tsb_energy_grad_spheres.restype = C.c_int
    lib.tsb_energy_grad_spheres.argtypes = [vp, vp, C.POINTER(tsb_terms_t), f32, vp, vp, vp, vp, vp]
    lib.tsb_hvp.restype = C.c_int
    lib.tsb_hvp.argtypes = [vp, vp, vp, f32, f32, i32, f32, vp, vp, vp, vp]
    lib.tsb_hvp_ex.restype = C.c_int
    lib.tsb_hvp_ex.argtypes = [vp, vp, vp, C.POINTER(tsb_terms_t), f32, vp, vp, vp, vp]
    lib.tsb_line_search.restype = C.c_int
    lib.tsb_line_search.argtypes = [vp, vp, vp, C.POINTER(tsb_terms_t), vp, i32, vp, vp, vp, vp, vp]
    lib.tsb_hess_diag.restype = C.c_int
    lib.tsb_hess_diag.argtypes = [vp, vp, C.POINTER(tsb_terms_t), f32, vp, vp, vp]
    lib.tsb_pcg_create.restype = C.c_int
    lib.tsb_pcg_create.argtypes = [vp, C.POINTER(vp)]
    lib.tsb_pcg_destroy.restype = None
    lib.tsb_pcg_destroy.argtypes = [vp]
    lib.tsb_pcg_last_error.restype = C.c_char_p
    lib.tsb_pcg_last_error.argtypes = [vp]
    lib.tsb_pcg_device_bytes.restype = i64
    lib.tsb_pcg_device_bytes.argtypes = [vp]
    lib.tsb_pcg_set_blocks.restype = C.c_int
    lib.tsb_pcg_set_blocks.argtypes = [vp, vp, f32, vp, vp]
    lib.tsb_pcg_solve.restype = C.c_int
    lib.tsb_pcg_solve.argtypes = [vp, vp, vp, C.POINTER(tsb_terms_t), C.POINTER(tsb_pcg_options_t), vp, vp,
                                  C.POINTER(C.c_int32), vp]
    lib.tsb_sphere_axpy.restype = C.c_int
    lib.tsb_sphere_axpy.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.tsb_pcg_set_blocks_ex.restype = C.c_int
    lib.tsb_pcg_set_blocks_ex.argtypes = [vp, vp, f32, vp, vp, vp]
    lib.tsb_pcg_solve_ex.restype = C.c_int
    lib.tsb_pcg_solve_ex.argtypes = [vp, vp, vp, C.POINTER(tsb_terms_t), C.POINTER(tsb_pcg_options_t), vp, vp, vp,
                                     C.POINTER(C.c_int32), vp]
    lib.tsb_pcg_enable_psd.restype = C.c_int
    lib.tsb_pcg_enable_psd.argtypes = [vp, vp, vp, i32]
    lib.tsb_pcg_hvp_psd.restype = C.c_int
    lib.tsb_pcg_hvp_psd.argtypes = [vp, vp, vp, C.POINTER(tsb_terms_t), vp, vp, vp]
    lib.tsb_pcg_solve_tr.restype = C.c_int
    lib.tsb_pcg_solve_tr.argtypes = [vp, vp, vp, C.POINTER(tsb_terms_t), C.POINTER(tsb_pcg_options_t), vp, vp, vp, vp,
                                     C.POINTER(C.c_int32), vp]
    lib.tsb_hessian_create.restype = C.c_int
    lib.tsb_hessian_create.argtypes = [vp, vp, vp, i32, C.POINTER(vp)]
    lib.tsb_hessian_destroy.restype = None
    lib.tsb_hessian_destroy.argtypes = [vp]
    lib.tsb_hessian_last_error.restype = C.c_char_p
    lib.tsb_hessian_last_error.argtypes = [vp]
    lib.tsb_hessian_device_bytes.restype = i64
    lib.tsb_hessian_device_bytes.argtypes = [vp]
    lib.tsb_hessian_pattern.restype = C.c_int
    lib.tsb_hessian_pattern.argtypes = [vp, C.POINTER(i64), vp, vp, vp]
    lib.tsb_hessian_assemble.restype = C.c_int
    lib.tsb_hessian_assemble.argtypes = [vp, vp, C.POINTER(tsb_terms_t), vp, vp]
    lib.tsb_pcg_enable_sgs.restype = C.c_int
    lib.tsb_pcg_enable_sgs.argtypes = [vp, vp]
    lib.tsb_pcg_set_matrix.restype = C.c_int
    lib.tsb_pcg_set_matrix.argtypes = [vp, vp, C.POINTER(tsb_terms_t), vp, vp]
    lib.tsb_pcg_apply_precond.restype = C.c_int
    lib.tsb_pcg_apply_precond.argtypes = [vp, vp, vp, vp]
    lib.tsb_pcg_sgs_colors.restype = C.c_int
    lib.tsb_pcg_sgs_colors.argtypes = [vp, vp, C.POINTER(C.c_int32)]
    lib.tsb_pcg_enable_coarse.restype = C.c_int
    lib.tsb_pcg_enable_coarse.argtypes = [vp, vp, vp, i32, C.c_float]
    lib.tsb_pcg_set_coarse.restype = C.c_int
    lib.tsb_pcg_set_coarse.argtypes = [vp, vp, C.POINTER(tsb_terms_t), vp]
    lib.tsb_pcg_coarse_matrix.restype = C.c_int
    lib.tsb_pcg_coarse_matrix.argtypes = [vp, vp]
    lib.tsb_newton_create.restype = C.c_int
    lib.tsb_newton_create.argtypes = [vp, C.POINTER(vp)]
    lib.tsb_newton_destroy.restype = None
    lib.tsb_newton_destroy.argtypes = [vp]
    lib.tsb_newton_last_error.restype = C.c_char_p
    lib.tsb_newton_last_error.argtypes = [vp]
    lib.tsb_newton_device_bytes.restype = i64
    lib.tsb_newton_device_bytes.argtypes = [vp]
    lib.tsb_newton_reset.restype = C.c_int
    lib.tsb_newton_reset.argtypes = [vp, vp]
    lib.tsb_newton_step.restype = C.c_int
    lib.tsb_newton_step.argtypes = [vp, vp, C.POINTER(tsb_terms_t), C.POINTER(tsb_newton_options_t), vp, vp]
    lib.tsb_newton_prox_step.restype = C.c_int
    lib.tsb_newton_prox_step.argtypes = [vp, vp, vp, vp, C.POINTER(tsb_terms_t), C.POINTER(tsb_newton_options_t), vp, vp]
    lib.tsb_newton_tr_step.restype = C.c_int
    lib.tsb_newton_tr_step.argtypes = [vp, vp, vp, vp, C.POINTER(tsb_terms_t), C.POINTER(tsb_newton_tr_options_t), vp, vp]
    lib.tsb_newton_tr_step_ex.restype = C.c_int
    lib.tsb_newton_tr_step_ex.argtypes = [vp, vp, vp, vp, C.POINTER(tsb_terms_t), C.POINTER(tsb_newton_tr_options_t),
                                          C.POINTER(tsb_newton_backtrack_t), vp, vp]
    lib.tsb_newton_lbfgs_step.restype = C.c_int
    lib.tsb_newton_lbfgs_step.argtypes = [vp, vp, vp, vp, C.POINTER(tsb_terms_t), C.POINTER(tsb_newton_lbfgs_options_t), vp, vp]
    lib.tsb_energy_grad_host.restype = C.c_int
    lib.tsb_energy_grad_host.argtypes = [vp, vp, f32, f32, i32, f32, vp, vp, vp]
    lib.tsb_scale.restype = C.c_int
    lib.tsb_scale.argtypes = [vp, i64, f32, vp, vp, vp]
    lib.tsb_grad_limit.restype = C.c_int
    lib.tsb_grad_limit.argtypes = [vp, i64, f32, f32, vp, vp]
    lib.tsb_adam_uniform_step.restype = C.c_int
    lib.tsb_adam_uniform_step.argtypes = [vp, vp, vp, vp, i64, C.c_double, C.c_double, C.c_double, i32, C.c_double, vp, vp]
    lib.tsb_surface_create.restype = C.c_int
    lib.tsb_surface_create.argtypes = [vp, i32, vp, i32, i32, C.c_int, C.POINTER(vp)]
    lib.tsb_surface_destroy.restype = None
    lib.tsb_surface_destroy.argtypes = [vp]
    lib.tsb_surface_last_error.restype = C.c_char_p
    lib.tsb_surface_last_error.argtypes = [vp]
    lib.tsb_surface_forward.restype = C.c_int
    lib.tsb_surface_forward.argtypes = [vp, vp, vp, vp, vp]
    lib.tsb_surface_backward.restype = C.c_int
    lib.tsb_surface_backward.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.tsb_surface_extract.restype = C.c_int
    lib.tsb_surface_extract.argtypes = [vp, C.c_int32, C.c_int32, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                        C.POINTER(C.POINTER(C.c_int32)), C.POINTER(C.POINTER(C.c_int32))]
    lib.tsb_free_host.restype = None
    lib.tsb_free_host.argtypes = [vp]
    lib.tsb_setup_last_error.restype = C.c_char_p
    lib.tsb_setup_last_error.argtypes = []
    return lib


lib = _load()


def last_error(handle=None) -> str:
    msg = lib.tsb_last_error(handle)
    return msg.decode("utf-8", "replace") if msg else ""


def check(rc: int, handle=None, what: str = "tssplat_b200") -> None:
    """Non-zero return codes become exceptions, like the reference's throw std::runtime_error
    (``tssplat_ext/tet_spheres/tet_spheres.cpp:152-202``)."""
    if rc == TSB_OK:
        return
    raise RuntimeError(f"{what}: {last_error(handle)} (code {rc})")
