"""ctypes binding of ``libbaybe_b200.so`` (the C ABI declared in ``include/baybe_b200.h``).

There is no CPU fallback: if the library is missing or cannot be loaded, every call raises.
"""

from __future__ import annotations

import ctypes as C
from pathlib import Path

LIB_PATH = Path(__file__).resolve().parent / "_C" / "libbaybe_b200.so"
ABI_VERSION = 4

# enums (mirror include/baybe_b200.h)
KERNEL_FAMILY = {"matern12": 0, "matern32": 1, "matern52": 2, "rbf": 3}
LAYOUT = {"row_f32": 0, "col_f32": 1, "row_f64": 2, "col_f64": 3, "bits_u8": 4}
HOST_FORMAT = {"rows_f32": 0, "rows_f64": 1, "codes4": 2, "codes8": 3}
ACQ_KIND = {
    "qLogEI": 0, "qEI": 1, "qUCB": 2, "qSR": 3, "qPI": 4,
    "UCB": 5, "EI": 6, "LogEI": 7, "PI": 8, "PM": 9, "PSTD": 10,
    "qEHVI": 11, "qLogEHVI": 12,
}
MC_KINDS = ("qLogEI", "qEI", "qUCB", "qSR", "qPI", "qEHVI", "qLogEHVI")
HVI_KINDS = ("qEHVI", "qLogEHVI")  # Pareto objectives: bb_hvi_score (baybe_b200/multiobjective.py)
HVI_MAX_TARGETS = 4
HVI_MAX_CELLS = 1024
# never by the fused kernels: hybrid spaces (qNEI only) by baybe_b200/hybrid.py (conditional form + bb_nei_reduce),
# discrete spaces by baybe_b200/noisy.py (bb_nei_score)
NEI_KINDS = ("qNEI", "qLogNEI")
# never by the fused kernels: Pareto objectives by random Chebyshev scalarisation, baybe_b200/parego.py
PAREGO_KINDS = ("qLogNParEGO",)
PAREGO_MAX_TARGETS = 8  # BB_OBJ_MAX_TARGETS
# never by the fused kernels: Pareto objectives with a sampled front, baybe_b200/nehvi.py (bb_hvi_decompose, then
# bb_hvi_score with the qEHVI kind)
NEHVI_KINDS = ("qNEHVI",)
# never by the fused kernels: integrated posterior variance over fixed integration points, baybe_b200/nipv.py
# (bb_nipv_score); no base samples, but batches and joint values go through the conditioning set like the MC kinds
NIPV_KINDS = ("qNIPV",)
NIPV_MAX_TRAIN = 256
MAX_PENDING = 31
MAX_TRAIN = 1024

BB_ERR_INVALID, BB_ERR_UNSUPPORTED, BB_ERR_CUDA, BB_ERR_NOT_PD, BB_ERR_WORKSPACE = -1, -2, -3, -4, -5

_dp = C.POINTER(C.c_double)


class ModelDesc(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("d", C.c_int32), ("family", C.c_int32), ("task_col", C.c_int32),
        ("n_tasks", C.c_int32), ("has_outputscale", C.c_int32), ("outputscale", C.c_double),
        ("train_x", _dp), ("train_y", _dp), ("lower", _dp), ("upper", _dp), ("lengthscale", _dp),
        ("noise", _dp), ("mean_const", _dp), ("task_covar", _dp),
    ]


class Model(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32),
        ("n", C.c_int32), ("n_pad", C.c_int32), ("d", C.c_int32), ("d_pad", C.c_int32),
        ("family", C.c_int32), ("task_col", C.c_int32), ("n_tasks", C.c_int32),
        ("n_chunks", C.c_int32), ("jitter_tries", C.c_int32),
        ("y_mean", C.c_float), ("y_std", C.c_float), ("prior_scale", C.c_float),
        ("r_scale", C.c_float), ("jitter", C.c_double),
        ("d_blob", C.c_void_p), ("blob_bytes", C.c_size_t),
        ("d_cand_scale", C.c_void_p), ("d_cand_shift", C.c_void_p), ("d_train_m2", C.c_void_p),
        ("d_train_sq", C.c_void_p), ("d_alpha", C.c_void_p), ("d_train_task", C.c_void_p),
        ("d_task_covar", C.c_void_p), ("d_mean_const", C.c_void_p), ("d_rimg", C.c_void_p),
        ("d_linv", C.c_void_p), ("d_alpha64", C.c_void_p), ("d_xn64", C.c_void_p),
        ("d_linv32", C.c_void_p),
        ("dist_scale_a", C.c_float), ("dist_scale_b", C.c_float),
        ("wide", C.c_int32), ("d_wide", C.c_int32), ("d_wimg", C.c_void_p),
        ("d_wimg_bits", C.c_void_p), ("d_wnorm_bits", C.c_void_p), ("d_wide_ws", C.c_void_p),
        ("wide_ws_rows", C.c_int64), ("dist_scale_w", C.c_float), ("pad_", C.c_int32),
        ("d_pend_img", C.c_void_p), ("d_pend_norm", C.c_void_p), ("d_pend_task", C.c_void_p),
        ("d_kpend_ws", C.c_void_p), ("dist_scale_p", C.c_float), ("dist_scale_wp", C.c_float),
        ("d_mc_table", C.c_void_p), ("d_timg_b", C.c_void_p), ("dist_k", C.c_int32),
        ("ts_sa", C.c_float), ("ts_aug_sq", C.c_float), ("ts_aug_one", C.c_float), ("ts_g", C.c_float),
        ("ts_kscale", C.c_float),
    ]


class AcqSpec(C.Structure):
    _fields_ = [
        ("kind", C.c_int32), ("maximize", C.c_int32), ("best_f", C.c_float), ("beta", C.c_float),
        ("obj_scale", C.c_float), ("obj_shift", C.c_float), ("tau_relu", C.c_float),
        ("tau_max", C.c_float), ("tau_pi", C.c_float),
    ]


OBJ_MAX_TARGETS, OBJ_MAX_OPS, OBJ_MAX_STACK = 8, 32, 4
OBJ_OP = {"AFFINE": 0, "CONST": 1, "CLAMP": 2, "TWO_SIDED": 3, "BELL": 4, "LOG": 5, "EXP": 6, "POW_INT": 7,
          "SIGMOID": 8, "DUP_INPUT": 9, "ADD": 10, "MUL": 11}
OBJ_SCALARIZER = {"NONE": 0, "MEAN": 1, "GEOM_MEAN": 2}


class ObjInstr(C.Structure):
    _fields_ = [("op", C.c_int32), ("arg", C.c_float * 3)]


class Objective(C.Structure):
    _fields_ = [("n_targets", C.c_int32), ("scalarizer", C.c_int32), ("n_ops", C.c_int32 * OBJ_MAX_TARGETS),
                ("weight", C.c_float * OBJ_MAX_TARGETS), ("prog", (ObjInstr * OBJ_MAX_OPS) * OBJ_MAX_TARGETS)]


class Best(C.Structure):
    _fields_ = [("val", C.c_float), ("pad_", C.c_int32), ("idx", C.c_int64)]


MAX_PEERS = 8


class PeerGroup(C.Structure):
    _fields_ = [("rank", C.c_int32), ("world", C.c_int32), ("d_key", C.c_void_p * MAX_PEERS),
                ("d_count", C.c_void_p * MAX_PEERS)]


class NativeLibraryError(RuntimeError):
    """The CUDA extension is missing or failed to load (there is no CPU fallback)."""


_lib = None

_vp, _i32, _i64, _sz = C.c_void_p, C.c_int32, C.c_int64, C.c_size_t
_SIGNATURES = {
    "bb_abi_version": (C.c_int, []),
    "bb_last_error": (C.c_char_p, []),
    "bb_model_blob_bytes": (_sz, [_i32, _i32, _i32]),
    "bb_model_build": (C.c_int, [C.POINTER(ModelDesc), _vp, _sz, C.POINTER(Model), _vp]),
    "bb_fit_workspace_bytes": (_sz, [_i32, _i32, _i32]),
    "bb_fit_setup": (C.c_int, [_vp, _sz, _i32, _i32, _i32, _dp, _dp, C.POINTER(C.c_int32), _vp]),
    "bb_fit_eval": (C.c_int, [_vp, _i32, _i32, _i32, _i32, _dp, _dp, _dp, C.POINTER(C.c_int32), _vp]),
    "bb_fit_eval_loo": (C.c_int, [_vp, _i32, _i32, _i32, _i32, _dp, _dp, _dp, C.POINTER(C.c_int32), _vp]),
    "bb_kernel_matrix": (C.c_int, [C.POINTER(Model), _vp, _i32, _i64, _i64, _vp, _i64, _vp]),
    "bb_posterior": (C.c_int, [C.POINTER(Model), _vp, _i32, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _i32, _vp]),
    "bb_pending_stats": (C.c_int, [C.POINTER(Model), _vp, _i32, _vp, _vp, _vp, _vp]),
    "bb_acq_score": (C.c_int, [C.POINTER(AcqSpec), _vp, _vp, _i64, _vp, _i32, _vp, _vp]),
    "bb_acq_score_joint": (C.c_int, [C.POINTER(AcqSpec), _vp, _vp, _vp, _i64, _vp, _vp, _i32, _vp, _i32, _vp, _vp]),
    "bb_score_fused": (C.c_int, [C.POINTER(Model), C.POINTER(AcqSpec), _vp, _i32, _i64, _i64, _vp, _vp, _i32, _vp, _vp, _i64, _vp]),
    "bb_best_init": (C.c_int, [_vp, _vp]),
    "bb_argmax": (C.c_int, [_vp, _vp, _i64, _i64, _vp, _vp]),
    "bb_best_decode": (C.c_int, [_vp, _vp, _vp]),
    "bb_topk": (C.c_int, [_vp, _vp, _i64, _i32, _vp, _vp, _vp, _vp, _vp]),
    "bb_score_fused_host": (C.c_int, [C.POINTER(Model), C.POINTER(AcqSpec), _vp, _i32, _i64, _i64, _vp, _i32,
                                      C.POINTER(_vp), C.POINTER(_vp), _i64, _vp, _vp, _i32, _vp, _vp, _i64, _vp, _vp]),
    "bb_score_fused_overlapped": (C.c_int, [C.POINTER(Model), C.POINTER(AcqSpec), _vp, _i32, _i64, _i64, _vp, _i32, _vp,
                                            _i64, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _i64, _vp, _vp]),
    "bb_nei_reduce": (C.c_int, [_vp, _i64, _i32, _i32, _vp, _vp, _vp, _vp, C.c_float, C.c_float, _i64, _vp, _vp]),
    "bb_hvi_score": (C.c_int, [C.POINTER(AcqSpec), _i32, C.POINTER(C.c_float), C.POINTER(C.c_float), _i64, _vp, _vp,
                               _i32, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp, _i32, _vp, _vp, _vp, _i64, _vp]),
    "bb_objective_score": (C.c_int, [C.POINTER(AcqSpec), C.POINTER(Objective), _i64, _vp, _vp, _i32, _vp, _vp, _vp,
                                     _vp, _vp, _i32, _vp, _vp, _vp, _i64, _vp]),
    "bb_joint_posterior": (C.c_int, [C.POINTER(Model), _vp, _i32, _vp, _vp, _vp, _vp, _sz, _vp]),
    "bb_nei_score": (C.c_int, [_i32, C.c_float, C.c_float, C.c_float, C.c_float, _i64, _vp, _vp, _i32, _vp, _vp, _vp,
                               _vp, _i32, _vp, _i32, _vp, _vp, _vp, _vp, _i64, _vp]),
    "bb_parego_score": (C.c_int, [_i32, C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_float, C.c_float, C.c_float,
                                  _i64, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _i32, _vp, _i32, _vp, _vp, _vp, _vp, _i64,
                                  _vp]),
    "bb_hvi_decompose": (C.c_int, [_i32, C.POINTER(C.c_double), _i32, _i32, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp]),
    "bb_nipv_score": (C.c_int, [C.POINTER(Model), C.POINTER(C.c_float), C.c_float, _vp, _i64, _vp, _i64, _vp, _i32,
                                _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _sz, _vp]),
    "bb_decode_codes":(C.c_int, [_vp, _i32, _i64, _i32, _i64, _vp, _i32, _vp, _i64, _vp]),
    "bb_peer_slots_init": (C.c_int, [_vp, _vp, _vp]),
    "bb_allreduce_best": (C.c_int, [C.POINTER(PeerGroup), _vp, C.c_uint32, _vp, _vp, _vp]),
    "bb_debug_posterior_simt": (C.c_int, [C.POINTER(Model), _vp, _i32, _i64, _i64, _vp, _vp, _vp]),
    "bb_debug_set_trace": (C.c_int, [_vp, _i64]),
}
EXPORTED_SYMBOLS = tuple(_SIGNATURES)


def load() -> C.CDLL:
    """Load the shared library (once) and type its entry points."""
    global _lib
    if _lib is not None:
        return _lib
    import os

    # diagnostic only (scripts/ab_kernel.py): time another build of the SAME library on the same box
    variant = os.environ.get("BB_LIB_VARIANT")
    path = LIB_PATH if not variant else LIB_PATH.parent / "variants" / f"{variant}.so"
    if not path.exists():
        raise NativeLibraryError(
            f"{path} not found: build it with `python -m baybe_b200.build` "
            "(baybe_b200 has no CPU fallback)"
        )
    try:
        lib = C.CDLL(str(path))
    except OSError as e:  # pragma: no cover - depends on the environment
        raise NativeLibraryError(f"cannot load {path}: {e}") from e
    for name, (res, args) in _SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            if variant:  # an older build may lack newer entry points
                continue
            raise
        fn.restype = res
        fn.argtypes = args
    if lib.bb_abi_version() != ABI_VERSION:
        raise NativeLibraryError(
            f"ABI mismatch: library reports {lib.bb_abi_version()}, binding expects {ABI_VERSION}"
        )
    _lib = lib
    return lib


def check(rc: int, what: str) -> None:
    """Map a bb_status to the exception types the reference's callers expect."""
    if rc == 0:
        return
    msg = load().bb_last_error().decode(errors="replace")
    text = f"{what}: {msg} (status {rc})"
    if rc in (BB_ERR_INVALID, BB_ERR_WORKSPACE):
        raise ValueError(text)
    if rc == BB_ERR_UNSUPPORTED:
        raise NotImplementedError(text)
    if rc == BB_ERR_NOT_PD:
        raise FloatingPointError(text)
    raise RuntimeError(text)
