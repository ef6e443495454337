"""ctypes binding of libb2gram.so (include/b2gram.h) and a thin object wrapper.

There is deliberately no CPU implementation behind these calls: if the shared library is missing
or no H100 is visible, every compute entry point raises ``RuntimeError`` (the reference's error
style, stage_1_train_model.py:74,125,142).
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional, Tuple

import numpy as np

from . import build as _build

F32, BF16, F64 = 0, 1, 2
MEM_DEVICE, MEM_HOST = 0, 1
KERNEL_AUTO, KERNEL_SIMT, KERNEL_TCGEN05, KERNEL_NARROW = 0, 1, 2, 3
PRECISION_SPLIT, PRECISION_BF16 = 0, 1
E_ARG = -1
E_SINGULAR = -4
E_COMM = -5
EXCHANGE_NONE, EXCHANGE_NCCL, EXCHANGE_PEER = 0, 1, 2
ABI_VERSION = 2
MAX_D = 128
MAX_ALPHAS = 64
GLM_LOG, GLM_IDENTITY = 0, 1
GLM_STEPS = 21
SVM_SQUARED_HINGE, SVM_SQUARED_EPSILON = 0, 1
MAX_CLASSES = 32
LOO_SQUARED, LOO_ACCURACY = 0, 1

_c_i64 = C.c_int64
_vp = C.c_void_p

# name -> (restype, argtypes); mirrors include/b2gram.h one to one
_SIGNATURES = {
    "b2_abi_version": (C.c_int, []),
    "b2_last_error": (C.c_char_p, []),
    "b2_device_count": (C.c_int, [C.POINTER(C.c_int)]),
    "b2_ctx_create": (C.c_int, [C.c_int, C.POINTER(_vp)]),
    "b2_ctx_destroy": (C.c_int, [_vp]),
    "b2_ctx_sync": (C.c_int, [_vp]),
    "b2_ctx_info": (C.c_int, [_vp, C.c_char_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_size_t)]),
    "b2_ctx_set_kernel": (C.c_int, [_vp, C.c_int]),
    "b2_ctx_set_drain_rows": (C.c_int, [_vp, C.c_int]),
    "b2_ctx_set_precision": (C.c_int, [_vp, C.c_int]),
    "b2_ctx_set_sm_limit": (C.c_int, [_vp, C.c_int]),
    "b2_dev_alloc": (C.c_int, [_vp, C.c_size_t, C.POINTER(_vp)]),
    "b2_dev_free": (C.c_int, [_vp, _vp]),
    "b2_host_alloc": (C.c_int, [_vp, C.c_size_t, C.POINTER(_vp)]),
    "b2_host_free": (C.c_int, [_vp, _vp]),
    "b2_copy_h2d": (C.c_int, [_vp, _vp, _vp, C.c_size_t]),
    "b2_copy_d2h": (C.c_int, [_vp, _vp, _vp, C.c_size_t]),
    "b2_dev_memset": (C.c_int, [_vp, _vp, C.c_int, C.c_size_t]),
    "b2_gram_reset": (C.c_int, [_vp, C.c_int]),
    "b2_gram_accumulate": (C.c_int, [_vp, _vp, C.c_int, _vp, _c_i64, C.c_int, _c_i64, C.c_int, _vp, C.c_int]),
    "b2_gram_allreduce": (C.c_int, [_vp]),
    "b2_gram_export": (C.c_int, [_vp, _vp, C.POINTER(_c_i64)]),
    "b2_gram_import": (C.c_int, [_vp, _vp, C.c_int]),
    "b2_split_mask": (C.c_int, [_c_i64, _c_i64, C.c_uint32, _vp]),
    "b2_copy_d2d": (C.c_int, [_vp, _vp, _vp, C.c_size_t]),
    "b2_pack_columns": (C.c_int, [_vp, _vp, C.c_int, _c_i64, C.c_int, _vp]),
    "b2_upload_columns": (C.c_int, [_vp, _vp, _vp, C.c_int, _c_i64, C.c_int, _vp]),
    "b2_fit": (C.c_int, [_vp, _vp, C.c_int, _vp, _c_i64, C.c_int, _c_i64, C.c_int, _vp, C.c_int, C.c_double, C.c_int, _vp,
                         C.POINTER(C.c_double)]),
    "b2_fit_refined": (C.c_int, [_vp, _vp, C.c_int, _vp, _c_i64, C.c_int, _c_i64, C.c_int, _vp, C.c_int, C.c_double,
                                 C.c_int, C.c_int, C.c_double, _vp, C.POINTER(C.c_double), C.POINTER(C.c_int),
                                 C.POINTER(C.c_double)]),
    "b2_solve": (C.c_int, [_vp, C.c_double, C.c_int, _vp, C.POINTER(C.c_double)]),
    "b2_solve_eigvals": (C.c_int, [_vp, C.c_double, C.c_int, _vp, C.POINTER(C.c_int), C.POINTER(_c_i64)]),
    "b2_solve_spectral": (C.c_int, [_vp, C.c_double, C.c_int, _vp, C.POINTER(C.c_double), _vp, C.POINTER(C.c_int)]),
    "b2_solve_eigh": (C.c_int, [_vp, C.c_int, _vp, _vp]),
    "b2_solve_enet_path": (C.c_int, [_vp, C.c_int, C.c_double, _vp, C.c_int, C.c_double, C.c_int, C.c_double, C.c_int,
                                     _vp, _vp, _vp, _vp, _vp, _vp, C.POINTER(C.c_double)]),
    "b2_gram_folds": (C.c_int, [_vp, _vp, C.c_int, _vp, _c_i64, C.c_int, _c_i64, C.c_int, _vp, C.c_int, _vp]),
    "b2_solve_enet_cv": (C.c_int, [_vp, _vp, C.c_int, C.c_int, _vp, C.c_int, _vp, C.c_int, C.c_double, C.c_int,
                                   C.c_double, C.c_int, _vp, _vp, _vp, _vp, _vp]),
    "b2_ridge_loo": (C.c_int, [_vp, _vp, C.c_int, _vp, _c_i64, C.c_int, _c_i64, C.c_int, _vp, C.c_int, _vp, C.c_int,
                               C.c_int, _vp, _vp, C.POINTER(C.c_int), _vp, C.POINTER(C.c_double)]),
    "b2_residual_moments": (C.c_int, [_vp, _vp, C.c_int, _vp, _c_i64, C.c_int, _c_i64, C.c_int, _vp, C.c_int, _vp,
                                      C.c_double, C.c_int, _vp]),
    "b2_solve_bayes_ridge": (C.c_int, [_vp, C.c_int, _vp, C.c_int, C.c_double, _vp, C.c_int, _vp,
                                       C.POINTER(C.c_double), C.POINTER(C.c_double), _vp, C.POINTER(C.c_int), _vp, _vp]),
    "b2_solve_ard": (C.c_int, [_vp, C.c_int, _vp, C.c_double, C.c_int, C.c_double, _vp, C.c_int, _vp,
                               C.POINTER(C.c_double), C.POINTER(C.c_double), _vp, C.POINTER(C.c_int), _vp, _vp]),
    "b2_score_std": (C.c_int, [_vp, _vp, C.c_int, _c_i64, C.c_int, _c_i64, C.c_int, _vp, _vp, C.c_double, _vp,
                               C.c_double, _vp, _vp]),
    "b2_glm_pass": (C.c_int, [_vp, _vp, C.c_int, _vp, _c_i64, C.c_int, _c_i64, C.c_int, _vp, C.c_int, C.c_int,
                              C.c_double, _vp, C.c_double, C.c_int, _vp, _vp]),
    "b2_glm_line_search": (C.c_int, [_vp, _vp, C.c_int, _vp, _c_i64, C.c_int, _c_i64, C.c_int, _vp, C.c_int, C.c_int,
                                     C.c_double, _vp, C.c_double, _vp, C.c_double, C.c_int, _vp]),
    "b2_glm_predict": (C.c_int, [_vp, _vp, C.c_int, _c_i64, C.c_int, _c_i64, C.c_int, C.c_int, _vp, C.c_double, _vp]),
    "b2_logistic_pass": (C.c_int, [_vp, _vp, C.c_int, _vp, _c_i64, C.c_int, _c_i64, C.c_int, _vp, C.c_int, C.c_double,
                                   C.c_double, _vp, C.c_double, C.c_int, _vp, _vp]),
    "b2_logistic_line_search": (C.c_int, [_vp, _vp, C.c_int, _vp, _c_i64, C.c_int, _c_i64, C.c_int, _vp, C.c_int,
                                          C.c_double, C.c_double, _vp, C.c_double, _vp, C.c_double, C.c_int, _vp]),
    "b2_logistic_predict": (C.c_int, [_vp, _vp, C.c_int, _c_i64, C.c_int, _c_i64, C.c_int, _vp, C.c_double, C.c_double,
                                      C.c_double, _vp, _vp, _vp]),
    "b2_label_scan": (C.c_int, [_vp, _vp, _c_i64, _vp, C.c_int, _vp]),
    "b2_class_sums": (C.c_int, [_vp, _vp, C.c_int, _vp, _c_i64, C.c_int, _c_i64, C.c_int, _vp, C.c_int, _vp, C.c_int,
                                _vp, _vp, _vp]),
    "b2_class_scatter": (C.c_int, [_vp, _vp, C.c_int, _vp, _c_i64, C.c_int, _c_i64, C.c_int, _vp, C.c_int, _vp, C.c_int,
                                   _vp, _vp, _vp, _vp]),
    "b2_class_scatters": (C.c_int, [_vp, _vp, C.c_int, _vp, _c_i64, C.c_int, _c_i64, C.c_int, _vp, C.c_int, _vp,
                                    C.c_int, _vp, _vp, _vp, _vp]),
    "b2_qda_decision": (C.c_int, [_vp, _vp, C.c_int, _vp, _c_i64, C.c_int, _c_i64, C.c_int, _vp, C.c_int, _vp, C.c_int,
                                  _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b2_solve_classes": (C.c_int, [_vp, C.c_double, C.c_int, _vp, C.c_int, _vp, _vp]),
    "b2_classify": (C.c_int, [_vp, _vp, C.c_int, _vp, _c_i64, C.c_int, _c_i64, C.c_int, _vp, C.c_int, _vp, _vp, C.c_int,
                              _vp, _vp, _vp, _vp]),
    "b2_label_values": (C.c_int, [_vp, _vp, _c_i64, _vp, C.c_int, C.c_int, _vp, C.POINTER(C.c_int),
                                  C.POINTER(C.c_int)]),
    "b2_multinomial_pass": (C.c_int, [_vp, _vp, C.c_int, _vp, _c_i64, C.c_int, _c_i64, C.c_int, _vp, C.c_int, _vp,
                                      C.c_int, _vp, C.c_int, _vp, _vp]),
    "b2_multinomial_line_search": (C.c_int, [_vp, _vp, C.c_int, _vp, _c_i64, C.c_int, _c_i64, C.c_int, _vp, C.c_int,
                                             _vp, C.c_int, _vp, _vp, C.c_int, _vp]),
    "b2_softmax_rows": (C.c_int, [_vp, _vp, _c_i64, C.c_int, C.c_int]),
    "b2_svm_pass": (C.c_int, [_vp, _vp, C.c_int, _vp, _c_i64, C.c_int, _c_i64, C.c_int, _vp, C.c_int, C.c_int,
                              C.c_double, _vp, C.c_double, _vp, C.c_double, C.c_int, _vp, _vp]),
    "b2_ridge_classifier_loo": (C.c_int, [_vp, _vp, C.c_int, _vp, _c_i64, C.c_int, _c_i64, C.c_int, _vp, C.c_int, _vp,
                                          C.c_int, _vp, C.c_int, C.c_int, C.c_int, _vp, _vp, _vp, C.POINTER(C.c_int), _vp,
                                          _vp, _vp]),
    "b2_score": (C.c_int, [_vp, _vp, C.c_int, _c_i64, C.c_int, _c_i64, C.c_int, _vp, C.c_double, _vp, _vp,
                           C.c_int, _vp, _vp]),
    "b2_score_allreduce": (C.c_int, [_vp, _vp]),
    "b2_metrics": (C.c_int, [_vp, _vp, _vp, C.c_int, _c_i64, C.c_int, _vp]),
    "b2_synth_tranche": (C.c_int, [_vp, C.c_uint64, _c_i64, C.c_int, C.c_double, C.c_double, _vp, _vp,
                                   C.POINTER(_c_i64)]),
    "b2_synth": (C.c_int, [_vp, C.c_uint64, _c_i64, _c_i64, C.c_int, _c_i64, C.c_int, C.c_double, C.c_double,
                           C.c_double, _vp, _vp]),
    "b2_comm_unique_id": (C.c_int, [C.c_char_p]),
    "b2_comm_init": (C.c_int, [_vp, C.c_int, C.c_int, C.c_char_p]),
    "b2_comm_destroy": (C.c_int, [_vp]),
    "b2_comm_barrier": (C.c_int, [_vp]),
    "b2_comm_p2p_export": (C.c_int, [_vp, C.c_char_p]),
    "b2_comm_p2p_attach": (C.c_int, [_vp, C.c_int, C.c_int, C.c_char_p]),
    "b2_comm_p2p_detach": (C.c_int, [_vp]),
    "b2_comm_p2p_attach_local": (C.c_int, [_vp, C.c_int, C.c_int, C.POINTER(_vp)]),
    "b2_comm_set_timeout_ms": (C.c_int, [_vp, _c_i64]),
    "b2_comm_info": (C.c_int, [_vp, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "b2_ctx_stats": (C.c_int, [_vp, C.POINTER(_c_i64)]),
    "b2_timer_start": (C.c_int, [_vp]),
    "b2_timer_stop": (C.c_int, [_vp, C.POINTER(C.c_double)]),
    "b2_last_kernel_ms": (C.c_int, [_vp, C.POINTER(C.c_double), C.POINTER(C.c_int)]),
    "b2_launch_count": (C.c_int, [_vp, C.POINTER(_c_i64)]),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)
_lib = None


def lib_path() -> str:
    return os.environ.get("B2_LIB_PATH") or _build.LIB_PATH   # B2_LIB_PATH: development override (kernel variants)


def load():
    """dlopen libb2gram.so (building it first if the sources are newer and nvcc is present)."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if os.environ.get("B2_LIB_PATH"):
        pass
    elif not os.path.exists(path) or (_build.is_stale() and os.environ.get("B2_NO_REBUILD") != "1"):
        try:
            _build.build()
        except Exception as exc:  # pragma: no cover - only without nvcc
            if not os.path.exists(path):
                raise RuntimeError(f"libb2gram.so is missing and could not be built: {exc}") from exc
    lib = C.CDLL(path)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here == header/library mismatch: fail loudly
        fn.restype = res
        fn.argtypes = args
    if lib.b2_abi_version() != ABI_VERSION:
        raise RuntimeError("libb2gram.so ABI version mismatch")
    _lib = lib
    return lib


def last_error() -> str:
    return load().b2_last_error().decode("utf-8", "replace")


def _check(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError(f"{what} failed (code {rc}): {last_error()}")


def _check_args(rc: int, what: str) -> None:
    """``_check``, with the library's refusal of an argument (E_ARG) raised as ``ValueError``."""
    if rc == E_ARG:
        raise ValueError(last_error())
    _check(rc, what)


def device_count() -> int:
    n = C.c_int(0)
    rc = load().b2_device_count(C.byref(n))
    return int(n.value) if rc == 0 else 0


def pack_columns(columns) -> np.ndarray:
    """1-D host columns (all float64 or all float32, any stride) -> row-major float32 (n, d): ``b2_pack_columns``, the
    multi-threaded gather + conversion ``Context.upload_columns`` runs on the way to the device (host only, no GPU)."""
    cols = [np.asarray(c) for c in columns]
    if not cols or any(c.ndim != 1 or c.shape != cols[0].shape or c.dtype != cols[0].dtype for c in cols) \
            or cols[0].dtype not in (np.dtype(np.float64), np.dtype(np.float32)):
        raise RuntimeError("pack_columns: 1-D columns of one length and one dtype (float64 or float32) expected")
    n, d = int(cols[0].shape[0]), len(cols)
    out = np.empty((n, d), dtype=np.float32)
    ptrs = (C.c_void_p * d)(*[c.ctypes.data for c in cols])
    strides = (C.c_int64 * d)(*[c.strides[0] if n > 1 else c.itemsize for c in cols])
    _check(load().b2_pack_columns(C.cast(ptrs, C.c_void_p), C.cast(strides, C.c_void_p),
                                  F64 if cols[0].dtype == np.float64 else F32, n, d, out.ctypes.data), "b2_pack_columns")
    return out


def to_bf16_bits(a: np.ndarray) -> np.ndarray:
    """float32 -> bfloat16 bit patterns (uint16), round-to-nearest-even."""
    u = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)
    rounded = u + (np.uint32(0x7FFF) + ((u >> np.uint32(16)) & np.uint32(1)))
    return (rounded >> np.uint32(16)).astype(np.uint16)


def from_bf16_bits(b: np.ndarray) -> np.ndarray:
    return (b.astype(np.uint32) << np.uint32(16)).view(np.float32)


class DeviceArray:
    """A caller-owned HBM buffer: pointer + shape + element kind ('f32' | 'bf16' | 'u8' | 'f64')."""
    _ITEM = {"f32": 4, "bf16": 2, "u8": 1, "f64": 8}
    _NP = {"f32": np.float32, "bf16": np.uint16, "u8": np.uint8, "f64": np.float64}

    def __init__(self, ctx: "Context", shape: Tuple[int, ...], kind: str):
        self.ctx, self.shape, self.kind = ctx, tuple(int(s) for s in shape), kind
        self.nbytes = int(np.prod(self.shape, dtype=np.int64)) * self._ITEM[kind]
        p = _vp()
        _check(load().b2_dev_alloc(ctx._h, max(self.nbytes, 1), C.byref(p)), "b2_dev_alloc")
        self.ptr = p.value

    def copy_from(self, host: np.ndarray) -> "DeviceArray":
        host = np.ascontiguousarray(host, dtype=self._NP[self.kind])
        assert host.nbytes == self.nbytes, (host.nbytes, self.nbytes)
        _check(load().b2_copy_h2d(self.ctx._h, self.ptr, host.ctypes.data, self.nbytes), "b2_copy_h2d")
        return self

    def to_host(self) -> np.ndarray:
        out = np.empty(self.shape, dtype=self._NP[self.kind])
        _check(load().b2_copy_d2h(self.ctx._h, out.ctypes.data, self.ptr, self.nbytes), "b2_copy_d2h")
        return out

    def free(self) -> None:
        if self.ptr:
            load().b2_dev_free(self.ctx._h, self.ptr)
            self.ptr = None

    def __del__(self):  # best effort
        try:
            if self.ptr and self.ctx._h:
                self.free()
        except Exception:
            pass


class PinnedArray:
    """Pinned host memory exposed as a numpy array (for B2_MEM_HOST streaming)."""

    def __init__(self, ctx: "Context", shape, dtype):
        self.ctx = ctx
        dtype = np.dtype(dtype)
        nbytes = int(np.prod(shape, dtype=np.int64)) * dtype.itemsize
        p = _vp()
        _check(load().b2_host_alloc(ctx._h, max(nbytes, 1), C.byref(p)), "b2_host_alloc")
        self.ptr = p.value
        buf = (C.c_char * max(nbytes, 1)).from_address(self.ptr)
        self.array = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape, dtype=np.int64))).reshape(shape)

    def free(self) -> None:
        if self.ptr:
            self.array = None
            load().b2_host_free(self.ctx._h, self.ptr)
            self.ptr = None


def _x_kind(X) -> Tuple[int, int, int, int, int]:
    """(ptr, x_dtype, mem_kind, n, d) of a DeviceArray or a host ndarray (float32 / uint16-as-bf16)."""
    if isinstance(X, DeviceArray):
        if X.kind not in ("f32", "bf16"):
            raise RuntimeError("X must be f32 or bf16")
        n, d = X.shape
        return X.ptr, (F32 if X.kind == "f32" else BF16), MEM_DEVICE, n, d
    if not isinstance(X, np.ndarray) or X.ndim != 2 or not X.flags.c_contiguous:
        raise RuntimeError("host X must be a C-contiguous 2-D ndarray")
    if X.dtype == np.float32:
        return X.ctypes.data, F32, MEM_HOST, X.shape[0], X.shape[1]
    if X.dtype == np.uint16:
        return X.ctypes.data, BF16, MEM_HOST, X.shape[0], X.shape[1]
    raise RuntimeError(f"host X must be float32 (or uint16 bf16 bits), got {X.dtype}")


def _vec_ptr(v, kind: str, mem_kind: int, n: int, what: str) -> Optional[int]:
    if v is None:
        return None
    if isinstance(v, DeviceArray):
        if mem_kind != MEM_DEVICE or v.kind != kind or int(np.prod(v.shape)) != n:
            raise RuntimeError(f"{what}: device buffer of kind {kind} and length {n} expected")
        return v.ptr
    want = np.float32 if kind == "f32" else np.uint8
    if mem_kind != MEM_HOST or not isinstance(v, np.ndarray) or v.dtype != want or v.size != n \
            or not v.flags.c_contiguous:
        raise RuntimeError(f"{what}: contiguous host {want.__name__} array of length {n} expected")
    return v.ctypes.data


def _row_args(X, y, row_mask, mask_what: str = "row_mask"):
    """(ptr, x_dtype, mem_kind, n, d, y_ptr, mask_ptr) of rows, their f32 targets and their u8 mask (either may be
    None), all three where X lives."""
    ptr, xdt, mk, n, d = _x_kind(X)
    return ptr, xdt, mk, n, d, _vec_ptr(y, "f32", mk, n, "y"), _vec_ptr(row_mask, "u8", mk, n, mask_what)


class Context:
    """One GPU: streams, the fp64 statistic S, scratch, (optionally) one NCCL communicator."""

    def __init__(self, device: int = 0):
        self._h = None
        h = _vp()
        _check(load().b2_ctx_create(int(device), C.byref(h)), "b2_ctx_create")
        self._h = h.value
        self.device = int(device)
        self.d = 0
        self.serial = 0      # bumped whenever the resident statistic S changes owner / content (estimators check it)

    # -- lifecycle -----------------------------------------------------------------------------
    def close(self) -> None:
        if self._h:
            load().b2_ctx_destroy(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def sync(self) -> None:
        _check(load().b2_ctx_sync(self._h), "b2_ctx_sync")

    def info(self) -> dict:
        name = C.create_string_buffer(128)
        sm, hbm = C.c_int(0), C.c_size_t(0)
        _check(load().b2_ctx_info(self._h, name, 128, C.byref(sm), C.byref(hbm)), "b2_ctx_info")
        return {"name": name.value.decode(), "sm_count": sm.value, "hbm_bytes": hbm.value}

    def set_kernel(self, kernel: int) -> None:
        _check(load().b2_ctx_set_kernel(self._h, int(kernel)), "b2_ctx_set_kernel")

    def set_precision(self, precision: int) -> None:
        """PRECISION_SPLIT (default, bf16 hi+lo operands) or PRECISION_BF16 (single bf16 operand, 'bf16-accum')."""
        _check(load().b2_ctx_set_precision(self._h, int(precision)), "b2_ctx_set_precision")

    def set_sm_limit(self, n_sms: int) -> None:
        _check(load().b2_ctx_set_sm_limit(self._h, int(n_sms)), "b2_ctx_set_sm_limit")

    def set_drain_rows(self, rows: int) -> None:
        _check(load().b2_ctx_set_drain_rows(self._h, int(rows)), "b2_ctx_set_drain_rows")

    # -- buffers ----------------------------------------------------------------------------------
    def empty(self, shape, kind: str) -> DeviceArray:
        return DeviceArray(self, tuple(np.atleast_1d(shape)), kind)

    def to_device(self, host: np.ndarray, kind: Optional[str] = None) -> DeviceArray:
        if kind is None:
            kind = {np.dtype(np.float32): "f32", np.dtype(np.uint16): "bf16", np.dtype(np.uint8): "u8",
                    np.dtype(np.float64): "f64"}[host.dtype]
        return DeviceArray(self, host.shape, kind).copy_from(host)

    def upload_columns(self, columns) -> DeviceArray:
        """1-D host columns (all float64 or all float32, any stride -- what ``DataFrame[c].to_numpy()`` returns) -> a
        row-major float32 (n, d) DeviceArray: gathered, converted and copied by ``b2_upload_columns`` (host threads + a
        pinned ring), without the transposing copy / conversion passes of ``DataFrame.to_numpy``."""
        cols = [np.asarray(c) for c in columns]
        if not cols or any(c.ndim != 1 or c.shape != cols[0].shape or c.dtype != cols[0].dtype for c in cols) \
                or cols[0].dtype not in (np.dtype(np.float64), np.dtype(np.float32)):
            raise RuntimeError("upload_columns: 1-D columns of one length and one dtype (float64 or float32) expected")
        n, d = int(cols[0].shape[0]), len(cols)
        out = DeviceArray(self, (n, d), "f32")
        ptrs = (C.c_void_p * d)(*[c.ctypes.data for c in cols])
        strides = (C.c_int64 * d)(*[c.strides[0] if n > 1 else c.itemsize for c in cols])
        _check(load().b2_upload_columns(self._h, C.cast(ptrs, C.c_void_p), C.cast(strides, C.c_void_p),
                                        F64 if cols[0].dtype == np.float64 else F32, n, d, out.ptr), "b2_upload_columns")
        return out

    def copy_bandwidth_gbs(self, nbytes: int = 2 << 30, reps: int = 10) -> float:
        """This GPU's device-to-device copy bandwidth (read + write bytes per second, GB/s, best of ``reps``) -- the quantity
        bench.py reports next to the data-sheet figure."""
        a, b = DeviceArray(self, (nbytes,), "u8"), DeviceArray(self, (nbytes,), "u8")
        try:
            _check(load().b2_dev_memset(self._h, a.ptr, 1, nbytes), "b2_dev_memset")
            best = 0.0
            for _ in range(reps + 2):
                self.sync(); self.timer_start()
                _check(load().b2_copy_d2d(self._h, b.ptr, a.ptr, nbytes), "b2_copy_d2d")
                ms = self.timer_stop()
                best = max(best, 2.0 * nbytes / (ms * 1e-3) / 1e9)
            return best
        finally:
            a.free(); b.free()

    def pinned(self, shape, dtype) -> PinnedArray:
        return PinnedArray(self, tuple(np.atleast_1d(shape)), dtype)

    def _out(self, mem_kind: int, shape, kind: str, want: bool = True):
        """(buffer, pointer) of an output the library fills, where the rows live: a ``DeviceArray`` of ``kind`` (f64 /
        f32) for device rows, a numpy array otherwise; (None, None) unless ``want``."""
        if not want:
            return None, None
        if mem_kind == MEM_DEVICE:
            a = self.empty(shape, kind)
            return a, a.ptr
        a = np.empty(shape, dtype=DeviceArray._NP[kind])
        return a, a.ctypes.data

    # -- Gram ----------------------------------------------------------------------------------------
    def gram_reset(self, d: int) -> None:
        _check(load().b2_gram_reset(self._h, int(d)), "b2_gram_reset")
        self.d = int(d)
        self.serial += 1

    def gram_accumulate(self, X, y, row_mask=None, mask_keep: int = 1) -> None:
        ptr, xdt, mk, n, d, yp, mp = _row_args(X, y, row_mask)
        if self.d == 0:
            self.gram_reset(d)
        self.serial += 1
        _check(load().b2_gram_accumulate(self._h, ptr, xdt, yp, n, d, d, mk, mp, int(mask_keep)),
               "b2_gram_accumulate")

    def gram_allreduce(self) -> None:
        _check(load().b2_gram_allreduce(self._h), "b2_gram_allreduce")

    def gram_export(self) -> np.ndarray:
        S = np.empty((self.d + 2, self.d + 2), dtype=np.float64)
        n = _c_i64(0)
        _check(load().b2_gram_export(self._h, S.ctypes.data, C.byref(n)), "b2_gram_export")
        return S

    def gram_import(self, S: np.ndarray) -> None:
        S = np.ascontiguousarray(S, dtype=np.float64)
        d = S.shape[0] - 2
        _check(load().b2_gram_import(self._h, S.ctypes.data, d), "b2_gram_import")
        self.d = d
        self.serial += 1

    def fit(self, X, y, row_mask=None, mask_keep: int = 1, alpha: float = 0.0,
            fit_intercept: bool = True) -> Tuple[np.ndarray, float]:
        """The whole fit in one C call (b2_fit): reset + accumulate + all-reduce + solve.  Device-resident rows on the
        tensor-core path run as four launches (shift sample, Gram, finalize + peer scatter, gather + solve).  Raises ``np.linalg.LinAlgError`` on a rank-deficient Gram."""
        ptr, xdt, mk, n, d, yp, mp = _row_args(X, y, row_mask)
        coef = np.empty(d, dtype=np.float64)
        b0 = C.c_double(0.0)
        rc = load().b2_fit(self._h, ptr, xdt, yp, n, d, d, mk, mp, int(mask_keep), float(alpha),
                           int(bool(fit_intercept)), coef.ctypes.data, C.byref(b0))
        self.d = int(d)
        self.serial += 1
        if rc == E_SINGULAR:
            raise np.linalg.LinAlgError(last_error())
        _check(rc, "b2_fit")
        return coef, float(b0.value)

    def fit_refined(self, X, y, row_mask=None, mask_keep: int = 1, alpha: float = 0.0, fit_intercept: bool = True,
                    max_passes: int = 2, tol: float = 1e-10) -> Tuple[np.ndarray, float, int, float]:
        """``fit``, then up to ``max_passes`` residual passes over the same rows (b2_fit_refined): each pass reads the
        rows once for the fp64 gradient and corrects the solution through the factor of the Gram.  Returns (coef,
        intercept, passes kept, last step); the step is max_j |dcoef_j| sigma_j / sigma_y.  Raises
        ``np.linalg.LinAlgError`` on a rank-deficient Gram."""
        ptr, xdt, mk, n, d, yp, mp = _row_args(X, y, row_mask)
        coef = np.empty(d, dtype=np.float64)
        b0, step, passes = C.c_double(0.0), C.c_double(0.0), C.c_int(0)
        rc = load().b2_fit_refined(self._h, ptr, xdt, yp, n, d, d, mk, mp, int(mask_keep), float(alpha),
                                   int(bool(fit_intercept)), int(max_passes), float(tol), coef.ctypes.data, C.byref(b0),
                                   C.byref(passes), C.byref(step))
        self.d = int(d)
        self.serial += 1
        if rc == E_SINGULAR:
            raise np.linalg.LinAlgError(last_error())
        _check(rc, "b2_fit_refined")
        return coef, float(b0.value), int(passes.value), float(step.value)

    # -- solve -----------------------------------------------------------------------------------------
    def solve(self, alpha: float = 0.0, fit_intercept: bool = True) -> Tuple[np.ndarray, float]:
        """Cholesky solve; raises ``np.linalg.LinAlgError`` when the Gram matrix is rank deficient."""
        coef = np.empty(self.d, dtype=np.float64)
        b0 = C.c_double(0.0)
        rc = load().b2_solve(self._h, float(alpha), int(bool(fit_intercept)), coef.ctypes.data, C.byref(b0))
        if rc == E_SINGULAR:
            raise np.linalg.LinAlgError(last_error())
        _check(rc, "b2_solve")
        return coef, float(b0.value)

    def solve_spectral(self, cond: float = 1e-6, fit_intercept: bool = True):
        coef = np.empty(self.d, dtype=np.float64)
        sing = np.empty(self.d, dtype=np.float64)
        b0, rank = C.c_double(0.0), C.c_int(0)
        _check(load().b2_solve_spectral(self._h, float(cond), int(bool(fit_intercept)), coef.ctypes.data,
                                        C.byref(b0), sing.ctypes.data, C.byref(rank)), "b2_solve_spectral")
        return coef, float(b0.value), sing, int(rank.value)

    def solve_eigvals(self, cond: float = 1e-6, fit_intercept: bool = True):
        """(singular_, rank_, rows): sqrt of the eigenvalues of the centred Gram, descending (no eigenvectors)."""
        sing = np.empty(self.d, dtype=np.float64)
        rank, rows = C.c_int(0), _c_i64(0)
        _check(load().b2_solve_eigvals(self._h, float(cond), int(bool(fit_intercept)), sing.ctypes.data,
                                       C.byref(rank), C.byref(rows)), "b2_solve_eigvals")
        return sing, int(rank.value), int(rows.value)

    def solve_eigh(self, fit_intercept: bool = True) -> Tuple[np.ndarray, np.ndarray]:
        """(lambda, Q): eigenvalues (ascending, negative rounding values as 0) and orthonormal eigenvectors (column k for
        eigenvalue k) of the centred Gram (uncentred without an intercept) of the resident statistic."""
        lam = np.empty(self.d, dtype=np.float64)
        Q = np.empty((self.d, self.d), dtype=np.float64)
        _check(load().b2_solve_eigh(self._h, int(bool(fit_intercept)), lam.ctypes.data, Q.ctypes.data), "b2_solve_eigh")
        return lam, Q

    def solve_enet_path(self, l1_ratio: float = 1.0, alphas=None, n_alphas: int = 100, eps: float = 1e-3,
                        max_iter: int = 1000, tol: float = 1e-4, positive: bool = False, coef_init=None,
                        fit_intercept: bool = True) -> dict:
        """The elastic-net path of the resident statistic in one launch (b2_solve_enet_path): coordinate descent on the
        centred Gram, as sklearn's enet_path(precompute=Gram).  ``alphas``: None for sklearn's grid of ``n_alphas``
        values, else the alphas in the order they are solved.  Returns a dict of numpy arrays: alphas, coefs
        (n_alphas, d), intercepts, gaps (dual gap / n), n_iter, and the scalar tol (tol ||yc||^2 / n).  Raises
        ``ValueError`` for bad arguments and for a statistic without rows."""
        d = self.d
        al = None
        if alphas is not None:
            al = np.ascontiguousarray(np.asarray(alphas, dtype=np.float64).ravel())
            n_alphas = al.size
        ci = None
        if coef_init is not None:
            ci = np.ascontiguousarray(np.asarray(coef_init, dtype=np.float64).ravel())
            if ci.size != d:
                raise ValueError(f"coef_init has {ci.size} entries, the statistic has {d} features")
        n_alphas = int(n_alphas)
        k = max(n_alphas, 1)
        out = {"alphas": np.empty(k), "coefs": np.empty((k, d)), "intercepts": np.empty(k), "gaps": np.empty(k),
               "n_iter": np.empty(k, dtype=np.int32)}
        tol_out = C.c_double(0.0)
        rc = load().b2_solve_enet_path(self._h, int(bool(fit_intercept)), float(l1_ratio),
                                       al.ctypes.data if al is not None else None, n_alphas, float(eps), int(max_iter),
                                       float(tol), int(bool(positive)), ci.ctypes.data if ci is not None else None,
                                       out["alphas"].ctypes.data, out["coefs"].ctypes.data,
                                       out["intercepts"].ctypes.data, out["gaps"].ctypes.data,
                                       out["n_iter"].ctypes.data, C.byref(tol_out))
        _check_args(rc, "b2_solve_enet_path")
        out["tol"] = float(tol_out.value)
        return out

    def gram_folds(self, X, y, fold_of_row, n_folds: int) -> np.ndarray:
        """The statistic of every fold in one call (b2_gram_folds): row r belongs to fold ``fold_of_row[r]`` (uint8, where
        X lives; ids >= n_folds drop the row).  Leaves S = the sum of the folds resident and the fold statistics in the
        context for ``solve_enet_cv``; returns them, (n_folds, d + 2, d + 2)."""
        ptr, xdt, mk, n, d, yp, fp = _row_args(X, y, fold_of_row, "fold_of_row")
        out = np.empty((int(n_folds), d + 2, d + 2), dtype=np.float64)
        self.serial += 1
        rc = load().b2_gram_folds(self._h, ptr, xdt, yp, n, d, d, mk, fp, int(n_folds), out.ctypes.data)
        _check_args(rc, "b2_gram_folds")
        self.d = d
        return out

    def solve_enet_cv(self, n_folds: int, l1_ratios=(1.0,), alphas=None, n_alphas: int = 100, eps: float = 1e-3,
                      max_iter: int = 1000, tol: float = 1e-4, positive: bool = False, fit_intercept: bool = True,
                      fold_S=None, want_coefs: bool = False) -> dict:
        """Every (l1_ratio, fold) path of a cross-validation and its held-out error in one launch (b2_solve_enet_cv), on
        the fold statistics of the last ``gram_folds`` or on ``fold_S`` ((n_folds, d + 2, d + 2), uploaded; S becomes
        their sum).  ``alphas``: None for sklearn's grid of the summed statistic per l1_ratio, else the alphas in the
        order they are solved, shared by every l1_ratio.  Returns a dict of numpy arrays: alphas (n_l1, n_alphas),
        mse (n_l1, n_alphas, n_folds), n_iter and gaps (n_l1, n_folds, n_alphas) and, with ``want_coefs``, coefs
        (n_l1, n_folds, n_alphas, d).  Raises ``ValueError`` for bad arguments."""
        l1 = np.ascontiguousarray(np.atleast_1d(np.asarray(l1_ratios, dtype=np.float64)).ravel())
        al = None
        if alphas is not None:
            al = np.ascontiguousarray(np.asarray(alphas, dtype=np.float64).ravel())
            n_alphas = al.size
        fs = None
        if fold_S is not None:
            fs = np.ascontiguousarray(np.asarray(fold_S, dtype=np.float64))
            if fs.ndim != 3 or fs.shape[0] != int(n_folds) or fs.shape[1] != fs.shape[2] or fs.shape[1] < 3:
                raise ValueError(f"fold_S must have shape ({int(n_folds)}, d + 2, d + 2), got {fs.shape}")
            if self.d != fs.shape[1] - 2:
                self.gram_reset(fs.shape[1] - 2)
            self.serial += 1
        d, L, K, A = self.d, l1.size, int(n_folds), max(int(n_alphas), 1)
        out = {"alphas": np.empty((L, A)), "mse": np.empty((L, A, K)), "n_iter": np.empty((L, K, A), dtype=np.int32),
               "gaps": np.empty((L, K, A))}
        if want_coefs:
            out["coefs"] = np.empty((L, K, A, d))
        rc = load().b2_solve_enet_cv(self._h, fs.ctypes.data if fs is not None else None, K, int(bool(fit_intercept)),
                                     l1.ctypes.data if L else None, L, al.ctypes.data if al is not None else None,
                                     int(n_alphas), float(eps), int(max_iter), float(tol), int(bool(positive)),
                                     out["alphas"].ctypes.data, out["mse"].ctypes.data, out["n_iter"].ctypes.data,
                                     out["gaps"].ctypes.data, out["coefs"].ctypes.data if want_coefs else None)
        _check_args(rc, "b2_solve_enet_cv")
        return out

    def ridge_loo(self, X, y, alphas, row_mask=None, mask_keep: int = 1, fit_intercept: bool = True,
                  store_cv: bool = False):
        """RidgeCV(alphas).fit's leave-one-out search in one call (b2_ridge_loo): returns (mse per alpha, index of the
        first smallest, coef, intercept at that alpha, cv) where cv is None or the (n, n_alphas) e^2 per row and alpha
        (NaN on rows not kept) -- a float64 ndarray for host rows, an f64 DeviceArray for device rows.  Up to MAX_ALPHAS
        alphas per call."""
        ptr, xdt, mk, n, d, yp, mp = _row_args(X, y, row_mask)
        al = np.ascontiguousarray(np.asarray(alphas, dtype=np.float64).ravel())
        mse = np.empty(max(al.size, 1), dtype=np.float64)
        coef = np.empty(d, dtype=np.float64)
        b0, best = C.c_double(0.0), C.c_int(0)
        cv, cv_ptr = self._out(mk, (n, al.size), "f64", store_cv)
        rc = load().b2_ridge_loo(self._h, ptr, xdt, yp, n, d, d, mk, mp, int(mask_keep), al.ctypes.data, int(al.size),
                                 int(bool(fit_intercept)), mse.ctypes.data, cv_ptr, C.byref(best), coef.ctypes.data,
                                 C.byref(b0))
        self.d = int(d)
        self.serial += 1
        _check(rc, "b2_ridge_loo")
        return mse[: al.size], int(best.value), coef, float(b0.value), cv

    def _f64_coef(self, coef, d: int) -> np.ndarray:
        w = np.ascontiguousarray(coef, dtype=np.float64).ravel()
        if w.size != d:
            raise ValueError(f"coef has {w.size} entries, X has {d} columns")
        return w

    # -- BayesianRidge / ARDRegression (DESIGN.md section 9) ---------------------------------------------------
    def residual_moments(self, X, y, coef, intercept: float, row_mask=None, mask_keep: int = 1,
                         fit_intercept: bool = True) -> np.ndarray:
        """One fp64 pass over the kept rows at (coef, intercept) (b2_residual_moments): returns the d + 2 values
        [sum (x - m) e, sum e, sum e^2], e = y - intercept - x.coef, m the column means of the resident statistic (0
        without an intercept).  [coef, result] is the anchor of ``solve_bayes_ridge`` / ``solve_ard``."""
        ptr, xdt, mk, n, d, yp, mp = _row_args(X, y, row_mask)
        w = self._f64_coef(coef, d)
        out = np.empty(d + 2, dtype=np.float64)
        _check(load().b2_residual_moments(self._h, ptr, xdt, yp, n, d, d, mk, mp, int(mask_keep), w.ctypes.data,
                                          float(intercept), int(bool(fit_intercept)), out.ctypes.data),
               "b2_residual_moments")
        return out

    def _bayes_call(self, fn, what: str, args_before, ard: bool, max_iter: int, anchor, compute_score: bool,
                    fit_intercept: bool, want_sigma: bool) -> dict:
        d = self.d
        n_lambda = d if ard else 1
        an = None
        if anchor is not None:
            an = np.ascontiguousarray(anchor, dtype=np.float64).ravel()
            if an.size != 2 * d + 2:
                raise ValueError(f"anchor has {an.size} entries, {2 * d + 2} expected")
        coef = np.empty(d, dtype=np.float64)
        lam = np.empty(n_lambda, dtype=np.float64)
        b0, alpha, n_iter = C.c_double(0.0), C.c_double(0.0), C.c_int(0)
        scores = np.empty(max(int(max_iter), 0) + 1, dtype=np.float64) if compute_score else None
        sigma = np.empty((d, d), dtype=np.float64) if want_sigma else None
        rc = fn(self._h, int(bool(fit_intercept)), *args_before, an.ctypes.data if an is not None else None,
                int(bool(compute_score)), coef.ctypes.data, C.byref(b0), C.byref(alpha), lam.ctypes.data,
                C.byref(n_iter), scores.ctypes.data if scores is not None else None,
                sigma.ctypes.data if sigma is not None else None)
        if rc == E_SINGULAR:
            raise np.linalg.LinAlgError(last_error())
        _check_args(rc, what)
        k = int(n_iter.value)
        return {"coef": coef, "intercept": float(b0.value), "alpha": float(alpha.value),
                "lambda": lam if ard else float(lam[0]), "n_iter": k,
                "scores": scores[: k if ard else k + 1] if scores is not None else None, "sigma": sigma}

    def solve_bayes_ridge(self, alpha_1: float = 1e-6, alpha_2: float = 1e-6, lambda_1: float = 1e-6,
                          lambda_2: float = 1e-6, alpha_init=None, lambda_init=None, max_iter: int = 300,
                          tol: float = 1e-3, anchor=None, compute_score: bool = False, fit_intercept: bool = True,
                          want_sigma: bool = True) -> dict:
        """BayesianRidge's evidence maximisation on the resident statistic (b2_solve_bayes_ridge).  ``anchor``: None or
        [w0 (d), g0 (d), s0, sse0] (w0 and ``residual_moments`` at w0).  Returns a dict: coef, intercept, alpha, lambda,
        n_iter, scores (n_iter + 1 values with compute_score, else None) and sigma (d, d).  Raises ``ValueError`` for bad
        arguments and a statistic without rows."""
        nan = float("nan")
        hyper = np.array([alpha_1, alpha_2, lambda_1, lambda_2, nan if alpha_init is None else alpha_init,
                          nan if lambda_init is None else lambda_init], dtype=np.float64)
        return self._bayes_call(load().b2_solve_bayes_ridge, "b2_solve_bayes_ridge",
                                (hyper.ctypes.data, int(max_iter), float(tol)), False, max_iter, anchor, compute_score,
                                fit_intercept, want_sigma)

    def solve_ard(self, alpha_1: float = 1e-6, alpha_2: float = 1e-6, lambda_1: float = 1e-6, lambda_2: float = 1e-6,
                  threshold_lambda: float = 1e4, max_iter: int = 300, tol: float = 1e-3, anchor=None,
                  compute_score: bool = False, fit_intercept: bool = True, want_sigma: bool = True) -> dict:
        """ARDRegression's iteration on the resident statistic (b2_solve_ard).  Returns ``solve_bayes_ridge``'s dict with
        lambda per feature, n_iter scores and sigma (d, d): the kept x kept sigma_ at the kept rows and columns, zeros elsewhere.
        Raises ``np.linalg.LinAlgError`` on a non-positive pivot."""
        hyper = np.array([alpha_1, alpha_2, lambda_1, lambda_2], dtype=np.float64)
        return self._bayes_call(load().b2_solve_ard, "b2_solve_ard",
                                (hyper.ctypes.data, float(threshold_lambda), int(max_iter), float(tol)), True,
                                max_iter, anchor, compute_score, fit_intercept, want_sigma)

    def score_std(self, X, mean, sigma, noise_var: float, coef, intercept: float, want_yhat: bool = True):
        """predict(X, return_std=True) of BayesianRidge / ARDRegression in one fp64 pass (b2_score_std): returns (yhat |
        None, ystd), ystd = sqrt(max((x - mean)^T sigma (x - mean), 0) + noise_var) -- float64 ndarrays for host rows,
        f64 DeviceArrays for device rows."""
        ptr, xdt, mk, n, d = _x_kind(X)
        w = np.ascontiguousarray(coef, dtype=np.float64).ravel()
        m = np.ascontiguousarray(mean, dtype=np.float64).ravel() if mean is not None else None
        sg = np.ascontiguousarray(sigma, dtype=np.float64)
        if w.size != d or sg.shape != (d, d) or (m is not None and m.size != d):
            raise ValueError(f"coef / mean need {d} entries and sigma shape ({d}, {d})")
        ystd, sp = self._out(mk, (n,), "f64")
        yhat, hp = self._out(mk, (n,), "f64", want_yhat)
        rc = load().b2_score_std(self._h, ptr, xdt, n, d, d, mk, m.ctypes.data if m is not None else None,
                                 sg.ctypes.data, float(noise_var), w.ctypes.data, float(intercept), hp, sp)
        _check_args(rc, "b2_score_std")
        return yhat, ystd

    # -- PoissonRegressor / GammaRegressor / TweedieRegressor (DESIGN.md section 10) --------------------------------
    def glm_pass(self, X, y, coef, intercept: float, *, link: int = GLM_LOG, power: float = 1.0, row_mask=None,
                 mask_keep: int = 1, fit_intercept: bool = True, hessian: bool = True) -> dict:
        """One pass of the Newton solver's statistics at (coef, intercept) over the kept rows (b2_glm_pass).  Returns
        a dict of unscaled sums: loss, const (constant_to_optimal_zero), sum_y, kept, y_out_of_range, h_nonpos,
        y_nonfinite (floats), grad ((d + 1,): sum g x_j, then sum g) and hessian ((d + 1, d + 1) sum |h| [x 1][x 1]^T,
        or None without ``hessian``).  Raises ``ValueError`` for bad arguments."""
        ptr, xdt, mk, n, d, yp, mp = _row_args(X, y, row_mask)
        w = self._f64_coef(coef, d)
        sums = np.empty(d + 8, dtype=np.float64)
        hess = np.empty((d + 1, d + 1), dtype=np.float64) if hessian else None
        rc = load().b2_glm_pass(self._h, ptr, xdt, yp, n, d, d, mk, mp, int(mask_keep), int(link), float(power),
                                w.ctypes.data, float(intercept), int(bool(fit_intercept)), sums.ctypes.data,
                                hess.ctypes.data if hess is not None else None)
        _check_args(rc, "b2_glm_pass")
        keys = ("loss", "const", "sum_y", "kept", "y_out_of_range", "h_nonpos", "y_nonfinite")
        out = {k: float(sums[i]) for i, k in enumerate(keys)}
        out["grad"] = sums[7:].copy()
        out["hessian"] = hess
        return out

    def glm_line_search(self, X, y, coef, intercept: float, step, step_intercept: float, *, link: int = GLM_LOG,
                        power: float = 1.0, n_steps: int = GLM_STEPS, row_mask=None, mask_keep: int = 1) -> np.ndarray:
        """The backtracking ladder in one pass (b2_glm_line_search): the summed loss over the kept rows at
        (coef, intercept) + 2^-k (step, step_intercept) for k < n_steps."""
        ptr, xdt, mk, n, d, yp, mp = _row_args(X, y, row_mask)
        w, s = self._f64_coef(coef, d), self._f64_coef(step, d)
        out = np.empty(max(int(n_steps), 1), dtype=np.float64)
        rc = load().b2_glm_line_search(self._h, ptr, xdt, yp, n, d, d, mk, mp, int(mask_keep), int(link), float(power),
                                       w.ctypes.data, float(intercept), s.ctypes.data, float(step_intercept),
                                       int(n_steps), out.ctypes.data)
        _check_args(rc, "b2_glm_line_search")
        return out

    def glm_predict(self, X, coef, intercept: float, *, link: int = GLM_LOG):
        """mu = exp(X coef + intercept) (GLM_LOG) or X coef + intercept per row in fp64 (b2_glm_predict): a float64
        ndarray for host rows, an f64 DeviceArray for device rows."""
        ptr, xdt, mk, n, d = _x_kind(X)
        w = self._f64_coef(coef, d)
        mu, mu_ptr = self._out(mk, (n,), "f64")
        rc = load().b2_glm_predict(self._h, ptr, xdt, n, d, d, mk, int(link), w.ctypes.data, float(intercept), mu_ptr)
        _check_args(rc, "b2_glm_predict")
        return mu

    # -- LogisticRegression, binary (DESIGN.md section 11) ----------------------------------------------------------
    def logistic_pass(self, X, y, coef, intercept: float, neg_label: float = 0.0, pos_label: float = 1.0, *,
                      row_mask=None, mask_keep: int = 1, fit_intercept: bool = True, hessian: bool = True) -> dict:
        """One pass of the Newton solver's statistics for HalfBinomialLoss at (coef, intercept) over the kept rows
        (b2_logistic_pass); y holds the labels as stored, the target is 1 where y == pos_label and 0 where y == neg_label.
        Returns ``glm_pass``'s dict (sum_y: the positive rows, y_out_of_range: the rows with neither label) and correct:
        the rows classified correctly by the sign of eta.  Raises ``ValueError`` for bad arguments."""
        ptr, xdt, mk, n, d, yp, mp = _row_args(X, y, row_mask)
        w = self._f64_coef(coef, d)
        sums = np.empty(d + 9, dtype=np.float64)
        hess = np.empty((d + 1, d + 1), dtype=np.float64) if hessian else None
        rc = load().b2_logistic_pass(self._h, ptr, xdt, yp, n, d, d, mk, mp, int(mask_keep), float(neg_label),
                                     float(pos_label), w.ctypes.data, float(intercept), int(bool(fit_intercept)),
                                     sums.ctypes.data, hess.ctypes.data if hess is not None else None)
        _check_args(rc, "b2_logistic_pass")
        keys = ("loss", "const", "sum_y", "kept", "y_out_of_range", "h_nonpos", "y_nonfinite")
        out = {k: float(sums[i]) for i, k in enumerate(keys)}
        out["grad"] = sums[7:8 + d].copy()
        out["correct"] = float(sums[8 + d])
        out["hessian"] = hess
        return out

    def logistic_line_search(self, X, y, coef, intercept: float, step, step_intercept: float, neg_label: float = 0.0,
                             pos_label: float = 1.0, *, n_steps: int = GLM_STEPS, row_mask=None,
                             mask_keep: int = 1) -> np.ndarray:
        """The backtracking ladder of a logistic Newton step in one pass (b2_logistic_line_search)."""
        ptr, xdt, mk, n, d, yp, mp = _row_args(X, y, row_mask)
        w, s = self._f64_coef(coef, d), self._f64_coef(step, d)
        out = np.empty(max(int(n_steps), 1), dtype=np.float64)
        rc = load().b2_logistic_line_search(self._h, ptr, xdt, yp, n, d, d, mk, mp, int(mask_keep), float(neg_label),
                                            float(pos_label), w.ctypes.data, float(intercept), s.ctypes.data,
                                            float(step_intercept), int(n_steps), out.ctypes.data)
        _check_args(rc, "b2_logistic_line_search")
        return out

    def logistic_predict(self, X, coef, intercept: float, neg_label: float = 0.0, pos_label: float = 1.0, *,
                         decision: bool = False, proba: bool = False, label: bool = False) -> dict:
        """The logistic model per row in one pass (b2_logistic_predict): the wanted ones of decision (eta, fp64), proba
        ((n, 2) [1 - p, p], fp64) and label (pos_label where eta > 0, else neg_label; fp32) -- ndarrays for host rows,
        DeviceArrays for device rows."""
        ptr, xdt, mk, n, d = _x_kind(X)
        w = self._f64_coef(coef, d)
        out, ptrs = {}, {}
        for name, want, shape, kind in (("decision", decision, (n,), "f64"), ("proba", proba, (n, 2), "f64"),
                                        ("label", label, (n,), "f32")):
            a, ptrs[name] = self._out(mk, shape, kind, want)
            if want:
                out[name] = a
        rc = load().b2_logistic_predict(self._h, ptr, xdt, n, d, d, mk, w.ctypes.data, float(intercept),
                                        float(neg_label), float(pos_label), ptrs["decision"], ptrs["proba"],
                                        ptrs["label"])
        _check_args(rc, "b2_logistic_predict")
        return out

    def label_scan(self, y, row_mask=None, mask_keep: int = 1) -> dict:
        """The labels of an f32 DeviceArray y over the kept rows (b2_label_scan): kept, nonfinite, nonintegral (finite y
        != rint(y)), min and max of the finite kept y (NaN without any), n_min and n_max (kept rows equal to each)."""
        if not isinstance(y, DeviceArray) or y.kind != "f32":
            raise RuntimeError("label_scan: y must be an f32 DeviceArray")
        n = int(np.prod(y.shape))
        mp = _vec_ptr(row_mask, "u8", MEM_DEVICE, n, "row_mask")
        st = np.empty(7, dtype=np.float64)
        rc = load().b2_label_scan(self._h, y.ptr, n, mp, int(mask_keep), st.ctypes.data)
        _check_args(rc, "b2_label_scan")
        return dict(zip(("kept", "nonfinite", "nonintegral", "min", "max", "n_min", "n_max"), st.tolist()))

    # -- RidgeClassifier (DESIGN.md section 12) -----------------------------------------------------------------------
    @staticmethod
    def _f32_classes(classes, k: int) -> np.ndarray:
        c = np.ascontiguousarray(classes, dtype=np.float32).ravel()
        if c.size != k:
            raise ValueError(f"{k} classes expected, got {c.size}")
        return c

    def class_sums(self, X, y, classes, center=None, *, row_mask=None, mask_keep: int = 1) -> dict:
        """One pass over the kept rows for the class sums of a ridge classifier (b2_class_sums): ``classes`` are K sorted
        fp32 values and a row's class is the index of its y among them.  Returns sums ((K, d + 1): per class the sum of
        x - center over its rows, then their count), kept, unmatched (kept rows of no class, NaN included) and nonfinite
        (kept rows with y not finite).  ``center``: d values, None for zeros.  Raises ``ValueError`` for bad arguments."""
        ptr, xdt, mk, n, d, yp, mp = _row_args(X, y, row_mask)
        cl = self._f32_classes(classes, np.size(classes))
        c = None if center is None else self._f64_coef(center, d)
        sums = np.empty((cl.size, d + 1), dtype=np.float64)
        counts = np.empty(3, dtype=np.float64)
        rc = load().b2_class_sums(self._h, ptr, xdt, yp, n, d, d, mk, mp, int(mask_keep), cl.ctypes.data, cl.size,
                                  c.ctypes.data if c is not None else None, sums.ctypes.data, counts.ctypes.data)
        _check_args(rc, "b2_class_sums")
        return {"sums": sums, "kept": float(counts[0]), "unmatched": float(counts[1]), "nonfinite": float(counts[2])}

    def class_scatter(self, X, y, classes, means, weights=None, *, row_mask=None, mask_keep: int = 1) -> dict:
        """The pooled within-class scatter of the kept rows in one fp64 pass (b2_class_scatter): ``classes`` are K
        sorted fp32 values and a row's class is the index of its y among them, ``means`` the (K, d) class means and
        ``weights`` K class weights (None: all 1).  Returns scatter ((d, d): sum over the rows of class k of
        w_k (x - m_k)(x - m_k)^T, exactly symmetric), kept, unmatched (kept rows of no class, NaN included) and nonfinite
        (kept rows with y not finite).  Raises ``ValueError`` for bad arguments."""
        ptr, xdt, mk, n, d, yp, mp = _row_args(X, y, row_mask)
        cl = self._f32_classes(classes, np.size(classes))
        m = np.ascontiguousarray(means, dtype=np.float64)
        if m.shape != (cl.size, d):
            raise ValueError(f"means must be ({cl.size}, {d}), got {m.shape}")
        w = None if weights is None else np.ascontiguousarray(weights, dtype=np.float64).ravel()
        if w is not None and w.size != cl.size:
            raise ValueError(f"weights has {w.size} entries, {cl.size} classes")
        scatter = np.empty((d, d), dtype=np.float64)
        counts = np.empty(3, dtype=np.float64)
        rc = load().b2_class_scatter(self._h, ptr, xdt, yp, n, d, d, mk, mp, int(mask_keep), cl.ctypes.data, cl.size,
                                     m.ctypes.data, w.ctypes.data if w is not None else None, scatter.ctypes.data,
                                     counts.ctypes.data)
        _check_args(rc, "b2_class_scatter")
        return {"scatter": scatter, "kept": float(counts[0]), "unmatched": float(counts[1]),
                "nonfinite": float(counts[2])}

    # -- QuadraticDiscriminantAnalysis (DESIGN.md section 17) ----------------------------------------------------------
    def class_scatters(self, X, y, classes, means, *, row_mask=None, mask_keep: int = 1) -> dict:
        """Every class's own scatter of the kept rows in one fp64 pass over the rows in class order (b2_class_scatters):
        ``classes`` are K sorted fp32 values and a row's class is the index of its y among them, ``means`` the (K, d)
        class means.  Returns scatters ((K, d, d): sum over the rows of class k of (x - m_k)(x - m_k)^T, exactly
        symmetric, zero for a class without rows), class_counts ((K,) kept rows per class), kept, unmatched (kept rows of
        no class, NaN included) and nonfinite (kept rows with y not finite).  Raises ``ValueError`` for bad arguments."""
        ptr, xdt, mk, n, d, yp, mp = _row_args(X, y, row_mask)
        cl = self._f32_classes(classes, np.size(classes))
        m = np.ascontiguousarray(means, dtype=np.float64)
        if m.shape != (cl.size, d):
            raise ValueError(f"means must be ({cl.size}, {d}), got {m.shape}")
        scatters = np.empty((cl.size, d, d), dtype=np.float64)
        nk = np.empty(cl.size, dtype=np.float64)
        counts = np.empty(3, dtype=np.float64)
        rc = load().b2_class_scatters(self._h, ptr, xdt, yp, n, d, d, mk, mp, int(mask_keep), cl.ctypes.data, cl.size,
                                      m.ctypes.data, scatters.ctypes.data, nk.ctypes.data, counts.ctypes.data)
        _check_args(rc, "b2_class_scatters")
        return {"scatters": scatters, "class_counts": nk, "kept": float(counts[0]), "unmatched": float(counts[1]),
                "nonfinite": float(counts[2])}

    def qda_decision(self, X, means, transforms, offsets, classes, y=None, *, row_mask=None, mask_keep: int = 1,
                     decision: bool = False, label: bool = False, diff: bool = False) -> dict:
        """The quadratic discriminant per row and class in one fp64 pass (b2_qda_decision):
        d_k = -1/2 |(x - m_k) W_k|^2 + c_k with ``means`` (K, d), ``transforms`` (K, d, d) and ``offsets`` (K,).  The
        wanted ones of decision ((n, K) fp64), label (classes[argmax_k d_k], the first largest; fp32) and diff (d_1 - d_0,
        two classes only; fp64) -- ndarrays for host rows, DeviceArrays for device rows -- and, with y, kept and correct
        (kept rows whose y equals their label)."""
        ptr, xdt, mk, n, d, yp, mp = _row_args(X, y, row_mask)
        cl = self._f32_classes(classes, np.size(classes))
        k = cl.size
        m = np.ascontiguousarray(means, dtype=np.float64)
        w = np.ascontiguousarray(transforms, dtype=np.float64)
        c = np.ascontiguousarray(offsets, dtype=np.float64).ravel()
        if m.shape != (k, d) or w.shape != (k, d, d) or c.size != k:
            raise ValueError(f"means, transforms and offsets must be ({k}, {d}), ({k}, {d}, {d}) and ({k},), got "
                             f"{m.shape}, {w.shape} and {c.shape}")
        out, ptrs = {}, {}
        for name, want, shape, kind in (("decision", decision, (n, k), "f64"), ("label", label, (n,), "f32"),
                                        ("diff", diff, (n,), "f64")):
            a, ptrs[name] = self._out(mk, shape, kind, want)
            if want:
                out[name] = a
        counts = np.zeros(2, dtype=np.float64) if y is not None else None
        rc = load().b2_qda_decision(self._h, ptr, xdt, yp, n, d, d, mk, mp, int(mask_keep), cl.ctypes.data, k,
                                    m.ctypes.data, w.ctypes.data, c.ctypes.data, ptrs["decision"], ptrs["label"],
                                    ptrs["diff"], counts.ctypes.data if counts is not None else None)
        _check_args(rc, "b2_qda_decision")
        if counts is not None:
            out["kept"], out["correct"] = float(counts[0]), float(counts[1])
        return out

    def solve_classes(self, class_sums, alpha: float = 1.0, fit_intercept: bool = True,
                      n_classes: Optional[int] = None) -> Tuple[np.ndarray, np.ndarray]:
        """(coef (T, d), intercept (T,)) of the ridge classifier of the resident statistic and the class sums
        (b2_solve_classes): ``class_sums`` the (K, d + 1) ``sums`` of ``class_sums``, or None for the context's last ones
        (then ``n_classes`` = K).  T = 1 for two classes, else K.  Raises ``np.linalg.LinAlgError`` when the LDL^T meets
        a non-positive pivot."""
        if class_sums is not None:
            cs = np.ascontiguousarray(class_sums, dtype=np.float64)
            if cs.ndim != 2 or cs.shape[1] != self.d + 1:
                raise ValueError(f"class_sums must be (K, {self.d + 1}), got {cs.shape}")
            k, cs_ptr = cs.shape[0], cs.ctypes.data
        else:
            k, cs_ptr = int(n_classes or 0), None
        t = 1 if k == 2 else max(k, 1)
        coef = np.empty((t, max(self.d, 1)), dtype=np.float64)
        b0 = np.empty(t, dtype=np.float64)
        rc = load().b2_solve_classes(self._h, float(alpha), int(bool(fit_intercept)), cs_ptr, k, coef.ctypes.data,
                                     b0.ctypes.data)
        if rc == E_SINGULAR:
            raise np.linalg.LinAlgError(last_error())
        _check_args(rc, "b2_solve_classes")
        return coef, b0

    def classify(self, X, coef, intercept, classes, y=None, *, row_mask=None, mask_keep: int = 1,
                 decision: bool = False, label: bool = False) -> dict:
        """The ridge classifier per row in one pass (b2_classify): eta = X coef^T + intercept for the T rows of coef.
        The wanted ones of decision ((n, T) fp64) and label (classes[argmax eta], the first largest; for T = 1
        classes[1] where eta > 0, else classes[0]; fp32) -- ndarrays for host rows, DeviceArrays for device rows -- and,
        with y, kept and correct (kept rows whose y equals their label)."""
        ptr, xdt, mk, n, d, yp, mp = _row_args(X, y, row_mask)
        w = np.ascontiguousarray(coef, dtype=np.float64)
        w = w.reshape(1, -1) if w.ndim == 1 else w
        if w.ndim != 2 or w.shape[1] != d:
            raise ValueError(f"coef must be (T, {d}), got {np.shape(coef)}")
        t = w.shape[0]
        b0 = np.ascontiguousarray(intercept, dtype=np.float64).ravel()
        if b0.size != t:
            raise ValueError(f"intercept has {b0.size} entries, coef {t} rows")
        cl = self._f32_classes(classes, max(t, 2))
        out, ptrs = {}, {}
        for name, want, shape, kind in (("decision", decision, (n, t), "f64"), ("label", label, (n,), "f32")):
            a, ptrs[name] = self._out(mk, shape, kind, want)
            if want:
                out[name] = a
        counts = np.zeros(2, dtype=np.float64) if y is not None else None
        rc = load().b2_classify(self._h, ptr, xdt, yp, n, d, d, mk, mp, int(mask_keep), w.ctypes.data, b0.ctypes.data,
                                t, cl.ctypes.data, ptrs["decision"], ptrs["label"],
                                counts.ctypes.data if counts is not None else None)
        _check_args(rc, "b2_classify")
        if counts is not None:
            out["kept"], out["correct"] = float(counts[0]), float(counts[1])
        return out

    def label_values(self, y, row_mask=None, mask_keep: int = 1, max_values: int = MAX_CLASSES):
        """(values, more): the distinct finite values of an f32 DeviceArray y over the kept rows, ascending (-0.0 as
        0.0), at most ``max_values`` of them, and whether there are more (b2_label_values)."""
        if not isinstance(y, DeviceArray) or y.kind != "f32":
            raise RuntimeError("label_values: y must be an f32 DeviceArray")
        n = int(np.prod(y.shape))
        mp = _vec_ptr(row_mask, "u8", MEM_DEVICE, n, "row_mask")
        vals = np.empty(max(int(max_values), 1), dtype=np.float32)
        found, more = C.c_int(0), C.c_int(0)
        rc = load().b2_label_values(self._h, y.ptr, n, mp, int(mask_keep), int(max_values), vals.ctypes.data,
                                    C.byref(found), C.byref(more))
        _check_args(rc, "b2_label_values")
        return vals[: found.value].copy(), bool(more.value)

    # -- LogisticRegression, multinomial (DESIGN.md section 14) ----------------------------------------------------
    @staticmethod
    def _f64_classes_coef(coef, k: int, d: int, what: str = "coef") -> np.ndarray:
        w = np.ascontiguousarray(coef, dtype=np.float64)
        if w.shape != (k, d + 1):
            raise ValueError(f"{what} must be ({k}, {d + 1}) (row k = [w_k, b_k]), got {w.shape}")
        return w

    def multinomial_pass(self, X, y, classes, coef, *, row_mask=None, mask_keep: int = 1, fit_intercept: bool = True,
                         hessian: bool = True) -> dict:
        """One pass of the Newton solver's statistics for HalfMultinomialLoss at coef ((K, d + 1), row k = [w_k, b_k])
        over the kept rows (b2_multinomial_pass); ``classes`` are K (3..MAX_CLASSES) sorted fp32 values and a row's class
        is the index of its y among them.  Returns a dict of unscaled sums: loss, kept, unmatched (kept rows of no class,
        NaN included), nonfinite (kept rows with y not finite), correct (kept rows whose first largest eta is their
        class), grad ((K, d + 1): sum g_k [x 1]) and hessian ((K, K, d + 1, d + 1) sum h_kl [x 1][x 1]^T, or None without
        ``hessian``).  Raises ``ValueError`` for bad arguments."""
        ptr, xdt, mk, n, d, yp, mp = _row_args(X, y, row_mask)
        cl = self._f32_classes(classes, np.size(classes))
        k = cl.size
        w = self._f64_classes_coef(coef, k, d)
        sums = np.empty(5 + k * (d + 1), dtype=np.float64)
        hess = np.empty((k, k, d + 1, d + 1), dtype=np.float64) if hessian else None
        rc = load().b2_multinomial_pass(self._h, ptr, xdt, yp, n, d, d, mk, mp, int(mask_keep), cl.ctypes.data, k,
                                        w.ctypes.data, int(bool(fit_intercept)), sums.ctypes.data,
                                        hess.ctypes.data if hess is not None else None)
        _check_args(rc, "b2_multinomial_pass")
        out = {key: float(sums[i]) for i, key in enumerate(("loss", "kept", "unmatched", "nonfinite", "correct"))}
        out["grad"] = sums[5:].reshape(k, d + 1).copy()
        out["hessian"] = hess
        return out

    def multinomial_line_search(self, X, y, classes, coef, step, *, n_steps: int = GLM_STEPS, row_mask=None,
                                mask_keep: int = 1) -> np.ndarray:
        """The backtracking ladder of a multinomial Newton step in one pass (b2_multinomial_line_search): the summed
        loss over the kept rows at coef + 2^-t step (both (K, d + 1)) for t < n_steps."""
        ptr, xdt, mk, n, d, yp, mp = _row_args(X, y, row_mask)
        cl = self._f32_classes(classes, np.size(classes))
        w = self._f64_classes_coef(coef, cl.size, d)
        s = self._f64_classes_coef(step, cl.size, d, "step")
        out = np.empty(max(int(n_steps), 1), dtype=np.float64)
        rc = load().b2_multinomial_line_search(self._h, ptr, xdt, yp, n, d, d, mk, mp, int(mask_keep), cl.ctypes.data,
                                               cl.size, w.ctypes.data, s.ctypes.data, int(n_steps), out.ctypes.data)
        _check_args(rc, "b2_multinomial_line_search")
        return out

    def softmax_rows(self, values) -> None:
        """Each row of a 2-D float64 array (an f64 ``DeviceArray`` or a C-contiguous ndarray) replaced in place by its
        softmax, as sklearn.utils.extmath.softmax computes it (b2_softmax_rows)."""
        if isinstance(values, DeviceArray):
            if values.kind != "f64" or len(values.shape) != 2:
                raise RuntimeError("softmax_rows: values must be a 2-D f64 DeviceArray")
            ptr, mk, (n, k) = values.ptr, MEM_DEVICE, values.shape
        else:
            if not isinstance(values, np.ndarray) or values.dtype != np.float64 or values.ndim != 2 \
                    or not values.flags.c_contiguous:
                raise RuntimeError("softmax_rows: host values must be a C-contiguous 2-D float64 ndarray")
            ptr, mk, (n, k) = values.ctypes.data, MEM_HOST, values.shape
        _check_args(load().b2_softmax_rows(self._h, ptr, int(n), int(k), mk), "b2_softmax_rows")

    # -- LinearSVC / LinearSVR (DESIGN.md section 15) ----------------------------------------------------------------
    def svm_pass(self, X, y, coef, intercept: float, *, loss: int = SVM_SQUARED_HINGE, param: float = 1.0,
                 coef_from=None, intercept_from: float = 0.0, row_mask=None, mask_keep: int = 1,
                 fit_intercept: bool = True, hessian: bool = True) -> dict:
        """One pass of liblinear's TRON statistics at the trial point (coef, intercept) over the kept rows (b2_svm_pass),
        ``param`` the positive label (SVM_SQUARED_HINGE) or epsilon (SVM_SQUARED_EPSILON).  Returns a dict of unscaled
        sums over the rows active at the trial point: loss, kept, active, entering and leaving (the rows that joined or
        left the active set since (coef_from, intercept_from); coef_from None: the empty set), positive (kept rows with
        y == param, squared hinge), y_nonfinite (floats), grad ((d + 1,): sum g [x 1]) and dhessian ((d + 1, d + 1)
        sum (active - active_from) [x 1][x 1]^T, or None without ``hessian``).  Raises ``ValueError`` for bad
        arguments."""
        ptr, xdt, mk, n, d, yp, mp = _row_args(X, y, row_mask)
        w = self._f64_coef(coef, d)
        wf = None if coef_from is None else self._f64_coef(coef_from, d)
        sums = np.empty(d + 8, dtype=np.float64)
        dh = np.empty((d + 1, d + 1), dtype=np.float64) if hessian else None
        rc = load().b2_svm_pass(self._h, ptr, xdt, yp, n, d, d, mk, mp, int(mask_keep), int(loss), float(param),
                                wf.ctypes.data if wf is not None else None, float(intercept_from), w.ctypes.data,
                                float(intercept), int(bool(fit_intercept)), sums.ctypes.data,
                                dh.ctypes.data if dh is not None else None)
        _check_args(rc, "b2_svm_pass")
        keys = ("loss", "kept", "active", "entering", "leaving", "positive", "y_nonfinite")
        out = {k: float(sums[i]) for i, k in enumerate(keys)}
        out["grad"] = sums[7:].copy()
        out["dhessian"] = dh
        return out

    # -- RidgeClassifierCV (DESIGN.md section 13) ------------------------------------------------------------------
    def ridge_classifier_loo(self, X, y, classes, alphas, row_mask=None, mask_keep: int = 1, *,
                             fit_intercept: bool = True, scoring: int = LOO_SQUARED, store_cv: bool = False) -> dict:
        """RidgeClassifierCV(alphas).fit's leave-one-out search in one call (b2_ridge_classifier_loo): ``classes`` are K
        sorted fp32 values (a row's class is the index of its y among them), up to MAX_ALPHAS alphas.  Returns a dict:
        mse and correct per alpha, best (the first smallest mse, or the first largest correct with LOO_ACCURACY), coef
        (T, d) and intercept (T,) at alphas[best] (T = 1 for two classes, else K), kept / unmatched / nonfinite (the
        class-sum pass's counts) and cv: None, or (n, T, n_alphas) e^2 (p = t - e with LOO_ACCURACY), NaN on rows not
        kept -- a float64 ndarray for host rows, an f64 DeviceArray for device rows.  Raises ``ValueError`` for bad
        arguments and no kept row, ``np.linalg.LinAlgError`` when the solve at alphas[best] meets a non-positive pivot
        (every other entry is then set: the dict rides on the exception as its ``result``)."""
        ptr, xdt, mk, n, d, yp, mp = _row_args(X, y, row_mask)
        cl = self._f32_classes(classes, np.size(classes))
        al = np.ascontiguousarray(np.asarray(alphas, dtype=np.float64).ravel())
        t = 1 if cl.size == 2 else max(cl.size, 1)
        mse = np.empty(max(al.size, 1), dtype=np.float64)
        correct = np.empty(max(al.size, 1), dtype=np.float64)
        coef = np.empty((t, max(d, 1)), dtype=np.float64)
        b0 = np.empty(t, dtype=np.float64)
        counts = np.zeros(3, dtype=np.float64)
        best = C.c_int(0)
        cv, cv_ptr = self._out(mk, (n, t, al.size), "f64", store_cv)
        rc = load().b2_ridge_classifier_loo(self._h, ptr, xdt, yp, n, d, d, mk, mp, int(mask_keep), cl.ctypes.data,
                                            cl.size, al.ctypes.data, int(al.size), int(bool(fit_intercept)),
                                            int(scoring), mse.ctypes.data, correct.ctypes.data, cv_ptr,
                                            C.byref(best), coef.ctypes.data, b0.ctypes.data, counts.ctypes.data)
        self.d = int(d)
        self.serial += 1
        out = {"mse": mse[: al.size], "correct": correct[: al.size], "best": int(best.value), "coef": coef,
               "intercept": b0, "kept": float(counts[0]), "unmatched": float(counts[1]),
               "nonfinite": float(counts[2]), "cv": cv}
        if rc == E_SINGULAR and "LDL" in last_error():
            exc = np.linalg.LinAlgError(last_error())
            exc.result = out
            raise exc
        if rc != 0 and isinstance(cv, DeviceArray):
            cv.free()
        _check_args(rc, "b2_ridge_classifier_loo")
        return out

    # -- scoring ------------------------------------------------------------------------------------------
    def metrics(self, y_actual, y_predicted) -> np.ndarray:
        """The ten reductions of b2_score on two vectors (b2_metrics); float64 inputs stay float64."""
        if isinstance(y_actual, DeviceArray):
            if not isinstance(y_predicted, DeviceArray) or y_actual.kind != y_predicted.kind \
                    or y_actual.kind not in ("f32", "f64") or y_actual.nbytes != y_predicted.nbytes:
                raise RuntimeError("metrics: two device vectors of the same kind (f32 / f64) and length expected")
            n = int(np.prod(y_actual.shape))
            a_ptr, p_ptr, dt, mk = y_actual.ptr, y_predicted.ptr, (F32 if y_actual.kind == "f32" else F64), MEM_DEVICE
        else:
            dtype = np.float32 if (np.asarray(y_actual).dtype == np.float32 and
                                   np.asarray(y_predicted).dtype == np.float32) else np.float64
            a = np.ascontiguousarray(np.asarray(y_actual, dtype=dtype).ravel())
            p = np.ascontiguousarray(np.asarray(y_predicted, dtype=dtype).ravel())
            if a.size != p.size:
                raise ValueError(f"Found input variables with inconsistent numbers of samples: [{a.size}, {p.size}]")
            n, a_ptr, p_ptr, dt, mk = a.size, a.ctypes.data, p.ctypes.data, (F32 if dtype == np.float32 else F64), MEM_HOST
        stats = np.zeros(10, dtype=np.float64)
        _check(load().b2_metrics(self._h, a_ptr, p_ptr, dt, n, mk, stats.ctypes.data), "b2_metrics")
        return stats

    def score(self, X, coef: np.ndarray, intercept: float, y=None, row_mask=None, mask_keep: int = 1,
              want_yhat: bool = True, out=None):
        """Returns (yhat | None, stats | None); stats = the ten reductions of include/b2gram.h b2_score
        ([sum_ape, sse, sum_y, sum_yy, max_abs_res, rows, sum_p, sum_pp, sum_yp, max_ape]).
        ``out``: a preallocated prediction buffer (DeviceArray f32 for device rows, float32 ndarray for host rows)
        to write into instead of allocating one per call."""
        ptr, xdt, mk, n, d, yp, mp = _row_args(X, y, row_mask)
        coef = np.ascontiguousarray(coef, dtype=np.float64).ravel()
        if coef.size != d:
            raise RuntimeError(f"coef has {coef.size} entries, X has {d} columns")
        if out is not None:
            if mk == MEM_DEVICE:
                if not isinstance(out, DeviceArray) or out.kind != "f32" or int(np.prod(out.shape)) != n:
                    raise RuntimeError("out must be an f32 DeviceArray with one element per row")
                yhat, yhat_ptr = out, out.ptr
            else:
                if not (isinstance(out, np.ndarray) and out.dtype == np.float32 and out.size == n
                        and out.flags.c_contiguous):
                    raise RuntimeError("out must be a C-contiguous float32 ndarray with one element per row")
                yhat, yhat_ptr = out, out.ctypes.data
        else:
            yhat, yhat_ptr = self._out(mk, (n,), "f32", want_yhat)
        stats = np.zeros(10, dtype=np.float64) if y is not None else None
        _check(load().b2_score(self._h, ptr, xdt, n, d, d, mk, coef.ctypes.data, float(intercept), yp, mp,
                               int(mask_keep), yhat_ptr, stats.ctypes.data if stats is not None else None),
               "b2_score")
        return yhat, stats

    def score_allreduce(self, stats: np.ndarray) -> np.ndarray:
        stats = np.ascontiguousarray(stats, dtype=np.float64)
        _check(load().b2_score_allreduce(self._h, stats.ctypes.data), "b2_score_allreduce")
        return stats

    # -- synthetic rows --------------------------------------------------------------------------------------
    def synth(self, n: int, d: int, seed: int = 1234, row_offset: int = 0, kind: str = "f32", alpha: float = 1.0,
              beta: float = 0.5, sigma: float = 10.0) -> Tuple[DeviceArray, DeviceArray]:
        X = self.empty((n, d), kind)
        y = self.empty((n,), "f32")
        _check(load().b2_synth(self._h, int(seed), int(row_offset), int(n), int(d), int(d),
                               F32 if kind == "f32" else BF16, float(alpha), float(beta), float(sigma), X.ptr,
                               y.ptr), "b2_synth")
        return X, y

    def synth_tranche(self, n: int, day: int, seed: int = 1234, beta: float = 0.5, sigma: float = 10.0):
        """One reference tranche (stage_3's generate_dataset: alpha(day), y >= 0 filter) -> (X (n, 1), y (n,), n_kept);
        the buffers hold ``n`` rows, the first ``n_kept`` are valid."""
        X = self.empty((n, 1), "f32")
        y = self.empty((n,), "f32")
        kept = _c_i64(0)
        _check(load().b2_synth_tranche(self._h, int(seed), int(n), int(day), float(beta), float(sigma), X.ptr, y.ptr,
                                       C.byref(kept)), "b2_synth_tranche")
        return X, y, int(kept.value)

    def stats(self) -> dict:
        out = (_c_i64 * 3)()
        _check(load().b2_ctx_stats(self._h, out), "b2_ctx_stats")
        return {"fused_fits": int(out[0]), "peer_exchanges": int(out[1]), "launches": int(out[2])}

    # -- multi-GPU -----------------------------------------------------------------------------------------------
    @staticmethod
    def comm_unique_id() -> bytes:
        buf = C.create_string_buffer(128)
        _check(load().b2_comm_unique_id(buf), "b2_comm_unique_id")
        return buf.raw

    def comm_init(self, n_ranks: int, rank: int, uid: bytes) -> None:
        _check(load().b2_comm_init(self._h, int(n_ranks), int(rank), C.create_string_buffer(uid, 128)),
               "b2_comm_init")

    def comm_p2p_export(self) -> bytes:
        """CUDA-IPC handle (64 bytes) of this rank's exchange buffer for the one-shot peer-memory all-reduce."""
        buf = C.create_string_buffer(64)
        _check(load().b2_comm_p2p_export(self._h, buf), "b2_comm_p2p_export")
        return buf.raw

    def comm_p2p_attach(self, n_ranks: int, rank: int, handles) -> None:
        """``handles``: the exported handles of all ranks, in rank order."""
        blob = b"".join(handles)
        if len(blob) != 64 * n_ranks:
            raise RuntimeError("need one 64-byte handle per rank")
        _check(load().b2_comm_p2p_attach(self._h, int(n_ranks), int(rank), C.create_string_buffer(blob, len(blob))),
               "b2_comm_p2p_attach")

    def comm_p2p_detach(self) -> None:
        _check(load().b2_comm_p2p_detach(self._h), "b2_comm_p2p_detach")

    @staticmethod
    def comm_p2p_attach_local(contexts) -> None:
        """Peer exchange between contexts of this process (rank = position in ``contexts``)."""
        arr = (_vp * len(contexts))(*[c._h for c in contexts])
        for rank, c in enumerate(contexts):
            _check(load().b2_comm_p2p_attach_local(c._h, len(contexts), rank, arr), "b2_comm_p2p_attach_local")

    def comm_set_timeout_ms(self, ms: int) -> None:
        _check(load().b2_comm_set_timeout_ms(self._h, int(ms)), "b2_comm_set_timeout_ms")

    def comm_info(self) -> dict:
        n, r, e = C.c_int(0), C.c_int(0), C.c_int(0)
        _check(load().b2_comm_info(self._h, C.byref(n), C.byref(r), C.byref(e)), "b2_comm_info")
        return {"n_ranks": n.value, "rank": r.value, "exchange": {0: "none", 1: "nccl", 2: "p2p"}[e.value]}

    def comm_barrier(self) -> None:
        _check(load().b2_comm_barrier(self._h), "b2_comm_barrier")

    # -- timing ---------------------------------------------------------------------------------------------------
    def timer_start(self) -> None:
        _check(load().b2_timer_start(self._h), "b2_timer_start")

    def timer_stop(self) -> float:
        ms = C.c_double(0.0)
        _check(load().b2_timer_stop(self._h, C.byref(ms)), "b2_timer_stop")
        return float(ms.value)

    def last_kernel_ms(self) -> Tuple[float, int]:
        ms, n = C.c_double(0.0), C.c_int(0)
        _check(load().b2_last_kernel_ms(self._h, C.byref(ms), C.byref(n)), "b2_last_kernel_ms")
        return float(ms.value), int(n.value)

    def launch_count(self) -> int:
        n = _c_i64(0)
        _check(load().b2_launch_count(self._h, C.byref(n)), "b2_launch_count")
        return int(n.value)
