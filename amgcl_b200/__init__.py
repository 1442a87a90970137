"""amgcl_b200 -- H100-native solve-phase backend for AMGCL.

The product is native:

  include/amgcl_b200.h              C ABI (the drop-in boundary)
  amgcl_b200/csrc/*.cu(h)           hand-written sm_90a kernels behind it
  include/amgcl/backend/b200.hpp    C++ binding to amgcl::backend (the reference is C++)
  amgcl_b200/host/dropin.cpp        AMGCL's own make_solver<amg<...>, cg|bicgstab>
                                    instantiated on that backend

This Python package is only the ctypes loader that bench.py and the tests use
to drive those libraries; it contains no numerical code and has NO CPU
fallback: constructing a :class:`Context` without a CUDA device raises.
"""
import ctypes
import os

import numpy as np

from . import build as _build

__all__ = ["lib", "dropin_lib", "Context", "Vector", "Csr", "Coarse", "Krylov", "DropinSolver",
           "poisson3d", "unstructured3d", "B200Error", "RELAX", "KRYLOV", "nccl_unique_id",
           "partition", "dist_split", "coarse_lu_plan"]

_c = ctypes
_i64 = _c.c_int64
_dbl = _c.c_double
_vp = _c.c_void_p
_P = _c.POINTER

RELAX = {"damped_jacobi": 0, "spai0": 1, "chebyshev": 2, "ilu0": 3}
KRYLOV = {"cg": 0, "bicgstab": 1, "gmres": 2, "bicgstabl": 3}


class B200Error(RuntimeError):
    pass


class ProfileEntry(_c.Structure):
    """b200_profile_entry (include/amgcl_b200.h)."""
    _fields_ = [("nrows", _i64), ("ncols", _i64), ("nnz", _i64), ("mode", _c.c_int),
                ("launches", _i64), ("total_ms", _dbl), ("min_ms", _dbl)]


class ProfileFormatEntry(_c.Structure):
    """b200_profile_format_entry (include/amgcl_b200_formats.h)."""
    _fields_ = [("entry", ProfileEntry), ("format", _c.c_int), ("value_bytes", _c.c_int)]


# column formats of a CSR operator (include/amgcl_b200_formats.h B200_FMT_*)
FORMAT_NAMES = ("plain", "window", "offset", "pattern", "col16", "col24", "pattern_values")


# vecK: element-wise pass over K+1 vector streams (reads + writes)
MODE_NAMES = {0: "spmv", 1: "spmv_acc", 2: "residual", 3: "relax", 4: "residual_scaled", 10: "vec1", 11: "vec2",
              12: "vec3", 13: "vec4", 14: "vec5", 15: "vec6", 16: "vec7",
              20: "dot", 21: "relax_zero", 22: "coarse_gemv", 23: "memset", 24: "coarse_tail", 25: "coarse_lu",
              30: "comm"}


_lib = None
_dropin = None


def lib():
    """ctypes handle of libamgcl_b200.so (built in-tree on first use)."""
    global _lib
    if _lib is not None:
        return _lib
    path = os.environ.get("B200_LIB") or _build.LIB_CUDA     # B200_LIB: experimental builds
    if not os.path.isfile(path):
        path = _build.build_cuda()
    L = _c.CDLL(path, mode=_c.RTLD_GLOBAL)
    L.b200_last_error.restype = _c.c_char_p
    L.b200_version.restype = _c.c_char_p
    sigs = {
        "b200_device_count": [],
        "b200_ctx_create": [_c.c_int, _P(_vp)],
        "b200_ctx_destroy": [_vp],
        "b200_ctx_default": [_P(_vp)],
        "b200_ctx_set_stream": [_vp, _vp],
        "b200_ctx_get_stream": [_vp, _P(_vp)],
        "b200_ctx_device": [_vp, _P(_c.c_int)],
        "b200_ctx_sync": [_vp],
        "b200_ctx_flush": [_vp],
        "b200_tail_stats": [_vp, _P(_c.c_uint64), _P(_c.c_uint64)],
        "b200_ctx_launch_count": [_vp, _P(_c.c_uint64)],
        "b200_ctx_reset_launch_count": [_vp],
        "b200_ctx_set_option": [_vp, _c.c_char_p, _i64],
        "b200_ctx_get_option": [_vp, _c.c_char_p, _P(_i64)],
        "b200_vec_create": [_vp, _c.c_size_t, _P(_vp)],
        "b200_vec_wrap": [_vp, _vp, _c.c_size_t, _P(_vp)],
        "b200_vec_destroy": [_vp],
        "b200_vec_size": [_vp, _P(_c.c_size_t)],
        "b200_vec_bytes": [_vp, _P(_c.c_size_t)],
        "b200_vec_data": [_vp, _P(_vp)],
        "b200_vec_upload": [_vp, _vp, _c.c_size_t],
        "b200_vec_download": [_vp, _vp, _c.c_size_t],
        "b200_vec_download_local": [_vp, _vp, _c.c_size_t],
        "b200_vec_local_range": [_vp, _P(_c.c_size_t), _P(_c.c_size_t)],
        # FP32 objects of the mixed-precision composition (b200<float> hierarchy)
        "b200_vec_create_f32": [_vp, _c.c_size_t, _P(_vp)],
        "b200_vec_upload_f32": [_vp, _vp, _c.c_size_t],
        "b200_vec_download_f32": [_vp, _vp, _c.c_size_t],
        "b200_vec_dtype": [_vp, _P(_c.c_int)],
        "b200_csr_create_i64_f32": [_vp, _i64, _i64, _vp, _vp, _vp, _P(_vp)],
        "b200_csr_create_i32_f32": [_vp, _i64, _i64, _vp, _vp, _vp, _P(_vp)],
        "b200_csr_dtype": [_vp, _P(_c.c_int)],
        "b200_coarse_create_i64_f32": [_vp, _i64, _vp, _vp, _vp, _P(_vp)],
        "b200_coarse_create_i32_f32": [_vp, _i64, _vp, _vp, _vp, _P(_vp)],
        "b200_csr_create_i64": [_vp, _i64, _i64, _vp, _vp, _vp, _P(_vp)],
        "b200_csr_create_i32": [_vp, _i64, _i64, _vp, _vp, _vp, _P(_vp)],
        "b200_csr_destroy": [_vp],
        "b200_csr_rows": [_vp, _P(_c.c_size_t)],
        "b200_csr_cols": [_vp, _P(_c.c_size_t)],
        "b200_csr_nonzeros": [_vp, _P(_c.c_size_t)],
        "b200_csr_bytes": [_vp, _P(_c.c_size_t)],
        "b200_csr_plan": [_vp, _P(_c.c_int), _P(_i64), _P(_i64)],
        "b200_spmv": [_vp, _dbl, _vp, _vp, _dbl, _vp],
        "b200_residual": [_vp, _vp, _vp, _vp, _vp],
        "b200_clear": [_vp, _vp],
        "b200_copy": [_vp, _vp, _vp],
        "b200_dot": [_vp, _vp, _vp, _P(_dbl)],
        "b200_axpby": [_vp, _dbl, _vp, _dbl, _vp],
        "b200_axpbypcz": [_vp, _dbl, _vp, _dbl, _vp, _dbl, _vp],
        "b200_vmul": [_vp, _dbl, _vp, _vp, _dbl, _vp],
        "b200_relax": [_vp, _vp, _vp, _vp, _vp, _vp, _dbl],
        "b200_coarse_create_i64": [_vp, _i64, _vp, _vp, _vp, _P(_vp)],
        "b200_coarse_create_i32": [_vp, _i64, _vp, _vp, _vp, _P(_vp)],
        "b200_coarse_destroy": [_vp],
        "b200_coarse_bytes": [_vp, _P(_c.c_size_t)],
        "b200_coarse_info": [_vp, _P(_c.c_int), _P(_i64), _P(_i64), _P(_i64)],
        "b200_coarse_lu_plan_i64": [_i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _P(_i64), _P(_c.c_int),
                                    _P(_i64), _P(_c.c_size_t), _P(_c.c_size_t)],
        "b200_coarse_solve": [_vp, _vp, _vp, _vp],
        "b200_nccl_unique_id": [_c.c_char_p, _c.c_size_t],
        "b200_dist_init": [_vp, _c.c_char_p, _c.c_size_t, _c.c_int, _c.c_int, _i64],
        "b200_dist_info": [_vp, _P(_c.c_int), _P(_c.c_int), _P(_i64), _P(_c.c_int)],
        "b200_partition": [_i64, _c.c_int, _c.c_int, _P(_i64), _P(_i64), _P(_i64)],
        "b200_dist_split_i64": [_c.c_int, _c.c_int, _c.c_int, _i64, _i64, _vp, _vp, _vp, _P(_vp)],
        "b200_split_info": [_vp, _P(_i64), _P(_i64), _P(_i64), _P(_i64), _P(_i64), _P(_i64)],
        "b200_split_copy": [_vp, _vp, _vp, _vp, _vp],
        "b200_split_destroy": [_vp],
        "b200_plan_i64": [_i64, _vp, _c.c_int, _c.c_int, _vp, _i64, _P(_i64), _P(_c.c_int),
                          _P(_c.c_int), _P(_i64)],
        "b200_ctx_largest_operator": [_vp, _P(_i64), _P(_c.c_int)],
        "b200_csr_patterns": [_vp, _P(_c.c_int), _P(_c.c_int), _P(_c.c_int)],
        "b200_pattern_plan_i64": [_i64, _i64, _vp, _vp, _vp, _vp, _vp, _P(_c.c_int), _P(_c.c_int), _P(_c.c_int)],
        "b200_pattern_value_plan_i64": [_i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _P(_c.c_int), _P(_c.c_int),
                                        _P(_c.c_int), _P(_c.c_int)],
        "b200_csr_offsets": [_vp, _P(_c.c_int), _P(_c.c_int)],
        "b200_offset_plan_i64": [_i64, _i64, _vp, _vp, _vp, _vp, _P(_c.c_int), _P(_c.c_int)],
        "b200_csr_narrow": [_vp, _P(_c.c_int)],
        "b200_csr_value_bytes": [_vp, _P(_c.c_int)],
        "b200_values_fit_f32": [_vp, _i64, _P(_c.c_int)],
        "b200_value_index_plan_i64": [_vp, _i64, _vp, _i64, _vp, _P(_c.c_int), _P(_c.c_int)],
        "b200_narrow_plan_i64": [_i64, _i64, _vp, _vp, _c.c_int, _c.c_int, _vp, _i64, _vp, _vp, _vp,
                                 _P(_i64), _P(_c.c_int)],
        "b200_csr_window": [_vp, _P(_c.c_int), _P(_c.c_int), _P(_c.c_int), _P(_i64)],
        "b200_window_plan_i64": [_i64, _i64, _vp, _vp, _c.c_int, _c.c_int, _c.c_int, _c.c_int, _c.c_int, _vp, _vp, _i64,
                                 _vp, _i64, _P(_i64), _P(_i64), _P(_c.c_int), _P(_c.c_int), _P(_c.c_int)],
        "b200_index_create_i64": [_vp, _vp, _c.c_size_t, _c.c_size_t, _P(_vp)],
        "b200_index_destroy": [_vp],
        "b200_index_size": [_vp, _P(_c.c_size_t)],
        "b200_gather": [_vp, _vp, _vp, _vp],
        "b200_gather_host": [_vp, _vp, _vp, _vp],
        "b200_scatter": [_vp, _vp, _vp, _vp],
        "b200_graph_begin": [_vp, _P(_c.c_int)],
        "b200_graph_end": [_vp, _P(_vp)],
        "b200_graph_abort": [_vp],
        "b200_graph_launch": [_vp, _vp, _P(_c.c_int)],
        "b200_graph_info": [_vp, _P(_i64), _P(_i64), _P(_i64), _P(_c.c_int)],
        "b200_graph_destroy": [_vp],
        # fused Krylov steps (device-resident scalars)
        "b200_krylov_create": [_vp, _c.c_size_t, _P(_vp)],
        "b200_krylov_destroy": [_vp],
        "b200_krylov_residual": [_vp, _vp, _vp, _vp, _vp, _P(_dbl)],
        "b200_krylov_scalars": [_vp, _vp, _c.c_int],
        "b200_cg_direction": [_vp, _vp, _vp, _vp],
        "b200_cg_step": [_vp, _vp, _vp, _vp, _vp, _vp, _P(_dbl)],
        "b200_bicg_start": [_vp, _vp, _vp],
        "b200_bicg_direction": [_vp, _vp, _vp, _vp],
        "b200_bicg_step_s": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _P(_dbl), _P(_dbl)],
        "b200_bicg_step_r": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _P(_dbl), _P(_dbl)],
        "b200_profile_begin": [_vp],
        "b200_profile_end": [_vp, _vp, _i64, _P(_i64)],
        "b200_profile_end_formats": [_vp, _vp, _i64, _P(_i64)],
    }
    for name, args in sigs.items():
        fn = getattr(L, name)
        fn.argtypes = args
        fn.restype = _c.c_int
    _lib = L
    return L


def dropin_lib():
    """ctypes handle of libamgcl_b200_dropin.so (AMGCL templates on backend::b200)."""
    global _dropin
    if _dropin is not None:
        return _dropin
    lib()   # libamgcl_b200.so first (RTLD_GLOBAL) so the dependency resolves
    path = _build.LIB_DROPIN
    if not os.path.isfile(path):
        path = _build.build_dropin()
    D = _c.CDLL(path)
    D.dropin_last_error.restype = _c.c_char_p
    D.dropin_create.argtypes = [_vp, _i64, _vp, _vp, _vp, _c.c_int, _c.c_int, _dbl, _c.c_int,
                                _c.c_int, _P(_vp)]
    D.dropin_create.restype = _c.c_int
    D.dropin_create_mixed.argtypes = D.dropin_create.argtypes
    D.dropin_create_mixed.restype = _c.c_int
    D.dropin_create_graph.argtypes = [_vp, _i64, _vp, _vp, _vp, _c.c_int, _c.c_int, _c.c_int, _dbl,
                                      _c.c_int, _c.c_int, _P(_vp)]
    D.dropin_create_graph.restype = _c.c_int
    D.dropin_graph_stats.argtypes = [_vp, _P(_i64), _P(_i64), _P(_i64)]
    D.dropin_graph_stats.restype = _c.c_int
    D.dropin_gather_scatter.argtypes = [_vp, _i64, _vp, _i64, _vp, _dbl, _vp, _vp, _vp]
    D.dropin_gather_scatter.restype = _c.c_int
    D.dropin_destroy.argtypes = [_vp]
    D.dropin_destroy.restype = None
    D.dropin_solve.argtypes = [_vp, _vp, _vp, _P(_i64), _P(_dbl)]
    D.dropin_solve.restype = _c.c_int
    D.dropin_solve_zero_guess.argtypes = [_vp, _vp, _vp, _P(_i64), _P(_dbl)]
    D.dropin_solve_zero_guess.restype = _c.c_int
    D.dropin_upload_rhs.argtypes = [_vp, _vp]
    D.dropin_upload_rhs.restype = _c.c_int
    D.dropin_solve_resident.argtypes = [_vp, _P(_i64), _P(_dbl)]
    D.dropin_solve_resident.restype = _c.c_int
    D.dropin_download_x.argtypes = [_vp, _vp]
    D.dropin_download_x.restype = _c.c_int
    D.dropin_apply_precond.argtypes = [_vp, _vp, _vp]
    D.dropin_apply_precond.restype = _c.c_int
    D.dropin_report.argtypes = [_vp, _c.c_char_p, _i64]
    D.dropin_report.restype = _i64
    D.dropin_bytes.argtypes = [_vp]
    D.dropin_bytes.restype = _i64
    D.dropin_set_num_threads.argtypes = [_c.c_int]
    D.dropin_set_num_threads.restype = None
    D.dropin_num_threads.restype = _c.c_int
    _dropin = D
    return D


def _check(rc, what=""):
    if rc != 0:
        msg = lib().b200_last_error().decode(errors="replace")
        raise B200Error("%s failed (%d): %s" % (what or "b200 call", rc, msg))


def _f64(a):
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a


def _ptr(a):
    return a.ctypes.data_as(_vp)


class Context:
    """Device + stream + scratch (b200_ctx_t)."""

    def __init__(self, device=0, stream=None):
        L = lib()
        if L.b200_device_count() <= 0:
            raise B200Error("amgcl_b200 requires a CUDA device (no CPU fallback)")
        self.h = _vp()
        _check(L.b200_ctx_create(int(device), _c.byref(self.h)), "b200_ctx_create")
        if stream is not None:
            self.set_stream(stream)

    def set_stream(self, cuda_stream):
        """cuda_stream: a cudaStream_t as int (torch: stream.cuda_stream).  0 means the
        legacy default stream (what torch's default stream is); None selects the
        context's own stream again."""
        if cuda_stream is None:
            handle = 0
        else:
            handle = int(cuda_stream) or 1     # (cudaStream_t)0x1 == cudaStreamLegacy
        _check(lib().b200_ctx_set_stream(self.h, _vp(handle)))

    def sync(self):
        _check(lib().b200_ctx_sync(self.h), "b200_ctx_sync")

    def flush(self):
        """Launch whatever was deferred into the coarse-tail list (option "coarse_tail")."""
        _check(lib().b200_ctx_flush(self.h), "b200_ctx_flush")

    def tail_stats(self):
        """(launches of the coarse-tail kernel, calls they executed) since context creation."""
        f, c = _c.c_uint64(), _c.c_uint64()
        _check(lib().b200_tail_stats(self.h, _c.byref(f), _c.byref(c)))
        return f.value, c.value

    def set_option(self, key, value):
        _check(lib().b200_ctx_set_option(self.h, key.encode(), int(value)), "b200_ctx_set_option")

    def get_option(self, key):
        v = _i64()
        _check(lib().b200_ctx_get_option(self.h, key.encode(), _c.byref(v)))
        return v.value

    @property
    def launches(self):
        v = _c.c_uint64()
        _check(lib().b200_ctx_launch_count(self.h, _c.byref(v)))
        return v.value

    def reset_launches(self):
        _check(lib().b200_ctx_reset_launch_count(self.h))

    # -- multi-GPU ---------------------------------------------------------
    def dist_init(self, unique_id, nranks, rank, dist_min_rows):
        """Join the NCCL communicator (one process per GPU).  Dimensions >= dist_min_rows
        are partitioned across the ranks from now on (see include/amgcl_b200.h)."""
        buf = _c.create_string_buffer(bytes(unique_id), 128)
        _check(lib().b200_dist_init(self.h, buf, 128, int(nranks), int(rank), int(dist_min_rows)),
               "b200_dist_init")

    def dist_info(self):
        r, n, p = _c.c_int(), _c.c_int(), _c.c_int()
        m = _i64()
        _check(lib().b200_dist_info(self.h, _c.byref(r), _c.byref(n), _c.byref(m), _c.byref(p)))
        return {"rank": r.value, "nranks": n.value, "dist_min_rows": m.value, "p2p": bool(p.value)}

    def largest_operator(self):
        """(non-zeros, column format) of the largest operator uploaded so far; format is one of
        one of FORMAT_NAMES."""
        nnz, fmt = _i64(), _c.c_int()
        _check(lib().b200_ctx_largest_operator(self.h, _c.byref(nnz), _c.byref(fmt)))
        return nnz.value, FORMAT_NAMES[fmt.value]

    def profile_begin(self):
        _check(lib().b200_profile_begin(self.h), "b200_profile_begin")

    def profile_end(self):
        """Per (matrix shape, mode, column format, value width) device times of the CSR kernels
        since profile_begin(); value_bytes is 1, 2, 4 or 8 for a CSR pass, 0 for the other kernels."""
        cap = 256
        buf = (ProfileFormatEntry * cap)()
        cnt = _i64()
        _check(lib().b200_profile_end_formats(self.h, buf, cap, _c.byref(cnt)), "b200_profile_end_formats")
        out = []
        for i in range(min(cap, cnt.value)):
            e, fmt, vb = buf[i].entry, buf[i].format, buf[i].value_bytes
            out.append({"nrows": e.nrows, "ncols": e.ncols, "nnz": e.nnz,
                        "mode": MODE_NAMES.get(e.mode, str(e.mode)), "launches": e.launches,
                        "total_ms": e.total_ms, "min_ms": e.min_ms, "format": FORMAT_NAMES[fmt],
                        "value_bytes": vb})
        return out

    def close(self):
        if self.h:
            lib().b200_ctx_destroy(self.h)
            self.h = _vp()

    # -- factories --------------------------------------------------------
    def vector(self, data_or_n):
        return Vector(self, data_or_n)

    def csr(self, nrows, ncols, ptr, col, val):
        return Csr(self, nrows, ncols, ptr, col, val)

    def coarse(self, n, ptr, col, val):
        return Coarse(self, n, ptr, col, val)

    # -- primitives (thin, 1:1 with the C ABI) ------------------------------
    def spmv(self, alpha, A, x, beta, y):
        _check(lib().b200_spmv(self.h, alpha, A.h, x.h, beta, y.h), "b200_spmv")

    def residual(self, f, A, x, r):
        _check(lib().b200_residual(self.h, f.h, A.h, x.h, r.h), "b200_residual")

    def clear(self, x):
        _check(lib().b200_clear(self.h, x.h), "b200_clear")

    def copy(self, x, y):
        _check(lib().b200_copy(self.h, x.h, y.h), "b200_copy")

    def dot(self, x, y):
        r = _dbl()
        _check(lib().b200_dot(self.h, x.h, y.h, _c.byref(r)), "b200_dot")
        return r.value

    def axpby(self, a, x, b, y):
        _check(lib().b200_axpby(self.h, a, x.h, b, y.h), "b200_axpby")

    def axpbypcz(self, a, x, b, y, c, z):
        _check(lib().b200_axpbypcz(self.h, a, x.h, b, y.h, c, z.h), "b200_axpbypcz")

    def vmul(self, alpha, x, y, beta, z):
        _check(lib().b200_vmul(self.h, alpha, x.h, y.h, beta, z.h), "b200_vmul")

    # -- index lists (Backend::gather / scatter) --
    def index(self, idx, size):
        """Device index list into a vector of `size` elements."""
        return Index(self, idx, size)

    def gather(self, I, src, dst):
        _check(lib().b200_gather(self.h, I.h, src.h, dst.h), "b200_gather")

    def gather_host(self, I, src):
        out = np.empty(I.n, dtype=np.float64)
        _check(lib().b200_gather_host(self.h, I.h, src.h, _ptr(out)), "b200_gather_host")
        return out

    def scatter(self, I, src, dst):
        _check(lib().b200_scatter(self.h, I.h, src.h, dst.h), "b200_scatter")

    # -- recorded call sequences (b200_graph_*) --
    def graph_begin(self):
        """Start recording; False when this context cannot record right now."""
        rec = _c.c_int(0)
        _check(lib().b200_graph_begin(self.h, _c.byref(rec)), "b200_graph_begin")
        return bool(rec.value)

    def graph_end(self):
        g = _vp()
        _check(lib().b200_graph_end(self.h, _c.byref(g)), "b200_graph_end")
        return Graph(self, g)

    def graph_abort(self):
        _check(lib().b200_graph_abort(self.h), "b200_graph_abort")

    def relax(self, A, rhs, x, tmp, diag, omega):
        _check(lib().b200_relax(self.h, A.h, rhs.h, x.h, tmp.h, diag.h, omega), "b200_relax")

    def coarse_solve(self, S, rhs, x):
        _check(lib().b200_coarse_solve(self.h, S.h, rhs.h, x.h), "b200_coarse_solve")


class Krylov:
    """Device-resident scalars of one Krylov solver (b200_krylov_t) + the fused steps."""

    SCALARS = ("rho", "qp", "alpha", "ts", "tt", "omega", "rr", "ss", "rho_next")

    def __init__(self, ctx, n):
        self.ctx = ctx
        self.h = _vp()
        _check(lib().b200_krylov_create(ctx.h, int(n), _c.byref(self.h)), "b200_krylov_create")

    def residual(self, rhs, A, x, r):
        out = _dbl()
        _check(lib().b200_krylov_residual(self.h, rhs.h, A.h, x.h, r.h, _c.byref(out)), "b200_krylov_residual")
        return out.value

    def scalars(self):
        buf = (_dbl * 9)()
        _check(lib().b200_krylov_scalars(self.h, buf, 9), "b200_krylov_scalars")
        return dict(zip(self.SCALARS, list(buf)))

    def cg_direction(self, r, s, p):
        _check(lib().b200_cg_direction(self.h, r.h, s.h, p.h), "b200_cg_direction")

    def cg_step(self, A, p, q, x, r):
        out = _dbl()
        _check(lib().b200_cg_step(self.h, A.h, p.h, q.h, x.h, r.h, _c.byref(out)), "b200_cg_step")
        return out.value

    def bicg_start(self, r, rh):
        _check(lib().b200_bicg_start(self.h, r.h, rh.h), "b200_bicg_start")

    def bicg_direction(self, r, v, p):
        _check(lib().b200_bicg_direction(self.h, r.h, v.h, p.h), "b200_bicg_direction")

    def bicg_step_s(self, A, rh, T, v, r, s, x):
        out = _dbl()
        _check(lib().b200_bicg_step_s(self.h, A.h, rh.h, T.h, v.h, r.h, s.h, x.h, _c.byref(out), None),
               "b200_bicg_step_s")
        return out.value

    def bicg_step_r(self, A, rh, T, t, s, r, x):
        out = _dbl()
        _check(lib().b200_bicg_step_r(self.h, A.h, rh.h, T.h, t.h, s.h, r.h, x.h, _c.byref(out), None),
               "b200_bicg_step_r")
        return out.value

    def close(self):
        if self.h:
            lib().b200_krylov_destroy(self.h)
            self.h = _vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Vector:
    """Device FP64 vector (b200_vec_t)."""

    def __init__(self, ctx, data_or_n):
        self.ctx = ctx
        self.h = _vp()
        if isinstance(data_or_n, (int, np.integer)):
            self.n = int(data_or_n)
            _check(lib().b200_vec_create(ctx.h, self.n, _c.byref(self.h)), "b200_vec_create")
        else:
            a = _f64(data_or_n)
            self.n = a.size
            _check(lib().b200_vec_create(ctx.h, self.n, _c.byref(self.h)), "b200_vec_create")
            self.upload(a)

    def upload(self, a):
        a = _f64(a)
        _check(lib().b200_vec_upload(self.h, _ptr(a), a.size), "b200_vec_upload")

    def numpy(self):
        out = np.empty(self.n, dtype=np.float64)
        _check(lib().b200_vec_download(self.h, _ptr(out), self.n), "b200_vec_download")
        return out

    def data_ptr(self):
        p = _vp()
        _check(lib().b200_vec_data(self.h, _c.byref(p)))
        return p.value or 0

    def __del__(self):
        try:
            if self.h:
                lib().b200_vec_destroy(self.h)
                self.h = _vp()
        except Exception:
            pass


class Csr:
    """Device CSR matrix + row-block plan (b200_csr_t)."""

    def __init__(self, ctx, nrows, ncols, ptr, col, val):
        self.ctx = ctx
        self.h = _vp()
        val = _f64(val)
        ptr = np.ascontiguousarray(ptr)
        col = np.ascontiguousarray(col)
        if ptr.dtype == np.int32 and col.dtype == np.int32:
            fn = lib().b200_csr_create_i32
        else:
            ptr = np.ascontiguousarray(ptr, dtype=np.int64)
            col = np.ascontiguousarray(col, dtype=np.int64)
            fn = lib().b200_csr_create_i64
        _check(fn(ctx.h, int(nrows), int(ncols), _ptr(ptr), _ptr(col), _ptr(val),
                  _c.byref(self.h)), "b200_csr_create")
        self.nrows, self.ncols, self.nnz = int(nrows), int(ncols), int(ptr[-1])

    def plan(self):
        lanes = _c.c_int()
        nb = _i64()
        nl = _i64()
        _check(lib().b200_csr_plan(self.h, _c.byref(lanes), _c.byref(nb), _c.byref(nl)))
        return {"lanes": lanes.value, "blocks": nb.value, "long_blocks": nl.value}

    def bytes(self):
        b = _c.c_size_t()
        _check(lib().b200_csr_bytes(self.h, _c.byref(b)))
        return b.value

    def patterns(self):
        """Pattern-indexed row storage of this operator (b200_csr_patterns)."""
        on, cnt, tot = _c.c_int(), _c.c_int(), _c.c_int()
        _check(lib().b200_csr_patterns(self.h, _c.byref(on), _c.byref(cnt), _c.byref(tot)))
        return {"pattern_indexed": bool(on.value), "count": cnt.value, "total": tot.value}

    def offsets(self):
        """Offset-indexed column storage of this operator (b200_csr_offsets)."""
        on, cnt = _c.c_int(), _c.c_int()
        _check(lib().b200_csr_offsets(self.h, _c.byref(on), _c.byref(cnt)))
        return {"offset_indexed": bool(on.value), "count": cnt.value}

    def narrow(self):
        """Width of this operator's block-relative columns: 16, 24, or 0 when it is not stored
        that way (b200_csr_narrow)."""
        w = _c.c_int()
        _check(lib().b200_csr_narrow(self.h, _c.byref(w)))
        return w.value

    def value_bytes(self):
        """Bytes per value the streaming passes read from this operator: 4 for an FP32 operator
        and for an FP64 one whose values are all exact FP32, 1 or 2 for an FP64 one streamed as
        indices into the table of its distinct values, else 8 (b200_csr_value_bytes).  For
        value-keyed patterns, the width of the pattern table's values the passes read."""
        b = _c.c_int()
        _check(lib().b200_csr_value_bytes(self.h, _c.byref(b)))
        return b.value

    def window(self):
        """Windowed storage of this operator (include/amgcl_b200.h: b200_csr_window)."""
        w, ms, mr, tot = _c.c_int(), _c.c_int(), _c.c_int(), _i64()
        _check(lib().b200_csr_window(self.h, _c.byref(w), _c.byref(ms), _c.byref(mr), _c.byref(tot)))
        return {"windowed": bool(w.value), "max_slots": ms.value, "max_runs": mr.value, "total_slots": tot.value}

    def __del__(self):
        try:
            if self.h and lib().b200_csr_destroy(self.h) == 0:
                self.h = _vp()      # (kept if the library refused, e.g. while a graph is recorded)
        except Exception:
            pass


def pattern_plan(nrows, ncols, ptr, col):
    """Host-only: the pattern-indexed row format b200_csr_create would build
    (b200_pattern_plan_i64).  None when the operator has too many row patterns."""
    ptr = np.ascontiguousarray(ptr, dtype=np.int64)
    col = np.ascontiguousarray(col, dtype=np.int64)
    pid = np.zeros(max(1, nrows), dtype=np.uint8)
    start = np.zeros(257, dtype=np.uint16)
    off = np.zeros(1024, dtype=np.int32)
    cnt, tot, ok = _c.c_int(), _c.c_int(), _c.c_int()
    _check(lib().b200_pattern_plan_i64(nrows, ncols, ptr.ctypes.data, col.ctypes.data, pid.ctypes.data,
                                       start.ctypes.data, off.ctypes.data, _c.byref(cnt), _c.byref(tot),
                                       _c.byref(ok)))
    if not ok.value:
        return None
    return {"pid": pid[:nrows], "start": start, "off": off, "count": cnt.value, "total": tot.value}


def pattern_value_plan(nrows, ncols, ptr, col, val):
    """Host-only: the value-keyed pattern format b200_csr_create tries first
    (b200_pattern_value_plan_i64): patterns of (col - row, value) pairs.  None when the operator
    has too many of them; else pattern_plan's fields plus "val" (the table's values, parallel to
    "off") and "exact_f32" (every table value survives double -> float -> double)."""
    ptr = np.ascontiguousarray(ptr, dtype=np.int64)
    col = np.ascontiguousarray(col, dtype=np.int64)
    val = np.ascontiguousarray(val, dtype=np.float64)
    pid = np.zeros(max(1, nrows), dtype=np.uint8)
    start = np.zeros(257, dtype=np.uint16)
    off = np.zeros(1024, dtype=np.int32)
    tab = np.zeros(1024, dtype=np.float64)
    cnt, tot, exact, ok = _c.c_int(), _c.c_int(), _c.c_int(), _c.c_int()
    _check(lib().b200_pattern_value_plan_i64(nrows, ncols, ptr.ctypes.data, col.ctypes.data, val.ctypes.data,
                                             pid.ctypes.data, start.ctypes.data, off.ctypes.data, tab.ctypes.data,
                                             _c.byref(cnt), _c.byref(tot), _c.byref(exact), _c.byref(ok)))
    if not ok.value:
        return None
    return {"pid": pid[:nrows], "start": start, "off": off, "val": tab, "count": cnt.value, "total": tot.value,
            "exact_f32": bool(exact.value)}


def offset_plan(nrows, ncols, ptr, col):
    """Host-only: the offset-indexed column format b200_csr_create would build
    (b200_offset_plan_i64).  None when the operator has more than 256 distinct col - row."""
    ptr = np.ascontiguousarray(ptr, dtype=np.int64)
    col = np.ascontiguousarray(col, dtype=np.int64)
    nnz = int(ptr[-1]) if nrows else 0
    idx8 = np.zeros(max(1, nnz), dtype=np.uint8)
    tab = np.zeros(256, dtype=np.int32)
    cnt, ok = _c.c_int(), _c.c_int()
    _check(lib().b200_offset_plan_i64(nrows, ncols, ptr.ctypes.data, col.ctypes.data, idx8.ctypes.data,
                                      tab.ctypes.data, _c.byref(cnt), _c.byref(ok)))
    if not ok.value:
        return None
    return {"idx8": idx8[:nnz], "tab": tab, "count": cnt.value}


def narrow_plan(nrows, ncols, ptr, col, lanes=0, nnz_cap=2048):
    """Host-only: the row-block plan's block-relative row pointers and narrow columns
    b200_csr_create would build for a single-GPU operator (b200_narrow_plan_i64).  A dict with
    nblocks, ptr16 [nrows] and width (16, 24, or 0 when the operator stays plain); when narrowed
    also base [nblocks], lo16 [nnz] and, width 24, hi8 [nnz]."""
    ptr = np.ascontiguousarray(ptr, dtype=np.int64)
    col = np.ascontiguousarray(col, dtype=np.int64)
    nnz = int(ptr[-1]) if nrows else 0
    cap = nrows // 4 + 2 + (nnz // 256 + 1)        # at least one block per quad or per 256 entries
    base = np.zeros(cap, dtype=np.int32)
    lo16 = np.zeros(max(1, nnz), dtype=np.uint16)
    hi8 = np.zeros(max(1, nnz), dtype=np.uint8)
    ptr16 = np.zeros(max(1, nrows), dtype=np.uint16)
    nb, w = _i64(), _c.c_int()
    _check(lib().b200_narrow_plan_i64(nrows, ncols, ptr.ctypes.data, col.ctypes.data, int(lanes), int(nnz_cap),
                                      base.ctypes.data, cap, lo16.ctypes.data, hi8.ctypes.data,
                                      ptr16.ctypes.data, _c.byref(nb), _c.byref(w)))
    out = {"nblocks": nb.value, "ptr16": ptr16[:nrows], "width": w.value}
    if w.value:
        out.update(base=base[:nb.value], lo16=lo16[:nnz])
        if w.value == 24:
            out["hi8"] = hi8[:nnz]
    return out


def values_fit_f32(val):
    """Host-only: whether every value keeps its bits through double -> float -> double, the rule
    b200_csr_create applies before it also stores an FP64 operator's values as FP32
    (b200_values_fit_f32)."""
    val = np.ascontiguousarray(val, dtype=np.float64)
    ok = _c.c_int()
    _check(lib().b200_values_fit_f32(val.ctypes.data, val.size, _c.byref(ok)))
    return bool(ok.value)


def value_index_plan(val):
    """Host-only: the index into the table of distinct values that b200_csr_create builds for an
    FP64 operator (b200_value_index_plan_i64).  Returns {"width": 8 or 16, "count", "table",
    "index"}, or {"width": 0, "count": 4097} when there are more than 4,096 distinct values."""
    val = np.ascontiguousarray(val, dtype=np.float64)
    tab = np.zeros(4096, dtype=np.float64)
    idx = np.zeros(max(1, 2 * val.size), dtype=np.uint8)
    cnt, w = _c.c_int(), _c.c_int()
    _check(lib().b200_value_index_plan_i64(val.ctypes.data, val.size, tab.ctypes.data, tab.size,
                                            idx.ctypes.data, _c.byref(cnt), _c.byref(w)))
    out = {"width": w.value, "count": cnt.value}
    if w.value:
        out["table"] = tab[:cnt.value]
        out["index"] = idx[:val.size] if w.value == 8 else idx[:2 * val.size].view(np.uint16)
    return out


def window_plan(nrows, ncols, ptr, col, lanes=0, nnz_cap=2048, slot_cap=1400, max_ratio=75, gap=2):
    """Host-only: the row-block plan and the windowed format b200_csr_create would build
    (b200_window_plan_i64).  Returns None when the operator does not qualify, else a dict with
    blk [nblocks,6], runs [nruns,2], col16 [nnz], max_slots, max_runs."""
    ptr = np.ascontiguousarray(ptr, dtype=np.int64)
    col = np.ascontiguousarray(col, dtype=np.int64)
    nnz = int(ptr[-1]) if nrows else 0
    nb, nr = _i64(), _i64()
    ms, mr, ok = _c.c_int(), _c.c_int(), _c.c_int()
    L = lib()
    _check(L.b200_window_plan_i64(nrows, ncols, ptr.ctypes.data, col.ctypes.data, lanes, nnz_cap, slot_cap,
                                  max_ratio, gap, None, None, 0, None, 0, _c.byref(nb), _c.byref(nr),
                                  _c.byref(ms), _c.byref(mr), _c.byref(ok)))
    if not ok.value:
        return None
    blk = np.zeros((nb.value, 6), dtype=np.int32)
    runs = np.zeros((max(1, nr.value), 2), dtype=np.int32)
    col16 = np.zeros(max(1, nnz), dtype=np.uint16)
    _check(L.b200_window_plan_i64(nrows, ncols, ptr.ctypes.data, col.ctypes.data, lanes, nnz_cap, slot_cap,
                                  max_ratio, gap, col16.ctypes.data, runs.ctypes.data, runs.shape[0],
                                  blk.ctypes.data, blk.shape[0], _c.byref(nb), _c.byref(nr),
                                  _c.byref(ms), _c.byref(mr), _c.byref(ok)))
    return {"blk": blk, "runs": runs[:nr.value], "col16": col16[:nnz], "max_slots": ms.value,
            "max_runs": mr.value}


def coarse_lu_plan(n, ptr, col):
    """Symbolic phase of the banded-LU coarse solver for a host matrix (b200_coarse_lu_plan_i64,
    no device needed): a dict with perm (perm[new] = old), lower / upper (per-row lower and
    per-column upper bandwidth of the permuted matrix), lfirst / ulast (per tile, the first
    and last tile its L and U panels reach), tile_rows, bandwidth, factor_bytes, setup_bytes."""
    L = lib()
    n = int(n)
    ptr = np.ascontiguousarray(ptr, dtype=np.int64)
    col = np.ascontiguousarray(col, dtype=np.int64)
    tiles, rows, bw = _i64(), _c.c_int(), _i64()
    fb, sb = _c.c_size_t(), _c.c_size_t()
    _check(L.b200_coarse_lu_plan_i64(n, _ptr(ptr), _ptr(col), None, None, None, None, None, 0,
                                     _c.byref(tiles), _c.byref(rows), _c.byref(bw), _c.byref(fb),
                                     _c.byref(sb)), "b200_coarse_lu_plan_i64")
    perm = np.empty(n, dtype=np.int32)
    lower = np.empty(n, dtype=np.int32)
    upper = np.empty(n, dtype=np.int32)
    lfirst = np.empty(tiles.value, dtype=np.int64)
    ulast = np.empty(tiles.value, dtype=np.int64)
    _check(L.b200_coarse_lu_plan_i64(n, _ptr(ptr), _ptr(col), _ptr(perm), _ptr(lower), _ptr(upper),
                                     _ptr(lfirst), _ptr(ulast), tiles.value, None, None, None, None, None),
           "b200_coarse_lu_plan_i64")
    return {"perm": perm, "lower": lower, "upper": upper, "lfirst": lfirst, "ulast": ulast,
            "tile_rows": rows.value, "bandwidth": bw.value, "factor_bytes": fb.value,
            "setup_bytes": sb.value}


class Coarse:
    """Coarsest-level device solver (b200_coarse_t): the dense inverse up to 16384 rows, a
    banded LU above."""

    def __init__(self, ctx, n, ptr, col, val):
        self.ctx = ctx
        self.h = _vp()
        ptr = np.ascontiguousarray(ptr, dtype=np.int64)
        col = np.ascontiguousarray(col, dtype=np.int64)
        val = _f64(val)
        _check(lib().b200_coarse_create_i64(ctx.h, int(n), _ptr(ptr), _ptr(col), _ptr(val),
                                            _c.byref(self.h)), "b200_coarse_create")
        self.n = int(n)

    COARSE_KINDS = ("dense_inverse", "banded_lu")

    def info(self):
        """{kind: 'dense_inverse' | 'banded_lu', n, bandwidth, tiles} (b200_coarse_info)."""
        k, n, bw, t = _c.c_int(), _i64(), _i64(), _i64()
        _check(lib().b200_coarse_info(self.h, _c.byref(k), _c.byref(n), _c.byref(bw), _c.byref(t)),
               "b200_coarse_info")
        return {"kind": self.COARSE_KINDS[k.value], "n": n.value, "bandwidth": bw.value, "tiles": t.value}

    def bytes(self):
        b = _c.c_size_t()
        _check(lib().b200_coarse_bytes(self.h, _c.byref(b)), "b200_coarse_bytes")
        return b.value

    def __del__(self):
        try:
            if self.h and lib().b200_coarse_destroy(self.h) == 0:
                self.h = _vp()      # (kept if the library refused, e.g. while a graph is recorded)
        except Exception:
            pass


class Index:
    """Device index list (b200_index_t)."""

    def __init__(self, ctx, idx, size):
        idx = np.ascontiguousarray(idx, dtype=np.int64)
        self.ctx = ctx
        self.n = idx.size
        self.h = _vp()
        _check(lib().b200_index_create_i64(ctx.h, _ptr(idx), idx.size, int(size), _c.byref(self.h)),
               "b200_index_create_i64")

    def __del__(self):
        try:
            if self.h and lib().b200_index_destroy(self.h) == 0:
                self.h = _vp()      # (kept if the library refused, e.g. while a graph is recorded)
        except Exception:
            pass


class Graph:
    """A recorded call sequence (b200_graph_t)."""

    def __init__(self, ctx, h):
        self.ctx = ctx
        self.h = h

    def launch(self):
        """Replay; False (and nothing done) when the vector state differs from recording time."""
        ok = _c.c_int(0)
        _check(lib().b200_graph_launch(self.ctx.h, self.h, _c.byref(ok)), "b200_graph_launch")
        return bool(ok.value)

    def info(self):
        k, n, r, st = _i64(), _i64(), _i64(), _c.c_int(0)
        _check(lib().b200_graph_info(self.h, _c.byref(k), _c.byref(n), _c.byref(r), _c.byref(st)))
        return {"kernels": k.value, "nodes": n.value, "replays": r.value, "stale": bool(st.value)}

    def close(self):
        if self.h:
            lib().b200_graph_destroy(self.h)
            self.h = _vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DropinSolver:
    """amgcl::make_solver<amg<backend::b200<double>, smoothed_aggregation, RELAX>, KRYLOV>
    -- the reference's own templates running on the H100 backend."""

    def __init__(self, ptr, col, val, relax="damped_jacobi", krylov="cg", tol=1e-8,
                 maxiter=100, coarse_enough=-1, ctx=None, precision="f64", graph=False):
        """precision: 'f64' (FP64 throughout) or 'mixed' (amg<backend::b200<float>> hierarchy
        under an FP64 Krylov solver, the reference's mixed-precision composition).
        graph: wrap the hierarchy in amgcl::preconditioner::b200_cycle_graph (every V-cycle
        is one CUDA graph launch); available for damped_jacobi|spai0 x cg|bicgstab and
        damped_jacobi + gmres."""
        D = dropin_lib()
        self.ptr = np.ascontiguousarray(ptr, dtype=np.int64)
        self.col = np.ascontiguousarray(col, dtype=np.int64)
        self.val = _f64(val)
        self.n = self.ptr.size - 1
        self.ctx = ctx
        self.h = _vp()
        if graph:
            rc = D.dropin_create_graph(ctx.h if ctx is not None else None, self.n, _ptr(self.ptr),
                                       _ptr(self.col), _ptr(self.val), RELAX[relax], KRYLOV[krylov],
                                       1 if precision == "mixed" else 0, float(tol), int(maxiter),
                                       int(coarse_enough), _c.byref(self.h))
        else:
            create = D.dropin_create_mixed if precision == "mixed" else D.dropin_create
            rc = create(ctx.h if ctx is not None else None, self.n, _ptr(self.ptr),
                        _ptr(self.col), _ptr(self.val), RELAX[relax], KRYLOV[krylov],
                        float(tol), int(maxiter), int(coarse_enough), _c.byref(self.h))
        if rc != 0:
            raise B200Error("dropin_create: " + D.dropin_last_error().decode(errors="replace"))

    def _err(self, what):
        raise B200Error(what + ": " + dropin_lib().dropin_last_error().decode(errors="replace"))

    def solve(self, rhs, x0=None):
        """End-to-end call with host buffers. Returns (x, iters, resid)."""
        rhs = _f64(rhs)
        x = np.zeros(self.n) if x0 is None else _f64(x0).copy()
        it = _i64()
        res = _dbl()
        if dropin_lib().dropin_solve(self.h, _ptr(rhs), _ptr(x), _c.byref(it), _c.byref(res)):
            self._err("dropin_solve")
        return x, it.value, res.value

    def solve_into(self, rhs, x):
        """Same as solve() but on caller-provided (e.g. pinned) host arrays; x is in/out."""
        it = _i64()
        res = _dbl()
        if dropin_lib().dropin_solve(self.h, _ptr(rhs), _ptr(x), _c.byref(it), _c.byref(res)):
            self._err("dropin_solve")
        return it.value, res.value

    def solve_zero_guess_into(self, rhs, x_out):
        """Host rhs in, host solution out, x0 = 0 created on the device (the tutorial's call
        pattern): one H2D and one D2H copy per solve."""
        it = _i64()
        res = _dbl()
        if dropin_lib().dropin_solve_zero_guess(self.h, _ptr(rhs), _ptr(x_out), _c.byref(it),
                                                _c.byref(res)):
            self._err("dropin_solve_zero_guess")
        return it.value, res.value

    def upload_rhs(self, rhs):
        rhs = _f64(rhs)
        if dropin_lib().dropin_upload_rhs(self.h, _ptr(rhs)):
            self._err("dropin_upload_rhs")

    def solve_resident(self):
        it = _i64()
        res = _dbl()
        if dropin_lib().dropin_solve_resident(self.h, _c.byref(it), _c.byref(res)):
            self._err("dropin_solve_resident")
        return it.value, res.value

    def download_x(self):
        x = np.empty(self.n)
        if dropin_lib().dropin_download_x(self.h, _ptr(x)):
            self._err("dropin_download_x")
        return x

    def apply_precond(self, f):
        f = _f64(f)
        x = np.empty(self.n)
        if dropin_lib().dropin_apply_precond(self.h, _ptr(f), _ptr(x)):
            self._err("dropin_apply_precond")
        return x

    def graph_stats(self):
        """(recorded graphs, kernels per replay, replays so far); zeros without graph=True."""
        g, k, r = _i64(), _i64(), _i64()
        dropin_lib().dropin_graph_stats(self.h, _c.byref(g), _c.byref(k), _c.byref(r))
        return g.value, k.value, r.value

    def report(self):
        need = dropin_lib().dropin_report(self.h, None, 0)
        buf = _c.create_string_buffer(int(need))
        dropin_lib().dropin_report(self.h, buf, need)
        return buf.value.decode(errors="replace")

    def close(self):
        if self.h:
            dropin_lib().dropin_destroy(self.h)
            self.h = _vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def set_setup_threads(n):
    """OpenMP threads for AMGCL's host-side hierarchy setup inside the drop-in library."""
    dropin_lib().dropin_set_num_threads(int(n))


def nccl_unique_id():
    """128-byte NCCL id (call on rank 0, ship to the other ranks, pass to Context.dist_init)."""
    buf = _c.create_string_buffer(128)
    _check(lib().b200_nccl_unique_id(buf, 128), "b200_nccl_unique_id")
    return bytes(buf.raw)


def partition(n, nranks, rank):
    """(block, lo, hi) of the uniform row-block partition the library uses."""
    b, lo, hi = _i64(), _i64(), _i64()
    _check(lib().b200_partition(int(n), int(nranks), int(rank), _c.byref(b), _c.byref(lo),
                                _c.byref(hi)), "b200_partition")
    return b.value, lo.value, hi.value


def dist_split(kind, nranks, rank, nrows, ncols, ptr, col, val):
    """Host view of one rank's share of an operator: always whole rows (the rank's block of
    the row partition).  kind 'halo': the vector the operator is applied to is partitioned --
    local columns become [0, n_loc), columns owned by rank o become n_loc + o*slots + position
    in o's send list; kind 'replicated': that vector is replicated, columns stay global.
    ('square' is an alias of 'halo'.)  Returns dict(nrows, ncols, n_loc, slots, ptr, col, val,
    send_idx)."""
    k = {"halo": 1, "square": 1, "replicated": 2}[kind]
    ptr = np.ascontiguousarray(ptr, dtype=np.int64)
    col = np.ascontiguousarray(col, dtype=np.int64)
    val = _f64(val)
    h = _vp()
    _check(lib().b200_dist_split_i64(k, int(nranks), int(rank), int(nrows), int(ncols), _ptr(ptr),
                                     _ptr(col), _ptr(val), _c.byref(h)), "b200_dist_split_i64")
    try:
        nr, nc, nnz, nl, S, ns = (_i64() for _ in range(6))
        _check(lib().b200_split_info(h, _c.byref(nr), _c.byref(nc), _c.byref(nnz), _c.byref(nl),
                                     _c.byref(S), _c.byref(ns)))
        p = np.zeros(nr.value + 1, dtype=np.int64)
        c = np.zeros(nnz.value, dtype=np.int64)
        v = np.zeros(nnz.value, dtype=np.float64)
        si = np.zeros(ns.value, dtype=np.int64)
        _check(lib().b200_split_copy(h, _ptr(p), _ptr(c), _ptr(v), _ptr(si)))
    finally:
        lib().b200_split_destroy(h)
    return {"nrows": nr.value, "ncols": nc.value, "n_loc": nl.value, "slots": S.value,
            "ptr": p, "col": c, "val": v, "send_idx": si}


def _morton_order(pts, bits=10):
    """Indices that sort 3-D points along a Z-order (Morton) curve: the locality a mesh
    generator's numbering typically has."""
    q = np.minimum((pts * (1 << bits)).astype(np.uint64), (1 << bits) - 1)
    code = np.zeros(pts.shape[0], dtype=np.uint64)
    for b in range(bits):
        for d in range(3):
            code |= ((q[:, d] >> np.uint64(b)) & np.uint64(1)) << np.uint64(3 * b + d)
    return np.argsort(code, kind="stable")


def unstructured3d(n, k=24, seed=0, order="morton"):
    """Synthetic stand-in for BASELINE.json config #4 (poisson3Db.mtx is not available offline):
    an SPD weighted graph Laplacian (+ small diagonal shift) on n random points of the unit
    cube, each connected to its k nearest neighbours with weight 1/d^2 (finite-element-like:
    near neighbours are strongly coupled), symmetrised -- an unstructured CSR with the row
    statistics of poisson3Db (85,623 rows, ~28 nnz/row at n = 85623, k = 24).  order="morton"
    numbers the points along a space-filling curve (mesh-like locality); order="random" keeps
    the random point order (worst case for the x-gathers).  Returns (ptr, col, val, rhs)."""
    import scipy.sparse as sp
    from scipy.spatial import cKDTree
    rng = np.random.default_rng(seed)
    pts = rng.uniform(0.0, 1.0, (int(n), 3))
    if order == "morton":
        pts = pts[_morton_order(pts)]
    dist, nbr = cKDTree(pts).query(pts, k=k + 1)
    rows = np.repeat(np.arange(n), k)
    cols = nbr[:, 1:].reshape(-1)
    h2 = float(np.median(dist[:, 1])) ** 2
    w = h2 / (dist[:, 1:].reshape(-1) ** 2 + 1e-3 * h2)
    W = sp.coo_matrix((w, (rows, cols)), shape=(n, n)).tocsr()
    W = W.maximum(W.T)                                 # symmetric weights
    deg = np.asarray(W.sum(axis=1)).ravel()
    A = (sp.diags(deg * (1.0 + 1e-3)) - W).tocsr()
    A.sort_indices()
    rhs = np.ones(n)
    return (A.indptr.astype(np.int64), A.indices.astype(np.int64),
            np.ascontiguousarray(A.data, dtype=np.float64), rhs)


def poisson3d(n, dtype_index=np.int64, anisotropy=1.0, convection=0.0):
    """3-D 7-point Poisson problem on an n^3 grid, natural ordering (i fastest),
    Dirichlet by truncation, rhs == 1: the same system the reference's tests generate
    (tests/sample_problem.hpp:11-82; hx = 1, hy = anisotropy, hz = anisotropy^2, so the
    default is diag 6, off-diag -1), built here with numpy.  convection > 0 adds a first-order
    upwind transport term with velocity (c, c/2, c/4) -- not in the reference's generator --
    which makes the matrix non-symmetric (for the BiCGStab / GMRES parity cases).
    Returns (ptr, col, val, rhs)."""
    n = int(n)
    n3 = n * n * n
    idx = np.arange(n3, dtype=np.int64)
    i = idx % n
    j = (idx // n) % n
    k = idx // (n * n)
    # neighbour order inside a row: k-1, j-1, i-1, diag, i+1, j+1, k+1
    offs = np.array([-n * n, -n, -1, 0, 1, n, n * n], dtype=np.int64)
    mask = np.empty((n3, 7), dtype=bool)
    mask[:, 0] = k > 0
    mask[:, 1] = j > 0
    mask[:, 2] = i > 0
    mask[:, 3] = True
    mask[:, 4] = i + 1 < n
    mask[:, 5] = j + 1 < n
    mask[:, 6] = k + 1 < n
    del i, j, k
    counts = mask.sum(axis=1)
    ptr = np.zeros(n3 + 1, dtype=np.int64)
    np.cumsum(counts, out=ptr[1:])
    cols = (idx[:, None] + offs[None, :])[mask]
    hx = 1.0
    hy = hx * float(anisotropy)
    hz = hy * float(anisotropy)
    ax, ay, az = 1.0 / (hx * hx), 1.0 / (hy * hy), 1.0 / (hz * hz)
    c = float(convection)
    stencil = np.array([-az - c / 4, -ay - c / 2, -ax - c,
                        (2 / (hx * hx) + 2 / (hy * hy) + 2 / (hz * hz)) + (c + c / 2 + c / 4),
                        -ax, -ay, -az])
    vals = np.broadcast_to(stencil, (n3, 7))[mask]
    rhs = np.ones(n3)
    return (ptr.astype(dtype_index), np.ascontiguousarray(cols, dtype=dtype_index),
            np.ascontiguousarray(vals, dtype=np.float64), rhs)
