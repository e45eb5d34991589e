"""ctypes binding of libls_b200.so (the C ABI declared in include/largesteps_b200.h; timing harnesses and per-phase
counters in include/largesteps_b200_diag.h).

There is NO CPU / torch fallback: if the shared library is missing the import of any operator fails loudly with
instructions to build it (`python -c "import __graft_entry__ as g; g.build()"` or `make -C csrc`).
"""
import ctypes
import os
from ctypes import c_int, c_int32, c_int64, c_uint32, c_uint64, c_size_t, c_float, c_void_p, c_char_p, POINTER

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("LS_LIB_PATH") or os.path.join(_HERE, "libls_b200.so")   # LS_LIB_PATH: A/B builds while tuning

LS_OK, LS_ERR_BAD_ARG, LS_ERR_CUDA, LS_ERR_BREAKDOWN, LS_ERR_NOT_CONVERGED, LS_ERR_UNSUPPORTED, \
    LS_ERR_INDEX_RANGE, LS_ERR_WORKSPACE = range(8)

# every symbol include/largesteps_b200.h and largesteps_b200_diag.h declare: name -> (restype, argtypes)
SYMBOLS = {
    "ls_version": (c_int, []),
    "ls_last_error": (c_char_p, []),
    "ls_status_string": (c_char_p, [c_int]),
    "ls_launch_count": (c_uint64, []),
    "ls_assemble_workspace_bytes": (c_int, [c_int64, c_int64, POINTER(c_size_t)]),
    "ls_assemble_count": (c_int, [c_void_p, c_int, c_int64, c_int64, c_void_p, c_size_t, POINTER(c_int64), c_void_p]),
    "ls_assemble_fill": (c_int, [c_void_p, c_int, c_void_p, c_int64, c_int64, c_int, c_float, c_float,
                                 c_void_p, c_size_t, c_int64, c_void_p, c_void_p, c_void_p,
                                 c_void_p, c_void_p, c_void_p, c_void_p]),
    "ls_laplacian_cot_bwd_scratch_bytes": (c_int, [c_int64, POINTER(c_size_t)]),
    "ls_laplacian_cot_bwd_f32": (c_int, [c_void_p, c_void_p, c_int, c_int64, c_int64, c_float, c_void_p, c_void_p, c_void_p,
                                         c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p]),
    "ls_cot_laplacian_product_scratch_bytes": (c_int, [c_int64, POINTER(c_size_t)]),
    "ls_cot_laplacian_product_f32": (c_int, [c_void_p, c_void_p, c_int, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_int,
                                             c_void_p, c_void_p, c_void_p]),
    "ls_cot_laplacian_product_bwd_f32": (c_int, [c_void_p, c_void_p, c_int, c_int64, c_int64, c_void_p, c_void_p, c_void_p,
                                                 c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "ls_coo_to_csr": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_void_p, c_void_p]),
    "ls_spmm_csr_f32": (c_int, [c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_int64, c_int, c_void_p]),
    "ls_spmm_csr_grad_val_f32": (c_int, [c_int64, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_int64, c_int, c_void_p,
                                         c_void_p]),
    "ls_pcg_workspace_bytes": (c_int, [c_int64, c_int64, c_int, POINTER(c_size_t)]),
    "ls_pcg_create": (c_int, [POINTER(c_void_p), c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                              c_void_p, c_size_t, c_void_p]),
    "ls_order_workspace_bytes": (c_int, [c_int64, POINTER(c_size_t)]),
    "ls_order_morton": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_size_t, c_void_p]),
    "ls_pcg_solve": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_float, c_int, c_void_p,
                             POINTER(c_float), c_void_p]),
    "ls_pcg_destroy": (c_int, [c_void_p]),
    "ls_pcg_set_refinement": (c_int, [c_void_p, c_int, c_float]),
    "ls_pcg_bench_spmm": (c_int, [c_void_p, c_int, c_int, c_void_p]),
    "ls_pcg_spmm_bytes": (c_int64, [c_void_p, c_int]),
    "ls_pcg_describe": (c_int, [c_void_p, POINTER(c_int64)]),
    "ls_pcg_bench": (c_int, [POINTER(c_void_p), c_int, c_int, c_int, c_int, c_void_p]),
    "ls_pcg_spmv_put": (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    "ls_pcg_spmv_get": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "ls_pcg_phase_cycles": (c_int, [c_void_p, POINTER(c_int64), c_int, c_void_p]),
    "ls_pcg_pattern_copy": (c_int, [c_void_p, POINTER(c_int64), POINTER(c_int32), POINTER(c_uint32), c_void_p]),
    "ls_pcg_batch_create": (c_int, [POINTER(c_void_p), POINTER(c_void_p), c_int, c_void_p]),
    "ls_pcg_batch_solve": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_float, c_int, c_void_p,
                                   POINTER(c_float), c_void_p]),
    "ls_pcg_batch_destroy": (c_int, [c_void_p]),
    "ls_pcg_batch_plan_ex": (c_int, [c_int, POINTER(c_int32), POINTER(c_int32), POINTER(c_int32), c_int, POINTER(c_int32),
                                     POINTER(c_int32), POINTER(c_int32), POINTER(c_int32)]),
    "ls_pcg_plan": (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_int, POINTER(c_int64)]),
    "ls_glue_scratch_bytes": (c_int, [POINTER(c_size_t)]),
    "ls_bucket_workspace_bytes": (c_int, [c_int64, POINTER(c_size_t)]),
    "ls_face_incidence": (c_int, [c_void_p, c_int, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "ls_index_buckets": (c_int, [c_void_p, c_int, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "ls_gather_rows_f32": (c_int, [c_void_p, c_void_p, c_int, c_int64, c_int, c_void_p, c_void_p]),
    "ls_gather_rows_bwd_f32": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p]),
    "ls_face_normals_f32": (c_int, [c_void_p, c_void_p, c_int, c_int64, c_void_p, c_void_p]),
    "ls_face_normals_bwd_f32": (c_int, [c_void_p, c_void_p, c_int, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "ls_vertex_normals_f32": (c_int, [c_void_p, c_void_p, c_int, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                      c_void_p, c_void_p, c_void_p]),
    "ls_vertex_normals_bwd_f32": (c_int, [c_void_p, c_void_p, c_int, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                          c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "ls_massmatrix_voronoi_f32": (c_int, [c_void_p, c_void_p, c_int, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_void_p]),
    "ls_massmatrix_voronoi_bwd_f32": (c_int, [c_void_p, c_void_p, c_int, c_int64, c_int64, c_void_p, c_void_p, c_void_p,
                                              c_void_p, c_void_p]),
    "ls_vertex_normals_batch_scratch_bytes": (c_int, [c_int, POINTER(c_size_t)]),
    "ls_vertex_normals_batch_f32": (c_int, [c_void_p, c_void_p, c_int, c_int64, c_int64, c_int, c_void_p, c_void_p,
                                            c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                            c_void_p, c_size_t, c_void_p]),
    "ls_vertex_normals_batch_bwd_f32": (c_int, [c_void_p, c_void_p, c_int, c_int64, c_int64, c_int, c_void_p, c_void_p,
                                                c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "ls_distance_bvh_bytes": (c_int, [c_int64, POINTER(c_size_t)]),
    "ls_distance_bvh_build": (c_int, [c_void_p, c_int64, c_void_p, c_int, c_int64, c_void_p, c_size_t, c_void_p]),
    "ls_distance_query_workspace_bytes": (c_int, [c_int64, POINTER(c_size_t)]),
    "ls_distance_query": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_size_t,
                                  c_void_p]),
    "ls_distance_result": (c_int, [c_void_p, POINTER(ctypes.c_double), c_void_p]),
    "ls_distance_grad_workspace_bytes": (c_int, [c_int64, c_int64, c_int64, POINTER(c_size_t)]),
    "ls_distance_grad_f32": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int, c_int64, c_void_p, c_void_p, c_void_p,
                                     c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "ls_distance_bvh_batch_bytes": (c_int, [c_int64, c_int64, POINTER(c_size_t)]),
    "ls_distance_bvh_batch_build": (c_int, [c_void_p, c_int64, c_void_p, c_int, c_int64, c_int64, c_void_p, c_void_p, c_size_t,
                                            c_void_p]),
    "ls_distance_query_batch_workspace_bytes": (c_int, [c_int64, c_int64, POINTER(c_size_t)]),
    "ls_distance_query_batch": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_int64, c_int64, c_void_p, c_void_p, c_void_p,
                                        c_void_p, c_void_p, c_int, c_void_p, c_size_t, c_void_p]),
    "ls_distance_segment_sum_f64": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_void_p, c_void_p]),
    "ls_remesh_workspace_bytes": (c_int, [c_int64, c_int64, POINTER(c_size_t)]),
    "ls_remesh_check": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_size_t, POINTER(c_uint32), c_void_p]),
    "ls_remesh_split": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, ctypes.c_double, c_void_p, c_size_t,
                                POINTER(c_int64), c_void_p]),
    "ls_remesh_collapse_round": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, ctypes.c_double, ctypes.c_double, c_void_p,
                                         c_size_t, POINTER(c_int64), c_void_p]),
    "ls_remesh_compact": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_size_t, POINTER(c_int64), POINTER(c_int64),
                                  c_void_p]),
    "ls_remesh_flip_round": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_size_t, POINTER(c_int64), c_void_p]),
    "ls_remesh_relax": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_int64, c_void_p, c_size_t, c_void_p]),
    "ls_remesh_split_v": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, ctypes.c_double, c_void_p, c_void_p,
                                  c_void_p, c_void_p, c_size_t, POINTER(c_int64), c_void_p]),
    "ls_remesh_collapse_round_v": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, ctypes.c_double, ctypes.c_double,
                                           c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, POINTER(c_int64), c_void_p]),
    "ls_remesh_compact_v": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t,
                                    POINTER(c_int64), POINTER(c_int64), c_void_p]),
    "ls_remesh_flip_round_v": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t,
                                       POINTER(c_int64), c_void_p]),
    "ls_remesh_relax_v": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p,
                                  c_size_t, c_void_p]),
    "ls_adam_uniform_step": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_float, c_float, c_float,
                                     c_float, c_float, c_float, c_float, c_void_p, c_void_p]),
    "ls_adam_uniform_step_multi": (c_int, [c_void_p, c_int, c_void_p, c_size_t, c_void_p]),
}

# one entry of ls_adam_uniform_step_multi's table (ls_adam_tensor): four pointers, the size, seven floats, padded to 8 bytes
ADAM_TENSOR = np.dtype([("param", np.uint64), ("grad", np.uint64), ("g1", np.uint64), ("g2", np.uint64), ("n", np.int64),
                        ("lr", np.float32), ("beta1", np.float32), ("beta2", np.float32), ("one_minus_beta1", np.float32),
                        ("one_minus_beta2", np.float32), ("c1", np.float32), ("c2", np.float32)], align=True)

_lib = None


class NativeLibraryMissing(ImportError):
    pass


def lib():
    """Load (once) and return the ctypes handle.  Raises NativeLibraryMissing if the .so is not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise NativeLibraryMissing(
                f"{LIB_PATH} not found: the CUDA library is not built. Build it with "
                "`python -c 'import __graft_entry__ as g; g.build()'` from the repo root "
                "(or `make -C large-steps-pytorch_b200/csrc`). There is no CPU fallback.")
        h = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(h, name)     # AttributeError if the header and the library drift apart
            fn.restype = res
            fn.argtypes = args
        _lib = h
    return _lib


def last_error():
    return lib().ls_last_error().decode("utf-8", "replace")


def check(rc, what=""):
    """Map an ls_status to the Python exception the reference surface would raise."""
    if rc == LS_OK:
        return
    msg = f"{what}: {last_error()}" if what else last_error()
    if rc == LS_ERR_BAD_ARG:
        raise ValueError(msg)
    if rc == LS_ERR_INDEX_RANGE:
        raise IndexError(msg)
    if rc == LS_ERR_NOT_CONVERGED:
        raise NotConverged(msg)
    if rc == LS_ERR_BREAKDOWN:
        raise Breakdown(msg)
    raise RuntimeError(f"[ls_status {rc}: {lib().ls_status_string(rc).decode()}] {msg}")


class NotConverged(RuntimeError):
    pass


class Breakdown(RuntimeError):
    pass


def stream_ptr(device=None):
    return c_void_p(torch.cuda.current_stream(device).cuda_stream)


def ptr(t):
    return c_void_p(t.data_ptr()) if t is not None else c_void_p(0)


def require_cuda(t, name):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor: largesteps_b200 runs on the GPU only (no CPU path)")


def launch_count():
    return int(lib().ls_launch_count())
