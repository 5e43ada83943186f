"""ctypes binding of libvpca.so (include/vpca.h) -- the Python twin of the JNI class ``NativePca``
shown in INTEGRATION.md.  One ``NativePca`` object = one ``vpca_ctx`` = one GPU.

There is no CPU fallback: importing this module never fails (so host logic stays testable without a
GPU), but constructing ``NativePca`` raises ``VpcaError`` when the CUDA library is missing or no
sm_90 device is usable.
"""
from __future__ import annotations

import ctypes
import os
from pathlib import Path
from typing import Optional, Tuple

import numpy as np

VPCA_OK = 0
VPCA_ERR_BAD_ARG = -1
VPCA_ERR_INDEX_OUT_OF_RANGE = -2
VPCA_ERR_CUDA = -3
VPCA_ERR_NCCL = -4
VPCA_ERR_OVERFLOW = -5
VPCA_ERR_STATE = -6
VPCA_ERR_NOMEM = -7
VPCA_ERR_UNSUPPORTED = -8
JOIN, MERGE = 0, 1    # vpca_join_rows modes (VPCA_JOIN / VPCA_MERGE)

DTYPE_I8 = 0
DTYPE_BF16 = 1
DTYPE_E2M1 = 2   # 4-bit cells, two per byte (cell j of a row in nibble j & 1 of byte j // 2; value m is the code 2 m)

_STATUS_NAMES = {
    -1: "BAD_ARG", -2: "INDEX_OUT_OF_RANGE", -3: "CUDA", -4: "NCCL", -5: "OVERFLOW", -6: "STATE",
    -7: "NOMEM", -8: "UNSUPPORTED",
}

# every symbol include/vpca.h declares (checked by tests/test_abi.py against the header)
EXPORTED_SYMBOLS = (
    "vpca_version", "vpca_create", "vpca_destroy", "vpca_last_error", "vpca_reset", "vpca_encode_calls",
    "vpca_accumulate_calls", "vpca_commit", "vpca_abort", "vpca_accumulate_dense", "vpca_gram_device_ptr",
    "vpca_finalize_gram", "vpca_get_gram", "vpca_set_gram", "vpca_compute_pca", "vpca_get_centered",
    "vpca_get_tridiagonal", "vpca_synth_dense_device", "vpca_get_stats", "vpca_debug_gram_profile",
    "vpca_gram_export_ipc", "vpca_gram_set_peers", "vpca_peer_barrier", "vpca_accumulate_panels",
    "vpca_synth_panels_device", "vpca_accumulate_calls_u16", "vpca_get_partial_gram", "vpca_load_partial_gram",
    "vpca_accumulate_bits", "vpca_gram_set_peer_mode", "vpca_gram_gather", "vpca_accumulate_bed",
    "vpca_synchronize", "vpca_host_alloc", "vpca_host_free", "vpca_gram_set_peers_local", "vpca_owner_row_bands",
    "vpca_get_gram_band", "vpca_variant_count", "vpca_debug_rebalance",
    "vpca_debug_lanczos_profile", "vpca_debug_max_clusters", "vpca_debug_band_tiles", "vpca_hash_keys", "vpca_join_rows", "vpca_join_fetch", "vpca_join_size", "vpca_accumulate_joined",
    "vpca_pool_create", "vpca_pool_destroy", "vpca_pool_size", "vpca_pool_ctx", "vpca_pool_last_error", "vpca_pool_reset",
    "vpca_pool_accumulate_calls", "vpca_pool_accumulate_calls_u16", "vpca_pool_accumulate_bits", "vpca_pool_accumulate_bed",
    "vpca_pool_commit", "vpca_pool_abort", "vpca_pool_reduce_and_finalize", "vpca_pool_get_gram", "vpca_pool_compute_pca",
    "vpca_pool_get_stats", "vpca_debug_tiles", "vpca_debug_plan", "vpca_debug_schedule",
    "vpca_loadings_calls", "vpca_loadings_bed", "vpca_loadings_panels", "vpca_project_begin", "vpca_project_calls",
    "vpca_project_bed", "vpca_project_panels", "vpca_project_get", "vpca_compute_pca_bands",
    "vpca_kinship_bed", "vpca_kinship_pairs", "vpca_compute_pca_subset", "vpca_ld_prune_bed",
    "vpca_ld_prune_bed_masked", "vpca_variant_qc_bed", "vpca_hwe_exact", "vpca_sample_missing_bed",
    "vpca_subset_bed_samples", "vpca_debug_device_bytes", "vpca_grm_bed", "vpca_grm_finalize", "vpca_get_grm",
    "vpca_compute_pca_grm", "vpca_grm_loadings_bed", "vpca_grm_project_bed", "vpca_glm_begin", "vpca_glm_linear_bed",
    "vpca_glm_logistic_begin", "vpca_glm_logistic_bed", "vpca_glm_firth_bed",
)

KINSHIP_MAX_SAMPLES = 21845   # vpca_kinship_*: the 3N x 3N plane Gram stays below 2^32 cells
LD_MAX_WINDOW = 4096          # vpca_ld_prune_bed: variants a window may reach back (VPCA_LD_MAX_WINDOW)
GRM_MAX_SAMPLES = 65535       # vpca_grm_* / vpca_compute_pca_grm: the sample limit of vpca_compute_pca
GLM_MAX_Q = 32                # vpca_glm_begin: covariate columns, the intercept included
GLM_ERRCODES = (".", "TOO_FEW_OBS", "CONST_ALLELE", "VIF_INFINITE", "NO_RESIDUAL",
                "LOGISTIC_CONVERGE_FAIL", "FIRTH_CONVERGE_FAIL")   # by VPCA_GLM_* value
GLM_FIRTH_MODES = {"fallback": 1, "always": 2}   # vpca_glm_firth_bed: VPCA_GLM_FIRTH_FALLBACK, VPCA_GLM_FIRTH_ALWAYS


class VpcaError(RuntimeError):
    """Raised for every negative vpca_status (the JNI shim rethrows the same way as RuntimeException)."""

    def __init__(self, code: int, message: str):
        super().__init__(f"vpca {_STATUS_NAMES.get(code, code)}: {message}")
        self.code = code


class IndexOutOfRange(VpcaError, IndexError):
    """Sample index outside [0, N): the reference throws at VariantsPca.scala:59 / :188."""


class VpcaConfig(ctypes.Structure):
    _fields_ = [
        ("struct_size", ctypes.c_uint32),
        ("n_samples", ctypes.c_int32),
        ("device", ctypes.c_int32),
        ("dtype", ctypes.c_int32),
        ("num_pc", ctypes.c_int32),
        ("max_multiplicity", ctypes.c_int32),
        ("partitions_in_flight", ctypes.c_int32),
        ("staging_lanes", ctypes.c_int32),
        ("chunk_variants", ctypes.c_int64),
        ("chunk_nnz", ctypes.c_int64),
        ("stream", ctypes.c_void_p),
        ("d_gram", ctypes.c_void_p),
        ("gram_band_row0", ctypes.c_int32),
        ("gram_band_rows", ctypes.c_int32),
    ]


class VpcaStats(ctypes.Structure):
    _fields_ = [
        ("variants_accumulated", ctypes.c_int64),
        ("gram_launches", ctypes.c_int64),
        ("kernel_launches", ctypes.c_int64),
        ("h2d_bytes", ctypes.c_int64),
        ("d2h_bytes", ctypes.c_int64),
        ("last_gram_ms", ctypes.c_float),
        ("last_eig_ms", ctypes.c_float),
        ("gram_cta_group", ctypes.c_int32),
        ("gram_resident", ctypes.c_int32),
        ("eig_method", ctypes.c_int32),
        ("eig_iterations", ctypes.c_int32),
    ]


_PKG = Path(__file__).resolve().parent
LIB_PATH = _PKG / "libvpca.so"
_lib: Optional[ctypes.CDLL] = None


def library_path() -> Path:
    return Path(os.environ.get("VPCA_LIBRARY", str(LIB_PATH)))


def load_library() -> ctypes.CDLL:
    """dlopen libvpca.so and declare the prototypes.  Raises VpcaError if the library is not built."""
    global _lib
    if _lib is not None:
        return _lib
    path = library_path()
    if not path.exists():
        raise VpcaError(VPCA_ERR_CUDA, f"{path} not found: build it with `python -c 'import __graft_entry__ as g; "
                        "g.build()'` (there is no CPU fallback)")
    L = ctypes.CDLL(str(path))
    vp, i64, i32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32
    L.vpca_version.restype = ctypes.c_int
    L.vpca_version.argtypes = []
    L.vpca_create.restype = ctypes.c_int
    L.vpca_create.argtypes = [ctypes.POINTER(VpcaConfig), ctypes.POINTER(vp)]
    L.vpca_destroy.restype = ctypes.c_int
    L.vpca_destroy.argtypes = [vp]
    L.vpca_last_error.restype = ctypes.c_char_p
    L.vpca_last_error.argtypes = [vp]
    L.vpca_reset.restype = ctypes.c_int
    L.vpca_reset.argtypes = [vp]
    L.vpca_encode_calls.restype = ctypes.c_int
    L.vpca_encode_calls.argtypes = [vp, vp, vp, i64, vp, i64]
    L.vpca_accumulate_calls.restype = ctypes.c_int
    L.vpca_accumulate_calls.argtypes = [vp, i64, vp, vp, i64]
    L.vpca_accumulate_calls_u16.restype = ctypes.c_int
    L.vpca_accumulate_calls_u16.argtypes = [vp, i64, vp, vp, i64]
    L.vpca_hash_keys.restype = ctypes.c_int
    L.vpca_hash_keys.argtypes = [vp, vp, vp, i64, vp]
    L.vpca_join_rows.restype = ctypes.c_int
    L.vpca_join_rows.argtypes = [vp, i32, i32, i64, vp, vp, vp, vp, i64, ctypes.POINTER(i64), ctypes.POINTER(i64)]
    L.vpca_join_size.restype = ctypes.c_int
    L.vpca_join_size.argtypes = [vp, ctypes.POINTER(i64), ctypes.POINTER(i64)]
    L.vpca_join_fetch.restype = ctypes.c_int
    L.vpca_join_fetch.argtypes = [vp, vp, vp]
    L.vpca_accumulate_joined.restype = ctypes.c_int
    L.vpca_accumulate_joined.argtypes = [vp, i64]
    L.vpca_accumulate_bits.restype = ctypes.c_int
    L.vpca_accumulate_bits.argtypes = [vp, i64, vp, i64, i64]
    L.vpca_accumulate_bed.restype = ctypes.c_int
    L.vpca_accumulate_bed.argtypes = [vp, i64, vp, i64, i64, ctypes.c_int32]
    L.vpca_commit.restype = ctypes.c_int
    L.vpca_commit.argtypes = [vp, i64]
    L.vpca_abort.restype = ctypes.c_int
    L.vpca_abort.argtypes = [vp, i64]
    L.vpca_accumulate_dense.restype = ctypes.c_int
    L.vpca_accumulate_dense.argtypes = [vp, vp, i64, i64, ctypes.c_int]
    L.vpca_gram_device_ptr.restype = ctypes.c_int
    L.vpca_gram_device_ptr.argtypes = [vp, ctypes.POINTER(vp)]
    L.vpca_finalize_gram.restype = ctypes.c_int
    L.vpca_finalize_gram.argtypes = [vp]
    L.vpca_get_gram.restype = ctypes.c_int
    L.vpca_get_gram.argtypes = [vp, vp]
    L.vpca_get_partial_gram.restype = ctypes.c_int
    L.vpca_get_partial_gram.argtypes = [vp, vp, ctypes.POINTER(i64)]
    L.vpca_load_partial_gram.restype = ctypes.c_int
    L.vpca_load_partial_gram.argtypes = [vp, vp, i64]
    L.vpca_variant_count.restype = i64
    L.vpca_variant_count.argtypes = [vp]
    L.vpca_synchronize.restype = ctypes.c_int
    L.vpca_synchronize.argtypes = [vp]
    L.vpca_host_alloc.restype = ctypes.c_int
    L.vpca_host_alloc.argtypes = [ctypes.c_size_t, ctypes.POINTER(vp)]
    L.vpca_host_free.restype = ctypes.c_int
    L.vpca_host_free.argtypes = [vp]
    L.vpca_gram_set_peers_local.restype = ctypes.c_int
    L.vpca_gram_set_peers_local.argtypes = [ctypes.POINTER(vp), i32]
    L.vpca_owner_row_bands.restype = ctypes.c_int
    L.vpca_owner_row_bands.argtypes = [i32, i32, ctypes.POINTER(i32)]
    L.vpca_get_gram_band.restype = ctypes.c_int
    L.vpca_get_gram_band.argtypes = [vp, i32, i32, vp]
    L.vpca_pool_create.restype = ctypes.c_int
    L.vpca_pool_create.argtypes = [ctypes.POINTER(VpcaConfig), i32, ctypes.POINTER(i32), ctypes.POINTER(vp)]
    L.vpca_pool_destroy.restype = ctypes.c_int
    L.vpca_pool_destroy.argtypes = [vp]
    L.vpca_pool_size.restype = i32
    L.vpca_pool_size.argtypes = [vp]
    L.vpca_pool_ctx.restype = vp
    L.vpca_pool_ctx.argtypes = [vp, i64]
    L.vpca_pool_last_error.restype = ctypes.c_char_p
    L.vpca_pool_last_error.argtypes = [vp]
    L.vpca_pool_reset.restype = ctypes.c_int
    L.vpca_pool_reset.argtypes = [vp]
    L.vpca_pool_accumulate_calls.restype = ctypes.c_int
    L.vpca_pool_accumulate_calls.argtypes = [vp, i64, vp, vp, i64]
    L.vpca_pool_accumulate_calls_u16.restype = ctypes.c_int
    L.vpca_pool_accumulate_calls_u16.argtypes = [vp, i64, vp, vp, i64]
    L.vpca_pool_accumulate_bits.restype = ctypes.c_int
    L.vpca_pool_accumulate_bits.argtypes = [vp, i64, vp, i64, i64]
    L.vpca_pool_accumulate_bed.restype = ctypes.c_int
    L.vpca_pool_accumulate_bed.argtypes = [vp, i64, vp, i64, i64, i32]
    L.vpca_pool_commit.restype = ctypes.c_int
    L.vpca_pool_commit.argtypes = [vp, i64]
    L.vpca_pool_abort.restype = ctypes.c_int
    L.vpca_pool_abort.argtypes = [vp, i64]
    L.vpca_pool_reduce_and_finalize.restype = ctypes.c_int
    L.vpca_pool_reduce_and_finalize.argtypes = [vp]
    L.vpca_pool_get_gram.restype = ctypes.c_int
    L.vpca_pool_get_gram.argtypes = [vp, vp]
    L.vpca_pool_compute_pca.restype = ctypes.c_int
    L.vpca_pool_compute_pca.argtypes = [vp, i32, vp, vp, ctypes.POINTER(i32)]
    L.vpca_pool_get_stats.restype = ctypes.c_int
    L.vpca_pool_get_stats.argtypes = [vp, ctypes.POINTER(VpcaStats)]
    L.vpca_debug_tiles.restype = ctypes.c_int
    L.vpca_debug_tiles.argtypes = [i32, i32, i32, vp, i32]
    L.vpca_debug_plan.restype = ctypes.c_int
    L.vpca_debug_plan.argtypes = [vp, i32, i32, i32, vp, i32]
    L.vpca_debug_schedule.restype = ctypes.c_int
    L.vpca_debug_schedule.argtypes = [i32, i32, i32, i32, i32, i32, ctypes.c_double, vp, i32, vp]
    L.vpca_debug_lanczos_profile.restype = ctypes.c_int
    L.vpca_debug_lanczos_profile.argtypes = [vp, vp, i32]
    L.vpca_debug_device_bytes.restype = i64
    L.vpca_debug_device_bytes.argtypes = []
    L.vpca_debug_rebalance.restype = ctypes.c_int
    L.vpca_debug_rebalance.argtypes = [vp, i32, i32, i32, i32, vp, vp, i32]
    L.vpca_set_gram.restype = ctypes.c_int
    L.vpca_set_gram.argtypes = [vp, vp]
    L.vpca_compute_pca.restype = ctypes.c_int
    L.vpca_compute_pca.argtypes = [vp, i32, vp, vp, ctypes.POINTER(i32)]
    L.vpca_compute_pca_bands.restype = ctypes.c_int
    L.vpca_compute_pca_bands.argtypes = [ctypes.POINTER(vp), i32, i32, vp, vp, ctypes.POINTER(i32)]
    L.vpca_get_centered.restype = ctypes.c_int
    L.vpca_get_centered.argtypes = [vp, vp]
    L.vpca_get_tridiagonal.restype = ctypes.c_int
    L.vpca_get_tridiagonal.argtypes = [vp, vp, vp]
    L.vpca_synth_dense_device.restype = ctypes.c_int
    L.vpca_synth_dense_device.argtypes = [vp, ctypes.c_uint64, i64, i64, ctypes.c_int, vp, i64]
    L.vpca_get_stats.restype = ctypes.c_int
    L.vpca_get_stats.argtypes = [vp, ctypes.POINTER(VpcaStats)]
    L.vpca_accumulate_panels.restype = ctypes.c_int
    L.vpca_accumulate_panels.argtypes = [vp, vp, i64, i64]
    L.vpca_synth_panels_device.restype = ctypes.c_int
    L.vpca_synth_panels_device.argtypes = [vp, ctypes.c_uint64, i64, i64, ctypes.c_int, vp, i64]
    L.vpca_gram_export_ipc.restype = ctypes.c_int
    L.vpca_gram_export_ipc.argtypes = [vp, vp]
    L.vpca_gram_set_peers.restype = ctypes.c_int
    L.vpca_gram_set_peers.argtypes = [vp, vp, i32, i32]
    L.vpca_peer_barrier.restype = ctypes.c_int
    L.vpca_peer_barrier.argtypes = [vp]
    L.vpca_gram_set_peer_mode.restype = ctypes.c_int
    L.vpca_gram_set_peer_mode.argtypes = [vp, ctypes.c_int32]
    L.vpca_gram_gather.restype = ctypes.c_int
    L.vpca_gram_gather.argtypes = [vp]
    L.vpca_debug_gram_profile.restype = ctypes.c_int
    L.vpca_debug_gram_profile.argtypes = [vp, vp, i32]
    L.vpca_loadings_calls.restype = ctypes.c_int
    L.vpca_loadings_calls.argtypes = [vp, i32, vp, vp, i64, vp, vp]
    L.vpca_loadings_bed.restype = ctypes.c_int
    L.vpca_loadings_bed.argtypes = [vp, i32, vp, i64, i64, i32, vp, vp]
    L.vpca_loadings_panels.restype = ctypes.c_int
    L.vpca_loadings_panels.argtypes = [vp, i32, vp, i64, i64, vp, vp]
    L.vpca_project_begin.restype = ctypes.c_int
    L.vpca_project_begin.argtypes = [vp, i32]
    L.vpca_project_calls.restype = ctypes.c_int
    L.vpca_project_calls.argtypes = [vp, vp, vp, i64, vp, vp]
    L.vpca_project_bed.restype = ctypes.c_int
    L.vpca_project_bed.argtypes = [vp, vp, i64, i64, i32, vp, vp]
    L.vpca_project_panels.restype = ctypes.c_int
    L.vpca_project_panels.argtypes = [vp, vp, i64, i64, vp, vp]
    L.vpca_project_get.restype = ctypes.c_int
    L.vpca_project_get.argtypes = [vp, vp, vp]
    L.vpca_kinship_bed.restype = ctypes.c_int
    L.vpca_kinship_bed.argtypes = [vp, vp, i64, i64]
    L.vpca_kinship_pairs.restype = ctypes.c_int
    L.vpca_kinship_pairs.argtypes = [vp, ctypes.c_double, i64, vp, vp, vp, ctypes.POINTER(i64)]
    L.vpca_ld_prune_bed.restype = ctypes.c_int
    L.vpca_ld_prune_bed.argtypes = [vp, vp, i64, i64, vp, ctypes.c_double, vp, i64, vp, vp, ctypes.POINTER(i64)]
    L.vpca_ld_prune_bed_masked.restype = ctypes.c_int
    L.vpca_ld_prune_bed_masked.argtypes = [vp, vp, i64, i64, vp, vp, ctypes.c_double, vp, i64, vp, vp, ctypes.POINTER(i64)]
    L.vpca_variant_qc_bed.restype = ctypes.c_int
    L.vpca_variant_qc_bed.argtypes = [vp, vp, i64, i64, vp, vp]
    L.vpca_hwe_exact.restype = ctypes.c_int
    L.vpca_hwe_exact.argtypes = [vp, vp, i64, vp]
    L.vpca_sample_missing_bed.restype = ctypes.c_int
    L.vpca_sample_missing_bed.argtypes = [vp, vp, i64, i64, i32, vp]
    L.vpca_subset_bed_samples.restype = ctypes.c_int
    L.vpca_subset_bed_samples.argtypes = [vp, vp, i64, i64, i32, vp, i32, vp, i64]
    L.vpca_compute_pca_subset.restype = ctypes.c_int
    L.vpca_compute_pca_subset.argtypes = [vp, vp, i32, vp, vp, ctypes.POINTER(i32)]
    L.vpca_grm_bed.restype = ctypes.c_int
    L.vpca_grm_bed.argtypes = [vp, vp, i64, i64]
    L.vpca_grm_finalize.restype = ctypes.c_int
    L.vpca_grm_finalize.argtypes = [vp, ctypes.POINTER(i64)]
    L.vpca_get_grm.restype = ctypes.c_int
    L.vpca_get_grm.argtypes = [vp, vp]
    L.vpca_compute_pca_grm.restype = ctypes.c_int
    L.vpca_compute_pca_grm.argtypes = [vp, i32, vp, vp]
    L.vpca_grm_loadings_bed.restype = ctypes.c_int
    L.vpca_grm_loadings_bed.argtypes = [vp, i32, vp, i64, i64, vp, vp]
    L.vpca_grm_project_bed.restype = ctypes.c_int
    L.vpca_grm_project_bed.argtypes = [vp, vp, i64, i64, vp, vp]
    L.vpca_glm_begin.restype = ctypes.c_int
    L.vpca_glm_begin.argtypes = [vp, vp, vp, i32, ctypes.POINTER(i64)]
    L.vpca_glm_linear_bed.restype = ctypes.c_int
    L.vpca_glm_linear_bed.argtypes = [vp, vp, i64, i64, i32, vp, vp]
    L.vpca_glm_logistic_begin.restype = ctypes.c_int
    L.vpca_glm_logistic_begin.argtypes = [vp, vp, vp, i32, ctypes.POINTER(i64)]
    L.vpca_glm_logistic_bed.restype = ctypes.c_int
    L.vpca_glm_logistic_bed.argtypes = [vp, vp, i64, i64, i32, vp, vp, vp]
    L.vpca_glm_firth_bed.restype = ctypes.c_int
    L.vpca_glm_firth_bed.argtypes = [vp, vp, i64, i64, i32, i32, vp, vp, vp, vp]
    _lib = L
    return L


def _host_ptr(a: np.ndarray) -> int:
    return a.ctypes.data


_NO_ROWS = np.zeros(1, np.uint8)   # the address passed for zero rows: vpca_ld_prune_bed refuses NULL rows even then


def _bed_rows(rows) -> Tuple[np.ndarray, int]:
    """(V, stride) uint8 rows as they are when already so (a .bed memmap is read in place), else a C-ordered copy, and
    their address, valid even for V = 0."""
    b = np.asarray(rows)
    if b.ndim != 2 or b.dtype != np.uint8 or not b.flags.c_contiguous:
        b = np.ascontiguousarray(b, dtype=np.uint8)
    if b.ndim != 2:
        raise VpcaError(VPCA_ERR_BAD_ARG, "rows must be (nv, stride_bytes)")
    return b, b.ctypes.data if b.size else _NO_ROWS.ctypes.data


class NativePca:
    """One GPU's VariantsPca state.  Method names follow the JNI class of INTEGRATION.md 1:1."""

    def __init__(self, n_samples: int, device: int = 0, dtype: int = DTYPE_I8, num_pc: int = 2,
                 max_multiplicity: int = 2, partitions_in_flight: int = 4, chunk_variants: int = 0,
                 chunk_nnz: int = 0, stream: int = 0, d_gram: int = 0, staging_lanes: int = 0,
                 gram_band: Optional[Tuple[int, int]] = None):
        self._lib = load_library()
        self.n = int(n_samples)
        self.dtype = int(dtype)
        self.elem_bits = {DTYPE_I8: 8, DTYPE_BF16: 16, DTYPE_E2M1: 4}[self.dtype]
        self.elem_bytes = self.elem_bits / 8
        self.max_multiplicity = int(max_multiplicity) if max_multiplicity > 0 else 2
        row0, rows = gram_band if gram_band is not None else (0, 0)
        cfg = VpcaConfig(ctypes.sizeof(VpcaConfig), n_samples, device, dtype, num_pc, max_multiplicity,
                         partitions_in_flight, staging_lanes, chunk_variants, chunk_nnz, stream or None, d_gram or None,
                         row0, rows)
        handle = ctypes.c_void_p()
        rc = self._lib.vpca_create(ctypes.byref(cfg), ctypes.byref(handle))
        self._h = handle if rc == VPCA_OK else None
        if rc != VPCA_OK:
            self._raise(rc, None)

    # -- error plumbing ------------------------------------------------------------------------
    def _raise(self, rc: int, handle):
        msg = self._lib.vpca_last_error(handle).decode("utf-8", "replace")
        if rc == VPCA_ERR_INDEX_OUT_OF_RANGE:
            raise IndexOutOfRange(rc, msg)
        raise VpcaError(rc, msg)

    def _check(self, rc: int):
        if rc != VPCA_OK:
            self._raise(rc, self._h)

    def close(self):
        if getattr(self, "_h", None) is not None:
            self._lib.vpca_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    # -- API -------------------------------------------------------------------------------------
    def reset(self):
        self._check(self._lib.vpca_reset(self._h))

    @staticmethod
    def _csr(offsets, sample_idx) -> Tuple[np.ndarray, np.ndarray]:
        off = np.ascontiguousarray(offsets, dtype=np.int64)
        idx = np.ascontiguousarray(sample_idx, dtype=np.int32)
        if off.ndim != 1 or len(off) < 1:
            raise VpcaError(VPCA_ERR_BAD_ARG, "offsets must be a 1-D array with nv+1 entries")
        return off, idx

    def encodeCalls(self, offsets, sample_idx) -> np.ndarray:
        """Device encode only (CSR rows -> dense sample-major tile), copied back: shape (n, nv)."""
        off, idx = self._csr(offsets, sample_idx)
        nv = len(off) - 1
        if self.elem_bits == 4:                      # packed: (n, ld / 2) bytes, ld a multiple of 128 cells
            ld = max(128, ((nv + 127) // 128) * 128)
            out = np.zeros((self.n, ld // 2), dtype=np.uint8)
            self._check(self._lib.vpca_encode_calls(self._h, _host_ptr(off), _host_ptr(idx) if len(idx) else None, nv,
                                                    _host_ptr(out), ld))
            return out
        out = np.zeros((self.n, max(nv, 1)), dtype=np.int8 if self.elem_bits == 8 else np.uint16)
        self._check(self._lib.vpca_encode_calls(self._h, _host_ptr(off), _host_ptr(idx) if len(idx) else None, nv,
                                                _host_ptr(out), out.shape[1]))
        return out[:, :nv]

    def accumulateCalls(self, partition_id: int, offsets, sample_idx):
        off, idx = self._csr(offsets, sample_idx)
        self._check(self._lib.vpca_accumulate_calls(self._h, int(partition_id), _host_ptr(off),
                                                    _host_ptr(idx) if len(idx) else None, len(off) - 1))

    # -- multi-dataset keying on the device (VariantsPca.scala:62-78, :115-148) --------------------------------------
    @staticmethod
    def _keys(keys):
        """list of bytes -> (payload uint8, key_offsets int64)"""
        lens = np.fromiter((len(k) for k in keys), dtype=np.int64, count=len(keys))
        koff = np.zeros(len(keys) + 1, dtype=np.int64)
        np.cumsum(lens, out=koff[1:])
        payload = np.frombuffer(b"".join(keys), dtype=np.uint8) if len(keys) else np.zeros(0, np.uint8)
        return np.ascontiguousarray(payload), koff

    def hashKeys(self, keys) -> np.ndarray:
        """MurmurHash3_x64_128 of every byte string in `keys`, computed on the GPU: (len(keys), 2) uint64 (h1, h2);
        `bytes(row).hex()` of a little-endian row is Guava's HashCode.toString (vpca_hash_keys)."""
        payload, koff = self._keys(keys)
        out = np.zeros((len(keys), 2), dtype=np.uint64)
        self._check(self._lib.vpca_hash_keys(self._h, _host_ptr(payload) if len(payload) else None, _host_ptr(koff),
                                             len(keys), _host_ptr(out) if len(keys) else None))
        return out

    def joinRows(self, mode: int, keys, offsets, sample_idx, n_left: int = 0, variant_set_count: int = 2):
        """Join (mode JOIN: rows [0, n_left) x rows [n_left, ...)) or merge (mode MERGE) of the rows of several datasets on
        their variant keys, on the GPU; the joined rows stay there (accumulateJoined / joinFetch).  Returns (rows, calls)."""
        payload, koff = self._keys(keys)
        off, idx = self._csr(offsets, sample_idx)
        if len(off) - 1 != len(keys):
            raise VpcaError(VPCA_ERR_BAD_ARG, "one key per row")
        rows, nnz = ctypes.c_int64(0), ctypes.c_int64(0)
        self._check(self._lib.vpca_join_rows(self._h, int(mode), int(variant_set_count), int(n_left),
                                             _host_ptr(payload) if len(payload) else None, _host_ptr(koff), _host_ptr(off),
                                             _host_ptr(idx) if len(idx) else None, len(keys), ctypes.byref(rows),
                                             ctypes.byref(nnz)))
        return int(rows.value), int(nnz.value)

    def joinSize(self):
        """(rows, calls) of the joined rows the context retains (vpca_join_size)."""
        rows, nnz = ctypes.c_int64(0), ctypes.c_int64(0)
        self._check(self._lib.vpca_join_size(self._h, ctypes.byref(rows), ctypes.byref(nnz)))
        return int(rows.value), int(nnz.value)

    def joinFetch(self, rows: int, nnz: int):
        """The joined rows of the last joinRows as a host CSR (offsets int64, sample indices int32)."""
        off = np.zeros(rows + 1, dtype=np.int64)
        idx = np.zeros(max(nnz, 1), dtype=np.int32)
        self._check(self._lib.vpca_join_fetch(self._h, _host_ptr(off), _host_ptr(idx)))
        return off, idx[:nnz]

    def lanczosProfile(self) -> np.ndarray:
        """(steps, 8) int64 ns timestamps of block 0 of the persistent Lanczos kernel (VPCA_LZ_PROF=1)."""
        out = np.zeros((32, 8), dtype=np.int64)
        cnt = self._lib.vpca_debug_lanczos_profile(self._h, _host_ptr(out), 32)
        if cnt < 0:
            self._check(cnt)
        return out[:cnt]

    def accumulateJoined(self, partition_id: int):
        """Encode + Gram of the joined rows of the last joinRows, straight from device memory (vpca_accumulate_joined)."""
        self._check(self._lib.vpca_accumulate_joined(self._h, int(partition_id)))

    def accumulateCallsRaw(self, partition_id: int, off_ptr: int, idx_ptr: int, nv: int, idx_bytes: int = 4):
        """Same, from raw host addresses (e.g. pinned torch tensors) -- no copies on the Python side.
        idx_bytes = 2: the indices are uint16 (vpca_accumulate_calls_u16)."""
        fn = self._lib.vpca_accumulate_calls if idx_bytes == 4 else self._lib.vpca_accumulate_calls_u16
        self._check(fn(self._h, int(partition_id), off_ptr, idx_ptr, int(nv)))

    def accumulateBits(self, partition_id: int, bits: np.ndarray):
        """bits: (nv, stride) uint8, bit s (LSB first) of row v = sample s carries variant v."""
        b = np.ascontiguousarray(bits, dtype=np.uint8)
        if b.ndim != 2:
            raise VpcaError(VPCA_ERR_BAD_ARG, "bits must be (nv, stride_bytes)")
        self._check(self._lib.vpca_accumulate_bits(self._h, int(partition_id), _host_ptr(b), b.shape[0], b.shape[1]))

    def accumulateBed(self, partition_id: int, rows: np.ndarray, counted_allele: int = 1):
        """rows: (nv, stride) uint8 PLINK .bed rows (2 bits per sample: 00 hom A1, 01 missing, 10 het, 11 hom A2);
        counted_allele 1: carriers of A1, 2: carriers of A2 (plink.py)."""
        b, ptr = _bed_rows(rows)
        self._check(self._lib.vpca_accumulate_bed(self._h, int(partition_id), ptr, b.shape[0], b.shape[1],
                                                  int(counted_allele)))

    def accumulateBitsRaw(self, partition_id: int, ptr: int, nv: int, stride_bytes: int):
        self._check(self._lib.vpca_accumulate_bits(self._h, int(partition_id), ptr, int(nv), int(stride_bytes)))

    def accumulateCalls16(self, partition_id: int, offsets, sample_idx):
        off = np.ascontiguousarray(offsets, dtype=np.int64)
        idx = np.ascontiguousarray(sample_idx, dtype=np.uint16)
        self._check(self._lib.vpca_accumulate_calls_u16(self._h, int(partition_id), _host_ptr(off),
                                                        _host_ptr(idx) if len(idx) else None, len(off) - 1))

    def commit(self, partition_id: int):
        self._check(self._lib.vpca_commit(self._h, int(partition_id)))

    def abort(self, partition_id: int):
        self._check(self._lib.vpca_abort(self._h, int(partition_id)))

    def accumulateDense(self, x: np.ndarray, nv: Optional[int] = None):
        """Host dense tile, shape (n, ld), int8 (or uint16 bf16 bits), of which the first `nv` columns (default: all)
        are cells; for DTYPE_E2M1 packed uint8 of shape (n, ld / 2) with ld % 128 == 0, `nv` valid cells per row and
        zero cells after them up to a multiple of 128."""
        x = np.asarray(x)
        if self.elem_bits == 4:
            if x.dtype != np.uint8 or x.ndim != 2 or x.shape[0] != self.n or (x.shape[1] * 2) % 128:
                raise VpcaError(VPCA_ERR_BAD_ARG, f"packed tile must be ({self.n}, ld/2) uint8 with ld % 128 == 0")
            x = np.ascontiguousarray(x)
            ld = x.shape[1] * 2
            self._check(self._lib.vpca_accumulate_dense(self._h, _host_ptr(x), ld if nv is None else int(nv), ld, 0))
            return
        want = np.int8 if self.elem_bits == 8 else np.uint16
        if x.dtype != want or x.ndim != 2 or x.shape[0] != self.n:
            raise VpcaError(VPCA_ERR_BAD_ARG, f"dense tile must be ({self.n}, ld) {np.dtype(want).name}")
        if not x.flags.c_contiguous:
            x = np.ascontiguousarray(x)
        ld = x.shape[1]
        self._check(self._lib.vpca_accumulate_dense(self._h, _host_ptr(x), ld if nv is None else int(nv), ld, 0))

    def accumulateDenseDevice(self, d_ptr: int, nv: int, ld: int):
        self._check(self._lib.vpca_accumulate_dense(self._h, d_ptr, int(nv), int(ld), 1))

    def accumulatePanels(self, d_ptr: int, nv: int, panel_variants: int):
        """Device-resident cohort in panel layout (see vpca.h): one Gram launch over all nv variants."""
        self._check(self._lib.vpca_accumulate_panels(self._h, d_ptr, int(nv), int(panel_variants)))

    def synthPanelsDevice(self, seed: int, v0: int, nv: int, mode: int, d_ptr: int, panel_variants: int):
        self._check(self._lib.vpca_synth_panels_device(self._h, ctypes.c_uint64(seed), int(v0), int(nv), int(mode),
                                                       d_ptr, int(panel_variants)))

    def panelBytes(self, nv: int, panel_variants: int) -> int:
        npanels = (int(nv) + panel_variants - 1) // panel_variants
        return npanels * self.n * panel_variants * self.elem_bits // 8

    def gramDevicePtr(self) -> int:
        p = ctypes.c_void_p()
        self._check(self._lib.vpca_gram_device_ptr(self._h, ctypes.byref(p)))
        return int(p.value)

    def exportIpcHandle(self) -> bytes:
        buf = ctypes.create_string_buffer(64)
        self._check(self._lib.vpca_gram_export_ipc(self._h, buf))
        return buf.raw

    def setPeers(self, handles, rank: int, mode: str = "replicate"):
        """handles: list of 64-byte handles of all ranks, in rank order.  mode: "replicate" (every flush into every
        rank's Gram) or "owner_rows" (reduce-scatter by Gram row bands; finish a pass with gatherGram())."""
        blob = ctypes.create_string_buffer(b"".join(handles), 64 * len(handles))
        self._check(self._lib.vpca_gram_set_peers(self._h, blob, len(handles), int(rank)))
        self._check(self._lib.vpca_gram_set_peer_mode(self._h, {"replicate": 0, "owner_rows": 1}[mode]))

    def gatherGram(self):
        """Closing step of a fused pass: all-rank barrier (+ pull of the other ranks' row bands in owner_rows mode)."""
        self._check(self._lib.vpca_gram_gather(self._h))

    def peerBarrier(self):
        self._check(self._lib.vpca_peer_barrier(self._h))

    def finalizeGram(self):
        self._check(self._lib.vpca_finalize_gram(self._h))

    def getGram(self) -> np.ndarray:
        out = np.empty((self.n, self.n), dtype=np.int32)
        self._check(self._lib.vpca_get_gram(self._h, _host_ptr(out)))
        return out

    def partialGram(self, with_count: bool = False):
        """The accumulated (not yet finalized) Gram: lower triangle meaningful.  Checkpoint payload (with_count: also
        the number of variants the counts stand for, which a resume hands back to loadPartialGram)."""
        out = np.empty((self.n, self.n), dtype=np.int32)
        nv = ctypes.c_int64(0)
        self._check(self._lib.vpca_get_partial_gram(self._h, _host_ptr(out), ctypes.byref(nv)))
        return (out, int(nv.value)) if with_count else out

    def loadPartialGram(self, gram: np.ndarray, variants_in_gram: int):
        """Restore a checkpointed partial Gram; accumulation continues on top of it (and keeps counting against the
        int32 bound of a similarity count from `variants_in_gram`)."""
        g = np.ascontiguousarray(gram, dtype=np.int32)
        if g.shape != (self.n, self.n):
            raise VpcaError(VPCA_ERR_BAD_ARG, "gram must be (n, n)")
        self._check(self._lib.vpca_load_partial_gram(self._h, _host_ptr(g), int(variants_in_gram)))

    def variantCount(self) -> int:
        v = int(self._lib.vpca_variant_count(self._h))
        if v < 0:
            self._raise(v, self._h)
        return v

    def synchronize(self):
        self._check(self._lib.vpca_synchronize(self._h))

    def gramBand(self, row0: int, rows: int) -> np.ndarray:
        """Rows [row0, row0 + rows) of the Gram as this context stores them (band-only contexts: their own band)."""
        out = np.empty((rows, self.n), dtype=np.int32)
        self._check(self._lib.vpca_get_gram_band(self._h, int(row0), int(rows), _host_ptr(out)))
        return out

    def setGram(self, gram: np.ndarray):
        g = np.ascontiguousarray(gram, dtype=np.int32)
        if g.shape != (self.n, self.n):
            raise VpcaError(VPCA_ERR_BAD_ARG, "gram must be (n, n)")
        self._check(self._lib.vpca_set_gram(self._h, _host_ptr(g)))

    def computePca(self, k: int = 2):
        """-> (vecs (n, k) with column c = PC c, evals (k,), nonZeroRows).  `vecs.T.ravel()` is the
        column-major array ``pca.toArray`` of VariantsPca.scala:227."""
        flat = np.empty(self.n * k, dtype=np.float64)
        evals = np.empty(k, dtype=np.float64)
        nz = ctypes.c_int32(0)
        self._check(self._lib.vpca_compute_pca(self._h, int(k), _host_ptr(flat), _host_ptr(evals), ctypes.byref(nz)))
        return flat.reshape(k, self.n).T.copy(), evals, int(nz.value)

    def getCentered(self) -> np.ndarray:
        out = np.empty((self.n, self.n), dtype=np.float64)
        self._check(self._lib.vpca_get_centered(self._h, _host_ptr(out)))
        return out

    def getTridiagonal(self):
        d = np.empty(self.n, dtype=np.float64)
        e = np.empty(self.n - 1, dtype=np.float64)
        self._check(self._lib.vpca_get_tridiagonal(self._h, _host_ptr(d), _host_ptr(e)))
        return d, e

    def synthDenseDevice(self, seed: int, v0: int, nv: int, mode: int, d_ptr: int, ld: int):
        self._check(self._lib.vpca_synth_dense_device(self._h, ctypes.c_uint64(seed), int(v0), int(nv), int(mode),
                                                      d_ptr, int(ld)))

    def gramProfile(self, max_ctas: int = 1024) -> np.ndarray:
        """(ctas, 4) int64 ns timestamps of the last Gram launch (needs VPCA_GRAM_PROF=1 at first launch)."""
        out = np.zeros((max_ctas, 4), dtype=np.int64)
        rc = self._lib.vpca_debug_gram_profile(self._h, _host_ptr(out), max_ctas)
        if rc < 0:
            self._raise(rc, self._h)
        return out[:rc]

    def stats(self) -> dict:
        st = VpcaStats()
        self._check(self._lib.vpca_get_stats(self._h, ctypes.byref(st)))
        return {name: getattr(st, name) for name, _ in VpcaStats._fields_}

    # -- variant loadings and projection onto computed principal coordinates (vpca.h, DESIGN.md 6) --------------------
    def loadingsCalls(self, k: int, offsets, sample_idx):
        """After computePca(k0 >= k), or a computePcaBands(..., k0 >= k) that named this context (band-only contexts
        included; the most recent solve wins): (w (nv, k) float64, count (nv,) int32) with w[v, c] = sum_s x[s][v] U[s, c]
        and count[v] = sum_s x[s][v] for the CSR rows given (rows without carriers allowed).  Without a valid U:
        VPCA_ERR_STATE on a full context, VPCA_ERR_UNSUPPORTED on a band-only one.  Above 65 535 samples the samples are
        summed in 4 fixed ranges (vpca.h); w[v] depends on column v, U and N only, whatever the input form."""
        off, idx = self._csr(offsets, sample_idx)
        nv = len(off) - 1
        w = np.zeros((max(nv, 1), int(k)), dtype=np.float64)
        cnt = np.zeros(max(nv, 1), dtype=np.int32)
        self._check(self._lib.vpca_loadings_calls(self._h, int(k), _host_ptr(off), _host_ptr(idx) if len(idx) else None, nv,
                                                  _host_ptr(w), _host_ptr(cnt)))
        return w[:nv], cnt[:nv]

    def loadingsBed(self, k: int, rows: np.ndarray, counted_allele: int = 1):
        """Same for PLINK .bed rows (see accumulateBed), with the same U and the same bits."""
        b, ptr = _bed_rows(rows)
        w = np.zeros((max(b.shape[0], 1), int(k)), dtype=np.float64)
        cnt = np.zeros(max(b.shape[0], 1), dtype=np.int32)
        self._check(self._lib.vpca_loadings_bed(self._h, int(k), ptr, b.shape[0], b.shape[1], int(counted_allele),
                                                _host_ptr(w), _host_ptr(cnt)))
        return w[:b.shape[0]], cnt[:b.shape[0]]

    def loadingsPanels(self, k: int, d_ptr: int, nv: int, panel_variants: int, d_w: int, d_count: int):
        """Device panels in, device outputs (nv x k float64, nv int32), ordered on the context's stream; U as for
        loadingsCalls, and the same bits whatever the panel width."""
        self._check(self._lib.vpca_loadings_panels(self._h, int(k), d_ptr, int(nv), int(panel_variants), d_w, d_count))

    def projectBegin(self, k: int):
        """Start a projection of this context's n samples onto k components (zeroes the accumulator)."""
        self._check(self._lib.vpca_project_begin(self._h, int(k)))
        self._proj_k = int(k)

    def projectCalls(self, offsets, sample_idx, w, mean):
        """Add sum_v (y[s][v] - mean[v]) w[v, :] for the CSR rows given; w (nv, k) and mean (nv,) align with the rows."""
        off, idx = self._csr(offsets, sample_idx)
        nv = len(off) - 1
        ww = np.ascontiguousarray(w, dtype=np.float64).reshape(nv, -1)
        mm = np.ascontiguousarray(mean, dtype=np.float64).reshape(nv)
        self._check(self._lib.vpca_project_calls(self._h, _host_ptr(off), _host_ptr(idx) if len(idx) else None, nv,
                                                 _host_ptr(ww), _host_ptr(mm)))

    def projectBed(self, rows: np.ndarray, w, mean, counted_allele: int = 1):
        b, ptr = _bed_rows(rows)
        ww = np.ascontiguousarray(w, dtype=np.float64).reshape(b.shape[0], -1)
        mm = np.ascontiguousarray(mean, dtype=np.float64).reshape(b.shape[0])
        self._check(self._lib.vpca_project_bed(self._h, ptr, b.shape[0], b.shape[1], int(counted_allele),
                                               _host_ptr(ww), _host_ptr(mm)))

    def projectPanels(self, d_ptr: int, nv: int, panel_variants: int, d_w: int, d_mean: int):
        self._check(self._lib.vpca_project_panels(self._h, d_ptr, int(nv), int(panel_variants), d_w, d_mean))

    def projectGet(self, evals) -> np.ndarray:
        """(n, k) projected coordinates: accumulated sums / evals[c] (evals of ones: the raw sums)."""
        k = getattr(self, "_proj_k", 0)        # 0: not begun, the library reports VPCA_ERR_STATE before reading evals
        ev = np.ascontiguousarray(evals, dtype=np.float64).reshape(-1)
        if k and len(ev) != k:
            raise VpcaError(VPCA_ERR_BAD_ARG, f"evals must have {k} entries")
        out = np.zeros(self.n * max(k, 1), dtype=np.float64)
        self._check(self._lib.vpca_project_get(self._h, _host_ptr(ev), _host_ptr(out)))
        return out.reshape(max(k, 1), self.n).T.copy()

    # -- KING-robust kinship between the samples (vpca.h, DESIGN.md 7) -------------------------------------------------
    def kinshipBed(self, rows: np.ndarray):
        """Add PLINK .bed rows ((nv, stride) uint8, see accumulateBed) to the kinship counts of every sample pair; calls
        add up, and the PCA Gram is not touched.  Synchronises."""
        b, ptr = _bed_rows(rows)
        self._check(self._lib.vpca_kinship_bed(self._h, ptr, b.shape[0], b.shape[1]))

    def kinshipPairs(self, min_kinship: float = float("-inf"), max_pairs: Optional[int] = None):
        """-> (ids (P, 2) int32 with a < b, counts (P, 5) int32 NSNP, HETHET, IBS0, HET1_HOM2, HET2_HOM1, kinship (P,)
        float64) of the pairs with KINSHIP >= min_kinship (-inf: every pair, NaN ones included), ordered by b then a.
        max_pairs: keep only the first max_pairs (None: all of them)."""
        total = ctypes.c_int64(0)
        self._check(self._lib.vpca_kinship_pairs(self._h, float(min_kinship), 0, None, None, None, ctypes.byref(total)))
        p = int(total.value) if max_pairs is None else min(int(total.value), int(max_pairs))
        ids = np.zeros((max(p, 1), 2), np.int32)
        counts = np.zeros((max(p, 1), 5), np.int32)
        kin = np.zeros(max(p, 1), np.float64)
        if p > 0:
            self._check(self._lib.vpca_kinship_pairs(self._h, float(min_kinship), p, _host_ptr(ids), _host_ptr(counts),
                                                     _host_ptr(kin), ctypes.byref(total)))
        return ids[:p], counts[:p], kin[:p]

    # -- LD pruning of the variants (vpca.h, DESIGN.md 9) --------------------------------------------------------------
    def ldPruneBed(self, rows: np.ndarray, window_lo, r2_max: float, max_pairs: int = 0, eligible=None):
        """Keep-first LD pruning of PLINK .bed rows ((V, stride) uint8; a .bed memmap is read in place, not copied) with
        window_lo[j] the first variant of j's window -> (keep (V,) bool, pairs (P, 2) int64 of (i, j), r2 (P,) float64):
        the first min(total, max_pairs) in-LD pairs in order of j, then i.  eligible ((V,) bool, e.g. the variant QC
        mask): only eligible variants are paired or kept -- the result of pruning the eligible rows alone, indexed over
        all V.  Synchronises."""
        b, rows_ptr = _bed_rows(rows)
        nv = b.shape[0]
        lo = np.ascontiguousarray(window_lo, dtype=np.int64).reshape(-1)
        if len(lo) != nv:
            raise VpcaError(VPCA_ERR_BAD_ARG, f"window_lo must have {nv} entries")
        keep = np.zeros(max(nv, 1), np.uint8)
        p = max(int(max_pairs), 0)
        pairs = np.zeros((max(p, 1), 2), np.int64)
        r2 = np.zeros(max(p, 1), np.float64)
        total = ctypes.c_int64(0)
        empty = np.zeros(1, np.int64)          # a valid address for zero variants
        lo_ptr = lo.ctypes.data if lo.size else _host_ptr(empty)
        if eligible is None:
            self._check(self._lib.vpca_ld_prune_bed(self._h, rows_ptr, nv, b.shape[1], lo_ptr, float(r2_max),
                                                    _host_ptr(keep), p, _host_ptr(pairs) if p else None,
                                                    _host_ptr(r2) if p else None, ctypes.byref(total)))
        else:
            el = np.ascontiguousarray(eligible, dtype=bool).reshape(-1)
            if len(el) != nv:
                raise VpcaError(VPCA_ERR_BAD_ARG, f"eligible must have {nv} entries")
            el = np.concatenate([el.view(np.uint8), np.zeros(1, np.uint8)])   # a valid address for zero variants
            self._check(self._lib.vpca_ld_prune_bed_masked(self._h, rows_ptr, nv, b.shape[1], lo_ptr, _host_ptr(el),
                                                           float(r2_max), _host_ptr(keep), p,
                                                           _host_ptr(pairs) if p else None,
                                                           _host_ptr(r2) if p else None, ctypes.byref(total)))
        got = min(int(total.value), p)
        return keep[:nv] != 0, pairs[:got], r2[:got]

    # -- variant QC (vpca.h, DESIGN.md 10) ---------------------------------------------------------------------------
    def variantQcBed(self, rows: np.ndarray, hwe: bool = True):
        """Genotype counts of PLINK .bed rows ((V, stride) uint8; a .bed memmap is read in place, not copied) ->
        (counts (V, 4) int32 of HOM_A1, HET, HOM_A2, MISSING; p (V,) float64 exact HWE p-values, or None without
        `hwe`).  Synchronises."""
        b, ptr = _bed_rows(rows)
        nv = b.shape[0]
        counts = np.zeros((max(nv, 1), 4), np.int32)
        p = np.zeros(max(nv, 1), np.float64)
        self._check(self._lib.vpca_variant_qc_bed(self._h, ptr, nv, b.shape[1],
                                                  _host_ptr(counts), _host_ptr(p) if hwe else None))
        return counts[:nv], (p[:nv] if hwe else None)

    # -- variance-standardized relationship matrix (vpca.h, DESIGN.md 13) ---------------------------------------------
    def grmBed(self, rows: np.ndarray):
        """Add PLINK .bed rows ((V, stride) uint8; a .bed memmap is read in place, not copied) to the GRM; calls add up,
        and the PCA Gram is not touched.  Synchronises."""
        b, ptr = _bed_rows(rows)
        self._check(self._lib.vpca_grm_bed(self._h, ptr, b.shape[0], b.shape[1]))

    def grmFinalize(self) -> int:
        """Finish the GRM -> M, the number of variants used (VPCA_ERR_STATE when M = 0)."""
        m = ctypes.c_int64(0)
        self._check(self._lib.vpca_grm_finalize(self._h, ctypes.byref(m)))
        return int(m.value)

    def getGrm(self) -> np.ndarray:
        """The finalized GRM, (n, n) float64, symmetric."""
        out = np.empty((self.n, self.n), dtype=np.float64)
        self._check(self._lib.vpca_get_grm(self._h, _host_ptr(out)))
        return out

    def computePcaGrm(self, k: int = 2):
        """-> (vecs (n, k) with column c = PC c of the GRM, evals (k,)): computePca's shapes and sign rule."""
        flat = np.empty(self.n * k, dtype=np.float64)
        evals = np.empty(k, dtype=np.float64)
        self._check(self._lib.vpca_compute_pca_grm(self._h, int(k), _host_ptr(flat), _host_ptr(evals)))
        return flat.reshape(k, self.n).T.copy(), evals

    def grmLoadingsBed(self, k: int, rows: np.ndarray):
        """GRM loadings of PLINK .bed rows ((V, stride) uint8; a .bed memmap is read in place) for the U of the last
        computePcaGrm -> (w (V, k) float64 = Z^T U, tab (V, 4) float64 z of each .bed code, zero for an unused variant).
        Pass the rows the GRM was built from: the tables are recomputed from them.  Synchronises."""
        b, ptr = _bed_rows(rows)
        nv = b.shape[0]
        w = np.zeros((max(nv, 1), int(k)), np.float64)
        tab = np.zeros((max(nv, 1), 4), np.float64)
        self._check(self._lib.vpca_grm_loadings_bed(self._h, int(k), ptr, nv,
                                                    b.shape[1], _host_ptr(w), _host_ptr(tab)))
        return w[:nv], tab[:nv]

    def projectGrmBed(self, rows: np.ndarray, tab, w):
        """Add sum_v tab[v][code(s, v)] w[v, :] of PLINK .bed rows ((V, stride) uint8 of this context's samples; a .bed
        memmap is read in place) to the projection begun by projectBegin; tab (V, 4) and w (V, k) of the reference align
        with the rows.  Read with projectGet(M * eigenvalues).  Synchronises."""
        b, ptr = _bed_rows(rows)
        nv = b.shape[0]
        tt = np.ascontiguousarray(tab, dtype=np.float64).reshape(nv, 4)
        ww = np.ascontiguousarray(w, dtype=np.float64).reshape(nv, -1)
        if nv and ww.shape[1] != getattr(self, "_proj_k", ww.shape[1]):
            raise VpcaError(VPCA_ERR_BAD_ARG, f"w must have {self._proj_k} columns")
        empty = np.zeros(4, np.float64)
        self._check(self._lib.vpca_grm_project_bed(self._h, ptr, nv, b.shape[1], _host_ptr(tt if nv else empty),
                                                   _host_ptr(ww if nv else empty)))

    # -- linear association tests (vpca.h, DESIGN.md 15) -----------------------------------------------------------------
    def glmBegin(self, pheno, covar=None) -> int:
        """Set the phenotype ((n,) float64, NaN = missing) and the covariates ((n, c) float64, NaN = missing; None for
        none) of the linear tests; the intercept is added.  Returns the regression samples (finite phenotype and
        covariates).  VPCA_ERR_BAD_ARG for +-Inf, more than 31 covariates, too few samples, a constant phenotype or a
        collinear covariate."""
        return self._glm_begin(self._lib.vpca_glm_begin, pheno, covar)

    def _glm_begin(self, fn, pheno, covar) -> int:
        y = np.ascontiguousarray(pheno, dtype=np.float64).reshape(-1)
        if y.shape[0] != self.n:
            raise VpcaError(VPCA_ERR_BAD_ARG, f"pheno must have {self.n} entries")
        c = np.zeros((self.n, 0)) if covar is None else np.ascontiguousarray(covar, dtype=np.float64).reshape(self.n, -1)
        m = ctypes.c_int64(0)
        self._check(fn(self._h, _host_ptr(y), _host_ptr(c) if c.shape[1] else None, c.shape[1], ctypes.byref(m)))
        return int(m.value)

    def _glm_bed(self, fn, rows, counted, *extra, dtypes=()):
        """Calls fn(ctx, rows, V, stride, counted, *extra, stats, err, *outputs) with outputs of dtypes -> (stats (V, 6),
        err (V,), *outputs (V,))."""
        b, ptr = _bed_rows(rows)
        nv = b.shape[0]
        outs = [np.zeros((max(nv, 1), 6), np.float64)] + [np.zeros(max(nv, 1), t) for t in (np.int32, *dtypes)]
        self._check(fn(self._h, ptr, nv, b.shape[1], int(counted), *extra, *(_host_ptr(o) for o in outs)))
        return tuple(o[:nv] for o in outs)

    def glmLinearBed(self, rows: np.ndarray, counted: int = 1):
        """Linear tests of PLINK .bed rows ((V, stride) uint8 of this context's samples; a .bed memmap is read in place)
        against the phenotype of glmBegin -> (stats (V, 6) float64: OBS_CT, A1_FREQ, BETA, SE, T_STAT, P, NaN where
        undefined; err (V,) int32: index into GLM_ERRCODES).  counted: 1 counts A1, 2 counts A2.  Synchronises."""
        return self._glm_bed(self._lib.vpca_glm_linear_bed, rows, counted)

    # -- logistic association tests (vpca.h, DESIGN.md 16) ---------------------------------------------------------------
    def glmLogisticBegin(self, pheno, covar=None) -> int:
        """Set the case/control phenotype ((n,) float64: 1 case, 0 control, NaN missing) and the covariates ((n, c)
        float64, NaN = missing; None for none) of the logistic tests; the intercept is added.  Returns the regression
        samples.  VPCA_ERR_BAD_ARG for what glmBegin refuses, a value outside {0, 1, NaN}, no case or no control, or a
        null model that does not converge."""
        return self._glm_begin(self._lib.vpca_glm_logistic_begin, pheno, covar)

    def glmLogisticBed(self, rows: np.ndarray, counted: int = 1):
        """Logistic tests of PLINK .bed rows ((V, stride) uint8 of this context's samples; a .bed memmap is read in
        place) against the phenotype of glmLogisticBegin -> (stats (V, 6) float64: OBS_CT, A1_FREQ, BETA, SE, Z, P, NaN
        where undefined; err (V,) int32: index into GLM_ERRCODES; passes (V,) int32: Newton passes).  counted: 1 counts
        A1, 2 counts A2.  Synchronises."""
        return self._glm_bed(self._lib.vpca_glm_logistic_bed, rows, counted, dtypes=(np.int32,))

    # -- Firth-penalized logistic tests (vpca.h, DESIGN.md 17) -----------------------------------------------------------
    def glmFirthBed(self, rows: np.ndarray, counted: int = 1, mode: str = "fallback"):
        """Logistic tests with Firth's penalized likelihood of PLINK .bed rows (as glmLogisticBed, on the state of
        glmLogisticBegin).  mode "fallback": the maximum-likelihood fit, and the Firth fit where it does not converge;
        "always": the Firth fit of every variant -> (stats (V, 6), err (V,), passes (V,) of the fit reported, firth (V,)
        uint8: 1 where the Firth fit ran).  Synchronises."""
        if mode not in GLM_FIRTH_MODES:
            raise VpcaError(VPCA_ERR_BAD_ARG, f"mode must be one of {', '.join(GLM_FIRTH_MODES)}, not {mode!r}")
        return self._glm_bed(self._lib.vpca_glm_firth_bed, rows, counted, GLM_FIRTH_MODES[mode],
                             dtypes=(np.int32, np.uint8))

    def hweExact(self, counts) -> np.ndarray:
        """Exact HWE p-values of (V, 4) int32 counts (HOM_A1, HET, HOM_A2, MISSING; MISSING ignored) -> (V,) float64."""
        c = np.ascontiguousarray(counts, dtype=np.int32).reshape(-1, 4)
        nv = c.shape[0]
        c = np.concatenate([c, np.zeros((1, 4), np.int32)])   # a valid address for zero variants
        p = np.zeros(nv + 1, np.float64)
        self._check(self._lib.vpca_hwe_exact(self._h, _host_ptr(c), nv, _host_ptr(p)))
        return p[:nv]

    # -- sample QC (vpca.h, DESIGN.md 11) ----------------------------------------------------------------------------

    def sampleMissingBed(self, rows: np.ndarray, n_samples: int) -> np.ndarray:
        """Missing calls of each of the n_samples samples of PLINK .bed rows ((V, stride) uint8; a .bed memmap is read in
        place, not copied) -> (n_samples,) int32.  The rows need not have this context's sample count.  Synchronises."""
        b, ptr = _bed_rows(rows)
        out = np.zeros(max(int(n_samples), 1), np.int32)
        self._check(self._lib.vpca_sample_missing_bed(self._h, ptr, b.shape[0],
                                                      b.shape[1], int(n_samples), _host_ptr(out)))
        return out[:int(n_samples)]

    def subsetBedSamples(self, rows: np.ndarray, n_samples: int, keep) -> np.ndarray:
        """PLINK .bed rows of n_samples samples ((V, stride) uint8; a .bed memmap is read in place, not copied) repacked to
        the samples keep (strictly increasing indices) -> (V, ceil(M / 4)) uint8, the rows of a fileset of those samples.
        The rows need not have this context's sample count.  Synchronises."""
        b, ptr = _bed_rows(rows)
        idx = np.ascontiguousarray(keep, dtype=np.int32).reshape(-1)
        m = len(idx)
        mb = (m + 3) // 4
        out = np.empty((b.shape[0], mb), np.uint8)
        empty = np.zeros(1, np.uint8)
        self._check(self._lib.vpca_subset_bed_samples(
            self._h, ptr, b.shape[0], b.shape[1], int(n_samples), _host_ptr(idx) if m else None, m,
            out.ctypes.data if out.size else _host_ptr(empty), mb))
        return out

    def computePcaSubset(self, keep, k: int = 2):
        """PCs of the samples with keep[s] true, from the Gram of all of them (DESIGN.md 8) -> (vecs (n, k), evals (k,),
        nonZeroRows of S[K, K]): kept rows hold their eigenvectors, removed rows their projection onto the same axes.
        Afterwards the loadings calls return the kept samples' loadings."""
        kb = np.ascontiguousarray(np.asarray(keep).reshape(-1) != 0, dtype=np.uint8)
        if kb.shape[0] != self.n:
            raise VpcaError(VPCA_ERR_BAD_ARG, f"keep must have {self.n} entries")
        flat = np.empty(self.n * k, dtype=np.float64)
        evals = np.empty(k, dtype=np.float64)
        nz = ctypes.c_int32(0)
        self._check(self._lib.vpca_compute_pca_subset(self._h, _host_ptr(kb), int(k), _host_ptr(flat), _host_ptr(evals),
                                                      ctypes.byref(nz)))
        return flat.reshape(k, self.n).T.copy(), evals, int(nz.value)


def debugTiles(n_samples: int, cta_group: int = 2, exact: bool = True) -> np.ndarray:
    """(tiles, 8) int32: the Gram kernel's tile list for n_samples (host-only, no GPU needed; see vpca_debug_tiles)."""
    L = load_library()
    cnt = L.vpca_debug_tiles(int(n_samples), int(cta_group), 1 if exact else 0, None, 0)
    if cnt < 0:
        raise VpcaError(cnt, L.vpca_last_error(None).decode("utf-8", "replace"))
    out = np.zeros((cnt, 8), dtype=np.int32)
    L.vpca_debug_tiles(int(n_samples), int(cta_group), 1 if exact else 0, _host_ptr(out), cnt)
    return out


def debugPlan(tiles: np.ndarray, workers: int, kb_window: int) -> np.ndarray:
    """(pieces, 6) int32 {worker, tile, kb_lo, kb_hi, acc_col, acc_cols_of_worker} of one window (vpca_debug_plan); the
    columns are B rows of the worker's register accumulator."""
    L = load_library()
    t = np.ascontiguousarray(tiles, dtype=np.int32)
    cap = 8 * int(workers) + 8
    out = np.zeros((cap, 6), dtype=np.int32)
    cnt = L.vpca_debug_plan(_host_ptr(t), len(t), int(workers), int(kb_window), _host_ptr(out), cap)
    if cnt < 0:
        raise VpcaError(VPCA_ERR_STATE, L.vpca_last_error(None).decode("utf-8", "replace"))
    return out[:cnt]


def debugSchedule(n_samples: int, cta_group: int, exact: bool, workers: int, kb_window: int, kb_total: int,
                  front_frac: float = -1.0):
    """Every piece each worker replays in one launch (vpca_debug_schedule): returns ((pieces, 6) int32 {worker, tile,
    kb_lo, kb_hi, first, flush} in launch order, schedule (0 waves, 1 resident, 2 front/tail), split point s)."""
    L = load_library()
    info = np.zeros(2, dtype=np.int32)
    args = (int(n_samples), int(cta_group), 1 if exact else 0, int(workers), int(kb_window), int(kb_total),
            float(front_frac))
    cnt = L.vpca_debug_schedule(*args, None, 0, _host_ptr(info))
    if cnt < 0:
        raise VpcaError(cnt, L.vpca_last_error(None).decode("utf-8", "replace"))
    out = np.zeros((cnt, 6), dtype=np.int32)
    L.vpca_debug_schedule(*args, _host_ptr(out), cnt, _host_ptr(info))
    return out, int(info[0]), int(info[1])


def debugBandTiles(n_samples: int, cta_group: int, row0: int, rows: int) -> np.ndarray:
    """Tiles of an owner-computes band context (vpca_debug_band_tiles), (tiles, 8) int32 like debugTiles."""
    L = load_library()
    L.vpca_debug_band_tiles.restype = ctypes.c_int
    L.vpca_debug_band_tiles.argtypes = [ctypes.c_int32] * 4 + [ctypes.c_void_p, ctypes.c_int32]
    cnt = L.vpca_debug_band_tiles(int(n_samples), int(cta_group), int(row0), int(rows), None, 0)
    if cnt < 0:
        raise VpcaError(cnt, L.vpca_last_error(None).decode("utf-8", "replace"))
    out = np.zeros((cnt, 8), dtype=np.int32)
    L.vpca_debug_band_tiles(int(n_samples), int(cta_group), int(row0), int(rows), _host_ptr(out), cnt)
    return out


def maxClusters(device: int, cluster_size: int) -> int:
    """Clusters of `cluster_size` Gram-kernel CTAs the device holds at once (vpca_debug_max_clusters)."""
    L = load_library()
    L.vpca_debug_max_clusters.restype = ctypes.c_int
    L.vpca_debug_max_clusters.argtypes = [ctypes.c_int32, ctypes.c_int32]
    c = L.vpca_debug_max_clusters(int(device), int(cluster_size))
    if c < 0:
        raise VpcaError(c, L.vpca_last_error(None).decode("utf-8", "replace"))
    return c


def debugRebalance(tiles: np.ndarray, workers: int, kb_window: int, cum: np.ndarray, col_limit: int = 512):
    """The rebalancer's repair of a candidate split (vpca_debug_rebalance): returns (repaired cum, pieces like debugPlan)."""
    L = load_library()
    t = np.ascontiguousarray(tiles, dtype=np.int32)
    c = np.ascontiguousarray(cum, dtype=np.float64).copy()
    assert c.shape == (workers + 1,)
    cap = 8 * int(workers) + 8
    out = np.zeros((cap, 6), dtype=np.int32)
    cnt = L.vpca_debug_rebalance(_host_ptr(t), len(t), int(workers), int(kb_window), int(col_limit), _host_ptr(c),
                                 _host_ptr(out), cap)
    if cnt < 0:
        raise VpcaError(cnt, L.vpca_last_error(None).decode("utf-8", "replace"))
    return c, out[:cnt]


def ownerRowBands(n_samples: int, world: int) -> list:
    """Row bands of VPCA_PEER_OWNER_ROWS: [(row0, rows)] per rank (vpca_owner_row_bands)."""
    L = load_library()
    ends = (ctypes.c_int32 * world)()
    rc = L.vpca_owner_row_bands(int(n_samples), int(world), ends)
    if rc != VPCA_OK:
        raise VpcaError(rc, L.vpca_last_error(None).decode("utf-8", "replace"))
    out, prev = [], 0
    for q in range(world):
        out.append((prev, int(ends[q]) - prev))
        prev = int(ends[q])
    return out


def computePcaBands(contexts, k: int = 2):
    """Top-k principal coordinates of a Gram held as row bands by `contexts` (rank order, bands covering [0, N); a context
    that stores the whole Gram is the band [0, N)) -> (vecs (N, k), evals (k,), nonZeroRows), like NativePca.computePca
    but with no 65 535-sample limit and no N x N workspace (vpca_compute_pca_bands).  Failures of the solver raise
    VpcaError with code VPCA_ERR_UNSUPPORTED; there is no fallback.  On success every context holds U (the first
    min(k, 16) columns) and the eigenvalues on its own device, so each rank can call loadings* on its variants; the call
    clears U on every context first, so after a failed solve they have none."""
    L = load_library()
    if not contexts:
        raise VpcaError(VPCA_ERR_BAD_ARG, "at least one context")
    n = contexts[0].n
    arr = (ctypes.c_void_p * len(contexts))(*[c._h.value if c._h is not None else None for c in contexts])
    flat = np.empty(n * max(int(k), 1), dtype=np.float64)
    evals = np.empty(max(int(k), 1), dtype=np.float64)
    nz = ctypes.c_int32(0)
    rc = L.vpca_compute_pca_bands(arr, len(contexts), int(k), _host_ptr(flat), _host_ptr(evals), ctypes.byref(nz))
    if rc != VPCA_OK:
        contexts[0]._raise(rc, contexts[0]._h)
    return flat[: n * k].reshape(k, n).T.copy(), evals[:k].copy(), int(nz.value)


def setPeersLocal(contexts, mode: str = "owner_rows"):
    """Wire NativePca objects that live in THIS process (any mix of devices) for the fused reduce
    (vpca_gram_set_peers_local); contexts[r] becomes rank r."""
    L = load_library()
    arr = (ctypes.c_void_p * len(contexts))(*[c._h.value for c in contexts])
    rc = L.vpca_gram_set_peers_local(arr, len(contexts))
    if rc != VPCA_OK:
        raise VpcaError(rc, L.vpca_last_error(None).decode("utf-8", "replace"))
    for c in contexts:
        c._check(L.vpca_gram_set_peer_mode(c._h, {"replicate": 0, "owner_rows": 1}[mode]))


class NativePcaPool:
    """One process driving all GPUs of the box: the ctypes twin of the JNI class ``NativePcaPool``
    (spark_examples_b200/jvm/NativePcaPool.scala).  Partition p is served by GPU p % n_gpus; every method except
    reset / reduceAndFinalize / getGram / computePca may be called from many threads at once."""

    def __init__(self, n_samples: int, n_gpus: int, devices=None, dtype: int = DTYPE_I8, num_pc: int = 2,
                 max_multiplicity: int = 2, partitions_in_flight: int = 4, staging_lanes: int = 0,
                 chunk_variants: int = 0, chunk_nnz: int = 0):
        self._lib = load_library()
        self.n = int(n_samples)
        cfg = VpcaConfig(ctypes.sizeof(VpcaConfig), n_samples, 0, dtype, num_pc, max_multiplicity, partitions_in_flight,
                         staging_lanes, chunk_variants, chunk_nnz, None, None, 0, 0)
        devs = None
        if devices is not None:
            devs = (ctypes.c_int32 * n_gpus)(*[int(d) for d in devices])
        h = ctypes.c_void_p()
        rc = self._lib.vpca_pool_create(ctypes.byref(cfg), int(n_gpus), devs, ctypes.byref(h))
        self._h = h if rc == VPCA_OK else None
        if rc != VPCA_OK:
            self._raise(rc)

    def _raise(self, rc: int):
        msg = self._lib.vpca_pool_last_error(self._h).decode("utf-8", "replace")
        if rc == VPCA_ERR_INDEX_OUT_OF_RANGE:
            raise IndexOutOfRange(rc, msg)
        raise VpcaError(rc, msg)

    def _check(self, rc: int):
        if rc != VPCA_OK:
            self._raise(rc)

    def close(self):
        if getattr(self, "_h", None) is not None:
            self._lib.vpca_pool_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    @property
    def size(self) -> int:
        return int(self._lib.vpca_pool_size(self._h))

    def reset(self):
        self._check(self._lib.vpca_pool_reset(self._h))

    def accumulateCalls(self, partition_id: int, offsets, sample_idx):
        off, idx = NativePca._csr(offsets, sample_idx)
        self._check(self._lib.vpca_pool_accumulate_calls(self._h, int(partition_id), _host_ptr(off),
                                                         _host_ptr(idx) if len(idx) else None, len(off) - 1))

    def accumulateCalls16(self, partition_id: int, offsets, sample_idx):
        off = np.ascontiguousarray(offsets, dtype=np.int64)
        idx = np.ascontiguousarray(sample_idx, dtype=np.uint16)
        self._check(self._lib.vpca_pool_accumulate_calls_u16(self._h, int(partition_id), _host_ptr(off),
                                                             _host_ptr(idx) if len(idx) else None, len(off) - 1))

    def accumulateBits(self, partition_id: int, bits: np.ndarray):
        b = np.ascontiguousarray(bits, dtype=np.uint8)
        self._check(self._lib.vpca_pool_accumulate_bits(self._h, int(partition_id), _host_ptr(b), b.shape[0], b.shape[1]))

    def accumulateBed(self, partition_id: int, rows: np.ndarray, counted_allele: int = 1):
        b, ptr = _bed_rows(rows)
        self._check(self._lib.vpca_pool_accumulate_bed(self._h, int(partition_id), ptr, b.shape[0], b.shape[1],
                                                       int(counted_allele)))

    def commit(self, partition_id: int):
        self._check(self._lib.vpca_pool_commit(self._h, int(partition_id)))

    def abort(self, partition_id: int):
        self._check(self._lib.vpca_pool_abort(self._h, int(partition_id)))

    def reduceAndFinalize(self):
        self._check(self._lib.vpca_pool_reduce_and_finalize(self._h))

    def getGram(self) -> np.ndarray:
        out = np.empty((self.n, self.n), dtype=np.int32)
        self._check(self._lib.vpca_pool_get_gram(self._h, _host_ptr(out)))
        return out

    def computePca(self, k: int = 2):
        flat = np.empty(self.n * k, dtype=np.float64)
        evals = np.empty(k, dtype=np.float64)
        nz = ctypes.c_int32(0)
        self._check(self._lib.vpca_pool_compute_pca(self._h, int(k), _host_ptr(flat), _host_ptr(evals), ctypes.byref(nz)))
        return flat.reshape(k, self.n).T.copy(), evals, int(nz.value)

    def stats(self) -> dict:
        st = VpcaStats()
        self._check(self._lib.vpca_pool_get_stats(self._h, ctypes.byref(st)))
        return {name: getattr(st, name) for name, _ in VpcaStats._fields_}
