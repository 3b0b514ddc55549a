"""ctypes binding of ``libpydeseq2_b200.so`` (the C ABI in ``include/pydeseq2_b200.h``).

This is the stub a maintainer of the reference would add to bind the CUDA backend
(INTEGRATION.md).  There is deliberately no CPU fallback: if the CUDA library has not been
built, or no sm_90 (H100) device is visible, the calls raise.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("PDQ_LIB") or os.path.join(_HERE, "libpydeseq2_b200.so")  # PDQ_LIB: tuning variants

c_ctx = C.c_void_p
c_design = C.c_void_p
c_dptr = C.c_void_p
f64p = C.POINTER(C.c_double)
i64p = C.POINTER(C.c_int64)

PDQ_MAX_P = 16
PDQ_MAX_P_WIDE = 64  # with pdq_set_wide_designs (B200Inference(wide_designs=True))
PDQ_MAX_P_LARGE = 128  # with pdq_set_large_designs as well (B200Inference(wide_designs=True, large_designs=True))
ALT_CODES = {None: 0, "greaterAbs": 1, "lessAbs": 2, "greater": 3, "less": 4}
UNIQUE_ID_BYTES = 128
PEER_HANDLE_BYTES = 64

STATUS = {0: "ok", -1: "cuda error", -2: "invalid argument", -3: "unsupported", -4: "nccl error", -5: "no sm_90 device"}


class B200Error(RuntimeError):
    """Raised for every non-zero ``pdq_status`` (environment errors: no device, CUDA/NCCL failure)."""


# name -> (restype, argtypes); mirrors include/pydeseq2_b200.h one to one
_SIGNATURES = {
    "pdq_version": (C.c_char_p, []),
    "pdq_device_count": (C.c_int, []),
    "pdq_ctx_create": (C.c_int, [C.c_int, C.POINTER(c_ctx)]),
    "pdq_ctx_destroy": (None, [c_ctx]),
    "pdq_last_error": (C.c_char_p, [c_ctx]),
    "pdq_device_info": (C.c_int, [c_ctx, C.c_char_p, C.c_size_t, C.POINTER(C.c_int), C.POINTER(C.c_size_t)]),
    "pdq_set_lanes_per_gene": (C.c_int, [c_ctx, C.c_int]),
    "pdq_set_debug_flags": (C.c_int, [c_ctx, C.c_int]),
    "pdq_set_wide_designs": (C.c_int, [c_ctx, C.c_int]),
    "pdq_set_wide_shrink": (C.c_int, [c_ctx, C.c_int]),
    "pdq_set_large_designs": (C.c_int, [c_ctx, C.c_int]),
    "pdq_set_large_shrink": (C.c_int, [c_ctx, C.c_int]),
    "pdq_design_pinv": (C.c_int, [f64p, C.c_int, C.c_int, f64p, C.POINTER(C.c_int)]),
    "pdq_design_pinv_large": (C.c_int, [f64p, C.c_int, C.c_int, f64p, C.POINTER(C.c_int)]),
    "pdq_launch_count": (C.c_int64, [c_ctx]),
    "pdq_buffer_epoch": (C.c_int64, [c_ctx]),
    "pdq_residency_stats": (C.c_int, [c_ctx, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "pdq_residency_clear": (C.c_int, [c_ctx]),
    "pdq_csv_scan": (C.c_int, [C.c_char_p, C.c_char, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_size_t)]),
    "pdq_csv_read_counts": (C.c_int, [C.c_char_p, C.c_char, C.c_int, i64p, C.c_int64, C.c_int64, C.c_int64, C.c_char_p, C.c_size_t,
                                      C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "pdq_malloc": (C.c_int, [c_ctx, C.c_size_t, C.POINTER(c_dptr)]),
    "pdq_free": (C.c_int, [c_ctx, c_dptr]),
    "pdq_host_alloc": (C.c_int, [c_ctx, C.c_size_t, C.POINTER(C.c_void_p)]),
    "pdq_host_free": (C.c_int, [c_ctx, C.c_void_p]),
    "pdq_memcpy_h2d": (C.c_int, [c_ctx, c_dptr, C.c_void_p, C.c_size_t]),
    "pdq_memcpy_d2h": (C.c_int, [c_ctx, C.c_void_p, c_dptr, C.c_size_t]),
    "pdq_memcpy_d2h_strided": (C.c_int, [c_ctx, C.c_void_p, c_dptr, C.c_size_t, C.c_size_t, C.c_size_t]),
    "pdq_memcpy_d2d": (C.c_int, [c_ctx, c_dptr, c_dptr, C.c_size_t]),
    "pdq_memcpy_d2h_side": (C.c_int, [c_ctx, C.c_void_p, c_dptr, C.c_size_t]),
    "pdq_side_join": (C.c_int, [c_ctx]),
    "pdq_memset": (C.c_int, [c_ctx, c_dptr, C.c_int, C.c_size_t]),
    "pdq_sync": (C.c_int, [c_ctx]),
    "pdq_event_record": (C.c_int, [c_ctx, C.c_int]),
    "pdq_event_elapsed_ms": (C.c_int, [c_ctx, C.c_int, C.c_int, C.POINTER(C.c_float)]),
    "pdq_capture_begin": (C.c_int, [c_ctx]),
    "pdq_capture_end": (C.c_int, [c_ctx, C.POINTER(C.c_void_p)]),
    "pdq_graph_launch": (C.c_int, [c_ctx, C.c_void_p]),
    "pdq_graph_destroy": (None, [c_ctx, C.c_void_p]),
    "pdq_design_create": (C.c_int, [c_ctx, f64p, f64p, C.c_int, C.c_int, C.POINTER(c_design)]),
    "pdq_design_destroy": (None, [c_ctx, c_design]),
    "pdq_lin_reg_mu": (C.c_int, [c_ctx, i64p, C.c_int64, C.c_int, C.c_int, f64p, f64p, C.c_int, C.c_double, f64p]),
    "pdq_irls": (C.c_int, [c_ctx, i64p, C.c_int64, C.c_int, C.c_int, f64p, f64p, C.c_int, f64p, C.c_double, C.c_double,
                           C.c_double, C.c_double, C.c_int, f64p, f64p, f64p, f64p, C.POINTER(C.c_int)]),
    "pdq_alpha_mle": (C.c_int, [c_ctx, i64p, C.c_int64, C.c_int, C.c_int, f64p, C.c_int, f64p, C.c_int64, f64p,
                                C.c_double, C.c_double, C.c_double, C.c_int, C.c_int, f64p, f64p]),
    "pdq_wald_test": (C.c_int, [c_ctx, f64p, C.c_int, C.c_int, f64p, f64p, f64p, C.c_int64, C.c_int, f64p, f64p,
                                C.c_double, C.c_int, f64p, f64p, f64p]),
    "pdq_wald_contrasts": (C.c_int, [c_ctx, f64p, f64p, C.c_int, C.c_int, f64p, f64p, C.c_int, f64p, C.c_int, f64p, f64p,
                                     C.POINTER(C.c_int), f64p, f64p, f64p, C.c_int64]),
    "pdq_fit_rough_dispersions": (C.c_int, [c_ctx, f64p, C.c_int64, C.c_int, C.c_int, f64p, C.c_int, f64p]),
    "pdq_fit_moments_dispersions": (C.c_int, [c_ctx, f64p, C.c_int64, C.c_int, C.c_int, f64p, f64p, f64p]),
    "pdq_lin_reg_mu_dev": (C.c_int, [c_ctx, c_design, c_dptr, C.c_int64, C.c_int, C.c_double, c_dptr, C.c_int64]),
    "pdq_irls_dev": (C.c_int, [c_ctx, c_design, c_dptr, C.c_int64, C.c_int, c_dptr, C.c_double, C.c_double, C.c_double,
                               C.c_double, C.c_int, c_dptr, c_dptr, c_dptr, C.c_int64, c_dptr, c_dptr]),
    "pdq_irls_wald_dev": (C.c_int, [c_ctx, c_design, c_dptr, C.c_int64, C.c_int, c_dptr, C.c_double, C.c_double, C.c_double,
                                    C.c_double, C.c_int, c_dptr, c_dptr, c_dptr, C.c_int64, c_dptr, c_dptr, f64p, f64p,
                                    C.c_double, C.c_int, c_dptr, c_dptr, c_dptr]),
    "pdq_map_irls_wald_dev": (C.c_int, [c_ctx, c_design, c_dptr, C.c_int64, C.c_int, c_dptr, C.c_int64, c_dptr, c_dptr, c_dptr, c_dptr,
                                        C.c_double, C.c_double, C.c_double, c_dptr, c_dptr, c_dptr, c_dptr, c_dptr, C.c_double,
                                        C.c_double, C.c_double, C.c_double, C.c_int, c_dptr, c_dptr, c_dptr, C.c_int64, c_dptr, f64p,
                                        f64p, C.c_double, C.c_int, c_dptr, c_dptr, c_dptr]),
    "pdq_map_irls_status": (C.c_int, [c_ctx, C.POINTER(C.c_uint64)]),
    "pdq_alpha_mle_dev": (C.c_int, [c_ctx, c_design, c_dptr, C.c_int64, C.c_int, c_dptr, C.c_int64, c_dptr, C.c_double,
                                    C.c_double, C.c_double, c_dptr, C.c_int, C.c_int, c_dptr, c_dptr]),
    "pdq_alpha_mle_hint_dev": (C.c_int, [c_ctx, c_design, c_dptr, C.c_int64, C.c_int, c_dptr, C.c_int64, c_dptr, C.c_double,
                                         C.c_double, C.c_double, c_dptr, C.c_int, C.c_int, c_dptr, c_dptr, c_dptr, c_dptr]),
    "pdq_wald_test_dev": (C.c_int, [c_ctx, c_design, c_dptr, c_dptr, c_dptr, C.c_int64, C.c_int, f64p, f64p, C.c_double,
                                    C.c_int, c_dptr, c_dptr, c_dptr]),
    "pdq_mom_dispersions_dev": (C.c_int, [c_ctx, c_design, c_dptr, C.c_int64, C.c_int, C.c_double, C.c_double, c_dptr,
                                          c_dptr, C.c_double, c_dptr, C.c_int64]),
    "pdq_mom_alpha_mle_dev": (C.c_int, [c_ctx, c_design, c_dptr, C.c_int64, C.c_int, C.c_double, C.c_double, C.c_double, c_dptr,
                                        c_dptr, c_dptr, C.c_int64, c_dptr, c_dptr, c_dptr]),
    "pdq_calculate_cooks": (C.c_int, [c_ctx, i64p, C.c_int64, C.c_int, C.c_int, f64p, f64p, C.c_int, f64p, f64p, C.c_int64,
                                      C.c_double, f64p, f64p, f64p, f64p]),
    "pdq_cooks_dev": (C.c_int, [c_ctx, c_design, c_dptr, C.c_int64, C.c_int, c_dptr, c_dptr, C.c_int64, C.c_double, c_dptr,
                                C.c_int64, c_dptr, c_dptr, c_dptr]),
    "pdq_size_factors": (C.c_int, [c_ctx, i64p, C.c_int64, C.c_int, C.c_int, f64p, f64p]),
    "pdq_fp64_peak_tflops": (C.c_int, [c_ctx, f64p]),
    "pdq_lfc_shrink_nbinom_glm": (C.c_int, [c_ctx, f64p, i64p, C.c_int64, C.c_int, C.c_int, C.c_int, f64p, f64p, C.c_double,
                                            C.c_double, C.c_int, f64p, f64p, f64p, C.POINTER(C.c_int)]),
    "pdq_lfc_shrink_dev": (C.c_int, [c_ctx, c_design, c_dptr, C.c_int64, C.c_int, c_dptr, C.c_double, C.c_double, C.c_int, c_dptr,
                                     c_dptr, c_dptr, c_dptr]),
    "pdq_size_factors_dev": (C.c_int, [c_ctx, c_dptr, C.c_int64, C.c_int, C.c_int, c_dptr, c_dptr]),
    "pdq_size_factors_ex": (C.c_int, [c_ctx, i64p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_void_p, f64p, f64p]),
    "pdq_size_factors_ex_dev": (C.c_int, [c_ctx, c_dptr, C.c_int64, C.c_int, C.c_int, C.c_int, c_dptr, c_dptr, c_dptr]),
    "pdq_size_factors_from_logmeans": (C.c_int, [c_ctx, i64p, C.c_int64, C.c_int, C.c_int, f64p, f64p]),
    "pdq_size_factors_from_logmeans_dev": (C.c_int, [c_ctx, c_dptr, C.c_int64, C.c_int, C.c_int, c_dptr, c_dptr]),
    "pdq_vst_transform": (C.c_int, [c_ctx, i64p, C.c_int64, C.c_int, C.c_int, f64p, C.c_int, C.c_double, C.c_double, f64p,
                                    C.c_int64]),
    "pdq_vst_transform_dev": (C.c_int, [c_ctx, c_dptr, C.c_int64, C.c_int, C.c_int, c_dptr, C.c_int, C.c_double, C.c_double,
                                        c_dptr, C.c_int64]),
    "pdq_padj_rejections": (C.c_int, [c_ctx, f64p, C.c_int, f64p, C.c_int64, C.c_int, f64p, C.c_int, C.c_double, f64p,
                                       C.POINTER(C.c_int)]),
    "pdq_padj_bh": (C.c_int, [c_ctx, f64p, C.c_int, f64p, C.c_int64, C.c_int, f64p, f64p, C.c_int64]),
    "pdq_dispersion_trend_gamma_glm": (C.c_int, [c_ctx, f64p, f64p, C.c_size_t, f64p, f64p, C.POINTER(C.c_int)]),
    "pdq_trend_prior": (C.c_int, [c_ctx, f64p, f64p, C.c_size_t, C.c_double, C.c_double, C.c_double, f64p, f64p]),
    "pdq_trend_fit_dev": (C.c_int, [c_ctx, c_dptr, c_dptr, C.c_size_t, C.c_double, C.c_double, C.c_double, c_dptr, c_dptr]),
    "pdq_gather_columns_dev": (C.c_int, [c_ctx, c_dptr, C.c_int64, C.c_int, c_dptr, C.c_int, c_dptr, C.c_int64]),
    "pdq_column_sums_dev": (C.c_int, [c_ctx, c_dptr, C.c_int64, C.c_int, C.c_int, c_dptr]),
    "pdq_scatter_rows_dev": (C.c_int, [c_ctx, c_dptr, c_dptr, c_dptr, C.c_int, C.c_int, C.c_int64, C.c_int]),
    "pdq_scatter_segments_dev": (C.c_int, [c_ctx, c_dptr, c_dptr, c_dptr, C.c_int, i64p]),
    "pdq_select_dispersions_dev": (C.c_int, [c_ctx, c_dptr, c_dptr, c_dptr, c_dptr, C.c_size_t, C.c_double, C.c_double, c_dptr,
                                             c_dptr]),
    "pdq_mu_from_lfc_dev": (C.c_int, [c_ctx, c_design, c_dptr, C.c_int, c_dptr, C.c_int64]),
    "pdq_comm_unique_id": (C.c_int, [c_ctx, C.c_void_p]),
    "pdq_comm_init": (C.c_int, [c_ctx, C.c_void_p, C.c_int, C.c_int]),
    "pdq_allgather_f64_dev": (C.c_int, [c_ctx, c_dptr, c_dptr, C.c_size_t]),
    "pdq_allgather_multi_f64_dev": (C.c_int, [c_ctx, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_size_t]),
    "pdq_comm_destroy": (C.c_int, [c_ctx]),
    "pdq_peer_window_alloc": (C.c_int, [c_ctx, C.c_size_t, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_void_p]),
    "pdq_peer_window_free": (C.c_int, [c_ctx, c_dptr]),
    "pdq_peer_group_open": (C.c_int, [c_ctx, c_dptr, C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_void_p)]),
    "pdq_peer_push_dev": (C.c_int, [c_ctx, C.c_void_p, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64), C.c_size_t]),
    "pdq_peer_status": (C.c_int, [c_ctx, C.c_void_p, C.POINTER(C.c_uint64)]),
    "pdq_peer_group_close": (C.c_int, [c_ctx, C.c_void_p]),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)
_lib = None


def load() -> C.CDLL:
    """Load the CUDA library; raise (never fall back) when it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise B200Error(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). pydeseq2_b200 has no CPU fallback."
        )
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here = header/library mismatch
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def as_f64p(a: np.ndarray):
    return a.ctypes.data_as(f64p)


def as_i64p(a: np.ndarray):
    return a.ctypes.data_as(i64p)


class Context:
    """Owns one ``pdq_ctx`` (one per backend object, not thread-safe -- like the reference's caller)."""

    def __init__(self, device: int = 0):
        self.lib = load()
        h = c_ctx()
        rc = self.lib.pdq_ctx_create(int(device), C.byref(h))
        if rc != 0:
            n = self.lib.pdq_device_count()
            raise B200Error(f"pdq_ctx_create(device={device}) failed: {STATUS.get(rc, rc)} ({n} CUDA device(s) visible); "
                            "this backend needs an sm_90 (H100) GPU and has no CPU fallback")
        self.h = h
        self.device = int(device)
        self.wide_designs = False  # pdq_set_wide_designs: designs of up to PDQ_MAX_P_WIDE columns
        self.wide_shrink = False   # pdq_set_wide_shrink: apeGLM shrinkage of those designs
        self.large_designs = False  # pdq_set_large_designs: designs of up to PDQ_MAX_P_LARGE columns (with wide_designs)
        self.large_shrink = False   # pdq_set_large_shrink: apeGLM shrinkage of those (with the three above)
        self._pin_pool = {}  # nbytes -> [addresses] of released page-locked blocks (cudaHostAlloc is expensive)

    def set_wide_designs(self, on: bool = True):
        """Accept designs of PDQ_MAX_P + 1 .. PDQ_MAX_P_WIDE columns on this context (off by default)."""
        self.check(self.lib.pdq_set_wide_designs(self.h, 1 if on else 0))
        self.wide_designs = bool(on)

    def set_wide_shrink(self, on: bool = True):
        """Run apeGLM shrinkage of designs of PDQ_MAX_P + 1 .. PDQ_MAX_P_WIDE columns on this context (off by default; needs
        :meth:`set_wide_designs` as well, or such designs are refused as without it)."""
        self.check(self.lib.pdq_set_wide_shrink(self.h, 1 if on else 0))
        self.wide_shrink = bool(on)

    def set_large_designs(self, on: bool = True):
        """Accept designs of PDQ_MAX_P_WIDE + 1 .. PDQ_MAX_P_LARGE columns on this context (off by default; needs
        :meth:`set_wide_designs` as well, or designs wider than PDQ_MAX_P are refused as without it)."""
        self.check(self.lib.pdq_set_large_designs(self.h, 1 if on else 0))
        self.large_designs = bool(on)

    def set_large_shrink(self, on: bool = True):
        """Run apeGLM shrinkage of designs of PDQ_MAX_P_WIDE + 1 .. PDQ_MAX_P_LARGE columns on this context (off by default;
        needs :meth:`set_wide_designs`, :meth:`set_wide_shrink` and :meth:`set_large_designs` as well, or such calls are
        refused as without it)."""
        self.check(self.lib.pdq_set_large_shrink(self.h, 1 if on else 0))
        self.large_shrink = bool(on)

    def check(self, rc: int):
        if rc != 0:
            msg = self.lib.pdq_last_error(self.h)
            raise B200Error(f"{STATUS.get(rc, rc)}: {msg.decode() if msg else ''}")

    def close(self):
        if getattr(self, "h", None):
            for blocks in self._pin_pool.values():
                for addr in blocks:
                    self.lib.pdq_host_free(self.h, C.c_void_p(addr))
            self._pin_pool = {}
            self.lib.pdq_ctx_destroy(self.h)
            self.h = None

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    # -- small conveniences used by the resident pipeline / bench --------------------------------
    def info(self):
        name = C.create_string_buffer(256)
        sm = C.c_int()
        mem = C.c_size_t()
        self.check(self.lib.pdq_device_info(self.h, name, 256, C.byref(sm), C.byref(mem)))
        return {"name": name.value.decode(), "sm_count": sm.value, "mem_bytes": mem.value}

    def malloc(self, nbytes: int) -> int:
        p = c_dptr()
        self.check(self.lib.pdq_malloc(self.h, int(nbytes), C.byref(p)))
        return p.value

    def free(self, dptr):
        if dptr:
            self.check(self.lib.pdq_free(self.h, c_dptr(dptr)))

    def h2d(self, dptr, arr: np.ndarray):
        assert arr.flags.c_contiguous
        self.check(self.lib.pdq_memcpy_h2d(self.h, c_dptr(dptr), arr.ctypes.data_as(C.c_void_p), arr.nbytes))

    def d2h(self, arr: np.ndarray, dptr):
        assert arr.flags.c_contiguous
        self.check(self.lib.pdq_memcpy_d2h(self.h, arr.ctypes.data_as(C.c_void_p), c_dptr(dptr), arr.nbytes))

    def d2h_side(self, arr: np.ndarray, dptr):
        """Like :meth:`d2h`, on a branch of the stream that overlaps the work enqueued after it; :meth:`side_join` ends the branch."""
        assert arr.flags.c_contiguous
        self.check(self.lib.pdq_memcpy_d2h_side(self.h, arr.ctypes.data_as(C.c_void_p), c_dptr(dptr), arr.nbytes))

    def side_join(self):
        """Order the stream behind every :meth:`d2h_side` copy since the previous join."""
        self.check(self.lib.pdq_side_join(self.h))

    def d2h_strided(self, arr: np.ndarray, dptr, stride: int):
        """arr[i] = the element at dptr + i * stride bytes (one element per `stride` bytes of device memory)."""
        assert arr.flags.c_contiguous and arr.ndim == 1
        self.check(self.lib.pdq_memcpy_d2h_strided(self.h, arr.ctypes.data_as(C.c_void_p), c_dptr(dptr), arr.itemsize, int(stride),
                                                   arr.size))

    def sync(self):
        self.check(self.lib.pdq_sync(self.h))

    def record(self, slot: int):
        self.check(self.lib.pdq_event_record(self.h, slot))

    def elapsed_ms(self, a: int, b: int) -> float:
        ms = C.c_float()
        self.check(self.lib.pdq_event_elapsed_ms(self.h, a, b, C.byref(ms)))
        return float(ms.value)

    def launches(self) -> int:
        return int(self.lib.pdq_launch_count(self.h))

    def residency_stats(self) -> dict:
        """Counters of the content-addressed residency cache of the host-buffer entry points."""
        v = [C.c_int64() for _ in range(4)]
        self.check(self.lib.pdq_residency_stats(self.h, *[C.byref(x) for x in v]))
        return dict(zip(("hits", "misses", "hit_bytes", "resident_bytes"), (x.value for x in v)))

    def residency_clear(self):
        self.check(self.lib.pdq_residency_clear(self.h))

    def fp64_peak_tflops(self) -> float:
        """Measured DFMA throughput of this device (TFLOP/s): the arithmetic roofline of the FP64-bound kernels."""
        out = np.zeros(1)
        self.check(self.lib.pdq_fp64_peak_tflops(self.h, as_f64p(out)))
        return float(out[0])

    def pinned_empty(self, shape, dtype=np.float64) -> np.ndarray:
        """numpy array backed by page-locked host memory (released when the array is collected)."""
        return np.asarray(_Pinned(self, tuple(int(s) for s in np.atleast_1d(shape)), np.dtype(dtype)))


class _Pinned:
    """Owner of one cudaHostAlloc block, exposed to numpy through ``__array_interface__``."""

    def __init__(self, ctx: Context, shape, dtype):
        n = max(int(np.prod(shape)) * dtype.itemsize, 1)
        pool = ctx._pin_pool.get(n)
        if pool:
            addr = pool.pop()
        else:
            p = C.c_void_p()
            ctx.check(ctx.lib.pdq_host_alloc(ctx.h, n, C.byref(p)))
            addr = p.value
        self._ctx = ctx  # keeps the context alive for as long as the block is
        self._addr = addr
        self._n = n
        self.__array_interface__ = {"shape": shape, "typestr": dtype.str, "data": (addr, False), "version": 3}

    def __del__(self):  # pragma: no cover
        try:
            if self._addr and self._ctx.h:
                pool = self._ctx._pin_pool.setdefault(self._n, [])
                if len(pool) < 6:
                    pool.append(self._addr)  # recycled by the next pinned_empty of the same size
                else:
                    self._ctx.lib.pdq_host_free(self._ctx.h, C.c_void_p(self._addr))
        except Exception:
            pass
