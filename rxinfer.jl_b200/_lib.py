"""ctypes binding of librxgauss.so (include/rxgauss.h).  Fails loudly: there is no CPU fallback.

This is the Python stand-in for the Julia ``ccall`` shim (julia/RxGaussB200.jl) -- Julia is not
available in the build image, so the host-side mirror of the reference interface is Python.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_longlong, c_size_t, c_uint, c_uint8, c_void_p

HERE = os.path.dirname(os.path.abspath(__file__))
# RXG_LIB selects an A/B build of the same library (tuning experiments); the product is librxgauss.so
LIB_PATH = os.environ.get("RXG_LIB") or os.path.join(HERE, "librxgauss.so")

RXG_OK, RXG_ERR_BAD_ARG, RXG_ERR_CUDA, RXG_ERR_NCCL = 0, 1, 2, 3
RXG_ERR_NOT_SPD, RXG_ERR_NAN, RXG_ERR_UNSUPPORTED, RXG_ERR_NO_DEVICE = 4, 5, 6, 7
STATUS_NAMES = {0: "OK", 1: "BAD_ARG", 2: "CUDA", 3: "NCCL", 4: "NOT_SPD", 5: "NAN", 6: "UNSUPPORTED", 7: "NO_DEVICE"}

PTR_DEVICE = 1 << 0
MODEL_PER_CHAIN = 1 << 1
ASYNC = 1 << 2
COV_SHARED_OUT = 1 << 3
PATH_PER_CHAIN = 1 << 4
TRANSITION_FIRST = 1 << 5
COV_REPLICATE = 1 << 6
MASK_SHARED = 1 << 7
U_SEQ_SHARED = 1 << 8      # u is one input sequence for every chain, a host array [rows, d]
U_SEQ_CHAIN = 1 << 9       # u is a per-chain input sequence, a device array [rows, d, batch]
RXG_DELTA_LINEARIZATION, RXG_DELTA_UNSCENTED = 0, 1

fp = POINTER(c_float)
u8p = POINTER(c_uint8)
i32p = POINTER(c_int32)

# name -> (restype, argtypes); the single source of truth checked against include/rxgauss.h by
# tests/test_abi.py
SIGNATURES = {
    "rxg_version": (c_int, []),
    "rxg_create": (c_int, [POINTER(c_void_p), c_int, c_uint]),
    "rxg_destroy": (c_int, [c_void_p]),
    "rxg_last_error": (c_char_p, [c_void_p]),
    "rxg_set_option": (c_int, [c_void_p, c_int, c_longlong]),
    "rxg_get_option": (c_int, [c_void_p, c_int, POINTER(c_longlong)]),
    "rxg_set_stream": (c_int, [c_void_p, c_void_p]),
    "rxg_sync": (c_int, [c_void_p]),
    "rxg_host_alloc": (c_int, [POINTER(c_void_p), c_size_t]),
    "rxg_host_free": (c_int, [c_void_p]),
    "rxg_supports": (c_int, [c_int, c_int]),
    "rxg_host_fill_threads": (c_int, []),
    "rxg_launch_count": (c_longlong, [c_void_p]),
    "rxg_set_profiling": (c_int, [c_void_p, c_int]),
    "rxg_profile_last_ms": (c_int, [c_void_p, POINTER(c_float), POINTER(c_float)]),
    "rxg_rule_mvnormal_meancov_out_f32": (c_int, [c_void_p, c_int64, c_int, fp, fp, fp, c_int, fp, fp, c_uint]),
    "rxg_rule_mvnormal_meancov_mean_f32": (c_int, [c_void_p, c_int64, c_int, fp, fp, fp, c_int, fp, fp, c_uint]),
    "rxg_rule_mvnormal_meancov_mean_data_f32": (c_int, [c_void_p, c_int64, c_int, fp, fp, c_int, fp, fp, c_uint]),
    "rxg_rule_mul_out_f32": (c_int, [c_void_p, c_int64, c_int, c_int, fp, c_int, fp, fp, fp, fp, c_uint]),
    "rxg_rule_mul_in_f32": (c_int, [c_void_p, c_int64, c_int, c_int, fp, c_int, fp, fp, fp, fp, i32p, c_uint]),
    "rxg_rule_add_out_f32": (c_int, [c_void_p, c_int64, c_int, fp, fp, fp, fp, fp, fp, c_uint]),
    "rxg_rule_add_in_f32": (c_int, [c_void_p, c_int64, c_int, fp, fp, fp, fp, fp, fp, c_uint]),
    "rxg_prod_gaussian_f32": (c_int, [c_void_p, c_int64, c_int, fp, fp, fp, fp, fp, fp, c_uint]),
    "rxg_meancov_to_wmp_f32": (c_int, [c_void_p, c_int64, c_int, fp, fp, fp, fp, i32p, c_uint]),
    "rxg_wmp_to_meancov_f32": (c_int, [c_void_p, c_int64, c_int, fp, fp, fp, fp, i32p, c_uint]),
    "rxg_marginal_gaussian_f32": (c_int, [c_void_p, c_int64, c_int, c_int, POINTER(fp), POINTER(fp), fp, fp, i32p, c_uint]),
    "rxg_rule_normal_precision_tau_f32": (c_int, [c_void_p, c_int64, fp, fp, fp, fp, fp, fp, c_uint]),
    "rxg_rule_normal_precision_out_f32": (c_int, [c_void_p, c_int64, fp, fp, fp, fp, fp, fp, c_uint]),
    "rxg_rule_normal_precision_tau_joint_f32": (c_int, [c_void_p, c_int64, fp, fp, fp, fp, c_uint]),
    "rxg_rule_mvnormal_precision_lambda_f32": (c_int, [c_void_p, c_int64, c_int, fp, fp, fp, fp, fp, fp, c_uint]),
    "rxg_prod_wishart_f32": (c_int, [c_void_p, c_int64, c_int, fp, fp, fp, fp, fp, fp, c_uint]),
    "rxg_wishart_mean_f32": (c_int, [c_void_p, c_int64, c_int, fp, fp, fp, i32p, c_uint]),
    "rxg_mv_iid_wishart_vmp_f32": (c_int, [c_void_p, c_int, c_int, c_int64, c_int, fp, fp, c_float, fp, fp, fp, fp, fp, fp, fp, i32p, c_uint]),
    "rxg_ar_vmp_f32": (c_int, [c_void_p, c_int, c_int, c_int64, c_int, c_float, c_float, c_float, c_float, c_float, fp, fp, fp, fp, fp, POINTER(c_double), c_uint]),
    "rxg_lar_vmp_f32": (c_int, [c_void_p, c_int, c_int, c_int64, c_int, fp, fp, fp, fp, fp, fp, fp, fp, POINTER(c_double), i32p, c_uint]),
    "rxg_gmm_vmp_f32": (c_int, [c_void_p, c_int, c_int, c_int, c_int64, c_int, fp, fp, fp, fp, fp, fp, fp, fp, fp, fp, fp, fp, fp, fp,
                                fp, fp, POINTER(c_double), fp, fp, fp, fp, fp, fp, i32p, c_uint]),
    "rxg_hmm_vmp_f32": (c_int, [c_void_p, c_int, c_int, c_int, c_int64, c_int, fp, fp, fp, fp, fp, fp, fp, u8p, fp, fp, fp, fp,
                                POINTER(c_double), fp, fp, fp, i32p, c_uint]),
    "rxg_hmm_gauss_vmp_f32": (c_int, [c_void_p, c_int, c_int, c_int, c_int64, c_int, fp, fp, fp, fp, fp, fp, fp, fp, fp, fp, fp, fp,
                                      fp, fp, fp, fp, fp, fp, fp, fp, POINTER(c_double), fp, fp, fp, fp, fp, fp, i32p, c_uint]),
    "rxg_binomial_polya_vmp_f32": (c_int, [c_void_p, c_int, c_int, c_int64, c_int, fp, fp, fp, i32p, i32p, fp, fp, POINTER(c_double),
                                           fp, fp, i32p, c_uint]),
    "rxg_multinomial_polya_vmp_f32": (c_int, [c_void_p, c_int, c_int, c_int64, c_int, fp, fp, i32p, fp, fp, POINTER(c_double),
                                              fp, fp, i32p, c_uint]),
    "rxg_multinomial_polya_online_f32": (c_int, [c_void_p, c_int, c_int, c_int64, c_int, fp, fp, POINTER(c_double),
                                                 POINTER(c_double), i32p, POINTER(c_double), POINTER(c_double), fp, fp,
                                                 POINTER(c_double), i32p, c_uint]),
    "rxg_prod_gamma_f32": (c_int, [c_void_p, c_int64, fp, fp, fp, fp, fp, fp, c_uint]),
    "rxg_prod_normal_f32": (c_int, [c_void_p, c_int64, fp, fp, fp, fp, fp, fp, c_uint]),
    "rxg_rule_gcv_out_f32": (c_int, [c_void_p, c_int64, fp, fp, fp, fp, c_float, c_float, fp, fp, c_uint]),
    "rxg_marginalrule_gcv_yx_f32": (c_int, [c_void_p, c_int64, fp, fp, fp, fp, fp, fp, c_float, c_float, fp, fp, c_uint]),
    "rxg_rule_gcv_z_prod_f32": (c_int, [c_void_p, c_int64, fp, fp, fp, fp, c_float, c_float, fp, fp, c_uint]),
    "rxg_lgssm_smooth_f32": (c_int, [c_void_p, c_int, c_int, c_int, c_int64, fp, fp, fp, fp, fp, fp, fp, fp, u8p, fp, fp, fp, i32p, c_uint]),
    "rxg_lgssm_smooth_predict_f32": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int64, fp, fp, fp, fp, fp, fp, fp, fp, u8p, fp, fp, fp,
                                             fp, fp, fp, fp, i32p, c_uint]),
    "rxg_lgssm_filter_f32": (c_int, [c_void_p, c_int, c_int, c_int, c_int64, fp, fp, fp, fp, fp, fp, fp, fp, u8p, fp, fp, fp, i32p, c_uint]),
    "rxg_lgssm_vmp_gamma_f32": (c_int, [c_void_p, c_int, c_int64, c_int, c_float, c_float, c_float, c_float, c_float, c_float, c_float, fp, fp, fp, fp, fp, c_uint]),
    "rxg_lgssm_vmp_gamma_fe_f32": (c_int, [c_void_p, c_int, c_int64, c_int, c_float, c_float, c_float, c_float, c_float, c_float, c_float, fp, fp, fp, fp, fp, fp, c_uint]),
    "rxg_lgssm_vmp_wishart_f32": (c_int, [c_void_p, c_int, c_int, c_int, c_int64, c_int, fp, fp, fp, fp, fp, fp, c_float, fp, fp, fp,
                                          u8p, fp, fp, fp, fp, POINTER(c_double), i32p, c_uint]),
    "rxg_lgssm_vmp_noise_f32": (c_int, [c_void_p, c_int, c_int, c_int, c_int64, c_int, fp, fp, fp, fp, fp, fp, c_float, fp, fp, fp,
                                        c_float, fp, fp, fp, u8p, fp, fp, fp, fp, fp, fp, POINTER(c_double), i32p, c_uint]),
    "rxg_lgssm_vmp_transition_f32": (c_int, [c_void_p, c_int, c_int, c_int, c_int64, c_int, fp, fp, fp, fp, fp, fp, fp, fp, fp, c_float,
                                             fp, fp, fp, c_float, fp, fp, fp, u8p, fp, fp, fp, fp, fp, fp, fp, fp, POINTER(c_double),
                                             i32p, c_uint]),
    "rxg_hgf_filter_f32": (c_int, [c_void_p, c_int, c_int64, c_int, c_float, c_float, c_float, c_float, fp, fp, fp, c_uint]),
    "rxg_hgf_filter_fe_f32": (c_int, [c_void_p, c_int, c_int64, c_int, c_float, c_float, c_float, c_float, fp, fp, fp, fp, fp, c_uint]),
    "rxg_hgf_vmp_learn_f32": (c_int, [c_void_p, c_int, c_int64, c_int, fp, c_float, c_float, fp, fp, fp, fp, fp, fp,
                                      POINTER(c_double), i32p, c_uint]),
    "rxg_lgssm_filter_chunk_f32": (c_int, [c_void_p, c_int, c_int, c_int, c_int64, fp, fp, fp, fp, fp, fp, fp, fp, fp, fp, fp, c_uint]),
    "rxg_hgf_filter_chunk_f32": (c_int, [c_void_p, c_int, c_int64, c_int, c_float, c_float, c_float, c_float, fp, fp, fp, c_uint]),
    "rxg_stream_vmp_gamma_f32": (c_int, [c_void_p, c_int, c_int64, c_int, c_float, fp, fp, fp, fp, fp, c_uint]),
    "rxg_selftest_umma_f32": (c_int, [c_void_p, fp, fp, fp, c_uint]),
    "rxg_selftest_umma_shape_f32": (c_int, [c_void_p, c_int, c_int, fp, fp, fp, c_uint]),
    "rxg_selftest_stream_f32": (c_int, [c_void_p, c_int64, c_int, c_int, fp, fp, c_uint]),
    "rxg_selftest_host_fill_gbs": (c_double, [fp, c_int64, c_int64, c_int, c_int]),
    "rxg_comm_unique_id": (c_int, [c_void_p]),
    "rxg_comm_init": (c_int, [c_void_p, c_int, c_int, c_void_p]),
    "rxg_allgather_posteriors": (c_int, [c_void_p, c_int, c_int, c_int64, fp, fp, fp, fp, c_uint]),
    "rxg_device_alloc": (c_int, [c_void_p, c_size_t, POINTER(c_void_p)]),
    "rxg_device_free": (c_int, [c_void_p, c_void_p]),
    "rxg_device_memset": (c_int, [c_void_p, c_void_p, c_int, c_size_t]),
    "rxg_memcpy_h2d": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t]),
    "rxg_memcpy_d2h": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t]),
    "rxg_peer_export": (c_int, [c_void_p, c_void_p, c_void_p]),
    "rxg_peer_open": (c_int, [c_void_p, c_void_p, POINTER(c_void_p)]),
    "rxg_peer_close": (c_int, [c_void_p, c_void_p]),
    "rxg_peer_group": (c_int, [c_void_p, c_int, c_int, POINTER(c_void_p)]),
    "rxg_peer_barrier": (c_int, [c_void_p, c_uint]),
    "rxg_peer_allgather_f32": (c_int, [c_void_p, c_int64, fp, POINTER(fp), c_uint]),
    "rxg_lgssm_smooth_gather_f32": (c_int, [c_void_p, c_int, c_int, c_int, c_int64, fp, fp, fp, fp, fp, fp, fp, fp, u8p,
                                            POINTER(fp), POINTER(fp), fp, i32p, c_uint]),
    "rxg_delta_check_source": (c_int, [c_char_p, c_char_p, c_char_p, c_int, c_int, c_int, POINTER(c_double), c_char_p,
                                       c_size_t]),
    "rxg_delta_model_create": (c_int, [c_void_p, c_char_p, c_char_p, c_char_p, c_int, c_int, c_int, POINTER(c_double),
                                       POINTER(c_void_p), c_char_p, c_size_t]),
    "rxg_delta_compile_count": (c_longlong, [c_void_p]),
    "rxg_delta_smooth_f32": (c_int, [c_void_p, c_void_p, c_int, c_int64, fp, fp, fp, fp, fp, fp, u8p, fp, fp, fp, fp, i32p,
                                     c_uint]),
    "rxg_delta_filter_chunk_f32": (c_int, [c_void_p, c_void_p, c_int, c_int64, fp, fp, fp, c_int, fp, u8p, fp, fp, fp, fp,
                                           fp, fp, i32p, c_uint]),
}


class RxGaussError(RuntimeError):
    def __init__(self, code, msg=""):
        self.code = code
        super().__init__(f"librxgauss error {code} ({STATUS_NAMES.get(code, '?')}): {msg}")


_lib = None
MISSING: list = []


def _missing_entry(name):
    def call(*a, **k):
        raise ImportError(f"{LIB_PATH} does not export {name}: rebuild it (python rxinfer.jl_b200/build.py)")
    return call


def _preload_nvrtc():
    """The Delta node compiles user functions with NVRTC, which the library opens as libnvrtc.so.12 on first use.  When
    the NVRTC wheel that PyTorch depends on is installed, load its copy globally so that this soname resolves even
    where no CUDA toolkit is on the loader's path."""
    import importlib.util
    try:
        spec = importlib.util.find_spec("nvidia.cuda_nvrtc")
    except (ImportError, ValueError):
        return
    for base in (spec.submodule_search_locations or []) if spec else []:
        path = os.path.join(base, "lib", "libnvrtc.so.12")
        if os.path.exists(path):
            ctypes.CDLL(path, mode=ctypes.RTLD_GLOBAL)
            return


def load():
    """Load the in-tree shared library.  Raises (never falls back) if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    _preload_nvrtc()
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python rxinfer.jl_b200/build.py` "
            "(nvcc, sm_90a).  There is no CPU fallback for the hot path.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            # a library older than this table (e.g. a stale build next to newer sources): everything it does export keeps
            # working, the missing entry fails loudly when it is CALLED; tests/test_abi.py requires MISSING to be empty
            MISSING.append(name)
            setattr(lib, name, _missing_entry(name))
            continue
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def as_fp(ptr_int):
    return ctypes.cast(c_void_p(int(ptr_int) if ptr_int else None), fp)
