"""ctypes binding of libdmosopt_b200.so (include/dmosopt_b200.h).

Thin layer: argument marshalling and error translation only.  Every function
takes/returns NumPy arrays (host) -- or, for inputs, anything exposing a CUDA
device pointer through ``data_ptr()`` (torch tensors) when the caller keeps
data resident.  There is deliberately NO CPU fallback: if the CUDA library is
missing or no GPU is present the import of the library / creation of the
context raises.
"""

import ctypes
import os
import threading
import weakref

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdmosopt_b200.so")

METRIC_NONE, METRIC_CROWDING, METRIC_EUCLIDEAN = 0, 1, 2
KERNEL_MATERN52, KERNEL_RBF = 0, 1
GP_FP64, GP_TENSOR, GP_AUTO = 0, 1, 2
POSTERIOR_GP, POSTERIOR_SVGP, POSTERIOR_DGP = 0, 1, 2  # dmo_nsga2_step_record_posterior, dmo_smpso_step_record: dmo_gp, dmo_svgp, dmo_dgp
GP_PREDICT_MAX_D = 64  # input dimensions of dmo_gp_create (csrc/gp.cu KS_DMAX) and of every tensor-core predict
GP_PREDICT_MAX_M = 16  # objectives of dmo_gp_create (csrc/gp.cu GP_MAX_M)
HV_MAX_OBJECTIVES = 8  # dmo_hypervolume: exact, chain sums for M <= 5 (csrc/hv.cu), limit-set recursion for 6 .. 8 (csrc/hv_many.cu)

_c_i64 = ctypes.c_int64
_c_u64 = ctypes.c_uint64
_c_int = ctypes.c_int
_c_dbl = ctypes.c_double
_vp = ctypes.c_void_p

# exported symbols -> (restype, argtypes); checked against the header by tests/test_abi.py
_SIGNATURES = {
    "dmo_version": (_c_int, []),
    "dmo_create": (_c_int, [_c_int, ctypes.POINTER(_vp)]),
    "dmo_destroy": (_c_int, [_vp]),
    "dmo_last_error": (ctypes.c_char_p, [_vp]),
    "dmo_synchronize": (_c_int, [_vp]),
    "dmo_stream": (_vp, [_vp]),
    "dmo_launch_count": (_c_i64, [_vp]),
    "dmo_wait_count": (_c_i64, [_vp]),
    "dmo_sm_count": (_c_int, [_vp]),
    "dmo_timer_begin": (_c_int, [_vp]),
    "dmo_timer_end": (_c_int, [_vp, ctypes.POINTER(ctypes.c_float)]),
    "dmo_host_alloc": (_c_int, [ctypes.POINTER(_vp), _c_u64]),
    "dmo_host_free": (_c_int, [_vp]),
    "dmo_device_alloc": (_c_int, [_vp, ctypes.POINTER(_vp), _c_u64]),
    "dmo_device_free": (_c_int, [_vp, _vp]),
    "dmo_memcpy": (_c_int, [_vp, _vp, _vp, _c_u64]),
    "dmo_flush_l2": (_c_int, [_vp]),
    "dmo_transfer_bytes": (_c_int, [_vp, ctypes.POINTER(_c_u64), ctypes.POINTER(_c_u64)]),
    "dmo_profile_enable": (_c_int, [_vp, _c_int]),
    "dmo_profile_report": (_c_int, [_vp, ctypes.c_char_p, _c_u64]),
    "dmo_round_f32": (_c_int, [_vp, _vp, _c_i64]),
    "dmo_rank_nd": (_c_int, [_vp, _vp, _c_i64, _c_int, _vp]),
    "dmo_crowding_distance": (_c_int, [_vp, _vp, _c_i64, _c_int, _vp]),
    "dmo_euclidean_distance": (_c_int, [_vp, _vp, _c_i64, _c_int, _vp]),
    "dmo_order_mo": (_c_int, [_vp, _vp, _c_i64, _c_int, _c_int, _vp, _c_int, _vp, _vp, _vp]),
    "dmo_remove_worst": (_c_int, [_vp, _vp, _vp, _c_i64, _c_int, _c_int, _c_int, _vp, _c_int, _c_i64, _vp, _vp, _vp, _vp]),
    "dmo_remove_worst_pair": (_c_int, [_vp, _vp, _vp, _c_i64, _vp, _vp, _c_i64, _c_int, _c_int, _c_int, _c_i64, _vp, _vp, _vp, _vp]),
    "dmo_remove_worst_pair_keys": (_c_int, [_vp, _vp, _vp, _c_i64, _vp, _vp, _c_i64, _c_int, _c_int, _c_int, _vp, _c_i64, _vp, _vp, _vp, _vp]),
    "dmo_tournament": (_c_int, [_vp, _vp, _vp, _c_i64, _c_i64, _c_u64, _c_u64, _vp, _vp]),
    "dmo_mutation_u": (_c_int, [_vp, _vp, _vp, _c_i64, _c_int, _vp, _vp, _vp, _c_dbl, _vp]),
    "dmo_sbx_u": (_c_int, [_vp, _vp, _vp, _vp, _c_i64, _c_int, _vp, _vp, _vp, _vp, _vp]),
    "dmo_nsga2_plan_length": (_c_i64, [_c_i64, _c_dbl, _c_dbl]),
    "dmo_nsga2_generate": (
        _c_int,
        [_vp, _vp, _c_i64, _c_int, _vp, _c_i64, _c_i64, _c_dbl, _c_dbl, _c_dbl, _vp, _vp, _vp, _vp, _c_u64, _c_u64, _vp, _vp, _vp, _vp],
    ),
    "dmo_gp_create": (_c_int, [_vp, _c_i64, _c_int, _c_int, _c_int, _vp, _vp, _vp, _c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, ctypes.POINTER(_vp)]),
    "dmo_gp_destroy": (_c_int, [_vp, _vp]),
    "dmo_gp_fit": (_c_int, [_vp, _c_i64, _c_int, _c_int, _c_int, _vp, _vp, _vp, _vp, _vp, _c_dbl, _vp, _vp, _vp]),
    "dmo_gp_set_linear_mean": (_c_int, [_vp, _vp, _vp, _vp]),
    "dmo_gp_predict": (_c_int, [_vp, _vp, _vp, _c_i64, _vp, _vp, _c_int]),
    "dmo_gp_auto_info": (_c_int, [_vp, _vp, ctypes.POINTER(_c_int), ctypes.POINTER(_c_int), ctypes.POINTER(_c_dbl), ctypes.POINTER(_c_dbl),
                                  ctypes.POINTER(_c_dbl), ctypes.POINTER(_c_i64)]),
    "dmo_gp_covariance_groups": (_c_int, [_vp, _vp, ctypes.POINTER(_c_int), _vp]),
    "dmo_mtgp_create": (_c_int, [_vp, _c_i64, _c_int, _c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, ctypes.POINTER(_c_dbl),
                                 ctypes.POINTER(_vp)]),
    "dmo_mtgp_predict": (_c_int, [_vp, _vp, _vp, _c_i64, _vp, _vp, _c_int]),
    "dmo_mtgp_destroy": (_c_int, [_vp, _vp]),
    "dmo_svgp_create": (_c_int, [_vp, _c_int, _c_int, _c_i64, _c_int, _vp, _vp, _vp, _vp, _vp, _vp, _c_dbl, _vp, _vp, _vp, _vp, _vp,
                                 ctypes.POINTER(_vp)]),
    "dmo_svgp_predict": (_c_int, [_vp, _vp, _vp, _c_i64, _vp, _vp, _c_int]),
    "dmo_svgp_groups": (_c_int, [_vp, _vp, ctypes.POINTER(_c_int), ctypes.POINTER(_c_int)]),
    "dmo_svgp_destroy": (_c_int, [_vp, _vp]),
    "dmo_svgp_optimal_q": (_c_int, [_vp, _c_i64, _c_i64, _c_int, _c_int, _vp, _vp, _vp, _vp, _vp, _vp, _c_dbl, _c_int, _vp, _vp]),
    "dmo_svgp_fit_create": (_c_int, [_vp, _c_i64, _c_int, _c_int, _c_int, _c_i64, _vp, _vp, _vp, _c_int, _c_dbl, ctypes.POINTER(_vp)]),
    "dmo_svgp_fit_destroy": (_c_int, [_vp, _vp]),
    "dmo_svgp_fit_natgrad": (_c_int, [_vp, _vp, _vp, _c_i64, _vp, _vp, _vp, _vp, _c_dbl]),
    "dmo_svgp_fit_elbo_grad": (_c_int, [_vp, _vp, _vp, _c_i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "dmo_svgp_fit_q": (_c_int, [_vp, _vp, _vp, _vp]),
    "dmo_dgp_create": (_c_int, [_vp, _c_int, _c_int, _c_int, _c_i64, _c_i64, _vp, _vp, _vp, _vp, _vp, _vp, _c_dbl, _vp, _vp, _vp, _vp, _vp,
                                _c_dbl, _vp, _c_dbl, _c_dbl, _c_int, _vp, _vp, _vp, _vp, _vp, ctypes.POINTER(_vp)]),
    "dmo_dgp_predict": (_c_int, [_vp, _vp, _vp, _c_i64, _c_u64, _c_u64, _vp, _vp, _vp, _c_int]),
    "dmo_dgp_destroy": (_c_int, [_vp, _vp]),
    "dmo_dgp_fit_create": (_c_int, [_vp, _c_i64, _c_int, _c_int, _c_int, _c_i64, _c_i64, _c_int, _c_int, _c_i64, _vp, _vp, _vp, _c_dbl, _c_dbl,
                                    ctypes.POINTER(_vp)]),
    "dmo_dgp_fit_destroy": (_c_int, [_vp, _vp]),
    "dmo_dgp_fit_set_params": (_c_int, [_vp, _vp, _vp, _c_i64]),
    "dmo_dgp_fit_get_params": (_c_int, [_vp, _vp, _vp, _c_i64]),
    "dmo_dgp_fit_loss_grad": (_c_int, [_vp, _vp, _vp, _c_i64, _c_u64, _c_u64, _vp, _vp, _vp, _vp]),
    "dmo_dgp_fit_adam_step": (_c_int, [_vp, _vp, _c_dbl]),
    "dmo_dgp_fit_epoch": (_c_int, [_vp, _vp, _vp, _c_i64, _c_dbl, _c_u64, _c_u64, _vp]),
    "dmo_mtgp_lml_grad": (_c_int, [_vp, _c_i64, _c_int, _c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "dmo_gp_lml_grad": (_c_int, [_vp, _c_i64, _c_int, _c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "dmo_nsga2_step": (_c_int, [_vp, _vp, _vp, _vp, _vp, _c_i64, _c_int, _c_int, _c_dbl, _c_dbl, _c_dbl, _vp, _vp, _vp, _vp, _c_u64, _c_u64,
                                _c_int, _c_int, _c_int, _c_int, _vp, _vp, _vp]),
    "dmo_nsga2_step_record": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _c_i64, _c_int, _c_int, _c_dbl, _c_dbl, _c_dbl, _vp, _vp, _vp, _vp,
                                       _c_u64, _c_u64, _c_int, _c_int, _c_int, _vp, _vp, _vp, _vp]),
    "dmo_nsga2_step_record_posterior": (_c_int, [_vp, _c_int, _vp, _c_u64, _c_u64, _vp, _vp, _vp, _vp, _c_i64, _c_int, _c_int, _c_dbl, _c_dbl,
                                                 _c_dbl, _vp, _vp, _vp, _vp, _c_u64, _c_u64, _c_int, _c_int, _c_int, _c_int, _vp, _vp, _vp,
                                                 _vp]),
    "dmo_hypervolume": (_c_int, [_vp, _vp, _c_i64, _c_int, _vp, ctypes.POINTER(_c_dbl)]),
    "dmo_hypervolume_ranked": (_c_int, [_vp, _vp, _c_i64, _c_int, _vp, _vp, ctypes.POINTER(_c_dbl)]),
    "dmo_nondominated_flags": (_c_int, [_vp, _vp, _c_i64, _c_int, _vp]),
    "dmo_hypervolume_mc": (_c_int, [_vp, _vp, _c_i64, _c_int, _vp, _c_int, _c_dbl, _c_dbl, _c_i64, _c_u64, _c_u64, ctypes.POINTER(_c_dbl),
                                    ctypes.POINTER(_c_i64), ctypes.POINTER(_c_i64), ctypes.POINTER(_c_int)]),
    "dmo_ehvi_select": (_c_int, [_vp, _vp, _c_i64, _vp, _vp, _c_i64, _c_int, _vp, _c_int, _c_i64, _vp, _vp]),
    "dmo_get_duplicates": (_c_int, [_vp, _vp, _c_i64, _c_int, _c_dbl, _vp]),
    "dmo_get_duplicates_pair": (_c_int, [_vp, _vp, _c_i64, _vp, _c_i64, _c_int, _c_dbl, _vp]),
    "dmo_epsilon_sort": (_c_int, [_vp, _vp, _c_i64, _c_int, _vp, _vp, ctypes.POINTER(_c_i64)]),
    "dmo_age_survival": (_c_int, [_vp, _vp, _vp, _c_i64, _c_int, _c_dbl, _vp, _c_int, _vp]),
    "dmo_smpso_velocity": (_c_int, [_vp, _vp, _vp, _vp, _vp, _c_int, _c_i64, _c_int, _c_dbl, _c_dbl, _c_dbl, _c_dbl, _c_dbl, _c_dbl, _vp, _vp, _vp]),
    "dmo_mutate_groups": (_c_int, [_vp, _vp, _c_i64, _c_i64, _c_i64, _c_int, _vp, _vp, _vp, _c_dbl, _c_u64, _c_u64, _vp, _vp]),
    "dmo_cmaes_sample": (_c_int, [_vp, _vp, _vp, _c_int, _vp, _c_i64, _vp, _vp, _c_i64, _c_int, _vp]),
    "dmo_cmaes_update_cholesky": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _c_i64, _c_int, _c_dbl, _c_dbl, _c_dbl]),
    "dmo_gather_rows": (_c_int, [_vp, _vp, _vp, _vp, _vp, _c_i64, _c_i64, _vp]),
    "dmo_cmaes_generate": (_c_int, [_vp, _vp, _vp, _c_int, _vp, _c_i64, _vp, _vp, _c_i64, _c_int, _vp, _vp, _vp]),
    "dmo_cmaes_step_z": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _c_i64, _c_int, _vp]),
    "dmo_scale_rows": (_c_int, [_vp, _vp, _c_i64, _c_i64, _vp, _vp, _vp, _c_i64]),
    "dmo_benchmark_eval": (_c_int, [_vp, _c_int, _vp, _c_i64, _c_int, _c_int, _c_dbl, _vp]),
    "dmo_sa_dgsm_design": (_c_int, [_vp, _vp, _c_i64, _c_int, _vp, _vp, _c_dbl, _vp]),
    "dmo_sa_fast_design": (_c_int, [_vp, _c_i64, _c_int, _vp, _vp, _vp, _vp, _vp]),
    "dmo_sa_dgsm_stats": (_c_int, [_vp, _vp, _vp, _c_i64, _c_int, _c_int, _vp, _vp, _vp, _c_int, _c_dbl, _vp, _vp, _vp, _vp]),
    "dmo_l2_discrepancy_terms": (_c_int, [_vp, _c_int, _vp, _c_i64, _c_int, _vp, _vp]),
    "dmo_glp_cd2_terms": (_c_int, [_vp, _vp, _c_i64, _c_int, _c_i64, _c_i64, _vp, _vp]),
    "dmo_glp_cd2_pairs": (_c_int, [_vp, _vp, _c_i64, _c_int, _c_i64, _c_i64, _vp]),
    "dmo_feas_fit": (_c_int, [_vp, _vp, _c_i64, _c_int, _c_int, _vp, _vp, _vp, _vp, _c_int, _vp, _c_int, _c_dbl, _vp, _vp, _vp, _vp, _vp, _vp,
                              _vp, _vp]),
    "dmo_feas_create": (_c_int, [_vp, _c_int, _c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, ctypes.POINTER(_vp)]),
    "dmo_feas_destroy": (_c_int, [_vp, _vp]),
    "dmo_feas_eval": (_c_int, [_vp, _vp, _vp, _c_i64, _c_int, _vp, _vp, _vp]),
    "dmo_smpso_generate": (_c_int, [_vp, _vp, _vp, _c_int, _c_i64, _c_int, _vp, _vp, _vp, _c_dbl, _c_u64, _c_u64, _vp, _vp]),
    "dmo_smpso_update": (_c_int, [_vp, _vp, _vp, _vp, _vp, _c_int, _vp, _c_int, _c_i64, _c_int, _c_int, _c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "dmo_smpso_step_record": (_c_int, [_vp, _c_int, _vp, _c_u64, _c_u64, _c_int, _vp, _vp, _vp, _c_int, _c_i64, _c_int, _c_int, _vp, _vp, _vp,
                                       _c_dbl, _c_u64, _c_u64, _c_int, _c_int, _c_int, _vp, _vp, _vp, _vp]),
    "dmo_cmaes_step_record": (_c_int, [_vp, _c_int, _vp, _c_u64, _c_u64, _c_int, _c_int, _c_int, _c_int, _vp, _vp, _c_int, _vp, _vp, _c_i64,
                                       _c_int, _c_int, _vp, _vp, _c_i64, _c_i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "dmo_cmaes_step_apply": (_c_int, [_vp, _vp, _vp, _c_int, _vp, _vp, _vp, _c_i64, _c_int, _c_int, _vp, _vp, _vp, _c_i64, _c_i64, _vp, _vp,
                                      _vp, _vp, _c_i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _c_dbl, _c_dbl, _c_dbl, _vp, _vp, _vp, _vp, _vp,
                                      _vp, _vp]),
}

_lib = None
_ctx = None
_ctx_device = None
_lock = threading.Lock()


class DmoError(RuntimeError):
    pass


def load_library(path=None):
    """Load the shared library and declare every prototype.  Raises if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    path = path or LIB_PATH
    if not os.path.exists(path):
        raise DmoError(
            f"dmosopt_b200: CUDA library {path} not found. Build it with `python -m dmosopt_b200.build` "
            "(nvcc, sm_90a). There is no CPU fallback."
        )
    lib = ctypes.CDLL(path)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def default_device():
    for k in ("DMOSOPT_B200_DEVICE", "LOCAL_RANK"):
        v = os.environ.get(k)
        if v is not None and v.strip() != "":
            return int(v)
    return 0


def context(device=None):
    """The process-wide context (one per process == one per GPU)."""
    global _ctx, _ctx_device
    with _lock:
        if _ctx is not None and (device is None or device == _ctx_device):
            return _ctx
        lib = load_library()
        dev = default_device() if device is None else int(device)
        h = _vp()
        st = lib.dmo_create(dev, ctypes.byref(h))
        if st != 0 or not h.value:
            raise DmoError(f"dmosopt_b200: dmo_create(device={dev}) failed with status {st}: no usable CUDA device (H100 required)")
        if _ctx is not None:
            lib.dmo_destroy(_ctx)
        _ctx, _ctx_device = h, dev
        return _ctx


def _check(st, what, ctx=None):
    if st != 0:
        msg = _lib.dmo_last_error(_ctx if ctx is None else ctx)
        raise DmoError(f"{what} failed (status {st}): {msg.decode() if msg else ''}")


# Additional contexts on the same GPU (own stream, own scratch): independent sub-problems of one call -- the swarms of an
# SMPSO update -- are issued from worker threads, one context each, so their latency-bound kernels (the rank chains)
# overlap on the device.  The C library is not re-entrant per context; different contexts may run concurrently.
_worker_ctx = []
_worker_pool = None


def worker_context(i):
    """The i-th worker context on the main context's GPU (created on first use)."""
    main = context()
    with _lock:
        while len(_worker_ctx) <= i:
            h = _vp()
            st = load_library().dmo_create(_ctx_device, ctypes.byref(h))
            if st != 0 or not h.value:
                raise DmoError(f"dmosopt_b200: dmo_create(device={_ctx_device}) failed for a worker context (status {st})")
            _worker_ctx.append(h)
    assert main is not None
    return _worker_ctx[i]


def worker_pool():
    global _worker_pool
    if _worker_pool is None:
        from concurrent.futures import ThreadPoolExecutor

        _worker_pool = ThreadPoolExecutor(max_workers=8, thread_name_prefix="dmosopt_b200_worker")
    return _worker_pool


def _ptr(a):
    """Raw pointer of a NumPy array, a torch CUDA tensor (data_ptr) or None."""
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    if hasattr(a, "data_ptr"):
        return int(a.data_ptr())
    if isinstance(a, int):
        return a
    raise TypeError(f"cannot pass {type(a)} to the CUDA library")


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _per_dim(v, d):
    """A scalar or (d,) distribution index as a (d,) float64 array."""
    return _f64(np.broadcast_to(np.asarray(v, dtype=np.float64), (d,)))


def _seed(seed):
    """A seed as the library's uint64."""
    return int(seed) & (2**64 - 1)


# --------------------------------------------------------------------------- context utilities
def synchronize():
    _check(load_library().dmo_synchronize(context()), "dmo_synchronize")


def stream_ptr():
    """The CUDA stream (cudaStream_t as an integer) every library call is issued on: wrap it with
    ``torch.cuda.ExternalStream`` to order torch / NCCL work with the library without device-wide synchronisation."""
    return int(load_library().dmo_stream(context()))


def launch_count():
    lib = load_library()
    return int(lib.dmo_launch_count(context())) + sum(int(lib.dmo_launch_count(c)) for c in _worker_ctx)


def wait_count():
    """Times the library has blocked the host on its stream (a stream synchronise or a blocking copy), all contexts."""
    lib = load_library()
    return int(lib.dmo_wait_count(context())) + sum(int(lib.dmo_wait_count(c)) for c in _worker_ctx)


def sm_count():
    return int(load_library().dmo_sm_count(context()))


def timer_begin():
    _check(load_library().dmo_timer_begin(context()), "dmo_timer_begin")


def timer_end():
    ms = ctypes.c_float()
    _check(load_library().dmo_timer_end(context(), ctypes.byref(ms)), "dmo_timer_end")
    return float(ms.value)


def flush_l2():
    _check(load_library().dmo_flush_l2(context()), "dmo_flush_l2")


def transfer_bytes():
    h2d = d2h = 0
    for c in [context()] + list(_worker_ctx):
        a, b = _c_u64(0), _c_u64(0)
        _check(load_library().dmo_transfer_bytes(c, ctypes.byref(a), ctypes.byref(b)), "dmo_transfer_bytes")
        h2d, d2h = h2d + int(a.value), d2h + int(b.value)
    return h2d, d2h


def profile_enable(on=True):
    _check(load_library().dmo_profile_enable(context(), 1 if on else 0), "dmo_profile_enable")


def profile_report():
    """{kernel name: (total ms, launches)} recorded since profile_enable(True)."""
    buf = ctypes.create_string_buffer(1 << 16)
    _check(load_library().dmo_profile_report(context(), buf, len(buf)), "dmo_profile_report")
    out = {}
    for line in buf.value.decode().splitlines():
        name, ms, cnt = line.rsplit(" ", 2)
        out[name] = (float(ms), int(cnt))
    return out


def round_f32(dev_ptr, n):
    _check(load_library().dmo_round_f32(context(), _ptr(dev_ptr), int(n)), "dmo_round_f32")


class DeviceArray:
    """A typed device buffer owned by the library context (for callers that keep populations resident)."""

    def __init__(self, shape, dtype=np.float64):
        self.shape = tuple(np.atleast_1d(shape).tolist()) if not isinstance(shape, tuple) else shape
        self.dtype = np.dtype(dtype)
        self.nbytes = int(np.prod(self.shape)) * self.dtype.itemsize
        p = _vp()
        _check(load_library().dmo_device_alloc(context(), ctypes.byref(p), max(self.nbytes, 1)), "dmo_device_alloc")
        self.ptr = p.value

    def data_ptr(self):
        return self.ptr

    def offset(self, nelem):
        """Raw pointer ``nelem`` elements into the buffer."""
        return self.ptr + int(nelem) * self.dtype.itemsize

    def upload(self, a):
        a = np.ascontiguousarray(a, dtype=self.dtype)
        assert a.nbytes <= self.nbytes
        _check(load_library().dmo_memcpy(context(), self.ptr, a.ctypes.data, a.nbytes), "dmo_memcpy")
        return self

    def download(self, count=None):
        n = int(np.prod(self.shape)) if count is None else int(count)
        out = np.empty(n, dtype=self.dtype)
        _check(load_library().dmo_memcpy(context(), out.ctypes.data, self.ptr, out.nbytes), "dmo_memcpy")
        return out.reshape(self.shape) if count is None else out

    def free(self):
        if self.ptr:
            load_library().dmo_device_free(context(), self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def memcpy(dst, src, nbytes):
    _check(load_library().dmo_memcpy(context(), _ptr(dst), _ptr(src), int(nbytes)), "dmo_memcpy")


# Page-locked host buffers are pooled: cudaHostAlloc of a population-sized block costs milliseconds, and the plugins
# hand out one offspring matrix per generation.  A block returns to the pool when the last NumPy view of it dies.
_pin_pool = {}
_pin_pool_bytes = 0
_PIN_POOL_LIMIT = 1 << 30
# page-locked bytes currently handed out (not pooled).  Callers such as MOASMO.optimize keep every offspring matrix of
# an epoch alive (x_new history): beyond this budget new offspring matrices are ordinary pageable arrays.
_pin_live_bytes = 0
_PIN_LIVE_LIMIT = int(os.environ.get("DMOSOPT_B200_PINNED_LIMIT", str(4 << 30)))
# Device mirrors of read-only host arrays the library itself produced (offspring matrix, population state):
# {host address: (nbytes, DeviceArray)}.  ``_in`` substitutes the device address, so data that was born on the GPU is
# not shipped back over PCIe when the caller hands it to the next call.  Only non-writeable arrays qualify: a
# caller who wants to edit must copy, and the copy has no mirror.
_mirrors = {}


def _pin_release(ptr, nbytes):
    global _pin_pool_bytes, _pin_live_bytes
    _pin_live_bytes -= nbytes
    _mirrors.pop(ptr, None)
    lst = _pin_pool.setdefault(nbytes, [])
    if len(lst) < 4 and _pin_pool_bytes + nbytes <= _PIN_POOL_LIMIT:
        lst.append(ptr)
        _pin_pool_bytes += nbytes
    elif _lib is not None:
        _lib.dmo_host_free(ptr)


def pinned_empty(shape, dtype=np.float64):
    """NumPy array backed by page-locked host memory (pooled; recycled when the last view is collected)."""
    global _pin_pool_bytes, _pin_live_bytes
    lib = load_library()
    context()
    dt = np.dtype(dtype)
    count = int(np.prod(shape))
    nbytes = (max(count * dt.itemsize, 1) + 4095) & ~4095
    lst = _pin_pool.get(nbytes)
    if lst:
        addr = lst.pop()
        _pin_pool_bytes -= nbytes
    else:
        p = _vp()
        if lib.dmo_host_alloc(ctypes.byref(p), nbytes) != 0:
            raise DmoError("dmo_host_alloc failed")
        addr = p.value
    buf = (ctypes.c_char * nbytes).from_address(addr)
    _pin_live_bytes += nbytes
    weakref.finalize(buf, _pin_release, addr, nbytes)
    return np.frombuffer(buf, dtype=dt, count=count).reshape(shape)


def mirror_register(host, dev):
    """Declare ``dev`` (DeviceArray) the device copy of the pinned array ``host`` (from pinned_empty)."""
    _mirrors[host.ctypes.data] = (host.nbytes, dev)


def _mirror_of(addr):
    """(base, nbytes, DeviceArray) of the registered host block that starts at or contains ``addr``, else None."""
    ent = _mirrors.get(addr)
    if ent is not None:
        return (addr,) + ent
    for base, (nbytes, dev) in list(_mirrors.items()):  # a finaliser may drop an entry while we look
        if base <= addr < base + nbytes:
            return base, nbytes, dev
    return None


def _mirrored_out(dev, nbytes=None):
    """Read-only host copy of ``dev`` (a DeviceArray the library has written; only its first ``nbytes`` are copied back
    when given) that keeps ``dev`` as its device mirror.  It is page-locked while the page-locked budget lasts; past it
    the caller is hoarding outputs, so it is pageable and its mirror is dropped with it."""
    if _pin_live_bytes < _PIN_LIVE_LIMIT:
        out = pinned_empty(dev.shape, dev.dtype)
    else:
        out = np.empty(dev.shape, dtype=dev.dtype)
        weakref.finalize(out, _mirrors.pop, out.ctypes.data, None)
    memcpy(out, dev.ptr, dev.nbytes if nbytes is None else nbytes)
    mirror_register(out, dev)
    out.flags.writeable = False
    return out


def mirror_drop(a):
    """Forget (and free) the device copy of ``a``: the host array stays valid, later uses simply upload it again.

    The optimizers call this once ``update`` has consumed an offspring matrix, so a caller that keeps every x_gen of an
    epoch (MOASMO.optimize's history) holds host memory only, not one HBM buffer per generation."""
    if not isinstance(a, np.ndarray):
        return
    m = _mirror_of(a.ctypes.data)
    if m is not None:
        _mirrors.pop(m[0], None)
        m[2].free()


def mirror_upload(host):
    """Refresh the device mirror of ``host`` after a host-side write through its writable base."""
    ent = _mirrors.get(host.ctypes.data)
    if ent is not None:
        ent[1].upload(host)


def mirror_ptr(a, require_readonly=True):
    """Device address mirroring the host array ``a`` (or an interior C-contiguous view of it), else None."""
    if not _mirrors or not isinstance(a, np.ndarray) or not a.flags.c_contiguous:
        return None
    if require_readonly and a.flags.writeable:
        return None
    m = _mirror_of(a.ctypes.data)
    if m is None:
        return None
    base, nbytes, dev = m
    off = a.ctypes.data - base
    return dev.ptr + off if dev.ptr and off + a.nbytes <= nbytes else None


def mirror_array(a):
    """The DeviceArray mirroring all of the host array ``a`` (same start, same size), else None."""
    if not isinstance(a, np.ndarray):
        return None
    ent = _mirrors.get(a.ctypes.data)
    if ent is None or ent[0] != a.nbytes or not ent[1].ptr:
        return None
    return ent[1]


def _in(a):
    """Pointer for an input array: the device mirror when the library holds one, else the host address."""
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        m = mirror_ptr(a)
        return m if m is not None else a.ctypes.data
    return _ptr(a)


def mirrored_readonly(a):
    """(read-only view, writable pinned base) of a page-locked, device-mirrored copy of ``a``.

    Returns (copy of a, None) when no CUDA context can be created (host-only unit tests)."""
    a = np.asarray(a)
    try:
        base = pinned_empty(a.shape, a.dtype)
        base[...] = a
        dev = DeviceArray(a.shape, a.dtype).upload(base)
    except DmoError:
        return np.array(a, copy=True), None
    mirror_register(base, dev)
    view = base.view()
    view.flags.writeable = False
    return view, base


def copy_into_pooled(a):
    """Writable copy of ``a`` in a pooled page-locked buffer; a plain ``a.copy()`` when no CUDA context exists."""
    a = np.asarray(a)
    if a.nbytes < (1 << 20):
        return a.copy()
    try:
        out = pinned_empty(a.shape, a.dtype)
    except DmoError:
        return a.copy()
    m = mirror_ptr(a)
    if m is not None:  # the DMA engine copies device -> pinned host faster than one host thread copies host -> host
        memcpy(out, m, a.nbytes)
    else:
        np.copyto(out, a)
    return out


def pinned_like(a):
    """Page-locked copy of ``a`` (same dtype / values); falls back to a plain copy when no context exists yet."""
    a = np.asarray(a)
    try:
        out = pinned_empty(a.shape, a.dtype)
    except DmoError:
        return np.array(a, copy=True)
    out[...] = a
    return out


# --------------------------------------------------------------------------- A1/A2
def rank_nd(Y):
    """dda.dda_ens (dmosopt/dda.py:97-152) -> int64 rank array (canonical non-dominated rank)."""
    Y = _f64(Y)
    n, M = Y.shape
    rank = np.empty(n, dtype=np.int32)
    _check(load_library().dmo_rank_nd(context(), _ptr(Y), n, M, _ptr(rank)), "dmo_rank_nd")
    return rank.astype(np.intp)


def nondominated_flags(Y):
    """int32 (n,) array: 0 for the rank-0 rows, 1 for the dominated ones -- the hypervolume / EHVI filter's own route."""
    Y = _f64(Y)
    n, M = Y.shape
    flags = np.empty(n, dtype=np.int32)
    _check(load_library().dmo_nondominated_flags(context(), _ptr(Y), n, M, _ptr(flags)), "dmo_nondominated_flags")
    return flags


# --------------------------------------------------------------------------- A3/A4
def crowding_distance(Y):
    Y = _f64(Y)
    n, M = Y.shape
    D = np.empty(n, dtype=np.float64)
    _check(load_library().dmo_crowding_distance(context(), _ptr(Y), n, M, _ptr(D)), "dmo_crowding_distance")
    return D


def euclidean_distance(Y):
    Y = _f64(Y)
    n, M = Y.shape
    D = np.empty(n, dtype=np.float64)
    _check(load_library().dmo_euclidean_distance(context(), _ptr(Y), n, M, _ptr(D)), "dmo_euclidean_distance")
    return D


# --------------------------------------------------------------------------- A5
def _extra_keys(extra):
    if not extra:
        return None, 0, []
    arrs = [_f64(e) for e in extra]
    tab = (ctypes.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
    return ctypes.cast(tab, ctypes.c_void_p), len(arrs), arrs


def order_mo(Y, metric=METRIC_NONE, extra_desc_keys=None):
    """(perm, rank[perm], dist[perm] or None): the ordering of MOEA.orderMO (dmosopt/MOEA.py:300-347)."""
    Y = _f64(Y)
    n, M = Y.shape
    perm = np.empty(n, dtype=np.int64)
    rank = np.empty(n, dtype=np.int32)
    dist = np.empty(n, dtype=np.float64) if metric != METRIC_NONE else None
    tab, nex, keep = _extra_keys(extra_desc_keys)
    _check(load_library().dmo_order_mo(context(), _ptr(Y), n, M, metric, tab, nex, _ptr(perm), _ptr(rank), _ptr(dist)), "dmo_order_mo")
    return perm, rank.astype(np.intp), dist


def remove_worst(X, Y, keep, metric=METRIC_NONE, extra_desc_keys=None):
    """First ``keep`` rows of the sortMO order (dmosopt/MOEA.py:398-423): (X, Y, rank, perm)."""
    X = _f64(X)
    Y = _f64(Y)
    n, d = X.shape
    M = Y.shape[1]
    keep = int(min(keep, n))
    Xo = np.empty((keep, d), dtype=np.float64)
    Yo = np.empty((keep, M), dtype=np.float64)
    rank = np.empty(keep, dtype=np.int32)
    perm = np.empty(keep, dtype=np.int64)
    tab, nex, hold = _extra_keys(extra_desc_keys)
    _check(
        load_library().dmo_remove_worst(context(), _ptr(X), _ptr(Y), n, d, M, metric, tab, nex, keep, _ptr(Xo), _ptr(Yo), _ptr(rank), _ptr(perm)),
        "dmo_remove_worst",
    )
    return Xo, Yo, rank.astype(np.intp), perm


def remove_worst_pair(Xa, Ya, Xb, Yb, keep, metric=METRIC_NONE, out_X=None, key=None):
    """remove_worst(vstack(Xa, Xb), vstack(Ya, Yb), keep) without the host-side concatenation.

    ``out_X`` (optional, float64 C-contiguous (keep, d)) receives the surviving rows directly; it may be the writable
    base of ``Xb``.  When ``out_X`` has a device mirror the survivors are written to the mirror and copied out once.
    ``key`` (optional FeasModel): its rank over [Xa; Xb], evaluated on the device, is the least significant descending
    key (MOEA.remove_worst with x_distance_metrics=[key.rank]).
    """
    Xa, Ya, Xb, Yb = _f64(Xa), _f64(Ya), _f64(Xb), _f64(Yb)
    na, d = Xa.shape
    nb = Xb.shape[0]
    M = Ya.shape[1]
    keep = int(min(keep, na + nb))
    if out_X is not None and (out_X.dtype != np.float64 or not out_X.flags.c_contiguous or out_X.shape != (keep, d)):
        out_X = None
    Xo = out_X if out_X is not None else pinned_empty((keep, d), np.float64)
    Yo = np.empty((keep, M), dtype=np.float64)
    rank = np.empty(keep, dtype=np.int32)
    perm = np.empty(keep, dtype=np.int64)
    xo_dev = mirror_ptr(Xo, require_readonly=False) if out_X is not None else None
    fn, keys = ("dmo_remove_worst_pair", ()) if key is None else ("dmo_remove_worst_pair_keys", (key._h,))
    _check(
        getattr(load_library(), fn)(context(), _in(Xa), _in(Ya), na, _in(Xb), _in(Yb), nb, d, M, metric, *keys, keep,
                                    xo_dev if xo_dev is not None else _ptr(Xo), _ptr(Yo), _ptr(rank), _ptr(perm)),
        fn,
    )
    if xo_dev is not None:
        memcpy(Xo, xo_dev, Xo.nbytes)
    return Xo, Yo, rank.astype(np.intp), perm


# --------------------------------------------------------------------------- A6
def tournament(rank, poolsize, seed, stream_id, crowd=None, return_uniforms=False):
    rank = np.ascontiguousarray(rank, dtype=np.int32)
    pop = rank.shape[0]
    cr = None if crowd is None else _f64(crowd)
    pool = np.empty(int(poolsize), dtype=np.int64)
    u = np.empty(pop, dtype=np.float64) if return_uniforms else None
    _check(
        load_library().dmo_tournament(context(), _ptr(rank), _ptr(cr), pop, int(poolsize), _seed(seed), int(stream_id), _ptr(pool), _ptr(u)),
        "dmo_tournament",
    )
    return (pool, u) if return_uniforms else pool


# --------------------------------------------------------------------------- A7/A8
def mutation_u(parents, u, di_mutation, xlb, xub, mutation_rate):
    parents = np.atleast_2d(_f64(parents))
    u = np.atleast_2d(_f64(u))
    n, d = parents.shape
    di = _per_dim(di_mutation, d)
    out = np.empty((n, d), dtype=np.float64)
    lb, ub = _f64(xlb), _f64(xub)  # named: the arrays must outlive the call
    _check(load_library().dmo_mutation_u(context(), _ptr(parents), _ptr(u), n, d, _ptr(di), _ptr(lb), _ptr(ub), float(mutation_rate), _ptr(out)), "dmo_mutation_u")
    return out


def sbx_u(parent1, parent2, u, di_crossover, xlb, xub):
    p1 = np.atleast_2d(_f64(parent1))
    p2 = np.atleast_2d(_f64(parent2))
    u = np.atleast_2d(_f64(u))
    n, d = p1.shape
    di = _per_dim(di_crossover, d)
    c1 = np.empty((n, d), dtype=np.float64)
    c2 = np.empty((n, d), dtype=np.float64)
    lb, ub = _f64(xlb), _f64(xub)
    _check(load_library().dmo_sbx_u(context(), _ptr(p1), _ptr(p2), _ptr(u), n, d, _ptr(di), _ptr(lb), _ptr(ub), _ptr(c1), _ptr(c2)), "dmo_sbx_u")
    return c1, c2


# --------------------------------------------------------------------------- A9
def nsga2_generate(pop_x, pool_idx, popsize, crossover_prob, mutation_prob, mutation_rate, di_crossover, di_mutation, xlb, xub, seed, stream_id, return_draws=False):
    """Offspring of the NSGA-II / AGE-MOEA variation loop (dmosopt/NSGA2.py:142-178).

    Returns (x_gen (P, d), child_kind (P,) int32 [0/1 = SBX child 1/2, 2 = mutant][, draws]).
    ``draws`` (if requested) is a dict with the random draws the kernel used, for replay on the
    CPU oracle: u_cross (T,), u_mut (T,), pair (T, 2), single (T,), u_genes (T, 2, d), T = dmo_nsga2_plan_length
    (2*popsize+64 for the default rates).
    """
    pop_x = _f64(pop_x)
    npop, d = pop_x.shape
    pool_idx = np.ascontiguousarray(pool_idx, dtype=np.int64)
    popsize = int(popsize)
    T = int(load_library().dmo_nsga2_plan_length(popsize, float(crossover_prob), float(mutation_prob)))
    if T <= 0:
        raise DmoError("nsga2_generate: crossover_prob / mutation_prob too small to plan the variation loop")
    # the offspring matrix stays on the device as the mirror of the (read-only, page-locked) array handed back
    x_dev = DeviceArray((popsize + 1, d), np.float64)
    kind = np.empty(popsize + 1, dtype=np.int32)
    nch = np.zeros(1, dtype=np.int64)
    draws = np.empty(T * (5 + 2 * d), dtype=np.float64) if return_draws else None
    dic, dim = _per_dim(di_crossover, d), _per_dim(di_mutation, d)
    lb, ub = _f64(xlb), _f64(xub)
    _check(
        load_library().dmo_nsga2_generate(
            context(), _in(pop_x), npop, d, _ptr(pool_idx), pool_idx.shape[0], popsize, float(crossover_prob), float(mutation_prob),
            float(mutation_rate), _ptr(dic), _ptr(dim), _ptr(lb), _ptr(ub), _seed(seed), int(stream_id),
            x_dev.ptr, _ptr(kind), _ptr(nch), _ptr(draws),
        ),
        "dmo_nsga2_generate",
    )
    P = int(nch[0])
    x_gen = _mirrored_out(x_dev, P * d * 8)
    if not return_draws:
        return x_gen[:P], kind[:P]
    dd = {
        "u_cross": draws[0:T],
        "u_mut": draws[T : 2 * T],
        "pair": draws[2 * T : 4 * T].reshape(T, 2).astype(np.int64),
        "single": draws[4 * T : 5 * T].astype(np.int64),
        "u_genes": draws[5 * T :].reshape(T, 2, d),
    }
    return x_gen[:P], kind[:P], dd


def nsga2_step_record(gp, pop_x, pop_y, rank, crossover_prob, mutation_prob, mutation_rate, di_crossover, di_mutation, xlb, xub,
                      seed, stream_id, precision, metric, round_to_f32, x_gen, y_gen, counts, key=None):
    """One resident NSGA-II generation, recorded (dmo_nsga2_step_record).  Returns the offspring count P.

    ``gp`` a GPHandle; ``pop_x`` (pop, d) float64, ``pop_y`` (pop, M) float64 and ``rank`` (pop,) int32 are device
    buffers (DeviceArray, a device address or a CUDA tensor), updated in place.  ``x_gen`` (pop+1, d), ``y_gen`` (pop+1, M)
    float64 and ``counts`` (4,) int64 receive the offspring, their posterior mean and the operator counts; into device or
    page-locked memory they are complete only after ``synchronize()``.  ``key`` (optional FeasModel): its rank of
    [children; parents] is the truncation's last key."""
    pop, d, M, dic, dim, lb, ub, nch = _step_record_args("nsga2_step_record", pop_x, pop_y, di_crossover, di_mutation, xlb, xub, x_gen,
                                                         y_gen, counts)
    _check(
        load_library().dmo_nsga2_step_record(
            context(), gp._h, None if key is None else key._h, _ptr(pop_x), _ptr(pop_y), _ptr(rank), pop, d, M, float(crossover_prob),
            float(mutation_prob), float(mutation_rate), _ptr(dic), _ptr(dim), _ptr(lb), _ptr(ub), _seed(seed), int(stream_id), int(precision),
            int(metric), 1 if round_to_f32 else 0, _ptr(x_gen), _ptr(y_gen), _ptr(counts), _ptr(nch),
        ),
        "dmo_nsga2_step_record",
    )
    return int(nch[0])


def nsga2_step_record_posterior(kind, posterior, draw_key, pop_x, pop_y, rank, crossover_prob, mutation_prob, mutation_rate, di_crossover,
                                di_mutation, xlb, xub, seed, stream_id, precision, metric, mean_f32, round_to_f32, x_gen, y_gen, counts,
                                key=None):
    """``nsga2_step_record`` on another posterior (dmo_nsga2_step_record_posterior): ``kind`` POSTERIOR_GP, _SVGP or _DGP and
    ``posterior`` the GPHandle, SVGPHandle or DGPHandle.  The offspring's objectives are the mean that handle's predict
    writes with return_var=True, rounded to float32 first when ``mean_f32``; ``draw_key`` (seed, stream_id) keys a deep
    GP's Monte Carlo draws.  Returns the offspring count P."""
    pop, d, M, dic, dim, lb, ub, nch = _step_record_args("nsga2_step_record_posterior", pop_x, pop_y, di_crossover, di_mutation, xlb, xub,
                                                         x_gen, y_gen, counts)
    draw_seed, draw_stream = draw_key
    _check(
        load_library().dmo_nsga2_step_record_posterior(
            context(), int(kind), posterior._h, _seed(draw_seed), int(draw_stream), None if key is None else key._h, _ptr(pop_x), _ptr(pop_y),
            _ptr(rank), pop, d, M, float(crossover_prob), float(mutation_prob), float(mutation_rate), _ptr(dic), _ptr(dim), _ptr(lb), _ptr(ub),
            _seed(seed), int(stream_id), int(precision), int(metric), 1 if mean_f32 else 0, 1 if round_to_f32 else 0, _ptr(x_gen), _ptr(y_gen),
            _ptr(counts), _ptr(nch),
        ),
        "dmo_nsga2_step_record_posterior",
    )
    return int(nch[0])


def _step_record_args(who, pop_x, pop_y, di_crossover, di_mutation, xlb, xub, x_gen, y_gen, counts):
    """(pop, d, M, di_crossover, di_mutation, xlb, xub, n_children buffer) of a recorded step, its host record checked."""
    pop, d = int(pop_x.shape[0]), int(pop_x.shape[1])
    M = int(pop_y.shape[1])
    for name, a, shape, dt in (("x_gen", x_gen, (pop + 1, d), np.float64), ("y_gen", y_gen, (pop + 1, M), np.float64), ("counts", counts, (4,), np.int64)):
        if isinstance(a, np.ndarray) and (a.shape != shape or a.dtype != dt or not a.flags.c_contiguous or not a.flags.writeable):
            raise ValueError(f"{who}: {name} must be a writable C-contiguous {np.dtype(dt).name} array of shape {shape}")
    return pop, d, M, _per_dim(di_crossover, d), _per_dim(di_mutation, d), _f64(xlb), _f64(xub), np.zeros(1, dtype=np.int64)


# --------------------------------------------------------------------------- N1: exact-GP fit for given hyper-parameters
def gp_fit(X_train, y, constant, length_scale, noise, kernel=KERNEL_MATERN52, jitter=1e-10, want_L=True, want_alpha=True):
    """(L (M,N,N) or None, alpha (M,N) or None, lml (M,)) of the exact GP with the given hyper-parameters, per objective:
    K = c k(X, X) + (noise + jitter) I, L = chol(K), alpha = K^-1 y, lml = log marginal likelihood (dmo_gp_fit).
    X_train (N,d) normalised inputs, y (M,N) normalised targets, length_scale (M,d)."""
    X_train = _f64(X_train)
    N, d = X_train.shape
    y = _f64(y)
    M = y.shape[0]
    ls = np.empty((M, d), dtype=np.float64)
    for m in range(M):
        ls[m, :] = np.asarray(length_scale[m], dtype=np.float64)
    cst, nz = _f64(constant), _f64(noise)
    assert y.shape == (M, N) and cst.shape == (M,) and nz.shape == (M,)
    L = np.empty((M, N, N), dtype=np.float64) if want_L else None
    alpha = np.empty((M, N), dtype=np.float64) if want_alpha else None
    lml = np.empty(M, dtype=np.float64)
    _check(load_library().dmo_gp_fit(context(), N, d, M, int(kernel), _ptr(X_train), _ptr(y), _ptr(cst), _ptr(ls), _ptr(nz), float(jitter), _ptr(L), _ptr(alpha),
                                     _ptr(lml)), "dmo_gp_fit")
    return L, alpha, lml


def mtgp_lml_grad(X_train, Y, length_scale, B, D, weight, bias):
    """(lml, grads) of the multitask exact GP (covariance K_x (x) B + I (x) diag(D), linear mean per task) for the given
    hyper-parameters (dmo_mtgp_lml_grad): lml = log p(Y), grads a dict of d lml / d {length_scale (d,), B (M,M) with
    independent entries, D (M,), weight (M,d), bias (M,)}.  X_train (N,d) normalised inputs, Y (N,M) normalised targets."""
    X_train, Y = _f64(X_train), _f64(Y)
    N, d = X_train.shape
    if Y.ndim == 1:
        Y = Y.reshape(-1, 1)
    M = Y.shape[1]
    assert Y.shape == (N, M), Y.shape
    ls = _per_dim(np.reshape(length_scale, -1), d)
    Bm, Dv, w, b = _f64(B).reshape(M, M), _f64(D).reshape(M), _f64(weight).reshape(M, d), _f64(bias).reshape(M)
    lml = np.empty(1)
    g = {"length_scale": np.empty(d), "B": np.empty((M, M)), "D": np.empty(M), "weight": np.empty((M, d)), "bias": np.empty(M)}
    _check(load_library().dmo_mtgp_lml_grad(context(), N, d, M, _ptr(X_train), _ptr(Y), _ptr(ls), _ptr(Bm), _ptr(Dv), _ptr(w), _ptr(b),
                                            _ptr(lml), _ptr(g["length_scale"]), _ptr(g["B"]), _ptr(g["D"]), _ptr(g["weight"]),
                                            _ptr(g["bias"])), "dmo_mtgp_lml_grad")
    return float(lml[0]), g


def gp_lml_grad(X_train, Y, length_scale, outputscale, noise, weight, bias):
    """(lml (M,), grads) of M independent exact GPs, K_m = s_m Matern52(X / l_m) + noise_m I with the linear prior mean
    X w_m + b_m (dmo_gp_lml_grad): lml_m = log p(y_m), grads a dict of d lml_m / d {length_scale (M,d), outputscale (M,),
    noise (M,), weight (M,d), bias (M,)}.  X_train (N,d) normalised inputs, Y (N,M) normalised targets."""
    X_train, Y = _f64(X_train), _f64(Y)
    N, d = X_train.shape
    if Y.ndim == 1:
        Y = Y.reshape(-1, 1)
    M = Y.shape[1]
    assert Y.shape == (N, M), Y.shape
    yt = _f64(Y.T)
    ls, w = _f64(length_scale).reshape(M, d), _f64(weight).reshape(M, d)
    s, nz, b = _f64(outputscale).reshape(M), _f64(noise).reshape(M), _f64(bias).reshape(M)
    lml = np.empty(M)
    g = {"length_scale": np.empty((M, d)), "outputscale": np.empty(M), "noise": np.empty(M), "weight": np.empty((M, d)), "bias": np.empty(M)}
    _check(load_library().dmo_gp_lml_grad(context(), N, d, M, _ptr(X_train), _ptr(yt), _ptr(ls), _ptr(s), _ptr(nz), _ptr(w), _ptr(b),
                                          _ptr(lml), _ptr(g["length_scale"]), _ptr(g["outputscale"]), _ptr(g["noise"]), _ptr(g["weight"]),
                                          _ptr(g["bias"])), "dmo_gp_lml_grad")
    return lml, g


# --------------------------------------------------------------------------- objects the library owns
class _LibObject:
    """Owns one library object: the handle ``_h`` (ctypes.c_void_p), released through the symbol ``_destroy`` by
    close() or on collection.  Nothing is destroyed once the library or the main context is gone (interpreter exit)."""

    _destroy = None
    _h = None

    def close(self):
        if self._h is not None and _lib is not None and _ctx is not None:
            getattr(_lib, self._destroy)(_ctx, self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _predict_io(X, width, return_var):
    """(X as (P, d) float64, page-locked mean (P, width), page-locked var (P, width) or None) of a posterior predict."""
    X = _f64(X)
    if X.ndim == 1:
        X = X.reshape(1, -1)
    mean = pinned_empty((X.shape[0], width), np.float64)
    var = pinned_empty((X.shape[0], width), np.float64) if return_var else None
    return X, mean, var


class _Posterior(_LibObject):
    """A resident posterior of ``M`` outputs whose predict symbol ``_predict`` takes (ctx, h, X, P, mean, var, precision)."""

    _predict = None

    def predict(self, X, return_var=True, precision=GP_FP64):
        X, mean, var = _predict_io(X, self.M, return_var)
        _check(getattr(load_library(), self._predict)(context(), self._h, _in(X), X.shape[0], _ptr(mean), _ptr(var), int(precision)),
               self._predict)
        return mean, var


# --------------------------------------------------------------------------- A18
class GPHandle(_Posterior):
    """Owns a dmo_gp object (posterior state resident in HBM)."""

    _destroy, _predict = "dmo_gp_destroy", "dmo_gp_predict"

    def __init__(self, X_train, alpha, factor, constant, length_scale, noise, y_mean, y_std, xlb, xub, kernel=KERNEL_MATERN52, factor_is_inverse=False):
        lib = load_library()
        X_train = _f64(X_train)
        N, d = X_train.shape
        alpha = _f64(alpha)
        M = alpha.shape[0]
        factor = _f64(factor)
        assert factor.shape == (M, N, N), factor.shape
        ls = np.empty((M, d), dtype=np.float64)
        for m in range(M):
            ls[m, :] = np.asarray(length_scale[m], dtype=np.float64)
        self.N, self.d, self.M = N, d, M
        cst, nz, ym, ys, lb, ub = _f64(constant), _f64(noise), _f64(y_mean), _f64(y_std), _f64(xlb), _f64(xub)
        assert cst.shape == (M,) and nz.shape == (M,) and ym.shape == (M,) and ys.shape == (M,) and lb.shape == (d,) and ub.shape == (d,)
        h = _vp()
        _check(
            lib.dmo_gp_create(
                context(), N, d, M, int(kernel), _ptr(X_train), _ptr(alpha), _ptr(factor), 1 if factor_is_inverse else 0, _ptr(cst),
                _ptr(ls), _ptr(nz), _ptr(ym), _ptr(ys), _ptr(lb), _ptr(ub), ctypes.byref(h),
            ),
            "dmo_gp_create",
        )
        self._h = h

    def set_linear_mean(self, weight, bias):
        """Prior mean w_m . x_n + b_m per objective (gpytorch LinearMean, A19); ``None, None`` removes it."""
        if weight is None and bias is None:
            _check(load_library().dmo_gp_set_linear_mean(context(), self._h, None, None), "dmo_gp_set_linear_mean")
            return
        w = _f64(np.asarray(weight, dtype=np.float64).reshape(self.M, self.d))
        b = _f64(np.asarray(bias, dtype=np.float64).reshape(self.M))
        _check(load_library().dmo_gp_set_linear_mean(context(), self._h, _ptr(w), _ptr(b)), "dmo_gp_set_linear_mean")

    def auto_info(self):
        """What precision=GP_AUTO does for this model (runs the one-off calibration if needed)."""
        mt, vt, rows = _c_int(0), _c_int(0), _c_i64(0)
        em, ev, th = _c_dbl(0.0), _c_dbl(0.0), _c_dbl(0.0)
        _check(load_library().dmo_gp_auto_info(context(), self._h, ctypes.byref(mt), ctypes.byref(vt), ctypes.byref(em), ctypes.byref(ev),
                                               ctypes.byref(th), ctypes.byref(rows)), "dmo_gp_auto_info")
        return {"mean_tensor": bool(mt.value & 1), "mean_only_tensor": bool(mt.value & 4),
                "var_tensor": bool(vt.value), "mean_err": em.value,
                "var_err": ev.value, "theta": th.value, "last_refined": int(rows.value)}

    def covariance_groups(self):
        """``(G, group_of)``: the number of distinct posterior covariances and, per objective, the group whose L^-1, K_*
        and variance contraction it shares (groups numbered in order of first appearance)."""
        n = _c_int(0)
        grp = np.zeros(self.M, dtype=np.int32)
        _check(load_library().dmo_gp_covariance_groups(context(), self._h, ctypes.byref(n), grp.ctypes.data_as(_vp)),
               "dmo_gp_covariance_groups")
        return int(n.value), [int(g) for g in grp]


# --------------------------------------------------------------------------- A19: multitask exact GP (MEGP_Matern)
class MTGPHandle(_Posterior):
    """Owns a dmo_mtgp object: the multitask posterior (covariance K_x (x) B + I (x) diag(D), linear mean per task)
    resident in HBM.  ``lml`` is the exact log marginal likelihood of the normalised targets."""

    _destroy, _predict = "dmo_mtgp_destroy", "dmo_mtgp_predict"

    def __init__(self, X_train, Y, length_scale, B, D, weight, bias, y_mean, y_std, xlb, xub):
        lib = load_library()
        X_train, Y = _f64(X_train), _f64(Y)
        N, d = X_train.shape
        if Y.ndim == 1:
            Y = Y.reshape(-1, 1)
        M = Y.shape[1]
        assert Y.shape == (N, M), Y.shape
        ls, Bm, Dv = _per_dim(np.reshape(length_scale, -1), d), _f64(B).reshape(M, M), _f64(D).reshape(M)
        w, b = _f64(weight).reshape(M, d), _f64(bias).reshape(M)
        ym, ys, lb, ub = _f64(y_mean).reshape(M), _f64(y_std).reshape(M), _f64(xlb).reshape(d), _f64(xub).reshape(d)
        self.N, self.d, self.M = N, d, M
        h, lml = _vp(), _c_dbl(0.0)
        _check(
            lib.dmo_mtgp_create(context(), N, d, M, _ptr(X_train), _ptr(Y), _ptr(ls), _ptr(Bm), _ptr(Dv), _ptr(w), _ptr(b), _ptr(ym), _ptr(ys),
                                _ptr(lb), _ptr(ub), ctypes.byref(lml), ctypes.byref(h)),
            "dmo_mtgp_create",
        )
        self._h = h
        self.lml = float(lml.value)


class SVGPHandle(_Posterior):
    """Owns a dmo_svgp object: the whitened variational GP posterior of L latent GPs (inducing points Zpts (L,Z,d),
    Matern-5/2 ARD kernels, q_mu (L,Z), lower-triangular q_sqrt (L,Z,Z)) mixed into M outputs by W (M,L) (None: the
    identity), resident in HBM.  ``y_var_scale`` (M,) multiplies the variance (None: y_std**2)."""

    _destroy, _predict = "dmo_svgp_destroy", "dmo_svgp_predict"

    def __init__(self, Zpts, variance, length_scale, q_mu, q_sqrt, y_mean, y_std, xlb, xrng, W=None, jitter=1e-2, y_var_scale=None):
        lib = load_library()
        Zp = _f64(Zpts)
        if Zp.ndim != 3:
            raise DmoError(f"dmo_svgp_create: Zpts must be (L, Z, d), got shape {Zp.shape}")
        L, Z, d = Zp.shape
        Wm = None if W is None else _f64(W)
        if Wm is not None and (Wm.ndim != 2 or Wm.shape[1] != L):
            raise DmoError(f"dmo_svgp_create: W must be (M, {L}), got shape {Wm.shape}")
        M = L if Wm is None else Wm.shape[0]
        s, ls, qm, qs = _f64(variance), _f64(length_scale), _f64(q_mu), _f64(q_sqrt)
        ym, ys, lb, rg = _f64(y_mean), _f64(y_std), _f64(xlb), _f64(xrng)
        vs = None if y_var_scale is None else _f64(y_var_scale)
        for name, a, shape in (("variance", s, (L,)), ("length_scale", ls, (L, d)), ("q_mu", qm, (L, Z)), ("q_sqrt", qs, (L, Z, Z)),
                               ("y_mean", ym, (M,)), ("y_std", ys, (M,)), ("xlb", lb, (d,)), ("xrng", rg, (d,)),
                               ("y_var_scale", vs, (M,))):
            if a is not None and a.shape != shape:
                raise DmoError(f"dmo_svgp_create: {name} must have shape {shape}, got {a.shape}")
        self.L, self.M, self.Z, self.d = L, M, Z, d
        h = _vp()
        _check(
            lib.dmo_svgp_create(context(), L, M, Z, d, _ptr(Zp), _ptr(s), _ptr(ls), _ptr(qm), _ptr(qs), _ptr(Wm), float(jitter), _ptr(ym),
                                _ptr(ys), _ptr(vs), _ptr(lb), _ptr(rg), ctypes.byref(h)),
            "dmo_svgp_create",
        )
        self._h = h

    def groups(self):
        """(distinct K_* planes, operator planes) that one predict produces and contracts."""
        g, p = _c_int(0), _c_int(0)
        _check(load_library().dmo_svgp_groups(context(), self._h, ctypes.byref(g), ctypes.byref(p)), "dmo_svgp_groups")
        return int(g.value), int(p.value)


def svgp_optimal_q(X, y, Zpts, variance, length_scale, noise, jitter=1e-2, inducing_is_data=False):
    """The optimal whitened q for a Gaussian likelihood (dmo_svgp_optimal_q): X (N,d), y (L,N), Zpts (L,Z,d), variance
    (L,), length_scale (L,d), noise (L,) -> q_mu (L,Z), lower-triangular q_sqrt (L,Z,Z).  inducing_is_data: GPflow's VGP
    (Z = X, f(X) = Lz v; Zpts is ignored and may be None)."""
    X = _f64(X)
    N, d = X.shape
    L = len(np.atleast_1d(variance))
    Zp = None if inducing_is_data else _f64(Zpts)
    Z = N if inducing_is_data else Zp.shape[1]
    y = _f64(y).reshape(L, N)
    s, ls, nz = _f64(variance).reshape(L), _f64(length_scale).reshape(L, d), _f64(noise).reshape(L)
    q_mu = np.empty((L, Z), np.float64)
    q_sqrt = np.empty((L, Z, Z), np.float64)
    _check(load_library().dmo_svgp_optimal_q(context(), N, Z, d, L, _ptr(X), _ptr(y), _ptr(Zp), _ptr(s), _ptr(ls), _ptr(nz), float(jitter),
                                             int(bool(inducing_is_data)), _ptr(q_mu), _ptr(q_sqrt)), "dmo_svgp_optimal_q")
    return q_mu, q_sqrt


class DGPHandle(_LibObject):
    """Owns a dmo_dgp: the two-layer deep GP posterior of gpytorch's DSPP / DeepGP (dmo_dgp_create), resident in HBM.
    Hidden layer: Z1pts (H,Z1,d), s1 (H,), ls1 (H,d), q_mu1 (H,Z1), q_sqrt1 (H,Z1,Z1), w1 (d,), b1; last layer: Z2pts
    (T,Z2,H), s2 (T,), ls2 (T,H), q_mu2 (T,Z2), q_sqrt2 (T,Z2,Z2), c2; noise (T,) task + global noise.  quad_sites (J,H)
    selects quadrature (DSPP); None means ``n_sites`` Monte Carlo draws per predict (DeepGP)."""

    _destroy = "dmo_dgp_destroy"

    def __init__(self, Z1pts, s1, ls1, q_mu1, q_sqrt1, w1, b1, Z2pts, s2, ls2, q_mu2, q_sqrt2, c2, noise, y_mean, y_std, xlb, xrng,
                 quad_sites=None, n_sites=None, jitter=1e-4, min_variance=1e-6):
        Z1p, Z2p = _f64(Z1pts), _f64(Z2pts)
        if Z1p.ndim != 3 or Z2p.ndim != 3:
            raise DmoError(f"dmo_dgp_create: Z1pts must be (H, Z1, d) and Z2pts (T, Z2, H), got {Z1p.shape} and {Z2p.shape}")
        H, Z1, d = Z1p.shape
        T, Z2 = Z2p.shape[:2]
        qs = None if quad_sites is None else _f64(quad_sites)
        if qs is not None:
            if qs.ndim != 2 or qs.shape[1] != H:
                raise DmoError(f"dmo_dgp_create: quad_sites must be (J, {H}), got shape {qs.shape}")
            n_sites = qs.shape[0]
        if n_sites is None:
            raise DmoError("dmo_dgp_create: n_sites is required without quad_sites")
        arrs = {"s1": (_f64(s1), (H,)), "ls1": (_f64(ls1), (H, d)), "q_mu1": (_f64(q_mu1), (H, Z1)), "q_sqrt1": (_f64(q_sqrt1), (H, Z1, Z1)),
                "w1": (_f64(w1), (d,)), "Z2pts": (Z2p, (T, Z2, H)), "s2": (_f64(s2), (T,)), "ls2": (_f64(ls2), (T, H)),
                "q_mu2": (_f64(q_mu2), (T, Z2)), "q_sqrt2": (_f64(q_sqrt2), (T, Z2, Z2)), "noise": (_f64(noise), (T,)),
                "y_mean": (_f64(y_mean), (T,)), "y_std": (_f64(y_std), (T,)), "xlb": (_f64(xlb), (d,)), "xrng": (_f64(xrng), (d,))}
        for name, (a, shape) in arrs.items():
            if a.shape != shape:
                raise DmoError(f"dmo_dgp_create: {name} must have shape {shape}, got {a.shape}")
        a = {k: v[0] for k, v in arrs.items()}
        self.d, self.H, self.T, self.J = d, H, T, int(n_sites)
        h = _vp()
        _check(load_library().dmo_dgp_create(
            context(), d, H, T, Z1, Z2, _ptr(Z1p), _ptr(a["s1"]), _ptr(a["ls1"]), _ptr(a["q_mu1"]), _ptr(a["q_sqrt1"]), _ptr(a["w1"]), float(b1),
            _ptr(Z2p), _ptr(a["s2"]), _ptr(a["ls2"]), _ptr(a["q_mu2"]), _ptr(a["q_sqrt2"]), float(c2), _ptr(a["noise"]), float(jitter),
            float(min_variance), self.J, _ptr(qs), _ptr(a["y_mean"]), _ptr(a["y_std"]), _ptr(a["xlb"]), _ptr(a["xrng"]), ctypes.byref(h)),
            "dmo_dgp_create")
        self._h = h

    def predict(self, X, seed=0, stream_id=0, return_var=True, return_eps=False, precision=GP_FP64):
        """(mean (P,T), var (P,T) or None[, eps (J,P,H)]) at the raw inputs X (P,d)."""
        X, mean, var = _predict_io(X, self.T, return_var)
        P = X.shape[0]
        eps = np.empty((self.J, P, self.H), np.float64) if return_eps else None
        _check(load_library().dmo_dgp_predict(context(), self._h, _in(X), P, int(seed), int(stream_id), _ptr(eps), _ptr(mean), _ptr(var),
                                              int(precision)), "dmo_dgp_predict")
        return (mean, var, eps) if return_eps else (mean, var)


class SVGPFitState(_LibObject):
    """Owns a dmo_svgp_fit: the training state of one GPflow variational model (L latents over the inducing points Zpts
    (Z,d), M outputs; inducing_is_data: VGP, Z = X) on X (N,d), Y (N,M), with q starting at N(0, I)."""

    _destroy = "dmo_svgp_fit_destroy"

    def __init__(self, X, Y, Zpts, L, jitter=1e-2, inducing_is_data=False):
        X = _f64(X)
        N, d = X.shape
        Yt = _f64(np.asarray(Y, dtype=np.float64).reshape(N, -1).T)
        M = Yt.shape[0]
        Zp = None if inducing_is_data else _f64(Zpts)
        Z = N if inducing_is_data else Zp.shape[0]
        if Zp is not None and Zp.shape != (Z, d):
            raise DmoError(f"dmo_svgp_fit_create: Zpts must be (Z, {d}), got shape {Zp.shape}")
        self.N, self.d, self.M, self.L, self.Z = N, d, M, int(L), Z
        h = _vp()
        _check(load_library().dmo_svgp_fit_create(context(), N, d, M, self.L, Z, _ptr(X), _ptr(Yt), _ptr(Zp), int(bool(inducing_is_data)),
                                                  float(jitter), ctypes.byref(h)), "dmo_svgp_fit_create")
        self._h = h

    def _args(self, batch, variance, length_scale, noise, W):
        b = np.ascontiguousarray(batch, dtype=np.int64).reshape(-1)
        s = _f64(variance).reshape(self.L)
        ls = _f64(length_scale).reshape(self.L, self.d)
        nz = _f64(noise).reshape(self.M)
        Wm = None if W is None else _f64(W).reshape(self.M, self.L)
        return b, s, ls, nz, Wm

    def natgrad(self, batch, variance, length_scale, noise, W=None, gamma=1.0):
        """One natural-gradient step on q (in place)."""
        b, s, ls, nz, Wm = self._args(batch, variance, length_scale, noise, W)
        _check(load_library().dmo_svgp_fit_natgrad(context(), self._h, _ptr(b), b.shape[0], _ptr(s), _ptr(ls), _ptr(nz), _ptr(Wm), float(gamma)),
               "dmo_svgp_fit_natgrad")

    def elbo_grad(self, batch, variance, length_scale, noise, W=None, grad=True):
        """(ell (M,), kl (L,), grads or None): grads a dict of d ELBO / d variance (L,), length_scale (L,d), noise (M,) and
        W (M,L) (when W is given) at the current q."""
        b, s, ls, nz, Wm = self._args(batch, variance, length_scale, noise, W)
        ell, kl = np.empty(self.M), np.empty(self.L)
        g = None
        if grad:
            g = {"variance": np.empty(self.L), "length_scale": np.empty((self.L, self.d)), "noise": np.empty(self.M),
                 "W": None if Wm is None else np.empty((self.M, self.L))}
        gp = (lambda k: None) if g is None else (lambda k: _ptr(g[k]))
        _check(load_library().dmo_svgp_fit_elbo_grad(context(), self._h, _ptr(b), b.shape[0], _ptr(s), _ptr(ls), _ptr(nz), _ptr(Wm), _ptr(ell),
                                                     _ptr(kl), gp("variance"), gp("length_scale"), gp("noise"), gp("W")),
               "dmo_svgp_fit_elbo_grad")
        return ell, kl, g

    def q(self):
        """(q_mu (L,Z), lower-triangular q_sqrt (L,Z,Z))."""
        q_mu = np.empty((self.L, self.Z))
        q_sqrt = np.empty((self.L, self.Z, self.Z))
        _check(load_library().dmo_svgp_fit_q(context(), self._h, _ptr(q_mu), _ptr(q_sqrt)), "dmo_svgp_fit_q")
        return q_mu, q_sqrt


class DGPFitState(_LibObject):
    """Owns a dmo_dgp_fit: the training state of the two-layer deep GP behind MDSPP_Matern (quadrature, n_sites sites)
    and MDGP_Matern (n_sites draws per row) on X (N,d) normalised inputs and Y (N,T) normalised targets, with H hidden
    units, Z1 / Z2 inducing points per layer and batches of at most batch_max rows.  The raw vector's layout is
    dmosopt_b200.h's (model_gpytorch.deepgp_flatten builds it); it starts at zero."""

    _destroy = "dmo_dgp_fit_destroy"

    def __init__(self, X, Y, H, Z1, Z2, n_sites, quadrature, batch_max, lengthscale_bounds=None, jitter=1e-4, min_variance=1e-6):
        X = _f64(X)
        N, d = X.shape
        Y = _f64(np.asarray(Y, dtype=np.float64).reshape(N, -1))
        T = Y.shape[1]
        lb = None if lengthscale_bounds is None else _f64(np.asarray(lengthscale_bounds, dtype=np.float64).reshape(2))
        self.N, self.d, self.H, self.T, self.Z1, self.Z2 = N, d, int(H), T, int(Z1), int(Z2)
        self.J, self.quadrature, self.batch_max = int(n_sites), bool(quadrature), int(batch_max)
        self.n_params = (self.Z1 * d + 2 * self.H + self.H * self.Z1 + self.H * self.Z1 * self.Z1 + d + 1 + T * self.Z2 * self.H + 2 * T
                         + T * self.Z2 + T * self.Z2 * self.Z2 + 1 + T + 1 + (self.J * self.H if self.quadrature else 0))
        h = _vp()
        _check(load_library().dmo_dgp_fit_create(context(), N, d, self.H, T, self.Z1, self.Z2, self.J, int(self.quadrature), self.batch_max,
                                                 _ptr(X), _ptr(Y), _ptr(lb), float(jitter), float(min_variance), ctypes.byref(h)),
               "dmo_dgp_fit_create")
        self._h = h

    def set_params(self, raw):
        r = _f64(raw).reshape(-1)
        _check(load_library().dmo_dgp_fit_set_params(context(), self._h, _ptr(r), r.shape[0]), "dmo_dgp_fit_set_params")

    def get_params(self):
        r = np.empty(self.n_params, np.float64)
        _check(load_library().dmo_dgp_fit_get_params(context(), self._h, _ptr(r), r.shape[0]), "dmo_dgp_fit_get_params")
        return r

    def loss_grad(self, batch, seed=0, step=0, eps=None, grad=True, return_eps=False):
        """(loss, grad (n_params,) or None[, eps (J,B,H)]) of the minibatch rows ``batch`` at the current parameters;
        ``eps`` (J,B,H) replaces MDGP's Philox draws keyed by (seed, step)."""
        b = np.ascontiguousarray(batch, dtype=np.int64).reshape(-1)
        e = None if eps is None else _f64(eps)
        loss = np.empty(1, np.float64)
        g = np.empty(self.n_params, np.float64) if grad else None
        eo = np.empty((self.J, b.shape[0], self.H), np.float64) if return_eps else None
        _check(load_library().dmo_dgp_fit_loss_grad(context(), self._h, _ptr(b), b.shape[0], int(seed), int(step), _ptr(e), _ptr(eo), _ptr(loss),
                                                    _ptr(g)), "dmo_dgp_fit_loss_grad")
        return (float(loss[0]), g, eo) if return_eps else (float(loss[0]), g)

    def adam_step(self, lr):
        _check(load_library().dmo_dgp_fit_adam_step(context(), self._h, float(lr)), "dmo_dgp_fit_adam_step")

    def epoch(self, perm, batch_size, lr, seed=0, step0=0):
        """The batch losses of one epoch over the permutation ``perm`` of range(N), one Adam step per batch."""
        p = np.ascontiguousarray(perm, dtype=np.int64).reshape(-1)
        if p.shape[0] != self.N:
            raise DmoError(f"dmo_dgp_fit_epoch: perm must have {self.N} entries, got {p.shape[0]}")
        out = np.empty(-(-self.N // int(batch_size)), np.float64)
        _check(load_library().dmo_dgp_fit_epoch(context(), self._h, _ptr(p), int(batch_size), float(lr), int(seed), int(step0), _ptr(out)),
               "dmo_dgp_fit_epoch")
        return out


# --------------------------------------------------------------------------- A16/A17
def hypervolume(F, ref, rank=None):
    """Exact hypervolume; ``rank`` (optional): non-dominated ranks of the rows within the superset they were selected from
    by rank (skips the non-dominated filter, see dmo_hypervolume_ranked)."""
    F = _f64(F)
    if F.ndim == 1:
        F = F.reshape(1, -1)
    n, M = F.shape
    ref = _f64(ref)
    out = _c_dbl(0.0)
    if rank is None:
        _check(load_library().dmo_hypervolume(context(), _ptr(F), n, M, _ptr(ref), ctypes.byref(out)), "dmo_hypervolume")
    else:
        rk = np.ascontiguousarray(rank, dtype=np.int32)
        assert rk.shape == (n,)
        _check(load_library().dmo_hypervolume_ranked(context(), _ptr(F), n, M, _ptr(ref), _ptr(rk), ctypes.byref(out)), "dmo_hypervolume_ranked")
    return float(out.value)


HVMC_ALGORITHMS = {"hybrid": 0, "fpras": 1, "mcm2rv": 2, "monte_carlo": 3}
HVMC_MAX_OBJECTIVES = 16  # dmo_hypervolume_mc (csrc/hv_mc.cu)
_HVMC_RAN = {1: "FPRAS", 2: "MCM2RV", 3: "MonteCarlo", 4: "Hybrid-FPRAS", 5: "Hybrid-MCM2RV"}


def hypervolume_mc(F, ref, algorithm="hybrid", epsilon=0.01, delta=0.25, n_samples=100000, seed=0, stream=0):
    """Monte-Carlo hypervolume estimate of the rows of F strictly inside ref (2 <= M <= 16), on the GPU.

    ``algorithm``: "hybrid", "fpras", "mcm2rv" (the (epsilon, delta) estimators of dmosopt/hv_adaptive.py) or
    "monte_carlo" (``n_samples`` uniform points, dmosopt/hv.py:191-241).  The result is a pure function of the filtered
    front, ``seed`` and ``stream`` (< 2^24).  Returns (value, info) with info = {"samples", "tests", "algorithm"}; "tests" counts
    the point-against-row tests performed (dmo_hypervolume_mc in include/dmosopt_b200.h says how that differs from the
    reference's num_comparisons for mcm2rv and monte_carlo)."""
    if algorithm not in HVMC_ALGORITHMS:
        raise ValueError(f"hypervolume_mc: unknown algorithm {algorithm!r} (one of {sorted(HVMC_ALGORITHMS)})")
    F = _f64(F)
    if F.ndim == 1:
        F = F.reshape(1, -1)
    n, M = F.shape
    ref = _f64(ref).reshape(-1)
    if ref.shape[0] != M:
        raise ValueError(f"hypervolume_mc: ref has {ref.shape[0]} coordinates, the points have {M}")
    out = _c_dbl(0.0)
    ns, nt, ran = _c_i64(0), _c_i64(0), _c_int(0)
    _check(
        load_library().dmo_hypervolume_mc(context(), _ptr(F), n, M, _ptr(ref), HVMC_ALGORITHMS[algorithm], float(epsilon), float(delta),
                                          int(n_samples), _seed(seed), int(stream), ctypes.byref(out), ctypes.byref(ns),
                                          ctypes.byref(nt), ctypes.byref(ran)),
        "dmo_hypervolume_mc",
    )
    return float(out.value), {"samples": int(ns.value), "tests": int(nt.value), "algorithm": _HVMC_RAN.get(ran.value)}


def ehvi_select(F, means, variances, ref, k, nds=True, return_scores=False):
    F = _f64(F)
    means = _f64(means)
    variances = _f64(variances)
    nf, M = F.shape
    nc = means.shape[0]
    k = int(min(k, nc))
    sel = np.empty(k, dtype=np.int64)
    score = np.empty(nc, dtype=np.float64) if return_scores else None
    ref = _f64(ref)
    _check(
        load_library().dmo_ehvi_select(context(), _ptr(F), nf, _ptr(means), _ptr(variances), nc, M, _ptr(ref), 1 if nds else 0, k, _ptr(sel), _ptr(score)),
        "dmo_ehvi_select",
    )
    return (sel, score) if return_scores else sel


# --------------------------------------------------------------------------- A21
def get_duplicates(X, eps=1e-16, Y=None):
    X = _f64(X)
    n, d = X.shape
    out = np.empty(n, dtype=np.uint8)
    if Y is None:
        _check(load_library().dmo_get_duplicates(context(), _in(X), n, d, float(eps), _ptr(out)), "dmo_get_duplicates")
    else:
        Y = _f64(Y)
        assert Y.ndim == 2 and Y.shape[1] == d, (X.shape, Y.shape)
        _check(load_library().dmo_get_duplicates_pair(context(), _in(X), n, _in(Y), Y.shape[0], d, float(eps), _ptr(out)), "dmo_get_duplicates_pair")
    return out.astype(bool)


ERR_OVERFLOW = 6  # DMO_ERR_OVERFLOW
EPSILON_MAX_OBJECTIVES = 16  # dmo_epsilon_sort (csrc/epsilon.cu)


def epsilon_sort(Y, eps):
    """Ascending int64 row indices of the epsilon-nondominated archive of Y's rows (MOEA.EpsilonSort fed every row in
    order, dmosopt/MOEA.py:470-595).  Rows sort on their first len(eps) columns; an eps of 0 or NaN counts as 1e-8.
    Raises OverflowError when some y / eps overflows, where the reference's math.floor does."""
    eps = _f64(eps).reshape(-1)
    M = eps.shape[0]
    Y = _f64(Y)
    if Y.ndim != 2 or Y.shape[1] < M:
        raise ValueError(f"epsilon_sort: Y must be (n, >= {M}) for {M} epsilons, got shape {Y.shape}")
    if Y.shape[1] != M:
        Y = np.ascontiguousarray(Y[:, :M])
    n = Y.shape[0]
    idx = np.empty(n, dtype=np.int64)
    count = _c_i64(0)
    st = load_library().dmo_epsilon_sort(context(), _ptr(Y), n, M, _ptr(eps), _ptr(idx), ctypes.byref(count))
    if st == ERR_OVERFLOW:
        raise OverflowError(_lib.dmo_last_error(_ctx).decode())
    _check(st, "dmo_epsilon_sort")
    return idx[: count.value]


# --------------------------------------------------------------------------- A11 AGE-MOEA
def age_survival(yn, nn, p, extreme):
    """Greedy part of AGEMOEA.survival_score (dmosopt/AGEMOEA.py:398-428) -> crowding values (m,)."""
    yn = _f64(yn)
    nn = _f64(nn)
    m, M = yn.shape
    ext = np.ascontiguousarray(extreme, dtype=np.int32)
    crowd = np.empty(m, dtype=np.float64)
    _check(load_library().dmo_age_survival(context(), _ptr(yn), _ptr(nn), m, M, float(p), _ptr(ext), ext.shape[0], _ptr(crowd)), "dmo_age_survival")
    return crowd


# --------------------------------------------------------------------------- A12 SMPSO
def smpso_velocity(position, velocity, leader1, leader2, w, c1, r1, c2, r2, chi, xlb, xub):
    f32_diff = 1 if (np.asarray(leader1).dtype == np.float32 and np.asarray(position).dtype == np.float32) else 0
    pos = np.ascontiguousarray(position, dtype=np.float32)
    vel = _f64(velocity)
    l1 = _f64(leader1)
    l2 = _f64(leader2)
    n, d = pos.shape
    lb, ub = _f64(xlb), _f64(xub)
    out = np.empty((n, d), dtype=np.float64)
    _check(
        load_library().dmo_smpso_velocity(context(), _ptr(pos), _ptr(vel), _ptr(l1), _ptr(l2), f32_diff, n, d, float(w), float(c1), float(r1), float(c2), float(r2),
                                          float(chi), _ptr(lb), _ptr(ub), _ptr(out)),
        "dmo_smpso_velocity",
    )
    return out


def mutate_groups(pop_x, group_size, n_groups, per_group, di_mutation, xlb, xub, mutation_rate, seed, stream_id, return_parents=False):
    pop_x = _f64(pop_x)
    d = pop_x.shape[1]
    total = int(n_groups) * int(per_group)
    di = _per_dim(di_mutation, d)
    lb, ub = _f64(xlb), _f64(xub)
    out = np.empty((total, d), dtype=np.float64)
    par = np.empty(total, dtype=np.int64) if return_parents else None
    _check(
        load_library().dmo_mutate_groups(context(), _ptr(pop_x), int(group_size), int(n_groups), int(per_group), d, _ptr(di), _ptr(lb), _ptr(ub),
                                         float(mutation_rate), _seed(seed), int(stream_id), _ptr(out), _ptr(par)),
        "dmo_mutate_groups",
    )
    return (out, par) if return_parents else out


BENCHMARKS = {"zdt1": 0, "zdt3": 1, "dtlz1": 10, "dtlz2": 11, "dtlz3": 12, "dtlz4": 13, "dtlz5": 14, "dtlz7": 16, "wfg1": 21, "wfg4": 24,
              "maf1": 31, "maf2": 32, "maf4": 34}


def benchmark_eval(name, X, n_obj, alpha=100.0):
    """Rows of X through one of the reference's benchmark functions (dmosopt/benchmarks/moo_benchmarks.py), on the GPU."""
    X = _f64(X)
    n, d = X.shape
    Y = np.empty((n, int(n_obj)), dtype=np.float64)
    _check(load_library().dmo_benchmark_eval(context(), BENCHMARKS[name], _in(X), n, d, int(n_obj), float(alpha), _ptr(Y)), "dmo_benchmark_eval")
    return Y


class SmpsoSwarms:
    """The swarm state of SMPSO resident in HBM (dmo_smpso_generate / dmo_smpso_update, csrc/smpso.cu): positions and
    objectives as float64 arrays holding float32-representable values, velocities in float64."""

    def __init__(self, parm, obj, vel, swarms, pop):
        parm, obj, vel = np.asarray(parm), np.asarray(obj), np.asarray(vel)
        self.swarms, self.pop, self.d, self.M = int(swarms), int(pop), parm.shape[1], obj.shape[1]
        n = self.swarms * self.pop
        assert parm.shape[0] == n and obj.shape[0] == n and vel.shape == (n, self.d)
        self.parm = DeviceArray((n, self.d)).upload(_f64(parm))
        self.obj = DeviceArray((n, self.M)).upload(_f64(obj))
        self.vel = DeviceArray((n, self.d)).upload(_f64(vel))

    def generate(self, di_mutation, xlb, xub, mutation_rate, seed, stream_id):
        """x_gen (2 * swarms * pop, d), laid out as SMPSO.py:163-184 does: the reference's float32 values, handed out as the
        float64 array MOEA.generate turns them into (np.clip against float64 bounds, MOEA.py:155) -- read-only, page-locked,
        with its device copy kept as a mirror so that evaluate(x_gen) / update(x_gen, ...) do not ship it back over PCIe."""
        di = _per_dim(di_mutation, self.d)
        lb, ub = _f64(xlb), _f64(xub)
        x_dev = DeviceArray((2 * self.swarms * self.pop, self.d), np.float64)
        _check(load_library().dmo_smpso_generate(context(), self.parm.ptr, self.vel.ptr, self.swarms, self.pop, self.d, _ptr(di), _ptr(lb), _ptr(ub),
                                                 float(mutation_rate), _seed(seed), int(stream_id), None, x_dev.ptr), "dmo_smpso_generate")
        return _mirrored_out(x_dev)

    def update(self, x_gen, y_gen, scalars, xlb, xub, metric, parm_out, obj_out):
        """One update_strategy (SMPSO.py:187-238) on the resident state; writes the new float32 state into parm_out /
        obj_out and returns (ranks (swarms, pop) intp, perm (swarms, pop) int64)."""
        n = self.swarms * self.pop
        x_gen = np.asarray(x_gen)
        if x_gen.dtype == np.float32:
            xg, is32 = np.ascontiguousarray(x_gen[:n]), 1
        else:
            xg, is32 = _f64(x_gen[:n]), 0  # a view of the caller's array: its device mirror (if any) is found by address
        yg = _f64(np.asarray(y_gen)[:n])
        sc = _f64(scalars)
        assert sc.shape == (self.swarms, 8) and xg.shape == (n, self.d) and yg.shape == (n, self.M)
        lb, ub = _f64(xlb), _f64(xub)
        ranks = np.empty(n, dtype=np.int32)
        perm = np.empty(n, dtype=np.int64)
        po = parm_out if (parm_out.dtype == np.float32 and parm_out.flags.c_contiguous) else np.empty((n, self.d), np.float32)
        oo = obj_out if (obj_out.dtype == np.float32 and obj_out.flags.c_contiguous) else np.empty((n, self.M), np.float32)
        lib = load_library()
        if self.swarms > 1 and os.environ.get("DMOSOPT_B200_SMPSO_THREADS", "1") != "0":
            # the swarms are independent (SMPSO.py:211-228): one worker context and thread per swarm, so the per-swarm
            # rank chains (latency bound, a fraction of the SMs each) overlap on the device
            synchronize()  # state and inputs produced on the main context's stream are complete
            pxg, pyg, psc, prk, ppm, ppo, poo = _in(xg), _in(yg), _ptr(sc), _ptr(ranks), _ptr(perm), _ptr(po), _ptr(oo)
            plb, pub = _ptr(lb), _ptr(ub)
            xsz = 4 if is32 else 8
            pop, d, M = self.pop, self.d, self.M

            def one(p):
                ctx, off = worker_context(p), p * pop
                st = lib.dmo_smpso_update(ctx, self.parm.ptr + off * d * 8, self.obj.ptr + off * M * 8, self.vel.ptr + off * d * 8, pxg + off * d * xsz, is32,
                                          pyg + off * M * 8, 1, pop, d, M, int(metric), psc + p * 64, plb, pub, prk + off * 4, ppm + off * 8,
                                          ppo + off * d * 4, poo + off * M * 4)
                return st, ctx

            for st, ctx in list(worker_pool().map(one, range(self.swarms))):
                _check(st, "dmo_smpso_update", ctx)
        else:
            _check(lib.dmo_smpso_update(context(), self.parm.ptr, self.obj.ptr, self.vel.ptr, _in(xg), is32, _in(yg), self.swarms, self.pop, self.d,
                                        self.M, int(metric), _ptr(sc), _ptr(lb), _ptr(ub), _ptr(ranks), _ptr(perm), _ptr(po), _ptr(oo)), "dmo_smpso_update")
        if po is not parm_out:
            parm_out[...] = po
        if oo is not obj_out:
            obj_out[...] = oo
        return ranks.astype(np.intp).reshape(self.swarms, self.pop), perm.reshape(self.swarms, self.pop)

    def step_record(self, kind, posterior, draw_key, var_route_mean, di_mutation, xlb, xub, mutation_rate, seed, stream_id, precision,
                    mean_f32, metric, scalars, ranks, x_gen, y_gen):
        """One resident SMPSO generation of MOASMO.optimize, recorded (dmo_smpso_step_record): generate, the posterior mean
        of every offspring row, update.  ``kind`` POSTERIOR_GP, _SVGP or _DGP and ``posterior`` its handle; ``draw_key``
        (seed, stream_id) keys a deep GP's draws.  ``var_route_mean`` False: the exact GP's mean-only predict (any
        precision); True: the mean its predict writes with return_var=True, rounded to float32 first when ``mean_f32``.
        ``scalars`` (swarms, 8) the host draws of the velocity update; ``ranks`` a (swarms * pop,) int32 DeviceArray that
        receives the survivors' ranks.  ``x_gen`` (2 * swarms * pop, d) and ``y_gen`` (2 * swarms * pop, M) float64
        receive the offspring and their mean; into page-locked memory they are complete only after ``synchronize()``."""
        P = 2 * self.swarms * self.pop
        for name, a, shape in (("x_gen", x_gen, (P, self.d)), ("y_gen", y_gen, (P, self.M))):
            if isinstance(a, np.ndarray) and (a.shape != shape or a.dtype != np.float64 or not a.flags.c_contiguous or not a.flags.writeable):
                raise ValueError(f"smpso_step_record: {name} must be a writable C-contiguous float64 array of shape {shape}")
        sc = _f64(scalars)
        if sc.shape != (self.swarms, 8):
            raise ValueError(f"smpso_step_record: scalars must have shape {(self.swarms, 8)}")
        draw_seed, draw_stream = draw_key
        di, lb, ub = _per_dim(di_mutation, self.d), _f64(xlb), _f64(xub)  # alive until the call returns
        _check(load_library().dmo_smpso_step_record(
            context(), int(kind), posterior._h, _seed(draw_seed), int(draw_stream), 1 if var_route_mean else 0, self.parm.ptr, self.obj.ptr,
            self.vel.ptr, self.swarms, self.pop, self.d, self.M, _ptr(di), _ptr(lb), _ptr(ub), float(mutation_rate), _seed(seed), int(stream_id),
            int(precision), 1 if mean_f32 else 0, int(metric), _ptr(sc), _ptr(ranks), _ptr(x_gen), _ptr(y_gen)), "dmo_smpso_step_record")

    def velocity_into(self, out):
        """Copy the resident velocities into ``out`` (float64, C-contiguous; page-locked state arrays take the DMA path)."""
        if out.dtype == np.float64 and out.flags.c_contiguous:
            memcpy(out, self.vel.ptr, out.nbytes)
        else:
            out[...] = self.vel.download()


# --------------------------------------------------------------------------- device-resident per-individual state
class ResidentRows:
    """(n, ...) float64 array that lives in HBM across generations (MO-CMA-ES keeps one (d, d) Cholesky factor, its
    inverse and one evolution path per parent: 604 MB at pop 131 072, d = 24).  NumPy sees it through ``__array__`` /
    indexing (a device -> host copy on demand), the kernels through ``ptr``."""

    def __init__(self, dev, shape):
        self.dev = dev
        self.shape = tuple(int(v) for v in shape)
        self.dtype = np.dtype(np.float64)
        self.ndim = len(self.shape)

    @property
    def ptr(self):
        return self.dev.ptr

    def data_ptr(self):
        return self.dev.ptr

    @property
    def row_elems(self):
        return int(np.prod(self.shape[1:])) if len(self.shape) > 1 else 1

    def __len__(self):
        return self.shape[0]

    def __array__(self, dtype=None, copy=None):
        n = int(np.prod(self.shape))
        a = self.dev.download(n).reshape(self.shape) if n else np.zeros(self.shape)
        return a if dtype is None else a.astype(dtype)

    def __getitem__(self, key):
        return np.asarray(self)[key]

    def copy(self):
        return gather_rows(self, np.arange(self.shape[0], dtype=np.int64))


def resident_rows(a):
    """Upload a host array as a ResidentRows (no-op for one)."""
    if isinstance(a, ResidentRows):
        return a
    a = _f64(a)
    return ResidentRows(DeviceArray(a.shape, np.float64).upload(a), a.shape)


def gather_rows(src, idx, alt=None, sel=None):
    """ResidentRows with rows ``(alt if sel[i] else src)[idx[i]]`` (dmo_gather_rows): device -> device."""
    idx = np.ascontiguousarray(idx, dtype=np.int64)
    n = idx.shape[0]
    shape = (n,) + src.shape[1:]
    out = ResidentRows(DeviceArray(shape, np.float64), shape)
    if n == 0:
        return out
    sl = None if sel is None else np.ascontiguousarray(sel, dtype=np.uint8)
    assert sel is None or (alt is not None and alt.shape[1:] == src.shape[1:] and sl.shape == (n,))
    _check(load_library().dmo_gather_rows(context(), src.ptr, None if alt is None else alt.ptr, _ptr(sl), _ptr(idx), n, src.row_elems, out.ptr), "dmo_gather_rows")
    return out


class _Borrowed:
    """Device memory owned by someone else (the mirror of a read-only host array) behind the DeviceArray surface."""

    def __init__(self, ptr, host):
        self.ptr, self.host = ptr, host

    def download(self, count=None):
        return np.array(self.host, dtype=np.float64).reshape(-1)[: None if count is None else int(count)]


def rows_of(a):
    """ResidentRows over ``a``: itself, the device mirror the library already holds for a read-only host array (no
    copy; valid while the mirror lives), or an upload."""
    if isinstance(a, ResidentRows):
        return a
    if isinstance(a, np.ndarray) and a.dtype == np.float64:
        m = mirror_ptr(a)
        if m is not None:
            return ResidentRows(_Borrowed(m, a), a.shape)
    return resident_rows(a)


def scale_rows(rows, factors, seg_row=None, seg_start=None):
    """In place on a ResidentRows: ``rows[seg_row[s]] *= factors[e]`` for e in [seg_start[s], seg_start[s+1]), one rounded
    multiplication after the other (dmo_scale_rows); without segments: ``rows[s] *= factors[s]``."""
    f = _f64(factors)
    sr = None if seg_row is None else np.ascontiguousarray(seg_row, dtype=np.int64)
    ss = None if seg_start is None else np.ascontiguousarray(seg_start, dtype=np.int64)
    n_seg = rows.shape[0] if sr is None else sr.shape[0]
    assert (ss is None or ss.shape[0] == n_seg + 1) and (ss is not None or f.shape[0] == n_seg)
    _check(load_library().dmo_scale_rows(context(), rows.ptr, rows.row_elems, n_seg, _ptr(sr), _ptr(ss), _ptr(f), f.shape[0]), "dmo_scale_rows")
    return rows


def identity_rows(n, d):
    """n copies of the d x d identity, resident (CMAES.py:137-141) -- built on the device from one uploaded matrix."""
    return gather_rows(resident_rows(np.identity(d)[None, :, :]), np.zeros(n, dtype=np.int64))


# --------------------------------------------------------------------------- A13 / A15 CMAES
def cmaes_sample(parents_x, sigmas, A, p_idx, z):
    px = _f64(parents_x)
    sg = _f64(sigmas)
    A = A if isinstance(A, ResidentRows) else _f64(A)
    z = _f64(z)
    pi = np.ascontiguousarray(p_idx, dtype=np.int64)
    n, d = z.shape
    cols = 1 if sg.ndim == 1 else sg.shape[1]
    out = np.empty((n, d), dtype=np.float64)
    _check(load_library().dmo_cmaes_sample(context(), _ptr(px), _ptr(sg), cols, A.ptr if isinstance(A, ResidentRows) else _ptr(A), px.shape[0], _ptr(pi), _ptr(z), n, d,
                                           _ptr(out)), "dmo_cmaes_sample")
    return out


def cmaes_generate(parents_x, sigmas, A, p_idx, z, xlb, xub):
    """Offspring of one MO-CMA-ES generation from the resident parent state: sample, global rescale, clip (CMAES.py:265-270,
    MOEA.py:155) in one call; returns a read-only page-locked (n, d) array whose device copy the next calls reuse."""
    z = _f64(z)
    pi = np.ascontiguousarray(p_idx, dtype=np.int64)
    n, d = z.shape
    px, sg = rows_of(parents_x), rows_of(sigmas)
    cols = 1 if sg.ndim == 1 else sg.shape[1]
    lb, ub = _f64(xlb), _f64(xub)
    x_dev = DeviceArray((n, d), np.float64)
    _check(load_library().dmo_cmaes_generate(context(), px.ptr, sg.ptr, cols, A.ptr, px.shape[0], _ptr(pi), _ptr(z), n, d, _ptr(lb), _ptr(ub), x_dev.ptr),
           "dmo_cmaes_generate")
    return _mirrored_out(x_dev)


def cmaes_step_z(x_gen, cand_idx, parents_x, par_idx, xlb, xub, steps):
    """z = ((x_gen[cand_idx] - parents_x[par_idx]) / (xub - xlb)) / steps on resident rows (CMAES.py:359)."""
    ci = np.ascontiguousarray(cand_idx, dtype=np.int64)
    pi = np.ascontiguousarray(par_idx, dtype=np.int64)
    n, d = ci.shape[0], parents_x.shape[1]
    out = ResidentRows(DeviceArray((n, d), np.float64), (n, d))
    if n:
        lb, ub = _f64(xlb), _f64(xub)
        _check(load_library().dmo_cmaes_step_z(context(), x_gen.ptr, _ptr(ci), parents_x.ptr, _ptr(pi), _ptr(lb), _ptr(ub), steps.ptr, n, d, out.ptr), "dmo_cmaes_step_z")
    return out


def cmaes_update_cholesky(A, Ainv, pc, z, psucc, cc, ccov, pthresh):
    """Batched CMAES.updateCholesky (dmosopt/CMAES.py:489-537); returns new (A, Ainv, pc).  ResidentRows are updated in
    place in HBM (no factor crosses the PCIe bus), host arrays are copied, staged and returned."""
    if isinstance(A, ResidentRows):
        n, d = pc.shape
        if n:
            z, ps = (z if isinstance(z, ResidentRows) else _f64(z)), _f64(psucc)
            _check(load_library().dmo_cmaes_update_cholesky(context(), A.ptr, Ainv.ptr, pc.ptr, _ptr(z), _ptr(ps), n, d, float(cc), float(ccov), float(pthresh)),
                   "dmo_cmaes_update_cholesky")
        return A, Ainv, pc
    A = np.array(A, dtype=np.float64, order="C")
    Ainv = np.array(Ainv, dtype=np.float64, order="C")
    pc = np.array(pc, dtype=np.float64, order="C")
    z = _f64(z)
    ps = _f64(psucc)
    n, d = pc.shape
    _check(load_library().dmo_cmaes_update_cholesky(context(), _ptr(A), _ptr(Ainv), _ptr(pc), _ptr(z), _ptr(ps), n, d, float(cc), float(ccov), float(pthresh)),
           "dmo_cmaes_update_cholesky")
    return A, Ainv, pc


class CmaesResident:
    """The device buffers of MOASMO's resident MO-CMA-ES generation (dmo_cmaes_step_record / dmo_cmaes_step_apply): the
    parent state in two halves, each (parents_x, sigmas, A, Ainv, pc) ResidentRows plus the float64 objectives and int32
    ranks, and the candidates of the current generation (offspring x, [y_gen; parents_y], their ranks).  ``cur`` is the
    half that holds the state; ``apply`` writes the other one and flips."""

    def __init__(self, parents_x, sigmas, A, Ainv, pc, parents_y, n_off):
        self.pop, self.d = parents_x.shape
        self.M = parents_y.shape[1]
        self.C = int(n_off)
        rows = (parents_x, sigmas, A, Ainv, pc)
        # half 0 is the plugin's own state (no copy), half 1 is allocated here
        self.halves = [rows + (DeviceArray((self.pop, self.M)).upload(_f64(parents_y)), DeviceArray((self.pop,), np.int32)),
                       tuple(ResidentRows(DeviceArray(r.shape, np.float64), r.shape) for r in rows)
                       + (DeviceArray((self.pop, self.M)), DeviceArray((self.pop,), np.int32))]
        self.cur = 0
        n = self.C + self.pop
        self.cand_x = DeviceArray((self.C, self.d))
        self.cand_y = DeviceArray((n, self.M))
        self.cand_rank = DeviceArray((n,), np.int32)
        self.codes = pinned_empty((n,), np.uint8)
        self.p_idx = pinned_empty((self.C,), np.int64)

    @property
    def state(self):
        """(parents_x, sigmas, A, Ainv, pc, parents_y, rank) of the current half."""
        return self.halves[self.cur]

    def step_record(self, kind, posterior, draw_key, var_route_mean, precision, mean_f32, cand_f32, arz, js, mu, xlb, xub, x_gen, y_gen):
        """The first half of a generation (dmo_cmaes_step_record): ``arz`` (C, d) normals and ``js`` (C,) parent draws from
        the host.  x_gen / y_gen (C, d) / (C, M) float64, ``self.codes`` and ``self.p_idx`` are complete after
        ``synchronize()``."""
        px, sg, A, _, _, py, _ = self.state
        z, j = _f64(arz), np.ascontiguousarray(js, dtype=np.int64)
        lb, ub = _f64(xlb), _f64(xub)
        if z.shape != (self.C, self.d) or j.shape != (self.C,):
            raise ValueError(f"cmaes_step_record: arz must have shape {(self.C, self.d)} and js {(self.C,)}")
        draw_seed, draw_stream = draw_key
        _check(load_library().dmo_cmaes_step_record(
            context(), int(kind), posterior._h, _seed(draw_seed), int(draw_stream), 1 if var_route_mean else 0, int(precision), 1 if mean_f32 else 0,
            1 if cand_f32 else 0, px.ptr, sg.ptr, sg.row_elems, A.ptr, py.ptr, self.pop, self.d, self.M, _ptr(z), _ptr(j), self.C, int(mu), _ptr(lb),
            _ptr(ub), self.cand_x.ptr, self.cand_y.ptr, self.cand_rank.ptr, _ptr(x_gen), _ptr(y_gen), _ptr(self.codes), _ptr(self.p_idx)),
            "dmo_cmaes_step_record")

    def step_apply(self, h, xlb, xub, cc, ccov, pthresh):
        """The second half (dmo_cmaes_step_apply) with the host's update arithmetic ``h`` (CMAES._strategy_scalars);
        the next parent set goes to the other half, which becomes the current one."""
        px, sg, A, Ainv, pc, _, _ = self.state
        out = self.halves[1 - self.cur]
        i64 = lambda a: np.ascontiguousarray(a, dtype=np.int64)  # noqa: E731
        oc, op, sr, ss, nc, ns = i64(h.ch_off), i64(h.par), i64(h.seg_row), i64(h.seg_start), i64(h.ch), i64(h.src_idx)
        ps, of, ef = _f64(h.off_psucc), _f64(h.off_fac), _f64(h.ev_fac)
        lb, ub = _f64(xlb), _f64(xub)
        _check(load_library().dmo_cmaes_step_apply(
            context(), px.ptr, sg.ptr, sg.row_elems, A.ptr, Ainv.ptr, pc.ptr, self.pop, self.d, self.M, self.cand_x.ptr, self.cand_y.ptr,
            self.cand_rank.ptr, self.C, oc.shape[0], _ptr(oc), _ptr(op), _ptr(ps), _ptr(of), sr.shape[0], _ptr(sr), _ptr(ss), _ptr(ef), _ptr(nc),
            _ptr(ns), _ptr(lb), _ptr(ub), float(cc), float(ccov), float(pthresh), *(a.ptr for a in out)), "dmo_cmaes_step_apply")
        self.cur = 1 - self.cur


# --------------------------------------------------------------------------- sensitivity analysis (SA_DGSM / SA_FAST)
def _design_out(shape, write, mirror):
    """(rows, d) design written by ``write(pointer)``: with ``mirror`` a read-only page-locked array whose device copy the
    library keeps (a surrogate predict of it uploads nothing), else an ordinary NumPy array."""
    if not mirror:
        out = np.empty(shape, dtype=np.float64)
        write(out.ctypes.data)
        return out
    dev = DeviceArray(shape, np.float64)
    write(dev.ptr)
    return _mirrored_out(dev)


def _bounds(xlb, xub, d):
    lb, ub = _f64(xlb).reshape(-1), _f64(xub).reshape(-1)
    if lb.shape != (d,) or ub.shape != (d,):
        raise ValueError(f"bounds must have {d} entries (got {lb.shape[0]} and {ub.shape[0]})")
    return lb, ub


def sa_dgsm_design(base, xlb, xub, delta=0.01, mirror=True):
    """(N (d+1), d) DGSM design from the base points ``base`` (N, d) in the unit cube (dmo_sa_dgsm_design): row i (d+1)
    is base_i, row i (d+1) + 1 + j is base_i + delta e_j, every row scaled to u (xub - xlb) + xlb."""
    B = _f64(base)
    if B.ndim != 2 or B.shape[0] < 1 or B.shape[1] < 1:
        raise ValueError(f"base must be a non-empty (N, d) array (got shape {B.shape})")
    N, d = B.shape
    lb, ub = _bounds(xlb, xub, d)
    write = lambda p: _check(load_library().dmo_sa_dgsm_design(context(), _ptr(B), N, d, _ptr(lb), _ptr(ub), float(delta), p), "dmo_sa_dgsm_design")
    return _design_out((N * (d + 1), d), write, mirror)


def sa_fast_design(N, omega, phi, xlb, xub, mirror=True):
    """(N d, d) eFAST design (dmo_sa_fast_design) for the frequencies ``omega`` (d,) and per-block phases ``phi`` (d,)."""
    w, ph = _f64(omega).reshape(-1), _f64(phi).reshape(-1)
    d, N = w.shape[0], int(N)
    if ph.shape != (d,):
        raise ValueError(f"phi must have {d} entries (got {ph.shape[0]})")
    lb, ub = _bounds(xlb, xub, d)
    write = lambda p: _check(load_library().dmo_sa_fast_design(context(), N, d, _ptr(w), _ptr(ph), _ptr(lb), _ptr(ub), p), "dmo_sa_fast_design")
    return _design_out((N * d, d), write, mirror)


def sa_dgsm_stats(X, Y, xlb, xub, boot_idx, conf_level=0.95):
    """{vi, vi_std, dgsm, conf}, each (M, d), of a DGSM design X (N (d+1), d) and its outputs Y (N (d+1), M)
    (dmo_sa_dgsm_stats).  X and Y may be host arrays (a mirrored design is read from its device copy) or device arrays
    (``data_ptr()``); boot_idx (R, N) are the base indices of the R bootstrap replicates."""
    from statistics import NormalDist

    xs, ys = tuple(X.shape), tuple(Y.shape)
    X = _f64(X) if isinstance(X, np.ndarray) else X
    Y = _f64(Y) if isinstance(Y, np.ndarray) else Y
    if len(xs) != 2 or xs[1] < 1 or xs[0] % (xs[1] + 1) != 0:
        raise ValueError(f"X must be a DGSM design of N (d+1) rows and d columns (got shape {xs})")
    d = xs[1]
    N = xs[0] // (d + 1)
    M = 1 if len(ys) == 1 else ys[1]
    if ys[0] != xs[0] or len(ys) > 2:
        raise ValueError(f"Y must have the design's {xs[0]} rows (got shape {ys})")
    idx = np.ascontiguousarray(boot_idx, dtype=np.int32)
    if idx.ndim != 2 or idx.shape[1] != N:
        raise ValueError(f"boot_idx must be (R, N={N}) (got shape {idx.shape})")
    lb, ub = _bounds(xlb, xub, d)
    z = NormalDist().inv_cdf(0.5 + conf_level / 2)
    out = {k: np.empty((M, d), dtype=np.float64) for k in ("vi", "vi_std", "dgsm", "conf")}
    _check(load_library().dmo_sa_dgsm_stats(context(), _in(X), _in(Y), N, d, M, _ptr(lb), _ptr(ub), _ptr(idx), idx.shape[0], float(z),
                                            _ptr(out["vi"]), _ptr(out["vi_std"]), _ptr(out["dgsm"]), _ptr(out["conf"])), "dmo_sa_dgsm_stats")
    return out


# --------------------------------------------------------------------------- uniform designs (discrepancy / GLP search)
L2_METRICS = {"MD2": 0, "CD2": 1, "SD2": 2, "WD2": 3}  # DMO_L2_*
GLP_MAX_CANDIDATES = 65535  # lattices per dmo_glp_cd2_terms / _pairs call (csrc/design.cu, one grid row each)
GLP_MAX_LATTICE = 2**31 - 1  # (k + 1) h stays below 2^62 in int64


def l2_discrepancy_terms(X, metric):
    """(D2, D3) of the design X (n, s) for ``metric`` in MD2 / CD2 / SD2 / WD2 (dmo_l2_discrepancy_terms)."""
    A = _f64(X)
    if A.ndim != 2 or A.shape[0] < 1 or A.shape[1] < 1:
        raise ValueError(f"X must be a non-empty (n, s) array (got shape {A.shape})")
    d2, d3 = np.empty(1), np.empty(1)
    _check(load_library().dmo_l2_discrepancy_terms(context(), L2_METRICS[metric], _ptr(A), A.shape[0], A.shape[1], _ptr(d2), _ptr(d3)),
           "dmo_l2_discrepancy_terms")
    return float(d2[0]), float(d3[0])


def _multipliers(H, lattice, rows):
    H = np.ascontiguousarray(H, dtype=np.int64)
    if H.ndim != 2 or H.shape[1] < 1:
        raise ValueError(f"H must be a (C, s) array of multipliers (got shape {H.shape})")
    if not 2 <= lattice <= GLP_MAX_LATTICE or not 1 <= rows <= lattice:
        raise ValueError(f"lattice {lattice} outside [2, 2^31 - 1] or rows {rows} outside [1, lattice]")
    return H


def glp_cd2_terms(H, lattice, rows):
    """CD2's (D2, D3), each (C,), of the rank-1 lattices with multipliers H (C, s) (dmo_glp_cd2_terms), in chunks of
    GLP_MAX_CANDIDATES."""
    H = _multipliers(H, lattice, rows)
    C, s = H.shape
    d2, d3 = np.empty(C), np.empty(C)
    for c0 in range(0, C, GLP_MAX_CANDIDATES):
        h = np.ascontiguousarray(H[c0 : c0 + GLP_MAX_CANDIDATES])
        _check(load_library().dmo_glp_cd2_terms(context(), _ptr(h), h.shape[0], s, int(lattice), int(rows), _ptr(d2[c0:]), _ptr(d3[c0:])),
               "dmo_glp_cd2_terms")
    return d2, d3


def glp_cd2_pairs(H, lattice, rows):
    """(L, rows^2) CD2 pair products of the lattices H (L, s) in the reference's operation order (dmo_glp_cd2_pairs)."""
    H = _multipliers(H, lattice, rows)
    if H.shape[0] > GLP_MAX_CANDIDATES:
        raise ValueError(f"at most {GLP_MAX_CANDIDATES} lattices per call (got {H.shape[0]})")
    P = np.empty((H.shape[0], rows * rows))
    _check(load_library().dmo_glp_cd2_pairs(context(), _ptr(H), H.shape[0], H.shape[1], int(lattice), int(rows), _ptr(P)), "dmo_glp_cd2_pairs")
    return P


# --------------------------------------------------------------------------- logistic feasibility model
FEAS_MAX_D = 90  # input dimensions of dmo_feas_fit / dmo_feas_create (csrc/feasibility.cu FEAS_MAX_D)
FEAS_MAX_J = 32  # constraints
FEAS_MAX_N = 65536  # training rows of dmo_feas_fit


def feas_fit(X, labels, folds, pca_mean, pca_comps, Cs, max_iter=100, tol=1e-11):
    """dmo_feas_fit: every (dataset, C, k) L1-logistic problem of J two-class constraints in one batch.

    X (N, d); labels (J, N) 0/1; folds (J, N) test-fold ids; pca_mean (6 J, d), pca_comps (6 J, d-1, d).  Returns a dict
    with scaler_mean / scaler_scale (6 J, d-1) and, per problem p = (s nC + c)(d-1) + k-1, coef (P, d), iters,
    objective, kkt, converged, correct."""
    X = _f64(X)
    N, d = X.shape
    labels = np.ascontiguousarray(labels, dtype=np.uint8)
    folds = np.ascontiguousarray(folds, dtype=np.int8)
    J = labels.shape[0]
    pca_mean, pca_comps, Cs = _f64(pca_mean), _f64(pca_comps), _f64(Cs)
    assert labels.shape == (J, N) and folds.shape == (J, N), "feas_fit: labels / folds must be (J, N)"
    assert pca_mean.shape == (6 * J, d) and pca_comps.shape == (6 * J, d - 1, d), "feas_fit: bad PCA shapes"
    nC = Cs.size
    P = 6 * J * nC * (d - 1)
    out = {
        "scaler_mean": np.empty((6 * J, d - 1)), "scaler_scale": np.empty((6 * J, d - 1)), "coef": np.empty((P, d)),
        "iters": np.empty(P, dtype=np.int32), "objective": np.empty(P), "kkt": np.empty(P),
        "converged": np.empty(P, dtype=np.int8), "correct": np.empty(P, dtype=np.int64),
    }
    _check(
        load_library().dmo_feas_fit(context(), _ptr(X), N, d, J, _ptr(labels), _ptr(folds), _ptr(pca_mean), _ptr(pca_comps), nC, _ptr(Cs),
                                    int(max_iter), float(tol), *[_ptr(out[k]) for k in ("scaler_mean", "scaler_scale", "coef", "iters",
                                                                                          "objective", "kkt", "converged", "correct")]),
        "dmo_feas_fit",
    )
    return out


class FeasModel(_LibObject):
    """A fitted feasibility model held on the device (dmo_feas): J constraints over d inputs."""

    _destroy = "dmo_feas_destroy"

    def __init__(self, k, mean, comps, smean, sscale, coef, intercept):
        k = np.ascontiguousarray(k, dtype=np.int32)
        mean = _f64(mean)
        J, d = mean.shape
        arrs = [_f64(a) for a in (comps, smean, sscale, coef, intercept)]
        assert k.shape == (J,) and arrs[0].shape == (J, d - 1, d) and arrs[4].shape == (J,)
        assert all(a.shape == (J, d - 1) for a in arrs[1:4])
        self.d, self.J = d, J
        h = _vp()
        _check(load_library().dmo_feas_create(context(), d, J, _ptr(k), _ptr(mean), *[_ptr(a) for a in arrs], ctypes.byref(h)),
               "dmo_feas_create")
        self._h = h

    def eval(self, X, rank=True, proba=False, decision=False):
        """(rank (n,), proba (J, n), decision (J, n)); the ones not asked for are None.  X may be a host array (its device
        mirror is read when it has one) or a device tensor."""
        if isinstance(X, np.ndarray) or not hasattr(X, "data_ptr"):
            X = np.ascontiguousarray(X, dtype=np.float64)
            n = X.shape[0]
            if X.ndim != 2 or X.shape[1] != self.d:
                raise ValueError(f"feasibility model: x must be (n, {self.d}), got {X.shape}")
        else:
            n = int(X.shape[0])
        r = np.empty(n) if rank else None
        p = np.empty((self.J, n)) if proba else None
        t = np.empty((self.J, n)) if decision else None
        _check(load_library().dmo_feas_eval(context(), self._h, _in(X), n, self.d, _ptr(r), _ptr(p), _ptr(t)), "dmo_feas_eval")
        return r, p, t
