"""ctypes binding of the C ABI in include/afl_b200.h (lib/libafl_b200.so).

There is no CPU fallback: if the shared library is missing, or a call fails, this raises.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libafl_b200.so")

AFL_OK, AFL_ERR_BAD_ARG, AFL_ERR_PRECONDITION, AFL_ERR_CUDA, AFL_ERR_UNSUPPORTED, AFL_ERR_WORKSPACE, AFL_ERR_NO_WINNER = range(7)
AFL_ERR_NAN_LOSS, AFL_ERR_NAN_DIST_LOSS = 7, 8
AFL_F32, AFL_BF16, AFL_F16 = 0, 1, 2
GRAM_AUTO, GRAM_FORCE_SIMT, GRAM_FORCE_TCGEN05, GRAM_SINGLE_PASS, GRAM_REWRITE_HI = 0, 1, 2, 4, 8
GRAM_TF32X2 = 16
GRAM_BF16X2 = 32
GRAM_NO_CENTER = 64

_vp, _i, _i64, _sz, _d, _f = C.c_void_p, C.c_int, C.c_int64, C.c_size_t, C.c_double, C.c_float

# name -> (restype, argtypes); mirrors include/afl_b200.h one to one
SIGNATURES = {
    "afl_version": (C.c_char_p, []),
    "afl_last_error": (C.c_char_p, []),
    "afl_device_info": (_i, [C.POINTER(_i), C.POINTER(_i), C.POINTER(_i), C.POINTER(_sz), C.POINTER(_sz)]),
    "afl_launch_count": (C.c_uint64, []),
    "afl_profile_enable": (_i, [_i]),
    "afl_profile_read": (_i, [C.c_char_p, C.POINTER(_d), C.POINTER(_i)]),
    "afl_mean": (_i, [_vp, _i, _i64, _i64, _i, _vp, _vp]),
    "afl_sqdist_workspace_bytes": (_sz, [_i, _i64, _i, _i]),
    "afl_sqdist_partial": (_i, [_vp, _i, _i64, _i64, _i, _vp, _vp, _sz, _i, _vp]),
    "afl_sqdist_to_dist": (_i, [_vp, _i, _vp, _vp]),
    "afl_select_workspace_bytes": (_sz, [_i]),
    "afl_krum_select": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "afl_krum_from_sqdist": (_i, [_vp, _i, _i, _i, _vp, _vp, _sz, _vp]),
    "afl_bulyan_select": (_i, [_vp, _i, _i, _i, _vp, _vp, _sz, _vp]),
    "afl_trimmed_mean": (_i, [_vp, _i, _i64, _i64, _i, _vp, _i, _i, _vp, _vp]),
    "afl_gather_row": (_i, [_vp, _i, _i64, _i64, _i, _vp, _vp, _vp]),
    "afl_alie": (_i, [_vp, _i, _i64, _i64, _i, _d, _vp, _vp, _vp, _vp, _i64, _vp]),
    "afl_alie_band": (_i, [_vp, _vp, _d, _vp, _vp, _i64, _vp]),
    "afl_momentum_step": (_i, [_vp, _vp, _vp, _i64, _f, _f, _vp]),
    "afl_momentum_step_batched": (_i, [_vp, _vp, _vp, _i, _i64, _f, _vp, _vp]),
    "afl_xgpu_create": (_i, [_i, _i, _i, C.POINTER(_vp)]),
    "afl_xgpu_handle": (_i, [_vp, C.c_char_p]),
    "afl_xgpu_connect": (_i, [_vp, C.c_char_p]),
    "afl_xgpu_destroy": (_i, [_vp]),
    "afl_krum_sharded": (_i, [_vp, _vp, _i, _i64, _i64, _i, _i, _i, _vp, _sz, _i, _vp, C.POINTER(C.POINTER(_i)),
                              C.POINTER(C.POINTER(_i)), C.POINTER(C.POINTER(_i))]),
    "afl_sqdist_allreduce": (_i, [_vp, _vp, _i, _i64, _i64, _i, _vp, _vp, _sz, _i, _vp, C.POINTER(C.POINTER(_i))]),
    "afl_defend_host": (_i, [C.c_char_p, _vp, _i, _i64, _i64, _i, _i, _vp, C.POINTER(_i), _i64]),
    "afl_sqdist_host": (_i, [_vp, _i, _i64, _i64, _vp, _i64]),
    "afl_bulyan_host": (_i, [_vp, _i, _i64, _i64, _i, _i, _vp, _vp, _i64]),
    "afl_alie_host": (_i, [_vp, _i, _i64, _d, _vp, _vp, _vp, _i64]),
    "afl_batched_workspace_bytes": (_sz, [C.c_char_p, _i, _i, _i64, _i]),
    "afl_defend_batched": (_i, [C.c_char_p, _vp, _i, _i64, _i, _i64, _i64, _i, _i, _i, _vp, _vp, _vp, _vp, _sz, _vp]),
    "afl_alie_batched": (_i, [_vp, _i, _i64, _i, _i64, _i64, _i, _d, _vp, _vp, _vp, _vp, _i64, _i64, _vp]),
    "afl_batched_each_workspace_bytes": (_sz, [C.c_char_p, _i, _i, _i64, _i]),
    "afl_defend_batched_each": (_i, [C.c_char_p, _vp, _i, _i64, _i, _i64, _i64, _i, _i, _vp, _vp, _vp, _vp, _vp, _sz,
                                     _vp]),
    "afl_alie_batched_each": (_i, [_vp, _i, _i64, _i, _i64, _i64, _i, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _vp,
                                   _sz, _vp]),
    "afl_metrics_workspace_bytes": (_sz, [_i, _i, _i64, _i]),
    "afl_attack_metrics_batched": (_i, [_vp, _i, _i64, _i, _i64, _i64, _i, _i, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp,
                                        _vp, _vp, _vp, _sz, _vp]),
    "afl_attack_metrics_batched_each": (_i, [_vp, _i, _i64, _i, _i64, _i64, _i, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp,
                                             _vp, _vp, _vp, _vp, _sz, _vp]),
    "afl_batched_rows_workspace_bytes": (_sz, [C.c_char_p, _i, _i, _i64, _i]),
    "afl_defend_batched_rows": (_i, [C.c_char_p, _vp, _i, _i64, _i, _i64, _i64, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                     _sz, _vp]),
    "afl_attack_metrics_batched_rows": (_i, [_vp, _i, _i64, _i, _i64, _i64, _i, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp,
                                             _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "afl_batched_large_workspace_bytes": (_sz, [C.c_char_p, _i, _i, _i64, _i]),
    "afl_defend_batched_large": (_i, [C.c_char_p, _vp, _i, _i64, _i, _i64, _i64, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                      _sz, _vp]),
    "afl_alie_batched_large": (_i, [_vp, _i, _i64, _i, _i64, _i64, _i, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _vp,
                                    _sz, _vp]),
    "afl_backdoor_start_batched": (_i, [_vp, _i, _i64, _i, _i64, _i64, _i, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp,
                                        _sz, _vp]),
    "afl_backdoor_finish_batched": (_i, [_i, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _i64, _i64, _vp,
                                         _sz, _vp]),
    "afl_batched_table_dev": (_i, [C.c_char_p, _i, _i, _vp, _i, _vp, _vp, _vp, _vp, _sz, _vp, _vp]),
    "afl_defend_batched_dev": (_i, [C.c_char_p, _vp, _i, _i64, _i, _i64, _i64, _i, _vp, _i, _vp, _vp, _vp, _vp, _vp, _i,
                                    _vp, _sz, _vp, _vp]),
    "afl_alie_batched_dev": (_i, [_vp, _i, _i64, _i, _i64, _i64, _i, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _sz,
                                  _vp, _vp]),
    "afl_attack_metrics_batched_dev": (_i, [_vp, _i, _i64, _i, _i64, _i64, _i, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp,
                                            _vp, _vp, _vp, _vp, _vp, _sz, _vp, _vp]),
    "afl_attack_trace_workspace_bytes": (_sz, [_i, _i64]),
    "afl_attack_trace_dev": (_i, [_vp, _i, _i64, _i, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _i, _vp, _i, _i64, _vp, _vp,
                                  _vp, _vp, _vp, _vp, _sz, _vp, _vp]),
    "afl_batched_large_dev_workspace_bytes": (_sz, [C.c_char_p, _i, _i, _i64, _i]),
    "afl_defend_batched_large_dev": (_i, [C.c_char_p, _vp, _i, _i64, _i, _i64, _i64, _i, _vp, _i, _vp, _vp, _vp, _vp, _vp,
                                          _i, _vp, _sz, _vp, _vp]),
    "afl_mnist_client_grads": (_i, [_vp, _i, _i64, _vp, _vp, _i, _i, _vp, _vp, _i, _i, _vp, _vp, _i64, _i64, _vp]),
    "afl_mnist_client_grads_sets": (_i, [_vp, _i, _i64, _vp, _vp, _i, _i, _vp, _vp, _vp, _i, _i, _vp, _vp, _i64, _i64,
                                         _vp]),
    "afl_mnist_evaluate_workspace_bytes": (_sz, [_i, _i, _i]),
    "afl_mnist_evaluate": (_i, [_vp, _i, _i64, _vp, _vp, _i, _i, _vp, _i, _vp, _i, _vp, _vp, _vp, _sz, _vp]),
    "afl_mnist_client_grads_each": (_i, [_vp, _i, _i64, _vp, _vp, _i, _i, _vp, _vp, _vp, _i, _vp, _i, _vp, _vp, _i64,
                                         _i64, _vp]),
    "afl_mnist_evaluate_each": (_i, [_vp, _i, _i64, _vp, _vp, _i, _i, _vp, _vp, _i, _i, _vp, _i, _vp, _vp, _vp, _sz,
                                     _vp]),
    "afl_backdoor_start_batched_dev": (_i, [_vp, _i, _i64, _i, _i64, _i64, _i, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp,
                                            _vp, _sz, _vp, _vp]),
    "afl_backdoor_finish_batched_dev": (_i, [_i, _i, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _i64,
                                             _i64, _vp, _sz, _vp, _vp]),
    "afl_mnist_backdoor_train": (_i, [_vp, _vp, _i, _i64, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _d, _i, _i, _vp]),
    "afl_mnist_backdoor_train_each": (_i, [_vp, _vp, _i, _i64, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i,
                                           _vp]),
    "afl_mnist_backdoor_test": (_i, [_vp, _i, _i64, _vp, _vp, _i, _i, _vp, _vp, _i, _vp, _i, _vp, _vp, _vp]),
    "afl_cifar10_client_grads": (_i, [_vp, _i, _i64, _vp, _vp, _i, _i, _vp, _vp, _i, _i, _vp, _vp, _i64, _i64, _vp]),
    "afl_cifar10_client_grads_sets": (_i, [_vp, _i, _i64, _vp, _vp, _i, _i, _vp, _vp, _vp, _i, _i, _vp, _vp, _i64,
                                           _i64, _vp]),
    "afl_cifar10_evaluate_workspace_bytes": (_sz, [_i, _i, _i]),
    "afl_cifar10_evaluate": (_i, [_vp, _i, _i64, _vp, _vp, _i, _i, _vp, _i, _vp, _i, _vp, _vp, _vp, _sz, _vp]),
    "afl_cifar10_client_grads_each": (_i, [_vp, _i, _i64, _vp, _vp, _i, _i, _vp, _vp, _vp, _i, _vp, _i, _vp, _vp, _i64,
                                           _i64, _vp]),
    "afl_cifar10_evaluate_each": (_i, [_vp, _i, _i64, _vp, _vp, _i, _i, _vp, _vp, _i, _i, _vp, _i, _vp, _vp, _vp, _sz,
                                       _vp]),
    "afl_cifar10_backdoor_train_workspace_bytes": (_sz, [_i]),
    "afl_cifar10_backdoor_train": (_i, [_vp, _vp, _i, _i64, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _d, _i, _i, _vp,
                                        _sz, _vp]),
    "afl_cifar10_backdoor_train_each": (_i, [_vp, _vp, _i, _i64, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                             _i, _vp, _sz, _vp]),
    "afl_cifar10_backdoor_test_workspace_bytes": (_sz, [_i, _i, _i]),
    "afl_cifar10_backdoor_test": (_i, [_vp, _i, _i64, _vp, _vp, _i, _i, _vp, _vp, _i, _vp, _i, _vp, _vp, _vp, _sz, _vp]),
}

_lib = None


class NativeError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"afl_b200 error {code}: {msg}")
        self.code = code


def lib():
    """Load (once) and return the shared library; raise if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} not found: build the CUDA extension first "
                "(python -c 'import __graft_entry__ as g; g.build()' at the repo root). "
                "This package has no CPU fallback.")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)          # AttributeError here == ABI drift, fail loudly
            fn.restype, fn.argtypes = res, args
        _lib = handle
    return _lib


def check(rc: int):
    """Map a status code to the reference's error behaviour: precondition -> AssertionError."""
    if rc == AFL_OK:
        return
    msg = lib().afl_last_error().decode("utf-8", "replace")
    if rc == AFL_ERR_PRECONDITION:
        raise AssertionError(msg)
    if rc == AFL_ERR_UNSUPPORTED:
        raise NotImplementedError(msg)
    if rc == AFL_ERR_BAD_ARG:
        raise ValueError(msg)
    if rc == AFL_ERR_NO_WINNER:
        raise KeyError(-1)                       # what `distances.pop(-1)` raises in the reference (defences.py:66)
    raise NativeError(rc, msg)


def launch_count() -> int:
    return int(lib().afl_launch_count())


def profile_enable(on):
    """False/0: off; True/1: every bracketed kernel; 2: only the dominant kernel of each rule."""
    check(lib().afl_profile_enable(int(on)))


def profile_read(kernel: str):
    """(total_ms, launches) of the recorded launches of `kernel`; clears them."""
    ms, cnt = _d(0.0), _i(0)
    check(lib().afl_profile_read(kernel.encode(), C.byref(ms), C.byref(cnt)))
    return ms.value, cnt.value


