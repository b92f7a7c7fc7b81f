"""ctypes binding of libb200mpi.so (include/b200mpi.h).

The library is the product; this module only declares its C ABI to Python.  It fails loudly when
the shared object is missing -- there is no Python or CPU fallback for any data call.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libb200mpi.so")

# enums of include/b200mpi.h
U8, I64, F32, F64 = 0, 1, 2, 3
SUM, MAX, MIN = 0, 1, 2
REPLACE, NO_OP = 3, 4                      # one-sided only
LOCK_EXCLUSIVE, LOCK_SHARED = 1, 2
HOST, DEVICE = 0, 1
COLL_ALLREDUCE, COLL_BCAST, COLL_ALLGATHER, COLL_REDUCE_SCATTER = 0, 1, 2, 3
ALGO_AUTO, ALGO_ONESHOT, ALGO_TWOSHOT, ALGO_RING, ALGO_NVLS, ALGO_TWOSHOT_SMEM, ALGO_LL, ALGO_HYBRID = 0, 1, 2, 3, 4, 5, 6, 7
ALGO_NAMES = {0: "auto", 1: "oneshot", 2: "twoshot", 3: "ring", 4: "nvls", 5: "twoshot_smem", 6: "ll", 7: "hybrid"}

OK = 0
ERR_ARG, ERR_NOT_INIT, ERR_BOOTSTRAP, ERR_PASSWORD, ERR_TIMEOUT, ERR_TAG_EXISTS = -1, -2, -3, -4, -5, -6
ERR_CUDA, ERR_NOMEM, ERR_TRUNCATE, ERR_NO_DEVICE, ERR_UNSUPPORTED, ERR_PEER = -7, -8, -9, -10, -11, -12

# every symbol include/b200mpi.h declares: name -> (restype, argtypes)
_c = ctypes
SYMBOLS = {
    "b200mpi_init": (_c.c_int, [_c.c_char_p, _c.c_char_p, _c.c_char_p, _c.c_int64, _c.c_int]),
    "b200mpi_finalize": (_c.c_int, []),
    "b200mpi_rank": (_c.c_int, []),
    "b200mpi_size": (_c.c_int, []),
    "b200mpi_device": (_c.c_int, []),
    "b200mpi_version": (_c.c_int, []),
    "b200mpi_last_error": (_c.c_char_p, []),
    "b200mpi_alloc": (_c.c_int, [_c.c_size_t, _c.POINTER(_c.c_void_p)]),
    "b200mpi_free": (_c.c_int, [_c.c_void_p]),
    "b200mpi_host_alloc": (_c.c_int, [_c.c_size_t, _c.POINTER(_c.c_void_p)]),
    "b200mpi_host_free": (_c.c_int, [_c.c_void_p]),
    "b200mpi_memcpy": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_size_t, _c.c_int]),
    "b200mpi_heap_info": (_c.c_int, [_c.POINTER(_c.c_size_t), _c.POINTER(_c.c_size_t), _c.POINTER(_c.c_int)]),
    "b200mpi_send": (_c.c_int, [_c.c_void_p, _c.c_size_t, _c.c_int, _c.c_int, _c.c_int, _c.c_int]),
    "b200mpi_isend": (_c.c_int, [_c.c_void_p, _c.c_size_t, _c.c_int, _c.c_int, _c.c_int, _c.c_int]),
    "b200mpi_wait": (_c.c_int, [_c.c_int, _c.c_int]),
    "b200mpi_recv": (_c.c_int, [_c.c_void_p, _c.c_size_t, _c.POINTER(_c.c_size_t), _c.c_int, _c.c_int, _c.c_int, _c.c_int]),
    "b200mpi_bcast": (_c.c_int, [_c.c_void_p, _c.c_size_t, _c.c_int, _c.c_int, _c.c_int]),
    "b200mpi_allreduce": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_size_t, _c.c_int, _c.c_int, _c.c_int]),
    "b200mpi_allgather": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_size_t, _c.c_int, _c.c_int]),
    "b200mpi_reduce_scatter": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_size_t, _c.c_int, _c.c_int, _c.c_int]),
    "b200mpi_reduce": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_size_t, _c.c_int, _c.c_int, _c.c_int, _c.c_int]),
    "b200mpi_alltoall": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_size_t, _c.c_int, _c.c_int]),
    "b200mpi_gather": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_size_t, _c.c_int, _c.c_int, _c.c_int]),
    "b200mpi_scatter": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_size_t, _c.c_int, _c.c_int, _c.c_int]),
    "b200mpi_gatherv": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.POINTER(_c.c_size_t), _c.c_int, _c.c_int, _c.c_int]),
    "b200mpi_scatterv": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.POINTER(_c.c_size_t), _c.c_int, _c.c_int, _c.c_int]),
    "b200mpi_allgatherv": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.POINTER(_c.c_size_t), _c.c_int, _c.c_int]),
    "b200mpi_alltoallv": (_c.c_int, [_c.c_void_p, _c.POINTER(_c.c_size_t), _c.c_void_p, _c.POINTER(_c.c_size_t), _c.c_int, _c.c_int]),
    "b200mpi_scan": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_size_t, _c.c_int, _c.c_int, _c.c_int]),
    "b200mpi_exscan": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_size_t, _c.c_int, _c.c_int, _c.c_int]),
    "b200mpi_reduce_scatterv": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.POINTER(_c.c_size_t), _c.c_int, _c.c_int, _c.c_int]),
    "b200mpi_allreduce_loc": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_size_t, _c.c_int, _c.c_int, _c.c_int]),
    "b200mpi_reduce_loc": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_size_t, _c.c_int, _c.c_int, _c.c_int, _c.c_int]),
    "b200mpi_win_create": (_c.c_int, [_c.c_void_p, _c.c_size_t, _c.POINTER(_c.c_int)]),
    "b200mpi_win_free": (_c.c_int, [_c.c_int]),
    "b200mpi_win_fence": (_c.c_int, [_c.c_int]),
    "b200mpi_put": (_c.c_int, [_c.c_void_p, _c.c_size_t, _c.c_int, _c.c_int, _c.c_size_t, _c.c_int, _c.c_int]),
    "b200mpi_get": (_c.c_int, [_c.c_void_p, _c.c_size_t, _c.c_int, _c.c_int, _c.c_size_t, _c.c_int, _c.c_int]),
    "b200mpi_accumulate": (_c.c_int, [_c.c_void_p, _c.c_size_t, _c.c_int, _c.c_int, _c.c_int, _c.c_size_t, _c.c_int, _c.c_int]),
    "b200mpi_win_lock": (_c.c_int, [_c.c_int, _c.c_int, _c.c_int]),
    "b200mpi_win_unlock": (_c.c_int, [_c.c_int, _c.c_int]),
    "b200mpi_get_accumulate": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_size_t, _c.c_int, _c.c_int, _c.c_int, _c.c_size_t, _c.c_int, _c.c_int]),
    "b200mpi_fetch_and_op": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_int, _c.c_int, _c.c_int, _c.c_size_t, _c.c_int]),
    "b200mpi_compare_and_swap": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_int, _c.c_int, _c.c_size_t, _c.c_int]),
    "b200mpi_win_post": (_c.c_int, [_c.c_void_p, _c.c_int, _c.c_int]),
    "b200mpi_win_start": (_c.c_int, [_c.c_void_p, _c.c_int, _c.c_int]),
    "b200mpi_win_complete": (_c.c_int, [_c.c_int]),
    "b200mpi_win_wait": (_c.c_int, [_c.c_int]),
    "b200mpi_win_test": (_c.c_int, [_c.c_int, _c.c_void_p]),
    "b200mpi_reduce_scatter_async": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_size_t, _c.c_int, _c.c_int]),
    "b200mpi_numa_node": (_c.c_int, []),
    "b200mpi_barrier": (_c.c_int, []),
    "b200mpi_bcast_async": (_c.c_int, [_c.c_void_p, _c.c_size_t, _c.c_int, _c.c_int]),
    "b200mpi_allreduce_async": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_size_t, _c.c_int, _c.c_int]),
    "b200mpi_allgather_async": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_size_t, _c.c_int]),
    "b200mpi_stream_sync": (_c.c_int, []),
    "b200mpi_set_algo": (_c.c_int, [_c.c_int, _c.c_int]),
    "b200mpi_get_algo": (_c.c_int, [_c.c_int, _c.c_size_t, _c.c_int]),
    "b200mpi_set_max_blocks": (_c.c_int, [_c.c_int]),
    "b200mpi_set_param": (_c.c_int, [_c.c_char_p, _c.c_int64]),
    "b200mpi_get_param": (_c.c_int, [_c.c_char_p, _c.POINTER(_c.c_int64)]),
    "b200mpi_get_stream": (_c.c_int, [_c.POINTER(_c.c_void_p)]),
    "b200mpi_set_stream": (_c.c_int, [_c.c_void_p]),
    "b200mpi_timer_start": (_c.c_int, []),
    "b200mpi_timer_stop": (_c.c_int, [_c.POINTER(_c.c_float)]),
    "b200mpi_pcie_probe": (_c.c_int, [_c.c_size_t, _c.c_int, _c.POINTER(_c.c_double), _c.POINTER(_c.c_double), _c.POINTER(_c.c_double)]),
    "b200mpi_link_probe": (_c.c_int, [_c.c_size_t, _c.c_int, _c.c_int, _c.POINTER(_c.c_float)]),
    "b200mpi_launch_count": (_c.c_int64, []),
}

_lib = None


def load():
    """Load libb200mpi.so (once) and type every entry point.  Raises if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "libb200mpi.so is not built (%s). Run `python -c 'import __graft_entry__ as g; g.build()'` "
            "or `make -C mpi_b200/csrc`. There is no fallback implementation." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH, mode=ctypes.RTLD_GLOBAL)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError here means header and library disagree
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def get_param(name):
    v = ctypes.c_int64()
    if load().b200mpi_get_param(name.encode(), ctypes.byref(v)):
        raise RuntimeError(last_error())
    return v.value


def last_error():
    return load().b200mpi_last_error().decode("utf-8", "replace")
