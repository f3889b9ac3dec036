"""ctypes binding of libluaradio_b200.so (include/lrb200.h).

This is the Python twin of the LuaJIT `ffi.cdef` + `platform.load` in lua/radio_b200/platform.lua
(reference pattern: radio/core/platform.lua:277-299).  There is no fallback: if the library is
missing, or no CUDA device is usable, every block's initialize() raises.
"""
import ctypes
import os
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_longlong, c_size_t, c_uint, c_uint32, c_uint64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("LRB200_LIB", os.path.join(_HERE, "libluaradio_b200.so"))   # override: A/B-testing kernel builds

LRB200_HOST = 0
LRB200_DEVICE = 1
FIR_AUTO, FIR_DIRECT, FIR_FFT = 0, 1, 2

_lib = None

_PROTOS = {
    # name: (restype, argtypes)
    "lrb200_init": (c_int, [c_int]),
    "lrb200_device_count": (c_int, []),
    "lrb200_current_device": (c_int, []),
    "lrb200_last_error": (c_char_p, []),
    "lrb200_version": (c_char_p, []),
    "lrb200_set_stream": (c_int, [c_void_p]),
    "lrb200_get_stream": (c_void_p, []),
    "lrb200_sync": (c_int, []),
    "lrb200_launch_count": (c_uint64, []),
    "lrb200_malloc": (c_void_p, [c_size_t]),
    "lrb200_free": (None, [c_void_p]),
    "lrb200_host_alloc": (c_void_p, [c_size_t]),
    "lrb200_host_free": (None, [c_void_p]),
    "lrb200_memcpy_h2d": (c_int, [c_void_p, c_void_p, c_size_t]),
    "lrb200_memcpy_d2h": (c_int, [c_void_p, c_void_p, c_size_t]),
    "lrb200_memset": (c_int, [c_void_p, c_int, c_size_t]),
    "lrb200_ipc_export": (c_int, [c_void_p, c_void_p]),
    "lrb200_ipc_import": (c_void_p, [c_void_p]),
    "lrb200_ipc_close": (c_int, [c_void_p]),
    "lrb200_memcpy_d2d": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p]),
    "lrb200_block_execute": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p, POINTER(c_size_t)]),
    "lrb200_block_execute_multi": (c_int, [c_void_p, POINTER(c_void_p), c_uint, c_size_t, POINTER(c_void_p), c_uint, POINTER(c_size_t)]),
    "lrb200_block_num_inputs": (c_uint, [c_void_p]),
    "lrb200_block_num_outputs": (c_uint, [c_void_p]),
    "lrb200_binary_create": (c_void_p, [c_char_p, c_uint, c_uint]),
    "lrb200_delay_create": (c_void_p, [c_uint, c_uint, c_uint]),
    "lrb200_pll_create": (c_void_p, [c_double, c_double, c_double, c_double, c_double, c_uint]),
    "lrb200_pll_set_mode": (c_int, [c_void_p, c_int]),
    "lrb200_pll_chunk_counts": (c_int, [c_void_p, POINTER(c_uint64), POINTER(c_uint64)]),
    "lrb200_agc_create": (c_void_p, [c_double, c_double, c_double, c_double, c_double, c_uint, c_uint]),
    "lrb200_powersquelch_create": (c_void_p, [c_double, c_double, c_double, c_uint, c_uint]),
    "lrb200_phasecorrector_create": (c_void_p, [c_uint, c_uint, c_uint]),
    "lrb200_psd_create": (c_void_p, [c_uint, c_void_p, c_double, c_uint, c_uint, c_uint]),
    "lrb200_block_max_output": (c_size_t, [c_void_p, c_size_t]),
    "lrb200_block_in_size": (c_size_t, [c_void_p]),
    "lrb200_block_out_size": (c_size_t, [c_void_p]),
    "lrb200_block_reset": (c_int, [c_void_p]),
    "lrb200_block_seek": (c_int, [c_void_p, c_uint64]),
    "lrb200_block_destroy": (None, [c_void_p]),
    "lrb200_block_name": (c_char_p, [c_void_p]),
    "lrb200_fir_create_crcf": (c_void_p, [c_void_p, c_uint, c_uint, c_uint]),
    "lrb200_fir_create_cccf": (c_void_p, [c_void_p, c_uint, c_uint, c_uint]),
    "lrb200_fir_create_rrrf": (c_void_p, [c_void_p, c_uint, c_uint, c_uint]),
    "lrb200_fir_execute": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p, POINTER(c_size_t)]),
    "lrb200_fir_reset": (c_int, [c_void_p]),
    "lrb200_fir_destroy": (None, [c_void_p]),
    "lrb200_fir_set_algorithm": (c_int, [c_void_p, c_int]),
    "lrb200_fir_get_algorithm": (c_int, [c_void_p]),
    "lrb200_hilbert_create": (c_void_p, [c_void_p, c_uint, c_uint]),
    "lrb200_rotator_create": (c_void_p, [c_double, c_uint]),
    "lrb200_discrim_create": (c_void_p, [c_float, c_uint]),
    "lrb200_downsample_create": (c_void_p, [c_uint, c_uint, c_uint]),
    "lrb200_iir_create_rrrf": (c_void_p, [c_void_p, c_uint, c_void_p, c_uint, c_uint]),
    "lrb200_iir_create_crcf": (c_void_p, [c_void_p, c_uint, c_void_p, c_uint, c_uint]),
    "lrb200_cmag_create": (c_void_p, [c_uint]),
    "lrb200_c2r_create": (c_void_p, [c_uint]),
    "lrb200_mulconst_create": (c_void_p, [c_float, c_float, c_uint, c_uint, c_uint]),
    "lrb200_upsample_create": (c_void_p, [c_uint, c_uint, c_uint]),
    "lrb200_iqconv_create": (c_void_p, [c_char_p, c_uint]),
    "lrb200_realconv_create": (c_void_p, [c_char_p, c_uint]),
    "lrb200_iqsink_create": (c_void_p, [c_char_p, c_uint]),
    "lrb200_realsink_create": (c_void_p, [c_char_p, c_uint]),
    "lrb200_graph_create": (c_void_p, []),
    "lrb200_graph_append": (c_int, [c_void_p, c_void_p]),
    "lrb200_graph_commit": (c_int, [c_void_p, c_int]),
    "lrb200_graph_execute": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p, POINTER(c_size_t)]),
    "lrb200_graph_execute_device": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p, POINTER(c_size_t)]),
    "lrb200_graph_max_output": (c_size_t, [c_void_p, c_size_t]),
    "lrb200_graph_set_superchunk": (c_int, [c_void_p, c_size_t]),
    "lrb200_graph_flush": (c_int, [c_void_p, c_void_p, POINTER(c_size_t)]),
    "lrb200_graph_halo": (c_longlong, [c_void_p]),
    "lrb200_graph_execute_shard": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_size_t, c_uint64, c_void_p, POINTER(c_size_t), c_void_p]),
    "lrb200_graph_reset": (c_int, [c_void_p]),
    "lrb200_graph_seek": (c_int, [c_void_p, c_uint64]),
    "lrb200_graph_num_stages": (c_int, [c_void_p]),
    "lrb200_graph_describe": (c_char_p, [c_void_p]),
    "lrb200_graph_stage_name": (c_char_p, [c_void_p, c_int]),
    "lrb200_graph_set_timing": (c_int, [c_void_p, c_int]),
    "lrb200_graph_stage_time_ms": (c_double, [c_void_p, c_int, POINTER(c_int)]),
    "lrb200_graph_destroy": (None, [c_void_p]),
    "lrb200_dag_create": (c_void_p, []),
    "lrb200_dag_add_block": (c_int, [c_void_p, c_void_p, POINTER(c_int), c_uint]),
    "lrb200_dag_add_graph": (c_int, [c_void_p, c_void_p, c_int]),
    "lrb200_dag_set_outputs": (c_int, [c_void_p, POINTER(c_int), c_uint]),
    "lrb200_dag_commit": (c_int, [c_void_p, c_int]),
    "lrb200_dag_execute": (c_int, [c_void_p, c_void_p, c_size_t, POINTER(c_void_p), POINTER(c_size_t)]),
    "lrb200_dag_execute_device": (c_int, [c_void_p, c_void_p, c_size_t, POINTER(c_void_p), POINTER(c_size_t)]),
    "lrb200_dag_max_output": (c_size_t, [c_void_p, c_uint, c_size_t]),
    "lrb200_dag_set_superchunk": (c_int, [c_void_p, c_size_t]),
    "lrb200_dag_flush": (c_int, [c_void_p, POINTER(c_void_p), POINTER(c_size_t)]),
    "lrb200_dag_reset": (c_int, [c_void_p]),
    "lrb200_dag_halo": (c_longlong, [c_void_p]),
    "lrb200_dag_seek": (c_int, [c_void_p, c_uint64]),
    "lrb200_dag_shard_record_bytes": (c_size_t, [c_void_p]),
    "lrb200_dag_shard_begin": (c_int, [c_void_p, c_void_p, c_size_t, c_size_t, c_uint64, POINTER(c_void_p), POINTER(c_size_t), c_void_p, c_size_t]),
    "lrb200_dag_shard_accepts": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t]),
    "lrb200_dag_shard_end": (c_int, [c_void_p, c_void_p, c_uint, POINTER(c_void_p), POINTER(c_size_t), c_void_p, c_size_t]),
    "lrb200_dag_describe": (c_char_p, [c_void_p]),
    "lrb200_dag_destroy": (None, [c_void_p]),
    "lrb200_synth_white_iq": (c_int, [c_void_p, c_uint64, c_size_t, c_uint32]),
    "lrb200_synth_fm_iq": (c_int, [c_void_p, c_uint64, c_size_t, c_uint32, c_double, c_double, c_double, c_float, c_float]),
}

EXPORTED_SYMBOLS = sorted(_PROTOS)


class LibraryError(RuntimeError):
    pass


def load():
    """dlopen the library and bind every prototype.  Raises LibraryError if the .so is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise LibraryError("libluaradio_b200.so not built (%s); run `python -m luaradio_b200.build`. "
                           "There is no CPU fallback." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in _PROTOS.items():
        fn = getattr(lib, name)       # AttributeError if a declared symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def last_error():
    return load().lrb200_last_error().decode("utf-8", "replace")


def check(rc, what=""):
    if rc != 0:
        raise LibraryError("%s failed: %s" % (what or "lrb200 call", last_error()))


def check_handle(h, what):
    if not h:
        raise LibraryError("Creating %s: %s" % (what, last_error()))
    return h


def require_device(device=None):
    """Initialise the library; raises LibraryError (loudly) when no GPU is usable.  Without an argument the device the
    process already selected (an earlier require_device(n), e.g. one rank per GPU) is kept -- re-initialising on device 0
    would move the library stream and leave every existing handle on the wrong GPU; an explicit `device` switches."""
    lib = load()
    if device is None:
        cur = lib.lrb200_current_device()
        if cur >= 0:
            return lib
        device = 0
    check(lib.lrb200_init(device), "lrb200_init(%d)" % device)
    return lib
