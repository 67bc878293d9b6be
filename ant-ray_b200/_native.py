"""ctypes binding of the C-ABI in include/b200coll.h (libb200coll.so, built in-tree).

This is the only place Python touches the native library.  It mirrors the call shape the
reference uses for cupy's NcclCommunicator (raw integer pointers, element counts, NCCL enum
values, raw stream pointer: nccl_collective_group.py:181-188).  There is deliberately no
fallback: if the library is missing, loading raises ImportError.
"""
import ctypes
import os
from ctypes import (POINTER, Structure, byref, c_char_p, c_float, c_int, c_int32, c_size_t, c_uint8,
                    c_uint32, c_uint64, c_void_p)

_LIB_NAME = "libb200coll.so"
_lib = None


class B200CollError(RuntimeError):
    """Native call failed.  `.status` holds the b200c_status_t code."""

    def __init__(self, status, message):
        super().__init__(message)
        self.status = status

    def __reduce__(self):  # keep (status, message) across process boundaries (Ray / test actors)
        return (B200CollError, (self.status, self.args[0] if self.args else ""))


# b200c_status_t
OK, EINVAL, ECUDA, ESTATE, EUNSUPPORTED, ETIMEOUT, EABORTED, EMISMATCH, ENOMEM = 0, -1, -2, -3, -4, -5, -6, -7, -8
# b200c_dtype_t (ncclDataType_t numbering)
INT8, UINT8, INT32, UINT32, INT64, UINT64, FLOAT16, FLOAT32, FLOAT64, BFLOAT16 = range(10)
# b200c_redop_t (ncclRedOp_t numbering)
SUM, PROD, MAX, MIN, AVG = range(5)
# b200c_algo_t
ALGO_AUTO, ALGO_ONESHOT, ALGO_TWOSHOT, ALGO_NVLS, ALGO_NVLS_PIPE, ALGO_LL, ALGO_NVLS_LANES, ALGO_NVLS_STREAMS = range(8)
# b200c_share_mode_t
SHARE_VMM_FD, SHARE_LEGACY_IPC = 0, 1
# b200c_act_t: the activation of a b200c_bn_*_act site
ACT_RELU6, ACT_SILU, ACT_HARDSWISH = 1, 2, 3
MAX_RANKS = 8


class Config(Structure):
    _fields_ = [("struct_size", c_uint32), ("share_mode", c_int32), ("staging_bytes", c_uint64),
                ("symmetric_bytes", c_uint64), ("p2p_slot_bytes", c_uint64), ("p2p_slots", c_uint32),
                ("max_blocks", c_uint32), ("oneshot_max_bytes", c_uint64), ("nvls_min_bytes", c_uint64),
                ("nvls_pipe_min_bytes", c_uint64), ("timeout_ms", c_uint64), ("granule_bytes", c_uint64),
                ("ll_max_bytes", c_uint64), ("bcast_rounds_min_bytes", c_uint64), ("nvls_blocks", c_uint32),
                ("nvls_lanes", c_uint32), ("lane_granule_bytes", c_uint64), ("nvls_lanes_min_bytes", c_uint64),
                ("nvls_unroll", c_uint32), ("rounds_order", c_uint32), ("nvls_streams_min_bytes", c_uint64),
                ("nvls_streams_piece_bytes", c_uint64)]


class Props(Structure):
    _fields_ = [("device", c_int32), ("sm_count", c_int32), ("cc_major", c_int32), ("cc_minor", c_int32),
                ("vmm_supported", c_int32), ("posix_fd_supported", c_int32), ("multicast_supported", c_int32),
                ("reserved", c_int32), ("total_mem", c_uint64)]


class Export(Structure):
    _fields_ = [("share_mode", c_int32), ("fd", c_int32), ("arena_bytes", c_uint64), ("layout_hash", c_uint64),
                ("pid", c_int32), ("device_uuid_lo", c_int32), ("ipc", c_uint8 * 64)]


# name -> (restype, argtypes).  Every symbol include/b200coll.h declares is listed here; the
# CPU test-suite checks the two stay in sync.
SYMBOLS = {
    "b200c_version": (c_int, []),
    "b200c_last_error": (c_char_p, []),
    "b200c_status_string": (c_char_p, [c_int]),
    "b200c_dtype_size": (c_size_t, [c_int]),
    "b200c_device_props": (c_int, [c_int, POINTER(Props)]),
    "b200c_default_config": (None, [POINTER(Config)]),
    "b200c_comm_create": (c_int, [c_int, c_int, c_int, POINTER(Config), POINTER(c_void_p)]),
    "b200c_comm_export": (c_int, [c_void_p, POINTER(Export)]),
    "b200c_comm_import": (c_int, [c_void_p, c_int, POINTER(Export)]),
    "b200c_comm_mc_create": (c_int, [c_void_p, POINTER(c_int)]),
    "b200c_comm_mc_import": (c_int, [c_void_p, c_int]),
    "b200c_comm_mc_add_device": (c_int, [c_void_p]),
    "b200c_comm_mc_bind": (c_int, [c_void_p]),
    "b200c_comm_mc_disable": (c_int, [c_void_p]),
    "b200c_comm_ready": (c_int, [c_void_p]),
    "b200c_comm_abort": (c_int, [c_void_p]),
    "b200c_comm_destroy": (c_int, [c_void_p]),
    "b200c_comm_check": (c_int, [c_void_p]),
    "b200c_comm_rank": (c_int, [c_void_p]),
    "b200c_comm_world": (c_int, [c_void_p]),
    "b200c_comm_has_multicast": (c_int, [c_void_p]),
    "b200c_comm_seq": (c_uint64, [c_void_p]),
    "b200c_comm_symmetric_base": (c_void_p, [c_void_p]),
    "b200c_comm_symmetric_bytes": (c_uint64, [c_void_p]),
    "b200c_pool_bind": (c_int, [c_void_p]),
    "b200c_pool_malloc": (c_void_p, [c_size_t, c_int, c_void_p]),
    "b200c_pool_free": (None, [c_void_p, c_size_t, c_int, c_void_p]),
    "b200c_allreduce": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_int, c_int, c_int, c_void_p]),
    "b200c_allreduce_scaled": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_int, c_int, c_float, c_int, c_void_p]),
    "b200c_reduce": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_int, c_int, c_int, c_void_p]),
    "b200c_broadcast": (c_int, [c_void_p, c_void_p, c_size_t, c_int, c_int, c_void_p]),
    "b200c_allgather": (c_int, [c_void_p, c_void_p, POINTER(c_void_p), c_size_t, c_int, c_void_p]),
    "b200c_reducescatter": (c_int, [c_void_p, POINTER(c_void_p), c_void_p, c_size_t, c_int, c_int, c_void_p]),
    "b200c_reducescatter_scaled": (c_int, [c_void_p, POINTER(c_void_p), c_void_p, c_size_t, c_int, c_int, c_float, c_void_p]),
    "b200c_send": (c_int, [c_void_p, c_void_p, c_size_t, c_int, c_void_p]),
    "b200c_recv": (c_int, [c_void_p, c_void_p, c_size_t, c_int, c_void_p]),
    "b200c_send_multi": (c_int, [c_void_p, c_void_p, c_size_t, POINTER(c_int), c_int, c_void_p]),
    "b200c_recv_multi": (c_int, [c_void_p, c_void_p, c_size_t, c_int, c_void_p]),
    "b200c_barrier": (c_int, [c_void_p, c_void_p]),
    "b200c_debug_fill_flags": (c_int, [c_void_p, c_uint32]),
    "b200c_bn_scratch_bytes": (c_size_t, [c_int]),
    "b200c_bn_forward": (c_int, [c_void_p] * 10 + [c_int, c_int, c_float, c_float, c_void_p, c_void_p]),
    "b200c_bn_forward_mask": (c_int, [c_void_p] * 11 + [c_int, c_int, c_float, c_float, c_void_p, c_void_p]),
    "b200c_bn_backward": (c_int, [c_void_p] * 10 + [c_int, c_int, c_void_p, c_void_p]),
    "b200c_bn_backward_mask": (c_int, [c_void_p] * 11 + [c_int, c_int, c_void_p, c_void_p]),
    "b200c_bn_dual_scratch_bytes": (c_size_t, [c_int]),
    "b200c_bn_forward_dual": (c_int, [c_void_p] * 11 + [c_float, c_float] + [c_void_p] * 7 + [c_float, c_float, c_int, c_int, c_void_p, c_void_p]),
    "b200c_bn_backward_dual": (c_int, [c_void_p] * 18 + [c_int, c_int, c_void_p, c_void_p]),
    "b200c_bn_forward_pool": (c_int, [c_void_p] * 10 + [c_int] * 4 + [c_float, c_float, c_void_p, c_void_p]),
    "b200c_bn_backward_pool": (c_int, [c_void_p] * 10 + [c_int] * 4 + [c_void_p, c_void_p]),
    "b200c_bn_infer": (c_int, [c_void_p] * 7 + [c_int, c_float, c_int, c_int, c_void_p]),
    "b200c_bn_infer_dual": (c_int, [c_void_p] * 7 + [c_float] + [c_void_p] * 4 + [c_float, c_int, c_int, c_int, c_void_p]),
    "b200c_bn_infer_pool": (c_int, [c_void_p] * 6 + [c_int, c_float] + [c_int] * 4 + [c_void_p]),
    "b200c_bn_forward_pool2": (c_int, [c_void_p] * 10 + [c_int] * 4 + [c_float, c_float, c_void_p, c_void_p]),
    "b200c_bn_backward_pool2": (c_int, [c_void_p] * 9 + [c_int] * 4 + [c_void_p, c_void_p]),
    "b200c_bn_infer_pool2": (c_int, [c_void_p] * 6 + [c_int, c_float] + [c_int] * 4 + [c_void_p]),
    "b200c_bn_forward_act": (c_int, [c_void_p] * 9 + [c_int, c_int, c_int, c_float, c_float, c_void_p, c_void_p]),
    "b200c_bn_backward_act": (c_int, [c_void_p] * 10 + [c_int, c_int, c_int, c_void_p, c_void_p]),
    "b200c_bn_infer_act": (c_int, [c_void_p] * 6 + [c_int, c_float, c_int, c_int, c_int, c_void_p]),
    "b200c_bn_forward_res": (c_int, [c_void_p] * 3 + [c_int] + [c_void_p] * 8 + [c_int, c_int, c_float, c_float, c_void_p, c_void_p]),
    "b200c_bn_backward_res": (c_int, [c_void_p] * 2 + [c_int] + [c_void_p] * 8 + [c_int, c_int, c_void_p, c_void_p]),
    "b200c_bn_infer_res": (c_int, [c_void_p] * 7 + [c_int, c_float, c_int, c_int, c_void_p]),
    "b200c_bn_forward_cat": (c_int, [POINTER(c_void_p), POINTER(c_int), c_int] + [c_void_p] * 9 + [c_int, c_int, c_float, c_float, c_void_p,
                                                                                              c_void_p]),
    "b200c_bn_backward_cat": (c_int, [c_void_p] * 2 + [POINTER(c_void_p), POINTER(c_int), c_int] + [c_void_p] * 6 + [c_int, c_int, c_void_p,
                                                                                                                  c_void_p]),
    "b200c_bn_infer_cat": (c_int, [POINTER(c_void_p), POINTER(c_int), c_int] + [c_void_p] * 5 + [c_int, c_float, c_int, c_int, c_void_p]),
    "b200c_bn_forward_slice": (c_int, [c_void_p, c_void_p, c_int] + [c_void_p] * 8 + [c_int, c_int, c_float, c_float, c_void_p, c_void_p]),
    "b200c_bn_backward_slice": (c_int, [c_void_p, c_int] + [c_void_p] * 8 + [c_int, c_int, c_void_p, c_void_p]),
    "b200c_bn_infer_slice": (c_int, [c_void_p, c_void_p, c_int] + [c_void_p] * 4 + [c_int, c_float, c_int, c_int, c_void_p]),
    "b200c_bn_shuffle_mask_bytes": (c_size_t, [c_int, c_int]),
    "b200c_bn_forward_shuffle": (c_int, [c_void_p, c_int] + [c_void_p] * 9 + [c_float, c_float] + [c_void_p] * 9
                                 + [c_float, c_float, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "b200c_bn_backward_shuffle": (c_int, [c_void_p] * 17 + [c_int, c_int, c_void_p, c_void_p]),
    "b200c_bn_infer_shuffle": (c_int, [c_void_p, c_int] + [c_void_p] * 5 + [c_float] + [c_void_p] * 5
                               + [c_float, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "b200c_se_scratch_bytes": (c_size_t, [c_int, c_int, c_int]),
    "b200c_se_pool": (c_int, [c_void_p] * 2 + [c_int] * 3 + [c_void_p, c_size_t, c_void_p]),
    "b200c_se_scale": (c_int, [c_void_p] * 3 + [c_int] * 3 + [c_void_p]),
    "b200c_se_backward_reduce": (c_int, [c_void_p] * 3 + [c_int] * 3 + [c_void_p, c_size_t, c_void_p]),
    "b200c_se_backward_elemt": (c_int, [c_void_p] * 4 + [c_int] * 3 + [c_void_p]),
    "b200c_bn_sync_scratch_bytes": (c_size_t, [c_int, c_int]),
    "b200c_bn_sync_forward": (c_int, [c_void_p] * 5 + [c_int] + [c_void_p] * 8 + [c_int, c_int, c_float, c_float, c_void_p, c_void_p]),
    "b200c_bn_sync_backward": (c_int, [c_void_p] * 5 + [c_int] + [c_void_p] * 9 + [c_int, c_int, c_void_p, c_void_p]),
    "b200c_launch_count": (c_uint64, []),
}


def library_path():
    override = os.environ.get("B200COLL_LIBRARY")
    if override:
        return override
    return os.path.join(os.path.dirname(os.path.abspath(__file__)), _LIB_NAME)


def load():
    """Load libb200coll.so once; raise ImportError if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    path = library_path()
    if not os.path.exists(path):
        raise ImportError(
            f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  ant_ray_b200 has no CPU or NCCL fallback.")
    lib = ctypes.CDLL(path, mode=ctypes.RTLD_LOCAL)
    for name, (restype, argtypes) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError here means header and library disagree
        fn.restype = restype
        fn.argtypes = argtypes
    if lib.b200c_version() < 200:
        raise ImportError("libb200coll.so is older than this Python package")
    _lib = lib
    return lib


def last_error():
    msg = load().b200c_last_error()
    return msg.decode(errors="replace") if msg else ""


def check(status):
    if status != OK:
        raise B200CollError(status, f"b200coll: {last_error()} (status {status})")


def default_config():
    cfg = Config()
    load().b200c_default_config(byref(cfg))
    return cfg


def device_props(device):
    p = Props()
    check(load().b200c_device_props(device, byref(p)))
    return p


def launch_count():
    return int(load().b200c_launch_count())
