"""ctypes binding of libmanatee_gpu.so (include/manatee_gpu.h).

The library is the product: if it is missing this module raises, loudly.  There
is no CPU fallback anywhere in ``manatee_b200`` (the CPU oracle lives under
``oracle/`` and is test infrastructure only).
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# MTZ_SO: load another build of the SAME library (kernel A/B experiments); default in-tree
SO_PATH = os.environ.get("MTZ_SO") or os.path.join(_HERE, "libmanatee_gpu.so")

OK, EINVAL, EAGAIN, ECUDA, EFORMAT, ECKSUM, ECODEC, ENOSPC, ENOMEM, EOF, ENOGPU, ECANCELED = \
    0, -1, -2, -3, -4, -5, -6, -7, -8, -9, -10, -11
MAX_DEVICES, MAX_PEERS = 16, 16
MODE_VERIFY, MODE_COMPRESS, MODE_DECOMPRESS, MODE_RECOMPRESS, MODE_PASSTHROUGH = 0, 1, 2, 3, 4
FLAG_DEFER_VERIFY = 1
FLAG_REENCODE_ALL = 2
FLAG_BLOCK_CKSUM = 4
FLAG_BLOCK_SHA256 = 8
FLAG_BLOCK_SHA512 = 16
FLAG_BLOCK_FRAMES = 32
FLAG_BLOCK_LZJB = 64
FLAG_BLOCK_LOGICAL = 128
XCHG_FIRST, XCHG_LAST = 1, 2
MODE_NAMES = {"verify": 0, "compress": 1, "decompress": 2, "recompress": 3, "passthrough": 4}


class MtzError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("libmanatee_gpu: %s (%d)" % (msg, code))
        self.code = code


class Config(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("device", C.c_int32), ("mode", C.c_uint32),
                ("flags", C.c_uint32), ("ring_bytes", C.c_uint64), ("out_ring_bytes", C.c_uint64),
                ("batch_bytes", C.c_uint64), ("record_bytes", C.c_uint32), ("n_slots", C.c_uint32),
                ("n_devices", C.c_uint32), ("devices", C.c_int32 * 16)]


class Stats(C.Structure):
    _fields_ = [("bytes_in", C.c_uint64), ("bytes_out", C.c_uint64), ("records", C.c_uint64),
                ("write_records", C.c_uint64), ("lz4_decoded", C.c_uint64),
                ("lz4_encoded", C.c_uint64), ("batches", C.c_uint64), ("bad_record", C.c_uint64),
                ("kernel_launches", C.c_uint64), ("gpu_ms", C.c_double), ("end_seen", C.c_uint64),
                ("k1_ms", C.c_double), ("codec_ms", C.c_double), ("k1_launches", C.c_uint64),
                ("k3_ms", C.c_double), ("k3_launches", C.c_uint64),
                ("lz4_certified", C.c_uint64)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class BlockStats(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("pad", C.c_uint32), ("logical_ok", C.c_uint64),
                ("frame_ok", C.c_uint64), ("frame_miss", C.c_uint64), ("skipped", C.c_uint64),
                ("first_frame_miss", C.c_uint64), ("sha256", C.c_uint64),
                ("sha512", C.c_uint64), ("frames_encoded", C.c_uint64),
                ("lzjb_encoded", C.c_uint64), ("zle_encoded", C.c_uint64),
                ("logical_checked", C.c_uint64)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_[2:]}


class Rec(C.Structure):
    _fields_ = [("off", C.c_uint64), ("payload", C.c_uint32), ("type", C.c_uint32),
                ("lsize", C.c_uint32), ("comp", C.c_uint32), ("resv", C.c_uint64)]


# every symbol include/manatee_gpu.h declares; tests/test_abi.py cross-checks the header
SYMBOLS = [
    "mtz_abi_version", "mtz_device_count", "mtz_open", "mtz_close", "mtz_last_error",
    "mtz_strerror", "mtz_ring_acquire", "mtz_ring_commit", "mtz_write", "mtz_flush",
    "mtz_out_peek", "mtz_out_consume", "mtz_read", "mtz_event_fd", "mtz_get_stats",
    "mtz_get_block_stats", "mtz_end_checksum", "mtz_host_alloc", "mtz_host_free", "mtz_process_host",
    "mtz_index_host", "mtz_dev_index", "mtz_dev_submit", "mtz_dev_aggregate",
    "mtz_dev_finish", "mtz_dev_reset", "mtz_dev_aggregate_async", "mtz_dev_finish_gathered", "mtz_set_carry",
    "mtz_k_lz4_decode", "mtz_k_lz4_encode",
    "mtz_fanout_attach", "mtz_out_peek_peer", "mtz_out_consume_peer", "mtz_read_peer", "mtz_cancel",
    "mtz_comm_unique_id", "mtz_comm_init", "mtz_comm_share", "mtz_dev_finish_exchange",
]

_lib = None


def lib():
    """Load libmanatee_gpu.so; raise if it has not been built (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(SO_PATH):
        raise ImportError(
            "libmanatee_gpu.so is not built: run `python -c 'import __graft_entry__ as g; "
            "g.build()'` (there is no CPU fallback for the snapshot stage)")
    # The library binds NCCL at run time (csrc/mtz_nccl.h).  In a Python process that will also
    # import torch, point it at the libnccl torch bundles: torch cannot import behind an older
    # libnccl.so.2 that somebody else loaded first under the same SONAME.
    if "MTZ_NCCL_LIB" not in os.environ:
        try:
            import importlib.util
            spec = importlib.util.find_spec("nvidia.nccl")
            for d in (spec.submodule_search_locations or []) if spec else []:
                cand = os.path.join(d, "lib", "libnccl.so.2")
                if os.path.exists(cand):
                    os.environ["MTZ_NCCL_LIB"] = cand
                    break
        except Exception:
            pass
    L = C.CDLL(SO_PATH)
    vp, sz, i32, u64 = C.c_void_p, C.c_size_t, C.c_int32, C.c_uint64
    H = vp
    L.mtz_abi_version.restype = i32
    L.mtz_device_count.restype = i32
    L.mtz_open.argtypes = [C.POINTER(Config), C.POINTER(H)]
    L.mtz_close.argtypes = [H]
    L.mtz_last_error.argtypes = [H]; L.mtz_last_error.restype = C.c_char_p
    L.mtz_strerror.argtypes = [i32]; L.mtz_strerror.restype = C.c_char_p
    L.mtz_ring_acquire.argtypes = [H, sz, C.POINTER(vp), C.POINTER(sz)]
    L.mtz_ring_commit.argtypes = [H, sz]
    L.mtz_write.argtypes = [H, vp, sz, i32]
    L.mtz_flush.argtypes = [H]
    L.mtz_out_peek.argtypes = [H, C.POINTER(vp), C.POINTER(sz)]
    L.mtz_out_consume.argtypes = [H, sz]
    L.mtz_read.argtypes = [H, vp, sz, C.POINTER(sz), i32]
    L.mtz_event_fd.argtypes = [H]
    L.mtz_get_stats.argtypes = [H, C.POINTER(Stats)]
    L.mtz_get_block_stats.argtypes = [H, C.POINTER(BlockStats)]
    L.mtz_end_checksum.argtypes = [H, C.POINTER(u64 * 4)]
    L.mtz_host_alloc.argtypes = [sz, C.POINTER(vp)]
    L.mtz_host_free.argtypes = [vp]
    L.mtz_process_host.argtypes = [H, vp, sz, vp, sz, C.POINTER(sz)]
    L.mtz_index_host.argtypes = [vp, sz, vp, sz, C.POINTER(sz), C.POINTER(sz)]
    L.mtz_dev_index.argtypes = [H, vp, sz, vp, sz, C.POINTER(sz), C.POINTER(sz), vp]
    L.mtz_dev_submit.argtypes = [H, vp, sz, vp, sz, vp, sz, vp]
    L.mtz_dev_aggregate.argtypes = [H, C.POINTER(u64 * 5)]
    L.mtz_dev_finish.argtypes = [H, vp, vp, C.POINTER(sz), C.POINTER(u64 * 4), C.POINTER(u64 * 4)]
    L.mtz_dev_reset.argtypes = [H]
    L.mtz_dev_aggregate_async.argtypes = [H, vp]
    L.mtz_dev_finish_gathered.argtypes = [H, vp, C.c_uint32, vp, C.POINTER(sz), C.POINTER(u64 * 4),
                                          C.POINTER(u64 * 4)]
    L.mtz_set_carry.argtypes = [H, vp, vp]
    L.mtz_fanout_attach.argtypes = [H, i32]
    L.mtz_out_peek_peer.argtypes = [H, i32, C.POINTER(vp), C.POINTER(sz)]
    L.mtz_out_consume_peer.argtypes = [H, i32, sz]
    L.mtz_read_peer.argtypes = [H, i32, vp, sz, C.POINTER(sz), i32]
    L.mtz_cancel.argtypes = [H]
    L.mtz_comm_unique_id.argtypes = [vp]
    L.mtz_comm_init.argtypes = [H, vp, i32, i32]
    L.mtz_comm_share.argtypes = [H, H]
    L.mtz_dev_finish_exchange.argtypes = [H, vp, C.c_uint32, C.POINTER(sz), C.POINTER(u64 * 4),
                                          C.POINTER(u64 * 4), C.POINTER(u64 * 4)]
    L.mtz_k_lz4_decode.argtypes = [H, vp, vp, vp, C.c_uint32, vp]
    L.mtz_k_lz4_encode.argtypes = [H, vp, vp, vp, C.c_uint32, vp]
    for s in SYMBOLS:
        getattr(L, s).restype = getattr(L, s).restype if s in (
            "mtz_last_error", "mtz_strerror") else i32
    _lib = L
    return L
