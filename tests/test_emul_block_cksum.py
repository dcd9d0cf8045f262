"""MTZ_FLAG_BLOCK_CKSUM on the CPU: the cases of tests/test_gpu_block_cksum.py run against the whole
library built for the SIMT emulator (tests/emul/make_emul_lib.py: the device code of
kernels_block.cuh and the library's launch sites, unchanged), including the device API across the
emulated build's codec sub-batch edge (700 records).  Test infrastructure only."""
import numpy as np
import pytest

import test_gpu_block_cksum as B


@pytest.fixture(scope="module")
def emul_library(emul_so):
    from manatee_b200 import _native as N
    saved = (N.SO_PATH, N._lib)
    N.SO_PATH, N._lib = emul_so, None
    try:
        yield N.lib()
    finally:
        N.SO_PATH, N._lib = saved


CASES = [
    ("raw_stream", B.test_raw_stream_every_block_matches_in_every_mode, ()),
    ("corrupted_then_restamped", B.test_corrupted_then_restamped_block_fails_only_with_the_flag, ()),
    ("flipped_key_bit", B.test_flipped_key_bit_fails, ()),
    ("lz4_on_disk-9-8192", B.test_lz4_on_disk_keys_match_the_encoder, (9, 8192)),
    ("lz4_on_disk-12-8192", B.test_lz4_on_disk_keys_match_the_encoder, (12, 8192)),
    ("frame_miss", B.test_frame_miss_is_counted_not_an_error, ()),
    ("send_c-9", B.test_send_c_stream_frames_checked_on_input, (9,)),
    ("send_c-12", B.test_send_c_stream_frames_checked_on_input, (12,)),
    ("skipped_classes", B.test_unverifiable_keys_are_skipped, ()),
    ("passthrough_einval", B.test_passthrough_with_the_flag_is_einval, ()),
    ("precedence", B.test_first_failing_record_in_stream_order_is_reported, ()),
    ("flag_changes_nothing", B.test_the_flag_changes_no_byte_and_no_stats_field, ()),
    ("ring_api-4093", B.test_ring_api, (4093,)),
    ("ring_api-1MiB", B.test_ring_api, (1 << 20,)),
    ("deferred_shards", B.test_deferred_shards, ()),
]


@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_block_cksum_case_on_the_emulated_library(emul_library, oracle, name):
    fn, args = {c[0]: (c[1], c[2]) for c in CASES}[name]
    fn(oracle, *args)


class HostMem(object):
    """device buffers for the emulated library: host memory is device memory there"""

    def put(self, a):
        a = np.ascontiguousarray(a).copy()
        return a, a.ctypes.data

    def zeros(self, n):
        a = np.zeros(n, dtype=np.uint8)
        return a, a.ctypes.data

    def get(self, a, n):
        return a[:n].copy()


def test_device_api_across_the_emulated_subbatch_edge(emul_library, oracle):
    B.device_api_subbatched(oracle, HostMem(), 1500)
