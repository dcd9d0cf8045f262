"""MTZ_FLAG_BLOCK_FRAMES on the CPU: the cases of tests/test_gpu_block_frames.py run against the whole
library built for the SIMT emulator (tests/emul/make_emul_lib.py: the device code of
kernels_frames.cuh, K3 and the library's launch sites, unchanged), including the device API across the
emulated build's sub-batch edge (700 records).  Test infrastructure only."""
import pytest

import test_gpu_block_frames as S
from test_emul_block_cksum import HostMem, emul_library  # noqa: F401  (fixture)

LZ4 = S.test_lz4_on_disk_keys_match_the_encoder_in_verify
CASES = [
    ("lz4_on_disk-9-512", LZ4, (9, 512)),
    ("lz4_on_disk-9-8192", LZ4, (9, 8192)),
    ("lz4_on_disk-12-8192", LZ4, (12, 8192)),
    ("lz4_on_disk-12-131072", LZ4, (12, 131072)),
    ("output_and_stats", S.test_the_output_and_the_stats_are_those_of_the_flag_off, ()),
    ("einval", S.test_the_flag_without_block_checksums_is_einval, ()),
    ("swapped_frame_keys", S.test_swapped_frame_keys_are_counted_not_errors, ()),
    ("corrupted_then_restamped", S.test_corrupted_then_restamped_records, ()),
    ("sha_keys-9", S.test_sha256_and_sha512_lz4_on_disk_keys, (9,)),
    ("sha_keys-12", S.test_sha256_and_sha512_lz4_on_disk_keys, (12,)),
    ("send_c", S.test_send_c_stream_the_flag_changes_nothing, ()),
    ("other_modes", S.test_the_other_modes_are_unchanged, ()),
    ("ring_api-4093", S.test_ring_api, (4093,)),
    ("ring_api-1MiB", S.test_ring_api, (1 << 20,)),
    ("deferred_shards", S.test_deferred_shards, ()),
]


@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_block_frames_case_on_the_emulated_library(emul_library, oracle, name):  # noqa: F811
    fn, args = {c[0]: (c[1], c[2]) for c in CASES}[name]
    fn(oracle, *args)


def test_device_api_across_the_emulated_subbatch_edge(emul_library, oracle):  # noqa: F811
    S.device_api_subbatched(oracle, HostMem(), 1500)
