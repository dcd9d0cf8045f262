"""MTZ_FLAG_BLOCK_SHA512 on the CPU: the cases of tests/test_gpu_block_sha512.py run against the whole
library built for the SIMT emulator (tests/emul/make_emul_lib.py: the device code of
kernels_sha512.cuh and the library's launch sites, unchanged), including the device API across the
emulated build's codec sub-batch edge (700 records).  Test infrastructure only."""
import pytest

import test_gpu_block_sha512 as S
from test_emul_block_cksum import HostMem, emul_library  # noqa: F401  (fixture)

MIXED = S.test_one_stream_mixing_fletcher4_sha256_sha512_and_skipped_keys
CASES = [
    ("every_mode", S.test_sha512_keys_match_in_every_mode, ()),
    ("corrupted_then_restamped", S.test_corrupted_then_restamped_block_fails_only_with_the_flag, ()),
    ("relabelled_keys", S.test_relabelled_keys_are_mismatches, ()),
    ("other_messages", S.test_fletcher4_and_sha256_failure_messages_are_unchanged, ()),
    ("lz4_on_disk-9", S.test_lz4_on_disk_sha512_keys, (9,)),
    ("lz4_on_disk-12", S.test_lz4_on_disk_sha512_keys, (12,)),
    ("swapped_frame_keys", S.test_swapped_frame_keys_are_counted_not_errors, ()),
    ("mixed_types-neither", MIXED, (False, False)),
    ("mixed_types-sha256", MIXED, (True, False)),
    ("mixed_types-sha512", MIXED, (False, True)),
    ("mixed_types-both", MIXED, (True, True)),
    ("record_size-512", S.test_record_sizes, (512,)),
    ("record_size-8192", S.test_record_sizes, (8192,)),
    ("record_size-131072", S.test_record_sizes, (131072,)),
    ("record_size-1MiB", S.test_record_sizes, (1 << 20,)),
    ("sixteen_mib_record", S.test_sixteen_mib_record, ()),
    ("precedence", S.test_first_failing_record_in_stream_order_is_reported, ()),
    ("ring_api-4093", S.test_ring_api, (4093,)),
    ("ring_api-1MiB", S.test_ring_api, (1 << 20,)),
    ("deferred_shards", S.test_deferred_shards, ()),
    ("einval", S.test_the_flag_without_block_checksums_is_einval, ()),
    ("flag_changes_nothing", S.test_the_flag_changes_nothing_without_sha512_keys, ()),
]


@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_block_sha512_case_on_the_emulated_library(emul_library, oracle, name):  # noqa: F811
    fn, args = {c[0]: (c[1], c[2]) for c in CASES}[name]
    fn(oracle, *args)


def test_device_api_across_the_emulated_subbatch_edge(emul_library, oracle):  # noqa: F811
    S.device_api_subbatched(oracle, HostMem(), 1500)
