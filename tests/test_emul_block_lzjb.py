"""MTZ_FLAG_BLOCK_LZJB on the CPU: the cases of tests/test_gpu_block_lzjb.py run against the whole
library built for the SIMT emulator (tests/emul/make_emul_lib.py: the device code of
kernels_lzjb.cuh and kernels_frames.cuh and the library's launch sites, unchanged), including the
device API across the emulated build's sub-batch edge (700 records).  Test infrastructure only."""
import pytest

import test_gpu_block_lzjb as S
from test_emul_block_cksum import HostMem, emul_library  # noqa: F401  (fixture)

KEYS = S.test_lzjb_and_zle_keys_match_the_encoders_in_verify
CASES = [
    ("keys-512-9", KEYS, (512, 9, False)),
    ("keys-8192-9", KEYS, (8192, 9, False)),
    ("keys-8192-9-frames", KEYS, (8192, 9, True)),
    ("keys-8192-12", KEYS, (8192, 12, False)),
    ("keys-131072-12-frames", KEYS, (131072, 12, True)),
    ("output_and_stats", S.test_the_output_and_the_stats_are_those_of_the_flag_off, ()),
    ("einval", S.test_the_flag_without_block_checksums_is_einval, ()),
    ("swapped_keys", S.test_swapped_keys_are_counted_not_errors, ()),
    ("corrupted_then_restamped", S.test_corrupted_then_restamped_records, ()),
    ("sha256_keys", S.test_sha256_and_sha512_keys, ("sha256",)),
    ("sha512_keys", S.test_sha256_and_sha512_keys, ("sha512",)),
    ("send_c-verify", S.test_send_c_stream_frames_checked_as_they_arrive, ("verify",)),
    ("send_c-recompress", S.test_send_c_stream_frames_checked_as_they_arrive, ("recompress",)),
    ("compress_decompress", S.test_compress_and_decompress_are_unchanged, ()),
    ("ring_api-4093", S.test_ring_api, (4093,)),
    ("ring_api-1MiB", S.test_ring_api, (1 << 20,)),
    ("deferred_shards", S.test_deferred_shards, ()),
]


@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_block_lzjb_case_on_the_emulated_library(emul_library, oracle, name):  # noqa: F811
    fn, args = {c[0]: (c[1], c[2]) for c in CASES}[name]
    fn(oracle, *args)


def test_device_api_across_the_emulated_subbatch_edge(emul_library, oracle):  # noqa: F811
    S.device_api_subbatched(oracle, HostMem(), 1500)
