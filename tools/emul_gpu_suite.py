#!/usr/bin/env python
"""Runs the gpu-marked parity tests against the WHOLE library built for the SIMT emulator
(tests/emul/make_emul_lib.py), on the CPU: the torch-free ones as they are, the ones that hold
device buffers in torch.cuda tensors with tests/emul/fake_torch.py standing in for torch (device
memory is host memory there).  One-off validation tool (minutes); the fast subset of the same
thing is part of the suite (tests/test_emul_library.py).
usage: tools/emul_gpu_suite.py [lib.so] [substring filter]"""
import inspect
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))
import fake_torch  # noqa: E402

sys.modules["torch"] = fake_torch                          # before anything imports torch

PARAMS = {
    "test_verify_end_checksum_matches_oracle": [(0, 131072), (1, 131072), (5, 512), (33, 4096), (64, 131072),
                                                (3, 1 << 20), (300, 131072)],
    "test_verify_batching_invariance": [(1 << 20,), (3 << 20,), (32 << 20,)],
    "test_corruption_reports_same_record_as_oracle": [("payload",), ("header",), ("embedded",), ("end",)],
    "test_verify_stream_identity": [(1 << 16,), (4093,), (1 << 20,), (7 << 20,)],
    "test_compress_matches_oracle": [(0,), (1 << 20,), (5 << 20,)],
    "test_transport_identity_compress_then_decompress": [(4096,), (65536,), (131072,), (1 << 20,)],
    "test_randomized_streams_all_modes": [(1,), (2,), (3,), (4,)],
    "test_lz4_on_disk_keys_match_the_encoder": [(9, 8192), (12, 8192), (12, 65536)],
    "test_send_c_stream_frames_checked_on_input": [(9,), (12,)],
    "test_ring_api": [(4093,), (1 << 20,)],
    "test_lz4_on_disk_sha256_keys": [(9,), (12,)],
    "test_record_sizes": [(512,), (8192,), (131072,), (1 << 20,)],
    "test_lz4_on_disk_sha512_keys": [(9,), (12,)],
    "test_one_stream_mixing_fletcher4_sha256_sha512_and_skipped_keys": [(False, False), (True, False),
                                                                        (False, True), (True, True)],
    "test_lz4_on_disk_keys_match_the_encoder_in_verify": [(9, 512), (9, 8192), (12, 8192), (12, 131072)],
    "test_sha256_and_sha512_lz4_on_disk_keys": [(9,), (12,)],
    "test_lzjb_and_zle_keys_match_the_encoders_in_verify": [(512, 9, False), (8192, 9, False), (8192, 12, True),
                                                            (131072, 9, True)],
    "test_sha256_and_sha512_keys": [("sha256",), ("sha512",)],
    "test_send_c_stream_frames_checked_as_they_arrive": [("verify",), ("recompress",)],
    "test_the_compressed_wire_counts_what_verify_counts": [(dict(sha256=False, sha512=False, lzjb=False),),
                                                           (dict(sha256=True, sha512=True, lzjb=True),)],
    "test_a_corrupted_raw_keyed_lz4_record_fails_the_recompress_relay": [("fletcher4",), ("sha256",), ("sha512",)],
}
SKIP = {"test_sixteen_mib_record": "16 MiB blocks take minutes per encode on the emulator",
        "test_size_independent_properties_at_2gib": "2 GiB of LZ4 work is out of reach for the emulator",
        "test_device_api_across_the_subbatch_edge": "66 000 records; tests/test_emul_block_cksum.py crosses the "
                                                    "emulated build's 700-record edge instead",
        "test_deferred_codec_shards": "its device buffers are torch tensors; tests/test_emul_block_logical.py runs it "
                                      "on host memory",
        "test_device_group": "needs two GPUs",
        "test_real_streams_with_lzjb_or_zle_keys": "tests/golden/real holds no stream with lzjb or zle keys"}


def main():
    so = sys.argv[1] if len(sys.argv) > 1 and sys.argv[1].endswith(".so") else None
    filt = sys.argv[-1] if len(sys.argv) > 1 and not sys.argv[-1].endswith(".so") else ""
    if so is None:
        so = os.path.join(tempfile.mkdtemp(prefix="emul_suite"), "libmanatee_gpu_emul.so")
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "emul", "make_emul_lib.py"), so])
        assert r.returncode == 0
    import oracle as O
    from manatee_b200 import _native as N
    N.SO_PATH, N._lib = so, None
    import test_gpu_block_cksum as B
    import test_gpu_block_sha256 as H
    import test_gpu_block_sha512 as W
    import test_gpu_block_frames as F
    import test_gpu_block_lzjb as J
    import test_gpu_block_logical as L
    import test_gpu_codec as K
    import test_gpu_lz4 as Z
    import test_gpu_stream as S
    import test_gpu_verify as V
    tot = fail = 0
    for mod in (V, S, Z, K, B, H, W, F, J, L):
        for name, fn in inspect.getmembers(mod, inspect.isfunction):
            if not name.startswith("test_") or filt not in name:
                continue
            if name in SKIP:
                print("skip  %s: %s" % (name, SKIP[name]))
                continue
            for args in PARAMS.get(name, [()]):
                t = time.time()
                try:
                    fn(O, *args)
                    res = "ok"
                except Exception as e:                      # noqa: BLE001
                    res = "FAIL %s: %s" % (type(e).__name__, str(e)[:200])
                    fail += 1
                tot += 1
                print("%-60s %-16s %6.1fs %s" % (name, args, time.time() - t, res), flush=True)
    print("TOTAL %d run, %d failed" % (tot, fail))
    return 1 if fail else 0


if __name__ == "__main__":
    sys.exit(main())
