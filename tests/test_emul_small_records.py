"""Metadata-heavy streams (tests/meta_streams.py) on the CPU: the K1 and scan kernels over more than
65 536 records, and the emulated library cutting batches on record count.  No GPU.

A batch whose records average under about 512 bytes fills its record table before its byte budget.
Then one scan covers more than 256 tiles of 256 records, and k_scan_spine goes round its loop more
than once.  The GPU twin of this file is tests/test_gpu_small_records.py."""
import pytest

import meta_streams as M
from test_emul_device_code import emu, _verify_on_emulator  # noqa: F401  (fixture)
from test_emul_library import emul_library  # noqa: F401  (fixture)

NONE = 0xffffffff
SCAN_TILE = 256                     # kernels_fletcher.cuh: records per scan tile and spine pass width
MAX_RECORD = (16 << 20) + 4096      # mtz_lib.cu MAX_RECORD_BYTES
BATCH = 16 << 20                    # 32 772 records a batch: ~400-byte records fill them in ~13 MB


def rec_cap(batch_bytes):
    """mtz_lib.cu ensure_slots: the record table of a batch slot"""
    return max(4096, (batch_bytes + MAX_RECORD) // 1024)


@pytest.fixture(scope="module")
def meta(oracle):
    """70 002 records, a 1 MiB and a 128 KiB WRITE among them (K1's G = 4 form cuts them in 128 KiB
    chunks); more than twice rec_cap(BATCH) records in fewer bytes than BATCH"""
    s = M.meta_stream(oracle, 11, 70000, big={1000: 1 << 20, 50000: 131072})
    cnt, offs = oracle.stream_index(s)
    assert cnt > 2 * rec_cap(BATCH) and cnt > 256 * SCAN_TILE
    return s, offs


def _flip(s, offs, k, byte=200):
    """one bit of record k's header (an unused byte of every type): record k's own checksum fails"""
    bad = s.copy()
    bad[int(offs[k]) + byte] ^= 0x10
    return bad


def test_k1_and_scan_over_more_than_65536_records(emu, oracle, meta):  # noqa: F811
    """K1 in the G = 4 form, the one launch_k1_kernel picks for these records (the one-warp-per-record
    form takes ten times as long on the emulator and sees the same scan)"""
    s, offs = meta
    rc, st = oracle.stream_verify(s)
    r = _verify_on_emulator(emu, s, 4)
    assert -(-r["nrec"] // SCAN_TILE) > SCAN_TILE                      # k_scan_spine: two passes
    assert r["bad"] == NONE and r["end_seen"] == 1 and r["end_ck"] == st.end_cksum.tuple()
    assert r["carry"] == oracle.fletcher4(s)
    whole = oracle.fletcher4_partial(s)
    assert r["agg"][1:] == whole[1:] and r["agg"][0] == whole[0] | (1 << 63)


def test_first_failing_record_past_65536(emu, oracle, meta):  # noqa: F811
    s, offs = meta
    bad = _flip(s, offs, 68001)
    rc, st = oracle.stream_verify(bad)
    assert rc == oracle.ECKSUM and st.bad_record == 68001
    r = _verify_on_emulator(emu, bad, 4)
    assert r["bad"] == st.bad_record


def _stage(mode):
    from manatee_b200 import GpuSnapshotStage
    return GpuSnapshotStage(mode, batch_bytes=BATCH)


def test_record_bound_batches_on_the_emulated_library(emul_library, oracle, meta):  # noqa: F811
    """batch_bytes = 16 MiB: every batch is cut at rec_cap records, long before its byte budget"""
    from manatee_b200._native import MtzError, ECKSUM
    s, offs = meta
    cap = rec_cap(BATCH)
    nb = -(-len(offs) // cap)
    assert nb >= 3
    rc, st = oracle.stream_verify(s)
    with _stage("verify") as g:
        g.process_host(s)
        assert g.stats()["batches"] == nb
        assert g.end_checksum() == st.end_cksum.tuple() and g.stats()["records"] == st.records
    k = cap + 12345                                                     # inside batch 2
    bad = _flip(s, offs, k)
    assert oracle.stream_verify(bad)[1].bad_record == k
    with _stage("verify") as g:
        with pytest.raises(MtzError) as ei:
            g.process_host(bad)
        assert ei.value.code == ECKSUM and g.stats()["bad_record"] == k
