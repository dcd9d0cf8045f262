"""GPU parity on metadata-heavy send streams (tests/meta_streams.py): long runs of 312..632-byte
DRR_OBJECT / DRR_FREE / DRR_FREEOBJECTS records, as a dataset with many files sends.  Bit-exact
against the oracle.

These streams reach code paths that depend only on how many records a batch holds or how small they
are:
  * batches cut on record count (batch_accept: `bc.cnt >= s.rec_cap`) instead of on bytes;
  * k_scan_spine going round its loop more than once (a scan over more than 256 tiles of 256);
  * device-API codec sub-batches split at 65 536 records;
  * the K1 form picked from the average record size, with 1 MiB and 16 MiB records inside;
  * the stamp chain's groups of STAMP_GROUP transitions with sub-stream edges at the group edges.
Every test asserts that it reached the shape it is named for, from the thresholds restated below,
so a change of those thresholds fails here instead of quietly testing byte-bound batches again."""
import numpy as np
import pytest

import block_ref as R
import meta_streams as M
from test_gpu_block_cksum import _pump, _run, _same, _want

pytestmark = pytest.mark.gpu

MAX_RECORD = (16 << 20) + 4096      # mtz_lib.cu MAX_RECORD_BYTES
VERIFY_BATCH = 32 << 20             # mtz_open: default batch_bytes of VERIFY
CODEC_BATCH = 256 << 20             # ... and of the re-encoding modes
SCAN_TILE = 256                     # kernels_fletcher.cuh: records per scan tile and spine pass width
DEV_SUBBATCH = 65536                # mtz_lib.cu: codec_alloc(h, h->dv_cb, 65536, ...)
STAMP_GROUP = 32                    # kernels_codec.cuh
K1_BANDS = {4: (0, 12 << 10), 8: (12 << 10, 24 << 10), 16: (24 << 10, 96 << 10), 32: (96 << 10, 1 << 40)}
K1_MAX_ROWS = 2048                  # MTZ_K1_MAX_ROWS: a K1 chunk is 2048 rows of 16 * G bytes


def rec_cap(batch_bytes):
    """mtz_lib.cu ensure_slots: the record table of a batch slot"""
    return max(4096, (batch_bytes + MAX_RECORD) // 1024)


def _nb(nrec, batch_bytes):
    return -(-nrec // rec_cap(batch_bytes))


@pytest.fixture(scope="module")
def meta(oracle):
    """600 002 records in under 256 MiB: more than twice rec_cap(256 MiB) = 278 532 records"""
    s = M.meta_stream(oracle, 21, 600000)
    cnt, offs = oracle.stream_index(s)
    assert s.size < CODEC_BATCH and cnt > 2 * rec_cap(CODEC_BATCH)
    return s, offs


def _stage(mode, **kw):
    from manatee_b200 import GpuSnapshotStage
    return GpuSnapshotStage(mode, **kw)


def _flip(s, offs, k, byte=200):
    """one bit of record k's header, in a byte no record type uses: record k's own checksum fails"""
    bad = s.copy()
    bad[int(offs[k]) + byte] ^= 0x10
    return bad


# ---- a. record-bound batches in VERIFY ---------------------------------------------------------------

@pytest.mark.parametrize("batch", [CODEC_BATCH, 64 << 20])
def test_record_bound_verify_batches(oracle, meta, batch):
    """256 MiB: three batches of 278 532 records.  64 MiB: batches of 81 924 records, 321 scan tiles,
    so k_scan_spine takes two passes in every batch"""
    s, offs = meta
    rc, st = oracle.stream_verify(s)
    assert _nb(len(offs), batch) > -(-s.size // batch)                  # more batches than bytes need
    if batch == 64 << 20:
        assert -(-rec_cap(batch) // SCAN_TILE) > SCAN_TILE
    with _stage("verify", batch_bytes=batch) as g:
        assert g.process_host(s) == s.size
        gs = g.stats()
        assert gs["batches"] == _nb(len(offs), batch) >= 3
        assert g.end_checksum() == st.end_cksum.tuple()
        assert gs["records"] == st.records and gs["bytes_in"] == s.size


@pytest.mark.parametrize("chunk", [4093, 1 << 20])
def test_record_bound_ring_api(oracle, meta, chunk):
    """the streaming engine at the default batch: 49 156 records a batch"""
    s, offs = meta
    rc, st = oracle.stream_verify(s)
    with _stage("verify") as g:
        out, err = _pump(g, s.tobytes(), chunk)
        assert not err, err
        assert out == s.tobytes()
        assert g.stats()["batches"] >= _nb(len(offs), VERIFY_BATCH) > s.size // VERIFY_BATCH + 1
        assert g.end_checksum() == st.end_cksum.tuple()


# ---- b. the first failing record -------------------------------------------------------------------

def test_first_failing_record_across_record_bound_batches(oracle, meta):
    from manatee_b200._native import MtzError, ECKSUM
    s, offs = meta
    cap = rec_cap(CODEC_BATCH)
    # last of batch 1, first of batch 2, past 65 536 within batch 2, past 2 * rec_cap (batch 3)
    for k in (cap - 1, cap, cap + DEV_SUBBATCH + 4321, 2 * cap + 123):
        bad = _flip(s, offs, k)
        rc, st = oracle.stream_verify(bad)
        assert rc == oracle.ECKSUM and st.bad_record == k
        with _stage("verify", batch_bytes=CODEC_BATCH) as g:
            with pytest.raises(MtzError) as ei:
                g.process_host(bad)
            assert ei.value.code == ECKSUM and g.stats()["bad_record"] == k, k


def test_deferred_verify_scans_every_batch_at_once(oracle, meta):
    """MTZ_FLAG_DEFER_VERIFY through process_host: the sums of all 13 batches meet in one scan of
    600 002 records (2 344 tiles, ten spine passes) at dev_finish"""
    from manatee_b200._native import FLAG_DEFER_VERIFY, MtzError, ECKSUM
    s, offs = meta
    rc, st = oracle.stream_verify(s)
    with _stage("verify", flags=FLAG_DEFER_VERIFY) as g:
        g.process_host(s)
        assert g.stats()["batches"] == _nb(len(offs), VERIFY_BATCH)
        a = g.dev_aggregate()
        whole = oracle.fletcher4_partial(s)
        assert a[0] == whole[0] | (1 << 63) and a[1:] == whole[1:]
        _, carry, _ = g.dev_finish(carry_in=(0, 0, 0, 0))
        assert carry == oracle.fletcher4(s) and g.end_checksum() == st.end_cksum.tuple()
    k = 2 * rec_cap(CODEC_BATCH) + 123
    bad = _flip(s, offs, k)
    with _stage("verify", flags=FLAG_DEFER_VERIFY) as g:
        g.process_host(bad)
        with pytest.raises(MtzError) as ei:
            g.dev_finish(carry_in=(0, 0, 0, 0))
        assert ei.value.code == ECKSUM and g.stats()["bad_record"] == k


# ---- c. the re-encoding modes at the default batch ---------------------------------------------------

def test_reencoding_modes_on_record_bound_batches(oracle, meta):
    s, offs = meta
    nb = _nb(len(offs), CODEC_BATCH)
    assert nb >= 3

    def run(mode, src, cap):
        out = np.zeros(cap, dtype=np.uint8)
        with _stage(mode) as g:
            n = g.process_host(src, out)
            gs = g.stats()
            assert gs["batches"] == nb, mode
            return out[:n], gs, g.end_checksum()

    rc, want_c, cst = oracle.stream_compress(s)
    assert rc == 0 and cst.lz4_out > 0
    c, gs, end = run("compress", s, s.size * 2 + (1 << 20))
    assert np.array_equal(c, want_c) and end == cst.end_cksum.tuple() and gs["lz4_encoded"] == cst.lz4_out
    rc, want_d, dst = oracle.stream_decompress(c)
    assert rc == 0
    d, gs, end = run("decompress", c, s.size + (1 << 20))
    assert np.array_equal(d, s), "DECOMPRESS(COMPRESS(x)) != x"
    assert np.array_equal(d, want_d) and end == dst.end_cksum.tuple() and gs["lz4_decoded"] == dst.lz4_in
    plain = oracle.wire_strip(c)
    rc, want_r, rst = oracle.stream_recompress(plain)
    assert rc == 0
    r, gs, end = run("recompress", plain, s.size + (1 << 20))
    assert np.array_equal(r, want_r) and end == rst.end_cksum.tuple() and gs["lz4_encoded"] == rst.lz4_out


# ---- d. the device API, more than 65 536 records in one submit ---------------------------------------

@pytest.fixture(scope="module")
def dev_meta(oracle):
    import torch
    from manatee_b200 import index_host
    s = M.meta_stream(oracle, 22, 160000)
    recs, used = index_host(s)
    assert used == s.size and len(recs) > 2 * DEV_SUBBATCH
    return s, recs, torch.from_numpy(s.copy()).cuda(), torch.from_numpy(recs.view(np.uint8).copy()).cuda()


def test_device_api_verify_one_submit(oracle, dev_meta):
    s, recs, d, d_recs = dev_meta
    rc, st = oracle.stream_verify(s)
    with _stage("verify") as g:
        g.dev_submit(d.data_ptr(), s.size, d_recs.data_ptr(), len(recs))
        a = g.dev_aggregate()
        whole = oracle.fletcher4_partial(s)
        assert a[0] == whole[0] | (1 << 63) and a[1:] == whole[1:]
        _, carry, _ = g.dev_finish()
        assert carry == oracle.fletcher4(s) and g.end_checksum() == st.end_cksum.tuple()


def test_device_api_codec_across_subbatches(oracle, dev_meta):
    """one COMPRESS and one RECOMPRESS submit of 160 002 records: three codec sub-batches"""
    import torch
    from manatee_b200 import index_host
    s, recs, d, d_recs = dev_meta
    rc, want_c, cst = oracle.stream_compress_plain(s)
    assert rc == 0
    d_out = torch.zeros(s.size + (1 << 20), dtype=torch.uint8, device="cuda")
    with _stage("compress") as g:
        g.dev_submit(d.data_ptr(), s.size, d_recs.data_ptr(), len(recs), d_out.data_ptr(), d_out.numel())
        ob, _, carry_out = g.dev_finish()
        assert np.array_equal(d_out[:ob].cpu().numpy(), want_c)
        assert g.end_checksum() == cst.end_cksum.tuple() and carry_out == oracle.fletcher4(want_c)
        assert g.stats()["lz4_encoded"] == cst.lz4_out
    rc, want_r, rst = oracle.stream_recompress(want_c)
    crecs, used = index_host(want_c)
    assert used == want_c.size and len(crecs) > 2 * DEV_SUBBATCH
    d_c = torch.from_numpy(want_c.copy()).cuda()
    d_crecs = torch.from_numpy(crecs.view(np.uint8).copy()).cuda()
    d_out.zero_()
    with _stage("recompress") as g:
        g.dev_submit(d_c.data_ptr(), want_c.size, d_crecs.data_ptr(), len(crecs), d_out.data_ptr(), d_out.numel())
        ob, _, _ = g.dev_finish()
        assert np.array_equal(d_out[:ob].cpu().numpy(), want_r)
        assert g.end_checksum() == rst.end_cksum.tuple()


def test_gpu_side_parse_of_varying_lengths(oracle, dev_meta):
    """k_index on 160 002 records whose lengths change at almost every record"""
    import torch
    from manatee_b200.stage import REC_DTYPE
    s, recs, d, _ = dev_meta
    d_recs = torch.zeros((len(recs) + 8) * 32, dtype=torch.uint8, device="cuda")
    with _stage("verify") as g:
        n, used = g.dev_index(d.data_ptr(), s.size, d_recs.data_ptr(), len(recs) + 8)
        assert n == len(recs) and used == s.size
        got = d_recs.cpu().numpy().view(REC_DTYPE)[:n]
        for f in ("off", "payload", "type", "lsize", "comp"):
            assert np.array_equal(got[f], recs[f]), f


# ---- e. the four K1 forms with large records inside ---------------------------------------------------

SMALL_PER_BAND = {4: 3000, 8: 990, 16: 366, 32: 100}


@pytest.mark.parametrize("G", [4, 8, 16, 32])
def test_k1_forms_with_large_records_inside(oracle, G):
    """One device-API VERIFY submit per K1 form.  launch_k1_kernel picks the form from the submit's
    average record size in_bytes / nrec: G = 32 at 96 KiB and more, 16 from 24 KiB, 8 from 12 KiB, 4
    below.  Each submit holds a 16 MiB and a 1 MiB WRITE and small records at every body alignment;
    one bit flipped on either side of a K1 chunk boundary inside the 16 MiB record is found."""
    import torch
    from manatee_b200 import index_host
    from manatee_b200._native import MtzError, ECKSUM
    m = SMALL_PER_BAND[G]
    i16, i1 = 65 + (m - 64) // 3, 65 + 2 * (m - 64) // 3
    s = M.meta_stream(oracle, 30 + G, m, big={i16: 16 << 20, i1: 1 << 20}, sweep=64)
    recs, used = index_host(s)
    lo, hi = K1_BANDS[G]
    assert lo <= s.size // len(recs) < hi
    small = recs["off"][recs["type"] != M.WRITE]
    assert M.body_residues(small, 16 * G) == set(range(0, 16 * G, 8))
    rc, st = oracle.stream_verify(s)
    d = torch.from_numpy(s.copy()).cuda()
    d_recs = torch.from_numpy(recs.view(np.uint8).copy()).cuda()
    assert d.data_ptr() % (16 * G) == 0

    def verify():
        """-> (error code, bad_record, END checksum) of one submit of `d`"""
        with _stage("verify") as g:
            g.dev_submit(d.data_ptr(), s.size, d_recs.data_ptr(), len(recs))
            try:
                g.dev_finish()
            except MtzError as e:
                return e.code, g.stats()["bad_record"], None
            return 0, None, g.end_checksum()

    assert verify() == (0, None, st.end_cksum.tuple())
    # K1 chunks of record i16 end at (its body start rounded down to a 16*G-byte row) + k * chunk
    chunk = K1_MAX_ROWS * 16 * G
    o = int(recs["off"][i16])
    row0 = (o + 280) & ~(16 * G - 1)
    for k in (1, (16 << 20) // chunk // 2):
        edge = row0 + k * chunk
        assert o + 312 < edge - 4 and edge < o + 312 + (16 << 20)
        for pos in (edge - 4, edge):
            bad = s.copy()
            bad[pos] ^= 0x04
            rc, bst = oracle.stream_verify(bad)
            assert rc == oracle.ECKSUM and bst.bad_record == i16 + 1
            d[pos] ^= 0x04
            got = verify()
            d[pos] ^= 0x04
            assert got == (ECKSUM, bst.bad_record, None), (k, pos - o)


# ---- f. sub-stream edges inside the stamp chain's groups ---------------------------------------------

def _cuts(recs, batch_bytes, begin_cuts):
    """batch_accept / the bulk loop of mtz_process_host, restated for the re-encoding modes: the
    [first, end) record ranges of the batches.  `begin_cuts`: a BEGIN opens a batch (a DECOMPRESS
    wire preamble does)"""
    cap, out, first, cnt, budget = batch_bytes + MAX_RECORD, [], 0, 0, 0
    for i, r in enumerate(recs):
        cost = 312 + max(int(r["payload"]), int(r["lsize"])) + 48
        if cnt > 0 and (budget + cost > cap or cnt >= rec_cap(batch_bytes) or (begin_cuts and r["type"] == 0)):
            out.append((first, i))
            first, cnt, budget = i, 0, 0
        cnt += 1
        budget += cost
        if budget >= batch_bytes:
            out.append((first, i + 1))
            first, cnt, budget = i + 1, 0, 0
    if cnt:
        out.append((first, len(recs)))
    return out


@pytest.mark.parametrize("t", [0, 30, 31, 32, 33, 63, 64])
def test_substream_edges_inside_stamp_groups(oracle, t):
    """The stamp chain takes transitions STAMP_GROUP at a time; a transition into BEGIN or END takes
    the generic step, and after transition 31 of a group the next step's weights come from padding
    slot 32.  A 1 MiB WRITE closes batch 1 on its byte budget (512 KiB), so batch 2 starts right
    behind it with t small records and then END.
      RECOMPRESS: BEGIN does not open a batch, so END -> BEGIN is transition t of batch 2.
      DECOMPRESS: the wire preamble in front of every BEGIN opens a batch, so batch 2 ends with END:
      its last transition (t - 1 -> t) is the generic one; at t = 0 the batch is END alone."""
    from manatee_b200 import index_host
    batch = 512 << 10
    raw = M.meta_stream(oracle, 100 + t, [t + 2, 40], big={2: 1 << 20})
    rc, wire, _ = oracle.stream_compress(raw)
    assert rc == 0
    plain = oracle.wire_strip(wire)
    recs, _ = index_host(plain)
    types = recs["type"]
    for mode, src, begin_cuts in (("recompress", plain, False), ("decompress", wire, True)):
        cuts = _cuts(recs, batch, begin_cuts)
        b0, b1 = cuts[1]
        assert cuts[0] == (0, 3) and types[b0 + t] == M.END
        if mode == "recompress":
            assert len(cuts) == 2 and types[b0 + t + 1] == M.BEGIN and b1 == len(recs)
        else:
            assert len(cuts) == 3 and b1 == b0 + t + 1
        rc, want, wst = getattr(oracle, "stream_" + mode)(src)
        assert rc == 0
        out = np.zeros(raw.size * 2 + (1 << 20), dtype=np.uint8)
        with _stage(mode, batch_bytes=batch) as g:
            n = g.process_host(src, out)
            assert g.stats()["batches"] == len(cuts), mode
            assert np.array_equal(out[:n], want), mode
            assert g.end_checksum() == wst.end_cksum.tuple(), mode
        if mode == "decompress":
            assert np.array_equal(out[:n], raw)


# ---- g. the block check on the record-bound stream -------------------------------------------------

def test_block_check_on_record_bound_batches(oracle, meta):
    s, offs = meta
    disk, dcs = R.as_on_disk(oracle, s)
    assert len(dcs) > 1000 and R.DC_LZ4 in dcs.values() and R.DC_OFF in dcs.values()
    for mode, batch in (("verify", VERIFY_BATCH), ("compress", CODEC_BATCH)):
        out, st, bs = _run(oracle, mode, disk)
        assert st["batches"] == _nb(len(offs), batch) >= 3, mode
        _, want = _want(oracle, mode, disk, out)
        assert want["logical_ok"] + want["frame_ok"] + want["skipped"] == len(dcs) and want["first_bad"] == R.NONE
        _same(bs, want)
