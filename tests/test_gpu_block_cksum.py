"""GPU: MTZ_FLAG_BLOCK_CKSUM through the C ABI -- every DRR_WRITE checked against the on-disk block
checksum its header carries (drr_key), on process_host, the ring API, the device API (sub-batched
and deferred) and a device group, against the reference model in tests/block_cksum_ref.py.

A block stored raw on disk must equal its logical bytes: a stream that was corrupted and then
re-stamped passes every stream checksum and fails here.  A block stored LZ4 on disk is compared with
the frame at hand and a mismatch is only counted.  With the flag off nothing changes."""
import threading

import numpy as np
import pytest

import block_cksum_ref as R

pytestmark = pytest.mark.gpu

MODES = {"verify": R.VERIFY, "compress": R.COMPRESS, "decompress": R.DECOMPRESS, "recompress": R.RECOMPRESS}
TIMING = ("gpu_ms", "k1_ms", "codec_ms", "k3_ms")
COUNTERS = ("logical_ok", "frame_ok", "frame_miss", "skipped", "first_frame_miss")


def _run(oracle, mode, s, flag=True, **kw):
    """process_host -> (output, stats, block stats); the output of VERIFY is the input"""
    from manatee_b200 import GpuSnapshotStage
    out = None if mode == "verify" else np.zeros(s.size * 3 + (1 << 20), dtype=np.uint8)
    with GpuSnapshotStage(mode, block_checksums=flag, **kw) as g:
        n = g.process_host(s, out)
        return (s if out is None else out[:n].copy()), g.stats(), g.block_stats()


def _want(oracle, mode, inp, out):
    """reference counters for a run of `mode` on `inp` that produced `out` (wire form)"""
    plain_in = oracle.wire_strip(inp) if mode == "decompress" else inp
    plain_out = None if mode == "verify" else oracle.wire_strip(out)
    return R.block_check(plain_in, plain_out, MODES[mode])


def _same(bs, want):
    assert {k: bs[k] for k in COUNTERS} == {k: want[k] for k in COUNTERS}, (bs, want)


def _raw_stream(oracle, n=24, recsize=8192):
    """a stream as the generator writes it: every key is the Fletcher-4 of the logical block"""
    return oracle.synth_stream(n, recsize=recsize, kind=oracle.PAYLOAD_PGPAGE)


def _mixed(oracle, n=30, recsize=8192, ashift=9):
    from test_gpu_codec import _mixed_stream
    return R.as_lz4_on_disk(oracle, _mixed_stream(oracle, n=n, recsize=recsize), ashift)


def _corrupt_restamped(oracle, s, k, byte=1234):
    """flip one payload bit of record k, then re-stamp: every stream checksum holds again"""
    s = s.copy()
    _, offs = oracle.stream_index(s)
    s[int(offs[k]) + 312 + byte] ^= 0x08
    assert oracle.stream_restamp(s)[0] == 0 and oracle.stream_verify(s)[0] == 0
    return s


def test_raw_stream_every_block_matches_in_every_mode(oracle):
    s = _raw_stream(oracle)
    for mode in ("verify", "compress", "recompress"):
        out, _, bs = _run(oracle, mode, s)
        _, want = _want(oracle, mode, s, out)
        assert want["logical_ok"] == 24 and want["first_bad"] == R.NONE
        _same(bs, want)
        if mode == "compress":
            c = out
    d, _, bs = _run(oracle, "decompress", c)
    assert np.array_equal(d, s)
    _, want = _want(oracle, "decompress", c, d)
    assert want["logical_ok"] == 24
    _same(bs, want)


def test_corrupted_then_restamped_block_fails_only_with_the_flag(oracle):
    """The case the check exists for: the stream checksums are all valid, the bytes are not the
    primary's.  Reported at the reference's record, with the object and offset, in every mode."""
    from manatee_b200._native import MtzError, ECKSUM
    s = _corrupt_restamped(oracle, oracle.synth_stream(40, recsize=16384, kind=oracle.PAYLOAD_PGPAGE), 17)
    _, want = R.block_check(s, None, R.VERIFY)
    assert want["first_bad"] == 17
    _run(oracle, "verify", s, flag=False)
    c, _, _ = _run(oracle, "compress", s, flag=False)
    for mode, src in (("verify", s), ("compress", s), ("recompress", s), ("decompress", c)):
        from manatee_b200 import GpuSnapshotStage
        out = np.zeros(s.size * 3 + (1 << 20), dtype=np.uint8)
        with GpuSnapshotStage(mode, block_checksums=True, batch_bytes=1 << 18) as g:
            with pytest.raises(MtzError) as ei:
                g.process_host(src, None if mode == "verify" else out)
            assert ei.value.code == ECKSUM, mode
            assert g.stats()["bad_record"] == 17, mode
            msg = str(ei.value)
            assert "block checksum" in msg and "object 8" in msg and "offset %d" % (15 * 16384) in msg, msg


def test_flipped_key_bit_fails(oracle):
    from manatee_b200._native import MtzError, ECKSUM
    s = _raw_stream(oracle).copy()
    _, offs = oracle.stream_index(s)
    s[int(offs[9]) + 56 + 17] ^= 0x40
    assert oracle.stream_restamp(s)[0] == 0
    _run(oracle, "verify", s, flag=False)
    from manatee_b200 import GpuSnapshotStage
    with GpuSnapshotStage("verify", block_checksums=True) as g:
        with pytest.raises(MtzError) as ei:
            g.process_host(s)
        assert ei.value.code == ECKSUM and "block checksum" in str(ei.value)
        assert g.stats()["bad_record"] == 9


@pytest.mark.parametrize("ashift,recsize", [(9, 8192), (12, 8192), (12, 65536)])
def test_lz4_on_disk_keys_match_the_encoder(oracle, ashift, recsize):
    """Keys of a dataset written with compression=lz4: the stage's encoder output equals every disk
    frame (the reference's encoder is the declared one), blocks ZFS stored raw match logically."""
    s, dcs = _mixed(oracle, n=24, recsize=recsize, ashift=ashift)
    nlz4 = sum(1 for v in dcs.values() if v == R.DC_LZ4)
    assert 0 < nlz4 < len(dcs)
    for mode in ("compress", "recompress", "verify"):
        out, _, bs = _run(oracle, mode, s)
        _, want = _want(oracle, mode, s, out)
        if mode == "verify":
            assert want["skipped"] == nlz4 and want["logical_ok"] == len(dcs) - nlz4
        else:
            assert want["frame_ok"] == nlz4 and want["frame_miss"] == 0
        _same(bs, want)


def test_frame_miss_is_counted_not_an_error(oracle):
    s, dcs = _mixed(oracle)
    lz4 = sorted(i for i, v in dcs.items() if v == R.DC_LZ4)
    _, offs = oracle.stream_index(s)
    s = s.copy()
    for i, j in zip(lz4[1:4], lz4[2:5]):      # the key of another valid frame
        _, key, p = R.get_key(s, int(offs[j]))
        R.set_key(s, int(offs[i]), key=key, ddk_prop=(p & ~0xffff) | (R.get_key(s, int(offs[i]))[2] & 0xffff))
    assert oracle.stream_restamp(s)[0] == 0
    for mode in ("compress", "recompress"):
        ref, _, _ = _run(oracle, mode, s, flag=False)
        out, _, bs = _run(oracle, mode, s)
        assert np.array_equal(out, ref)
        _, want = _want(oracle, mode, s, out)
        assert want["frame_miss"] == 3 and want["first_frame_miss"] == lz4[1]
        _same(bs, want)


@pytest.mark.parametrize("ashift", [9, 12])
def test_send_c_stream_frames_checked_on_input(oracle, ashift):
    s, dcs = _mixed(oracle, ashift=ashift)
    c = R.as_send_c(oracle, s, ashift)
    assert oracle.stream_verify(c)[0] == 0
    for mode in ("verify", "recompress"):
        ref, _, _ = _run(oracle, mode, c, flag=False)
        out, _, bs = _run(oracle, mode, c)
        assert np.array_equal(out, ref)
        _, want = _want(oracle, mode, c, out)
        assert want["frame_ok"] == sum(1 for v in dcs.values() if v == R.DC_LZ4) and want["frame_miss"] == 0
        _same(bs, want)


def test_unverifiable_keys_are_skipped(oracle):
    s = _raw_stream(oracle, n=12).copy()
    _, offs = oracle.stream_index(s)
    o = [int(offs[k]) for k in (3, 5, 7, 9)]
    R.set_key(s, o[0], ctype=R.SHA256)
    R.set_key(s, o[1], ddk_prop=R.prop(8192, 8192, R.DC_OFF, crypt=1))
    R.set_key(s, o[2], ddk_prop=R.prop(8192, 4096, R.DC_ZSTD))
    R.set_key(s, o[3], ddk_prop=0)
    assert oracle.stream_restamp(s)[0] == 0
    _, _, bs = _run(oracle, "verify", s)
    _, want = R.block_check(s, None, R.VERIFY)
    assert want["skipped"] == 4 and want["logical_ok"] == 8
    _same(bs, want)


def test_passthrough_with_the_flag_is_einval(oracle):
    from manatee_b200 import GpuSnapshotStage
    from manatee_b200._native import MtzError, EINVAL
    with pytest.raises(MtzError) as ei:
        GpuSnapshotStage("passthrough", block_checksums=True)
    assert ei.value.code == EINVAL


def test_first_failing_record_in_stream_order_is_reported(oracle):
    """One batch holds a block failure and a stream failure: the earlier record is reported; a record
    failing both reports its stream checksum."""
    from manatee_b200 import GpuSnapshotStage
    from manatee_b200._native import MtzError, ECKSUM
    base = oracle.synth_stream(20, recsize=8192, kind=oracle.PAYLOAD_PGPAGE)
    _, offs = oracle.stream_index(base)
    cases = []
    s = _corrupt_restamped(oracle, base, 5)
    s[int(offs[11]) + 24] ^= 1                     # header of record 11, not re-stamped
    cases.append((s, 5, "block checksum"))
    s = _corrupt_restamped(oracle, base, 12)
    s[int(offs[4]) + 24] ^= 1
    cases.append((s, 4, "stream checksum"))
    s = base.copy()
    s[int(offs[7]) + 60] ^= 1                      # the key of record 7, not re-stamped
    cases.append((s, 7, "stream checksum"))
    for s, rec, what in cases:
        assert oracle.stream_verify(s)[1].bad_record == rec or what == "block checksum"
        with GpuSnapshotStage("verify", block_checksums=True) as g:
            with pytest.raises(MtzError) as ei:
                g.process_host(s)
            assert ei.value.code == ECKSUM and what in str(ei.value), (rec, str(ei.value))
            assert g.stats()["bad_record"] == rec


def test_the_flag_changes_no_byte_and_no_stats_field(oracle):
    s, _ = _mixed(oracle)
    c, _, _ = _run(oracle, "compress", s, flag=False)
    for mode, src in (("verify", s), ("compress", s), ("recompress", s), ("decompress", c),
                      ("recompress", R.as_send_c(oracle, s))):
        a, sa, _ = _run(oracle, mode, src, flag=False, batch_bytes=1 << 18)
        b, sb, bs = _run(oracle, mode, src, flag=True, batch_bytes=1 << 18)
        assert np.array_equal(a, b), mode
        for k in TIMING:
            sa.pop(k); sb.pop(k)
        assert sa == sb, mode
        assert bs["logical_ok"] + bs["frame_ok"] > 0
    _, _, off = _run(oracle, "verify", s, flag=False)
    assert all(v == 0 for v in off.values())


def _pump(stage, data, chunk):
    err, got = [], []

    def prod():
        try:
            for i in range(0, len(data), chunk):
                stage.write(np.frombuffer(data[i:i + chunk], dtype=np.uint8))
            stage.flush()
        except Exception as e:  # noqa: BLE001
            err.append(e)

    t = threading.Thread(target=prod)
    t.start()
    try:
        while True:
            b = stage.read(1 << 20)
            if b is None:
                break
            got.append(b)
    except Exception as e:  # noqa: BLE001
        err.append(e)
    finally:
        t.join()
    return b"".join(got), err


@pytest.mark.parametrize("chunk", [4093, 1 << 20])
def test_ring_api(oracle, chunk):
    from manatee_b200 import GpuSnapshotStage
    from manatee_b200._native import MtzError, ECKSUM
    s, _ = _mixed(oracle)
    c = R.as_send_c(oracle, s)
    for mode in ("verify", "recompress"):
        with GpuSnapshotStage(mode, block_checksums=True, batch_bytes=1 << 18) as g:
            out, err = _pump(g, c.tobytes(), chunk)
            assert not err, err
            _, want = _want(oracle, mode, c, np.frombuffer(out, dtype=np.uint8))
            _same(g.block_stats(), want)
    # a failing block: no byte of its batch reaches the consumer
    bad = _corrupt_restamped(oracle, _raw_stream(oracle, n=40), 20)
    _, offs = oracle.stream_index(bad)
    with GpuSnapshotStage("verify", block_checksums=True, batch_bytes=1 << 16) as g:
        out, err = _pump(g, bad.tobytes(), chunk)
        assert any(isinstance(e, MtzError) and e.code == ECKSUM for e in err), err
        assert len(out) <= int(offs[20]) and g.stats()["bad_record"] == 20


class TorchMem(object):
    """device buffers for the device API: torch.cuda tensors"""

    def put(self, a):
        import torch
        t = torch.from_numpy(np.ascontiguousarray(a).copy()).cuda()
        return t, t.data_ptr()

    def zeros(self, n):
        import torch
        t = torch.zeros(n, dtype=torch.uint8, device="cuda")
        return t, t.data_ptr()

    def get(self, t, n):
        return t[:n].cpu().numpy()


def device_api_subbatched(oracle, mem, nrec):
    """DECOMPRESS on the device API over more records than one codec sub-batch holds: records that
    arrive LZ4 are checked on the decoded output, the ones stored raw on the input."""
    from manatee_b200 import GpuSnapshotStage, index_host
    s = oracle.synth_stream(nrec, recsize=4096, kind=oracle.PAYLOAD_PGPAGE)
    rc, c, _ = oracle.stream_compress_plain(s)
    assert rc == 0
    recs, used = index_host(c)
    d_in, p_in = mem.put(c)
    d_recs, p_recs = mem.put(recs.view(np.uint8))
    cap = s.size + (1 << 20)
    d_out, p_out = mem.zeros(cap)
    with GpuSnapshotStage("decompress", block_checksums=True) as g:
        g.dev_submit(p_in, c.size, p_recs, len(recs), p_out, cap)
        ob, _, _ = g.dev_finish()
        out = mem.get(d_out, ob)
        _, want = R.block_check(c, out, R.DECOMPRESS)
        assert want["logical_ok"] == nrec
        _same(g.block_stats(), want)
    from manatee_b200._native import MtzError, ECKSUM
    bad = _corrupt_restamped(oracle, s, nrec - 3, byte=100)
    rc, cb, _ = oracle.stream_compress_plain(bad)
    rb, _ = index_host(cb)
    d_in2, p_in2 = mem.put(cb)
    d_r2, p_r2 = mem.put(rb.view(np.uint8))
    with GpuSnapshotStage("decompress", block_checksums=True) as g:
        g.dev_submit(p_in2, cb.size, p_r2, len(rb), p_out, cap)
        with pytest.raises(MtzError) as ei:
            g.dev_finish()
        assert ei.value.code == ECKSUM and g.stats()["bad_record"] == nrec - 3


def test_device_api_across_the_subbatch_edge(oracle):
    device_api_subbatched(oracle, TorchMem(), 66000)


def test_deferred_shards(oracle):
    """MTZ_FLAG_DEFER_VERIFY: the block verdict of a shard surfaces at mtz_dev_finish, with the
    stream verdict, at the stream-wide record index."""
    from manatee_b200 import GpuSnapshotStage, index_host
    from manatee_b200._native import FLAG_DEFER_VERIFY, MtzError, ECKSUM
    s = oracle.synth_stream(60, recsize=16384, kind=oracle.PAYLOAD_PGPAGE)
    recs, _ = index_host(s)
    cut = int(recs["off"][31])
    for bad_rec, fails in ((None, None), (40, 1), (12, 0)):
        src = s if bad_rec is None else _corrupt_restamped(oracle, s, bad_rec)
        gs = [GpuSnapshotStage("verify", batch_bytes=1 << 18, flags=FLAG_DEFER_VERIFY, block_checksums=True)
              for _ in range(2)]
        try:
            gs[0].process_host(src[:cut]); gs[1].process_host(src[cut:])
            a0 = gs[0].dev_aggregate()
            c1 = oracle.fletcher4_apply((0, 0, 0, 0), (a0[0] & ((1 << 63) - 1),) + a0[1:])
            for k, carry in ((0, (0, 0, 0, 0)), (1, c1)):
                if fails == k:
                    with pytest.raises(MtzError) as ei:
                        gs[k].dev_finish(carry_in=carry)
                    assert ei.value.code == ECKSUM and "block checksum" in str(ei.value)
                    assert gs[k].stats()["bad_record"] + 31 * k == bad_rec
                else:
                    gs[k].dev_finish(carry_in=carry)
            if fails is None:
                assert gs[0].block_stats()["logical_ok"] + gs[1].block_stats()["logical_ok"] == 60
        finally:
            for g in gs:
                g.close()


def test_device_group(oracle):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    s, _ = _mixed(oracle)
    c = R.as_send_c(oracle, s)
    for mode in ("verify", "recompress"):
        out, _, bs = _run(oracle, mode, c, devices=[0, 1], batch_bytes=1 << 18)
        _, want = _want(oracle, mode, c, out)
        _same(bs, want)
