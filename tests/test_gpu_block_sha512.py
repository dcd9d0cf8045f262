"""GPU: MTZ_FLAG_BLOCK_SHA512 through the C ABI -- the block-checksum check (MTZ_FLAG_BLOCK_CKSUM)
extended to SHA-512/256 keys (checksum=sha512), hashed on the device by k_block_sha512, on
process_host, the ring API, the device API (sub-batched and deferred) and a device group.  Every
counter is the reference model's (tests/block_sha512_ref.py, hashlib), and the semantics are the
fletcher4 check's: a block stored raw on disk must equal its logical bytes, a frame is only counted.
The flag is independent of MTZ_FLAG_BLOCK_SHA256; without it sha512 keys are skipped, and on a stream
without sha512 keys it changes nothing."""
import numpy as np
import pytest

import block_sha512_ref as R
import test_gpu_block_cksum as B

pytestmark = pytest.mark.gpu

MODES = B.MODES
COUNTERS = B.COUNTERS + ("sha256", "sha512")


def _stage(mode, sha=True, sha256=False, **kw):
    from manatee_b200 import GpuSnapshotStage
    return GpuSnapshotStage(mode, block_checksums=True, block_sha256=sha256, block_sha512=sha, **kw)


def _run(oracle, mode, s, sha=True, sha256=False, **kw):
    """process_host -> (output, stats, block stats); the output of VERIFY is the input"""
    out = None if mode == "verify" else np.zeros(s.size * 3 + (1 << 20), dtype=np.uint8)
    with _stage(mode, sha, sha256, **kw) as g:
        n = g.process_host(s, out)
        return (s if out is None else out[:n].copy()), g.stats(), g.block_stats()


def _want(oracle, mode, inp, out, sha=True, sha256=False):
    plain_in = oracle.wire_strip(inp) if mode == "decompress" else inp
    plain_out = None if mode == "verify" else oracle.wire_strip(out)
    return R.block_check(plain_in, plain_out, MODES[mode], sha256=sha256, sha512=sha)


def _same(bs, want):
    assert {k: bs[k] for k in COUNTERS} == {k: want[k] for k in COUNTERS}, (bs, want)


def _sha_raw(oracle, n=24, recsize=8192, kind=None):
    """a generator stream re-keyed as written with checksum=sha512, compression=off"""
    s = oracle.synth_stream(n, recsize=recsize, kind=kind or oracle.PAYLOAD_PGPAGE).copy()
    for off, _, pl, t in R.records(s):
        if t == 3 and R.get_key(s, off)[2] == 0:      # the generator's 512-byte blocks carry prop 0
            R.set_key(s, off, ddk_prop=R.prop(pl, pl, R.DC_OFF))
    return R.as_sha512(oracle, s)


def _sha_mixed(oracle, n=30, recsize=8192, ashift=9):
    s, dcs = B._mixed(oracle, n=n, recsize=recsize, ashift=ashift)
    return R.as_sha512(oracle, s), dcs


def _fails(mode, src, rec, **kw):
    """the stage fails `src` with ECKSUM at record `rec`; returns the message"""
    from manatee_b200._native import MtzError, ECKSUM
    out = np.zeros(src.size * 4 + (1 << 20), dtype=np.uint8)
    with _stage(mode, **kw) as g:
        with pytest.raises(MtzError) as ei:
            g.process_host(src, None if mode == "verify" else out)
        assert ei.value.code == ECKSUM, mode
        assert g.stats()["bad_record"] == rec, mode
        return str(ei.value)


def test_sha512_keys_match_in_every_mode(oracle):
    s = _sha_raw(oracle)
    for mode in ("verify", "compress", "recompress"):
        out, _, bs = _run(oracle, mode, s)
        _, want = _want(oracle, mode, s, out)
        assert want["logical_ok"] == want["sha512"] == 24 and want["skipped"] == 0
        _same(bs, want)
        if mode == "compress":
            c = out
    d, _, bs = _run(oracle, "decompress", c)
    assert np.array_equal(d, s)
    _, want = _want(oracle, "decompress", c, d)
    assert want["logical_ok"] == want["sha512"] == 24 and want["skipped"] == 0
    _same(bs, want)


def test_corrupted_then_restamped_block_fails_only_with_the_flag(oracle):
    s = B._corrupt_restamped(oracle, _sha_raw(oracle, n=40, recsize=16384), 17)
    _, want = R.block_check(s, None, R.VERIFY, sha512=True)
    assert want["first_bad"] == 17
    # BLOCK_CKSUM alone, or with BLOCK_SHA256: every record is skipped, the stream passes
    for sha256 in (False, True):
        _, _, bs = _run(oracle, "verify", s, sha=False, sha256=sha256)
        _, want = R.block_check(s, None, R.VERIFY, sha256=sha256)
        assert want["skipped"] == 40 and bs["sha512"] == 0
        _same(bs, want)
    c, _, _ = _run(oracle, "compress", s, sha=False)
    for mode, src in (("verify", s), ("compress", s), ("recompress", s), ("decompress", c)):
        msg = _fails(mode, src, 17, batch_bytes=1 << 18)
        assert "block checksum mismatch at record 17 (object 8, offset %d)" % (15 * 16384) in msg, msg
        assert "the bytes differ from the block on disk (sha512 key)" in msg, msg


def test_relabelled_keys_are_mismatches(oracle):
    """a sha256 key labelled 11 and a sha512 key labelled 8 are compared by the other hash: the
    byte orders differ as well as the hashes"""
    base = B._raw_stream(oracle, n=12, recsize=8192).copy()
    _, offs = oracle.stream_index(base)
    a = R.as_sha256(oracle, base)
    R.set_key(a, int(offs[3]), ctype=R.SHA512)
    b = R.as_sha512(oracle, base)
    R.set_key(b, int(offs[5]), ctype=R.SHA256)
    for x, bad, name in ((a, 3, "sha512"), (b, 5, "sha256")):
        assert oracle.stream_restamp(x)[0] == 0
        _, want = R.block_check(x, None, R.VERIFY, sha256=True, sha512=True)
        assert want["first_bad"] == bad
        msg = _fails("verify", x, bad, sha256=True)
        assert "on disk (%s key)" % name in msg, msg


def test_fletcher4_and_sha256_failure_messages_are_unchanged(oracle):
    s = B._corrupt_restamped(oracle, B._raw_stream(oracle, n=12), 5)
    msg = _fails("verify", s, 5, sha256=True)
    assert "offset 24576): the bytes differ from the block on disk" in msg and "key)" not in msg, msg
    s = B._corrupt_restamped(oracle, R.as_sha256(oracle, B._raw_stream(oracle, n=12)), 5)
    msg = _fails("verify", s, 5, sha256=True)
    assert "the bytes differ from the block on disk (sha256 key)" in msg, msg


@pytest.mark.parametrize("ashift", [9, 12])
def test_lz4_on_disk_sha512_keys(oracle, ashift):
    """frame_ok for the stage's encoder output (COMPRESS, RECOMPRESS) and for `send -c` input
    (VERIFY, RECOMPRESS), including frames shorter than PSIZE that end inside a 128-byte block or on
    its boundary"""
    s, dcs = _sha_mixed(oracle, n=24, ashift=ashift)
    nlz4 = sum(1 for v in dcs.values() if v == R.DC_LZ4)
    assert 0 < nlz4 < len(dcs)
    for mode in ("compress", "recompress"):
        out, _, bs = _run(oracle, mode, s)
        _, want = _want(oracle, mode, s, out)
        assert want["frame_ok"] == nlz4 and want["frame_miss"] == 0 and want["sha512"] == len(dcs)
        _same(bs, want)
    c = R.as_send_c(oracle, s, ashift)
    for src in (c, R.trim_frames_to(oracle, c, 8), R.trim_frames_to(oracle, c, 128)):
        for mode in ("verify", "recompress"):
            ref, _, _ = _run(oracle, mode, src, sha=False)
            out, _, bs = _run(oracle, mode, src)
            assert np.array_equal(out, ref)
            _, want = _want(oracle, mode, src, out)
            assert want["frame_ok"] == nlz4 and want["frame_miss"] == 0
            _same(bs, want)


def test_swapped_frame_keys_are_counted_not_errors(oracle):
    s, dcs = _sha_mixed(oracle)
    lz4 = sorted(i for i, v in dcs.items() if v == R.DC_LZ4)
    _, offs = oracle.stream_index(s)
    s = s.copy()
    for i, j in zip(lz4[1:4], lz4[2:5]):
        _, key, p = R.get_key(s, int(offs[j]))
        R.set_key(s, int(offs[i]), key=key, ddk_prop=(p & ~0xffff) | (R.get_key(s, int(offs[i]))[2] & 0xffff))
    assert oracle.stream_restamp(s)[0] == 0
    for mode in ("compress", "recompress"):
        ref, _, _ = _run(oracle, mode, s, sha=False)
        out, _, bs = _run(oracle, mode, s)
        assert np.array_equal(out, ref)
        _, want = _want(oracle, mode, s, out)
        assert want["frame_miss"] == 3 and want["first_frame_miss"] == lz4[1]
        _same(bs, want)


def _mixed_types(oracle):
    """fletcher4, sha256 and sha512 keys and every skipped class in one stream"""
    f, dcs = B._mixed(oracle, n=40)
    h256, h512 = R.as_sha256(oracle, f), R.as_sha512(oracle, f)
    s = f.copy()
    recs = R.records(s)
    w = [i for i, r in enumerate(recs) if r[3] == 3]
    for h, picks in ((h256, w[1::3]), (h512, w[2::3])):
        for i in picks:
            s[recs[i][0] + 48:recs[i][0] + 88] = h[recs[i][0] + 48:recs[i][0] + 88]
    R.set_key(s, recs[w[3]][0], ddk_prop=0)
    R.set_key(s, recs[w[5]][0], ddk_prop=R.prop(8192, 4096, R.DC_ZSTD))
    R.set_key(s, recs[w[6]][0], ddk_prop=R.prop(8192, 8192, R.DC_OFF, crypt=1))
    R.set_key(s, recs[w[9]][0], ctype=12)          # skein: salted, never checked
    assert oracle.stream_restamp(s)[0] == 0
    return s


@pytest.mark.parametrize("sha256,sha512", [(False, False), (True, False), (False, True), (True, True)])
def test_one_stream_mixing_fletcher4_sha256_sha512_and_skipped_keys(oracle, sha256, sha512):
    s = _mixed_types(oracle)
    c, _, _ = _run(oracle, "compress", s, sha=False)
    for mode, src in (("verify", s), ("compress", s), ("recompress", s), ("decompress", c),
                      ("verify", R.as_send_c(oracle, s)), ("recompress", R.as_send_c(oracle, s))):
        out, _, bs = _run(oracle, mode, src, sha=sha512, sha256=sha256, batch_bytes=1 << 17)
        _, want = _want(oracle, mode, src, out, sha=sha512, sha256=sha256)
        assert (want["sha256"] > 0) == sha256 and (want["sha512"] > 0) == sha512
        assert want["skipped"] >= 4 and want["logical_ok"] + want["frame_ok"] > want["sha256"] + want["sha512"]
        _same(bs, want)


@pytest.mark.parametrize("recsize", [512, 8192, 131072, 1 << 20])
def test_record_sizes(oracle, recsize):
    s = _sha_raw(oracle, n=6, recsize=recsize)
    for mode in ("verify", "compress"):
        out, _, bs = _run(oracle, mode, s)
        _, want = _want(oracle, mode, s, out)
        assert want["logical_ok"] == want["sha512"] == 6
        _same(bs, want)
    msg = _fails("verify", B._corrupt_restamped(oracle, s, 4, byte=recsize - 1), 4)
    assert "sha512" in msg


def test_sixteen_mib_record(oracle):
    """the largest ZFS block: one thread hashes 16 MiB + one padding block"""
    s = _sha_raw(oracle, n=1, recsize=16 << 20, kind=oracle.PAYLOAD_PCG)
    _, _, bs = _run(oracle, "verify", s, batch_bytes=32 << 20)
    _, want = R.block_check(s, None, R.VERIFY, sha512=True)
    assert want["logical_ok"] == want["sha512"] == 1
    _same(bs, want)
    _fails("verify", B._corrupt_restamped(oracle, s, 2, byte=(16 << 20) - 8), 2, batch_bytes=32 << 20)


def test_first_failing_record_in_stream_order_is_reported(oracle):
    base = _sha_raw(oracle, n=20)
    _, offs = oracle.stream_index(base)
    cases = []
    s = B._corrupt_restamped(oracle, base, 5)
    s[int(offs[11]) + 24] ^= 1
    cases.append((s, 5, "block checksum"))
    s = B._corrupt_restamped(oracle, base, 12)
    s[int(offs[4]) + 24] ^= 1
    cases.append((s, 4, "stream checksum"))
    s = base.copy()
    s[int(offs[7]) + 60] ^= 1
    cases.append((s, 7, "stream checksum"))
    for s, rec, what in cases:
        assert what in _fails("verify", s, rec)


@pytest.mark.parametrize("chunk", [4093, 1 << 20])
def test_ring_api(oracle, chunk):
    from manatee_b200._native import MtzError, ECKSUM
    s, _ = _sha_mixed(oracle)
    c = R.as_send_c(oracle, s)
    for mode in ("verify", "recompress"):
        with _stage(mode, batch_bytes=1 << 18) as g:
            out, err = B._pump(g, c.tobytes(), chunk)
            assert not err, err
            _, want = _want(oracle, mode, c, np.frombuffer(out, dtype=np.uint8))
            assert want["sha512"] > 0
            _same(g.block_stats(), want)
    bad = B._corrupt_restamped(oracle, _sha_raw(oracle, n=40), 20)
    _, offs = oracle.stream_index(bad)
    with _stage("verify", batch_bytes=1 << 16) as g:
        out, err = B._pump(g, bad.tobytes(), chunk)
        assert any(isinstance(e, MtzError) and e.code == ECKSUM for e in err), err
        assert len(out) <= int(offs[20]) and g.stats()["bad_record"] == 20


def device_api_subbatched(oracle, mem, nrec):
    """DECOMPRESS on the device API over more records than one codec sub-batch holds: records that
    arrive LZ4 are hashed from the decoded output (the output base of their sub-batch)"""
    from manatee_b200 import index_host
    from manatee_b200._native import MtzError, ECKSUM
    s = _sha_raw(oracle, n=nrec, recsize=4096)
    for src, bad in ((s, None), (B._corrupt_restamped(oracle, s, nrec - 3, byte=100), nrec - 3)):
        rc, c, _ = oracle.stream_compress_plain(src)
        assert rc == 0
        recs, _ = index_host(c)
        d_in, p_in = mem.put(c)
        d_recs, p_recs = mem.put(recs.view(np.uint8))
        cap = s.size + (1 << 20)
        d_out, p_out = mem.zeros(cap)
        with _stage("decompress") as g:
            g.dev_submit(p_in, c.size, p_recs, len(recs), p_out, cap)
            if bad is None:
                ob, _, _ = g.dev_finish()
                _, want = R.block_check(c, mem.get(d_out, ob), R.DECOMPRESS, sha512=True)
                assert want["logical_ok"] == want["sha512"] == nrec
                _same(g.block_stats(), want)
            else:
                with pytest.raises(MtzError) as ei:
                    g.dev_finish()
                assert ei.value.code == ECKSUM and "(sha512 key)" in str(ei.value)
                assert g.stats()["bad_record"] == bad


def test_device_api_across_the_subbatch_edge(oracle):
    device_api_subbatched(oracle, B.TorchMem(), 66000)


def test_deferred_shards(oracle):
    from manatee_b200 import index_host
    from manatee_b200._native import FLAG_DEFER_VERIFY, MtzError, ECKSUM
    s = _sha_raw(oracle, n=60, recsize=16384)
    recs, _ = index_host(s)
    cut = int(recs["off"][31])
    for bad_rec, fails in ((None, None), (40, 1), (12, 0)):
        src = s if bad_rec is None else B._corrupt_restamped(oracle, s, bad_rec)
        gs = [_stage("verify", batch_bytes=1 << 18, flags=FLAG_DEFER_VERIFY) for _ in range(2)]
        try:
            gs[0].process_host(src[:cut]); gs[1].process_host(src[cut:])
            a0 = gs[0].dev_aggregate()
            c1 = oracle.fletcher4_apply((0, 0, 0, 0), (a0[0] & ((1 << 63) - 1),) + a0[1:])
            for k, carry in ((0, (0, 0, 0, 0)), (1, c1)):
                if fails == k:
                    with pytest.raises(MtzError) as ei:
                        gs[k].dev_finish(carry_in=carry)
                    assert ei.value.code == ECKSUM and "(sha512 key)" in str(ei.value)
                    assert gs[k].stats()["bad_record"] + 31 * k == bad_rec
                else:
                    gs[k].dev_finish(carry_in=carry)
            if fails is None:
                assert sum(g.block_stats()["sha512"] for g in gs) == 60
                assert sum(g.block_stats()["logical_ok"] for g in gs) == 60
        finally:
            for g in gs:
                g.close()


def test_device_group(oracle):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    s, _ = _sha_mixed(oracle)
    c = R.as_send_c(oracle, s)
    for mode in ("verify", "recompress"):
        out, _, bs = _run(oracle, mode, c, devices=[0, 1], batch_bytes=1 << 18)
        _, want = _want(oracle, mode, c, out)
        _same(bs, want)


def test_the_flag_without_block_checksums_is_einval(oracle):
    from manatee_b200 import GpuSnapshotStage
    from manatee_b200._native import MtzError, EINVAL, FLAG_BLOCK_SHA256, FLAG_BLOCK_SHA512
    for mode in ("verify", "compress", "passthrough"):
        for kw in (dict(block_sha512=True), dict(block_sha256=True, block_sha512=True),
                   dict(flags=FLAG_BLOCK_SHA512), dict(flags=FLAG_BLOCK_SHA256 | FLAG_BLOCK_SHA512)):
            with pytest.raises(MtzError) as ei:
                GpuSnapshotStage(mode, **kw)
            assert ei.value.code == EINVAL, (mode, kw)
    with pytest.raises(MtzError) as ei:
        _stage("passthrough")
    assert ei.value.code == EINVAL


def test_the_flag_changes_nothing_without_sha512_keys(oracle):
    f, _ = B._mixed(oracle)
    for sha256, s in ((False, f), (True, R.as_sha256(oracle, f))):
        c, _, _ = _run(oracle, "compress", s, sha=False)
        for mode, src in (("verify", s), ("compress", s), ("recompress", s), ("decompress", c),
                          ("recompress", R.as_send_c(oracle, s))):
            a, sa, ba = _run(oracle, mode, src, sha=False, sha256=sha256, batch_bytes=1 << 18)
            b, sb, bb = _run(oracle, mode, src, sha=True, sha256=sha256, batch_bytes=1 << 18)
            assert np.array_equal(a, b), mode
            for k in B.TIMING:
                sa.pop(k); sb.pop(k)
            assert sa == sb, mode
            assert ba == bb and bb["sha512"] == 0, mode
            assert bb["logical_ok"] + bb["frame_ok"] > 0 and (bb["sha256"] > 0) == sha256
