"""GPU: MTZ_FLAG_BLOCK_SHA256 through the C ABI -- the block-checksum check (MTZ_FLAG_BLOCK_CKSUM)
extended to SHA-256 keys (checksum=sha256), hashed on the device by k_block_sha256, on
process_host, the ring API, the device API (sub-batched and deferred) and a device group.  Every
counter is the reference model's (tests/block_ref.py, hashlib), and the semantics are the
fletcher4 check's: a block stored raw on disk must equal its logical bytes, a frame is only counted.
Without the new flag sha256 keys are skipped, and on a fletcher-only stream the flag changes nothing."""
import numpy as np
import pytest

import block_ref as R
import test_gpu_block_cksum as B

pytestmark = pytest.mark.gpu


def _sha_raw(oracle, n=24, recsize=8192, kind=None):
    """a generator stream re-keyed as written with checksum=sha256, compression=off"""
    s = oracle.synth_stream(n, recsize=recsize, kind=kind or oracle.PAYLOAD_PGPAGE).copy()
    for off, _, pl, t in R.records(s):
        if t == 3 and R.get_key(s, off)[2] == 0:      # the generator's 512-byte blocks carry prop 0
            R.set_key(s, off, ddk_prop=R.prop(pl, pl, R.DC_OFF))
    return R.as_sha(oracle, s, "sha256")


def _sha_mixed(oracle, n=30, recsize=8192, ashift=9):
    s, dcs = B._mixed(oracle, n=n, recsize=recsize, ashift=ashift)
    return R.as_sha(oracle, s, "sha256"), dcs


def test_sha256_keys_match_in_every_mode(oracle):
    s = _sha_raw(oracle)
    for mode in ("verify", "compress", "recompress"):
        out, _, bs = B._run(oracle, mode, s, sha256=True)
        _, want = B._want(oracle, mode, s, out, sha256=True)
        assert want["logical_ok"] == want["sha256"] == 24 and want["skipped"] == 0
        B._same(bs, want)
        if mode == "compress":
            c = out
    d, _, bs = B._run(oracle, "decompress", c, sha256=True)
    assert np.array_equal(d, s)
    _, want = B._want(oracle, "decompress", c, d, sha256=True)
    assert want["logical_ok"] == want["sha256"] == 24 and want["skipped"] == 0
    B._same(bs, want)


def test_corrupted_then_restamped_block_fails_only_with_the_flag(oracle):
    s = B._corrupt_restamped(oracle, _sha_raw(oracle, n=40, recsize=16384), 17)
    _, want = R.block_check(oracle, s, R.VERIFY, sha256=True)
    assert want["first_bad"] == 17
    # BLOCK_CKSUM alone: every record is skipped, the stream passes
    _, _, bs = B._run(oracle, "verify", s)
    _, want = R.block_check(oracle, s, R.VERIFY)
    assert want["skipped"] == 40 and bs["sha256"] == 0
    B._same(bs, want)
    c, _, _ = B._run(oracle, "compress", s)
    for mode, src in (("verify", s), ("compress", s), ("recompress", s), ("decompress", c)):
        msg = B._fails(mode, src, 17, batch_bytes=1 << 18, sha256=True)
        assert "block checksum mismatch at record 17 (object 8, offset %d)" % (15 * 16384) in msg, msg
        assert "sha256" in msg, msg
    # a fletcher4 key labelled sha256 (tests/test_gpu_block_cksum.py's skipped class) is compared now
    f = B._raw_stream(oracle, n=12).copy()
    _, offs = oracle.stream_index(f)
    R.set_key(f, int(offs[3]), ctype=R.SHA256)
    assert oracle.stream_restamp(f)[0] == 0
    B._run(oracle, "verify", f)
    B._fails("verify", f, 3, sha256=True)


def test_fletcher4_failure_message_names_no_type(oracle):
    s = B._corrupt_restamped(oracle, B._raw_stream(oracle, n=12), 5)
    msg = B._fails("verify", s, 5, sha256=True)
    assert "offset 24576): the bytes differ from the block on disk" in msg and "sha256" not in msg, msg


@pytest.mark.parametrize("ashift", [9, 12])
def test_lz4_on_disk_sha256_keys(oracle, ashift):
    """frame_ok for the stage's encoder output (COMPRESS, RECOMPRESS) and for `send -c` input
    (VERIFY, RECOMPRESS), including frames shorter than PSIZE that end inside a 64-byte block"""
    s, dcs = _sha_mixed(oracle, n=24, ashift=ashift)
    nlz4 = sum(1 for v in dcs.values() if v == R.DC_LZ4)
    assert 0 < nlz4 < len(dcs)
    for mode in ("compress", "recompress"):
        out, _, bs = B._run(oracle, mode, s, sha256=True)
        _, want = B._want(oracle, mode, s, out, sha256=True)
        assert want["frame_ok"] == nlz4 and want["frame_miss"] == 0 and want["sha256"] == len(dcs)
        B._same(bs, want)
    c = R.as_send_c(oracle, s, ashift)
    for src in (c, R.trim_frames(oracle, c)):
        for mode in ("verify", "recompress"):
            ref, _, _ = B._run(oracle, mode, src)
            out, _, bs = B._run(oracle, mode, src, sha256=True)
            assert np.array_equal(out, ref)
            _, want = B._want(oracle, mode, src, out, sha256=True)
            assert want["frame_ok"] == nlz4 and want["frame_miss"] == 0
            B._same(bs, want)


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
        ref, _, _ = B._run(oracle, mode, s)
        out, _, bs = B._run(oracle, mode, s, sha256=True)
        assert np.array_equal(out, ref)
        _, want = B._want(oracle, mode, s, out, sha256=True)
        assert want["frame_miss"] == 3 and want["first_frame_miss"] == lz4[1]
        B._same(bs, want)


def _mixed_types(oracle):
    """fletcher4 keys, sha256 keys and every skipped class in one stream"""
    f, dcs = B._mixed(oracle, n=40)
    h = R.as_sha(oracle, f, "sha256")
    s = f.copy()
    recs = R.records(s)
    w = [i for i, r in enumerate(recs) if r[3] == 3]
    for i in w[1::2]:                              # every other record: its sha256 key
        s[recs[i][0] + 48:recs[i][0] + 88] = h[recs[i][0] + 48:recs[i][0] + 88]
    R.set_key(s, recs[w[3]][0], ddk_prop=0)
    R.set_key(s, recs[w[5]][0], ddk_prop=R.prop(8192, 4096, R.DC_ZSTD))
    R.set_key(s, recs[w[6]][0], ddk_prop=R.prop(8192, 8192, R.DC_OFF, crypt=1))
    R.set_key(s, recs[w[8]][0], ctype=9)           # sha512: not checked
    assert oracle.stream_restamp(s)[0] == 0
    return s


def test_one_stream_mixing_fletcher4_sha256_and_skipped_keys(oracle):
    s = _mixed_types(oracle)
    c, _, _ = B._run(oracle, "compress", s)
    for mode, src in (("verify", s), ("compress", s), ("recompress", s), ("decompress", c),
                      ("verify", R.as_send_c(oracle, s)), ("recompress", R.as_send_c(oracle, s))):
        out, _, bs = B._run(oracle, mode, src, batch_bytes=1 << 17, sha256=True)
        _, want = B._want(oracle, mode, src, out, sha256=True)
        assert want["sha256"] > 0 and want["skipped"] >= 4 and want["logical_ok"] + want["frame_ok"] > want["sha256"]
        B._same(bs, want)


@pytest.mark.parametrize("recsize", [512, 8192, 131072, 1 << 20])
def test_record_sizes(oracle, recsize):
    s = _sha_raw(oracle, n=6, recsize=recsize)
    for mode in ("verify", "compress"):
        out, _, bs = B._run(oracle, mode, s, sha256=True)
        _, want = B._want(oracle, mode, s, out, sha256=True)
        assert want["logical_ok"] == want["sha256"] == 6
        B._same(bs, want)
    msg = B._fails("verify", B._corrupt_restamped(oracle, s, 4, byte=recsize - 1), 4, sha256=True)
    assert "sha256" in msg


def test_sixteen_mib_record(oracle):
    """the largest ZFS block: one thread hashes 16 MiB + one padding block"""
    s = _sha_raw(oracle, n=1, recsize=16 << 20, kind=oracle.PAYLOAD_PCG)
    _, _, bs = B._run(oracle, "verify", s, batch_bytes=32 << 20, sha256=True)
    _, want = R.block_check(oracle, s, R.VERIFY, sha256=True)
    assert want["logical_ok"] == want["sha256"] == 1
    B._same(bs, want)
    B._fails("verify", B._corrupt_restamped(oracle, s, 2, byte=(16 << 20) - 8), 2, batch_bytes=32 << 20, sha256=True)


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
        assert what in B._fails("verify", s, rec, sha256=True)


@pytest.mark.parametrize("chunk", [4093, 1 << 20])
def test_ring_api(oracle, chunk):
    from manatee_b200._native import MtzError, ECKSUM
    s, _ = _sha_mixed(oracle)
    c = R.as_send_c(oracle, s)
    for mode in ("verify", "recompress"):
        with B._stage(mode, batch_bytes=1 << 18, sha256=True) as g:
            out, err = B._pump(g, c.tobytes(), chunk)
            assert not err, err
            _, want = B._want(oracle, mode, c, np.frombuffer(out, dtype=np.uint8), sha256=True)
            assert want["sha256"] > 0
            B._same(g.block_stats(), want)
    bad = B._corrupt_restamped(oracle, _sha_raw(oracle, n=40), 20)
    _, offs = oracle.stream_index(bad)
    with B._stage("verify", batch_bytes=1 << 16, sha256=True) as g:
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
        with B._stage("decompress", sha256=True) as g:
            g.dev_submit(p_in, c.size, p_recs, len(recs), p_out, cap)
            if bad is None:
                ob, _, _ = g.dev_finish()
                _, want = R.block_check(oracle, c, R.DECOMPRESS, mem.get(d_out, ob), sha256=True)
                assert want["logical_ok"] == want["sha256"] == nrec
                B._same(g.block_stats(), want)
            else:
                with pytest.raises(MtzError) as ei:
                    g.dev_finish()
                assert ei.value.code == ECKSUM and "sha256" in str(ei.value)
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
        gs = [B._stage("verify", batch_bytes=1 << 18, flags=FLAG_DEFER_VERIFY, sha256=True) for _ in range(2)]
        try:
            gs[0].process_host(src[:cut]); gs[1].process_host(src[cut:])
            a0 = gs[0].dev_aggregate()
            c1 = oracle.fletcher4_apply((0, 0, 0, 0), (a0[0] & ((1 << 63) - 1),) + a0[1:])
            for k, carry in ((0, (0, 0, 0, 0)), (1, c1)):
                if fails == k:
                    with pytest.raises(MtzError) as ei:
                        gs[k].dev_finish(carry_in=carry)
                    assert ei.value.code == ECKSUM and "sha256" in str(ei.value)
                    assert gs[k].stats()["bad_record"] + 31 * k == bad_rec
                else:
                    gs[k].dev_finish(carry_in=carry)
            if fails is None:
                assert sum(g.block_stats()["sha256"] for g in gs) == 60
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
        out, _, bs = B._run(oracle, mode, c, devices=[0, 1], batch_bytes=1 << 18, sha256=True)
        _, want = B._want(oracle, mode, c, out, sha256=True)
        B._same(bs, want)


def test_the_flag_without_block_checksums_is_einval(oracle):
    from manatee_b200 import GpuSnapshotStage
    from manatee_b200._native import MtzError, EINVAL, FLAG_BLOCK_SHA256
    for mode in ("verify", "compress", "passthrough"):
        with pytest.raises(MtzError) as ei:
            GpuSnapshotStage(mode, block_sha256=True)
        assert ei.value.code == EINVAL
        with pytest.raises(MtzError) as ei:
            GpuSnapshotStage(mode, flags=FLAG_BLOCK_SHA256)
        assert ei.value.code == EINVAL
    with pytest.raises(MtzError) as ei:
        B._stage("passthrough", sha256=True)
    assert ei.value.code == EINVAL


def test_the_flag_changes_nothing_on_a_fletcher_only_stream(oracle):
    s, _ = B._mixed(oracle)
    c, _, _ = B._run(oracle, "compress", s)
    for mode, src in (("verify", s), ("compress", s), ("recompress", s), ("decompress", c),
                      ("recompress", R.as_send_c(oracle, s))):
        a, sa, ba = B._run(oracle, mode, src, batch_bytes=1 << 18)
        b, sb, bb = B._run(oracle, mode, src, sha256=True, batch_bytes=1 << 18)
        assert np.array_equal(a, b), mode
        assert sa == sb, mode
        assert ba == bb and bb["sha256"] == 0, mode
        assert bb["logical_ok"] + bb["frame_ok"] > 0
