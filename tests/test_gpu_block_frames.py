"""GPU: MTZ_FLAG_BLOCK_FRAMES through the C ABI -- in VERIFY, a block that arrives raw while its key
covers an LZ4 frame on disk is encoded by the declared encoder (K3) beside the batch and compared as
COMPRESS compares its own output, on process_host, the ring API, the device API (sub-batched and
deferred) and a device group.  Every counter is the reference model's (tests/block_ref.py)
and that of a COMPRESS run of the same stream; the output bytes and the non-timing mtz_stats fields
are those of the flag off.  In the other modes the flag changes nothing."""
import numpy as np
import pytest

import block_ref as R
import test_gpu_block_cksum as B

pytestmark = pytest.mark.gpu


def _verify_matches_model_and_compress(oracle, s, nlz4, sha256=False, sha512=False, **kw):
    """VERIFY + frames on `s`: the model's counters, COMPRESS's counters, frame_ok == nlz4"""
    flags = dict(sha256=sha256, sha512=sha512)
    _, _, bs = B._run(oracle, "verify", s, frames=True, **flags, **kw)
    _, want = R.block_check(oracle, s, R.VERIFY, frames=True, **flags)
    B._same(bs, want)
    assert bs["frame_ok"] == bs["frames_encoded"] == nlz4 and bs["skipped"] == 0 and bs["frame_miss"] == 0
    _, _, cs = B._run(oracle, "compress", s, **flags, **kw)
    assert {k: bs[k] for k in R.TRANSFER} == {k: cs[k] for k in R.TRANSFER}
    return bs


@pytest.mark.parametrize("ashift", [9, 12])
@pytest.mark.parametrize("recsize", [512, 8192, 131072, 1 << 20])
def test_lz4_on_disk_keys_match_the_encoder_in_verify(oracle, ashift, recsize):
    s, dcs = B._mixed(oracle, n=12 if recsize >= 131072 else 30, recsize=recsize, ashift=ashift)
    nlz4 = sum(1 for v in dcs.values() if v == R.DC_LZ4)
    assert recsize == 512 or 0 < nlz4 < len(dcs)
    _verify_matches_model_and_compress(oracle, s, nlz4)


def test_sixteen_mib_record(oracle):
    """the largest ZFS block: one K3 warp, and frame sums over several warp_fletcher chunks"""
    s, dcs = R.as_on_disk(oracle, oracle.synth_stream(2, recsize=16 << 20, kind=oracle.PAYLOAD_PGPAGE))
    nlz4 = sum(1 for v in dcs.values() if v == R.DC_LZ4)
    assert nlz4 == 2
    _verify_matches_model_and_compress(oracle, s, nlz4, batch_bytes=64 << 20)


def test_the_output_and_the_stats_are_those_of_the_flag_off(oracle):
    s, _ = B._mixed(oracle)
    for kw in (dict(batch_bytes=1 << 18), {}):
        a, sa, ba = B._run(oracle, "verify", s, **kw)
        b, sb, bb = B._run(oracle, "verify", s, frames=True, **kw)
        assert np.array_equal(a, b)
        assert sa == sb
        assert ba["frames_encoded"] == 0 and bb["frames_encoded"] == ba["skipped"] > 0
        assert bb["logical_ok"] == ba["logical_ok"]


def test_the_flag_without_block_checksums_is_einval(oracle):
    from manatee_b200 import GpuSnapshotStage
    from manatee_b200._native import MtzError, EINVAL, FLAG_BLOCK_FRAMES, FLAG_BLOCK_SHA256
    for mode in ("verify", "compress", "decompress", "recompress", "passthrough"):
        for kw in (dict(block_frames=True), dict(flags=FLAG_BLOCK_FRAMES),
                   dict(flags=FLAG_BLOCK_FRAMES | FLAG_BLOCK_SHA256)):
            with pytest.raises(MtzError) as ei:
                GpuSnapshotStage(mode, **kw)
            assert ei.value.code == EINVAL, (mode, kw)
    with pytest.raises(MtzError) as ei:
        B._stage("passthrough", frames=True)
    assert ei.value.code == EINVAL


def test_swapped_frame_keys_are_counted_not_errors(oracle):
    s, dcs = B._mixed(oracle)
    lz4 = sorted(i for i, v in dcs.items() if v == R.DC_LZ4)
    _, offs = oracle.stream_index(s)
    s = s.copy()
    for i, j in zip(lz4[1:4], lz4[2:5]):
        _, key, p = R.get_key(s, int(offs[j]))
        R.set_key(s, int(offs[i]), key=key, ddk_prop=(p & ~0xffff) | (R.get_key(s, int(offs[i]))[2] & 0xffff))
    assert oracle.stream_restamp(s)[0] == 0
    _, st, bs = B._run(oracle, "verify", s, frames=True)
    _, want = R.block_check(oracle, s, R.VERIFY, frames=True)
    assert want["frame_miss"] == 3 and want["first_frame_miss"] == lz4[1]
    B._same(bs, want)
    assert st["bad_record"] == R.NONE
    _, _, cs = B._run(oracle, "compress", s)
    assert {k: bs[k] for k in R.TRANSFER} == {k: cs[k] for k in R.TRANSFER}


def test_corrupted_then_restamped_records(oracle):
    """an LZ4-keyed record is a frame miss at its index; a record ZFS stored raw still fails with
    the object / offset message"""
    from manatee_b200._native import MtzError, ECKSUM
    s, dcs = B._mixed(oracle, n=40)
    lz4 = sorted(i for i, v in dcs.items() if v == R.DC_LZ4)
    raw = sorted(i for i, v in dcs.items() if v != R.DC_LZ4)
    k = lz4[len(lz4) // 2]
    c = B._corrupt_restamped(oracle, s, k, byte=100)
    _, st, bs = B._run(oracle, "verify", c, batch_bytes=1 << 18, frames=True)
    _, want = R.block_check(oracle, c, R.VERIFY, frames=True)
    assert want["frame_miss"] == 1 and want["first_frame_miss"] == k
    B._same(bs, want)
    assert st["bad_record"] == R.NONE
    k = raw[len(raw) // 2]
    c = B._corrupt_restamped(oracle, s, k, byte=100)
    _, offs = oracle.stream_index(c)
    w = np.frombuffer(c[int(offs[k]) + 8:int(offs[k]) + 32].tobytes(), dtype="<u8")
    obj, off = int(w[0]), int(w[2])                # drr_object, drr_offset
    with B._stage("verify", batch_bytes=1 << 18, frames=True) as g:
        with pytest.raises(MtzError) as ei:
            g.process_host(c)
        assert ei.value.code == ECKSUM and g.stats()["bad_record"] == k
        assert "block checksum mismatch at record %d (object %d, offset %d)" % (k, obj, off) in str(ei.value)


@pytest.mark.parametrize("ashift", [9, 12])
def test_sha256_and_sha512_lz4_on_disk_keys(oracle, ashift):
    s, dcs = B._mixed(oracle, n=24, ashift=ashift)
    nlz4 = sum(1 for v in dcs.values() if v == R.DC_LZ4)
    for name, src in (("sha256", R.as_sha(oracle, s, "sha256")), ("sha512", R.as_sha(oracle, s, "sha512"))):
        bs = _verify_matches_model_and_compress(oracle, src, nlz4, **{name: True})
        assert bs[name] == len(dcs)
        # without the hash's flag the records stay skipped: nothing is encoded for them
        _, _, off = B._run(oracle, "verify", src, frames=True)
        assert off["frames_encoded"] == 0 and off["skipped"] == len(dcs)


def test_send_c_stream_the_flag_changes_nothing(oracle):
    s, _ = B._mixed(oracle)
    c = R.as_send_c(oracle, s)
    a, sa, ba = B._run(oracle, "verify", c)
    b, sb, bb = B._run(oracle, "verify", c, frames=True)
    assert np.array_equal(a, b)
    assert sa == sb and ba == bb and bb["frames_encoded"] == 0 and bb["frame_ok"] > 0


def test_the_other_modes_are_unchanged(oracle):
    s, _ = B._mixed(oracle)
    c, _, _ = B._run(oracle, "compress", s)
    for mode, src in (("compress", s), ("recompress", s), ("decompress", c),
                      ("recompress", R.as_send_c(oracle, s))):
        a, sa, ba = B._run(oracle, mode, src, batch_bytes=1 << 18)
        b, sb, bb = B._run(oracle, mode, src, frames=True, batch_bytes=1 << 18)
        assert np.array_equal(a, b), mode
        assert sa == sb and ba == bb and bb["frames_encoded"] == 0, mode


@pytest.mark.parametrize("chunk", [4093, 1 << 20])
def test_ring_api(oracle, chunk):
    s, dcs = B._mixed(oracle)
    nlz4 = sum(1 for v in dcs.values() if v == R.DC_LZ4)
    _, want = R.block_check(oracle, s, R.VERIFY, frames=True)
    for kw in (dict(batch_bytes=1 << 18), {}):
        with B._stage("verify", frames=True, **kw) as g:
            out, err = B._pump(g, s.tobytes(), chunk)
            assert not err, err
            assert out == s.tobytes()
            B._same(g.block_stats(), want)
            assert want["frames_encoded"] == nlz4


def device_api_subbatched(oracle, mem, nrec):
    """VERIFY on the device API over more records than one frame sub-batch holds, and a frame miss
    and a logical mismatch near the end"""
    from manatee_b200 import index_host
    from manatee_b200._native import MtzError, ECKSUM
    s, dcs = B._mixed(oracle, n=nrec, recsize=4096)
    lz4 = sorted(i for i, v in dcs.items() if v == R.DC_LZ4)
    raw = sorted(i for i, v in dcs.items() if v != R.DC_LZ4)
    miss = B._corrupt_restamped(oracle, s, lz4[-2], byte=100)
    bad = B._corrupt_restamped(oracle, s, raw[-2], byte=100)
    for src, fails in ((s, False), (miss, False), (bad, True)):
        recs, _ = index_host(src)
        d_in, p_in = mem.put(src)
        d_recs, p_recs = mem.put(recs.view(np.uint8))
        with B._stage("verify", frames=True) as g:
            g.dev_submit(p_in, src.size, p_recs, len(recs))
            if fails:
                with pytest.raises(MtzError) as ei:
                    g.dev_finish()
                assert ei.value.code == ECKSUM and g.stats()["bad_record"] == raw[-2]
            else:
                g.dev_finish()
                _, want = R.block_check(oracle, src, R.VERIFY, frames=True)
                assert want["frames_encoded"] == len(lz4)
                B._same(g.block_stats(), want)


def test_device_api_across_the_subbatch_edge(oracle):
    device_api_subbatched(oracle, B.TorchMem(), 66000)


def test_deferred_shards(oracle):
    from manatee_b200 import index_host
    from manatee_b200._native import FLAG_DEFER_VERIFY, MtzError, ECKSUM
    s, dcs = B._mixed(oracle, n=60)
    lz4 = sorted(i for i, v in dcs.items() if v == R.DC_LZ4)
    raw = sorted(i for i, v in dcs.items() if v != R.DC_LZ4)
    recs, _ = index_host(s)
    cut = int(recs["off"][31])
    _, want = R.block_check(oracle, s, R.VERIFY, frames=True)
    late_lz4 = [i for i in lz4 if i > 31][0]
    late_raw = [i for i in raw if i > 31][0]
    for bad_rec, miss in ((None, None), (late_raw, None), (None, late_lz4)):
        src = s
        if bad_rec is not None:
            src = B._corrupt_restamped(oracle, s, bad_rec)
        if miss is not None:
            src = B._corrupt_restamped(oracle, s, miss, byte=100)
        gs = [B._stage("verify", batch_bytes=1 << 18, flags=FLAG_DEFER_VERIFY, frames=True) for _ in range(2)]
        try:
            gs[0].process_host(src[:cut]); gs[1].process_host(src[cut:])
            a0 = gs[0].dev_aggregate()
            c1 = oracle.fletcher4_apply((0, 0, 0, 0), (a0[0] & ((1 << 63) - 1),) + a0[1:])
            gs[0].dev_finish(carry_in=(0, 0, 0, 0))
            if bad_rec is not None:
                with pytest.raises(MtzError) as ei:
                    gs[1].dev_finish(carry_in=c1)
                assert ei.value.code == ECKSUM and "block checksum" in str(ei.value)
                assert gs[1].stats()["bad_record"] + 31 == bad_rec
                continue
            gs[1].dev_finish(carry_in=c1)
            b0, b1 = gs[0].block_stats(), gs[1].block_stats()
            assert b0["frames_encoded"] + b1["frames_encoded"] == len(lz4)
            if miss is None:
                assert b0["frame_ok"] + b1["frame_ok"] == want["frame_ok"] == len(lz4)
            else:
                assert b1["frame_miss"] == 1 and b1["first_frame_miss"] + 31 == miss
        finally:
            for g in gs:
                g.close()


def test_device_group(oracle):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    s, _ = B._mixed(oracle)
    _, want = R.block_check(oracle, s, R.VERIFY, frames=True)
    _, _, bs = B._run(oracle, "verify", s, devices=[0, 1], batch_bytes=1 << 18, frames=True)
    B._same(bs, want)
