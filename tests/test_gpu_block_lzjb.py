"""GPU: MTZ_FLAG_BLOCK_LZJB through the C ABI -- keys over an lzjb (on-disk compression 3) or zle (14)
frame.  In VERIFY a block that arrives raw is encoded by the declared encoders (k_lzjb_encode,
k_zle_encode) beside the batch and compared as the LZ4 frames of MTZ_FLAG_BLOCK_FRAMES are; a block
that arrives as its frame (`send -c`) is compared as it is, in VERIFY and RECOMPRESS.  Covered on
process_host, the ring API, the device API (sub-batched and deferred) and a device group.  Every
counter is the reference model's (tests/block_ref.py); the output bytes and the non-timing
mtz_stats fields are those of the flag off."""
import glob
import os

import numpy as np
import pytest

import block_ref as R
import test_gpu_block_cksum as B

pytestmark = pytest.mark.gpu


def _mixed(oracle, n=30, recsize=8192, ashift=9, codec=R.mixed_codecs):
    """pg-page records with incompressible and all-zero ones mixed in, keyed by lzjb, zle, lz4 and
    logical keys in turn"""
    from test_gpu_codec import _mixed_stream
    return R.as_on_disk(oracle, _mixed_stream(oracle, n=n, recsize=recsize), ashift, codec)


def _count(dcs, dc):
    return sum(1 for v in dcs.values() if v == dc)


def _verify_matches_model(oracle, s, dcs, frames=False, sha256=False, sha512=False, **kw):
    """VERIFY + lzjb on `s`: the model's counters; every lzjb / zle key is frame_ok"""
    flags = dict(lzjb=True, frames=frames, sha256=sha256, sha512=sha512)
    _, st, bs = B._run(oracle, "verify", s, **flags, **kw)
    _, want = R.block_check(oracle, s, R.VERIFY, **flags)
    B._same(bs, want)
    assert bs["lzjb_encoded"] == _count(dcs, R.DC_LZJB) and bs["zle_encoded"] == _count(dcs, R.DC_ZLE)
    assert bs["frames_encoded"] == (_count(dcs, R.DC_LZ4) if frames else 0)
    assert bs["frame_miss"] == 0 and st["bad_record"] == R.NONE
    return bs


@pytest.mark.parametrize("frames", [False, True])
@pytest.mark.parametrize("ashift", [9, 12])
@pytest.mark.parametrize("recsize", [512, 8192, 131072, 1 << 20])
def test_lzjb_and_zle_keys_match_the_encoders_in_verify(oracle, recsize, ashift, frames):
    s, dcs = _mixed(oracle, n=12 if recsize >= 131072 else 30, recsize=recsize, ashift=ashift)
    if recsize > 512 and not (ashift == 12 and recsize == 8192):
        assert _count(dcs, R.DC_LZJB) > 0 and _count(dcs, R.DC_ZLE) > 0
    bs = _verify_matches_model(oracle, s, dcs, frames=frames)
    assert bs["skipped"] == (0 if frames else _count(dcs, R.DC_LZ4))


def test_sixteen_mib_record(oracle):
    """the largest ZFS block: one encoder warp per record, frame sums over several warp_fletcher chunks"""
    for codec in (R.DC_LZJB, R.DC_ZLE):
        src = oracle.synth_stream(2, recsize=16 << 20, kind=oracle.PAYLOAD_PGPAGE)
        s, dcs = R.as_on_disk(oracle, src, 9, codec)
        assert _count(dcs, codec) == 2
        _verify_matches_model(oracle, s, dcs, batch_bytes=64 << 20)


def test_the_output_and_the_stats_are_those_of_the_flag_off(oracle):
    s, dcs = _mixed(oracle)
    for kw in (dict(batch_bytes=1 << 18), {}):
        a, sa, ba = B._run(oracle, "verify", s, **kw)
        b, sb, bb = B._run(oracle, "verify", s, lzjb=True, **kw)
        assert np.array_equal(a, b)
        assert sa == sb
        assert ba["lzjb_encoded"] == ba["zle_encoded"] == 0
        assert bb["lzjb_encoded"] + bb["zle_encoded"] == ba["skipped"] - bb["skipped"] > 0
        assert bb["logical_ok"] == ba["logical_ok"]


def test_the_flag_without_block_checksums_is_einval(oracle):
    from manatee_b200 import GpuSnapshotStage
    from manatee_b200._native import MtzError, EINVAL, FLAG_BLOCK_FRAMES, FLAG_BLOCK_LZJB
    for mode in ("verify", "compress", "decompress", "recompress", "passthrough"):
        for kw in (dict(block_lzjb=True), dict(flags=FLAG_BLOCK_LZJB), dict(flags=FLAG_BLOCK_LZJB | FLAG_BLOCK_FRAMES)):
            with pytest.raises(MtzError) as ei:
                GpuSnapshotStage(mode, **kw)
            assert ei.value.code == EINVAL, (mode, kw)
    with pytest.raises(MtzError) as ei:
        B._stage("passthrough", lzjb=True)
    assert ei.value.code == EINVAL


def test_swapped_keys_are_counted_not_errors(oracle):
    s, dcs = _mixed(oracle, n=40)
    comp = sorted(i for i, v in dcs.items() if v in (R.DC_LZJB, R.DC_ZLE))
    _, offs = oracle.stream_index(s)
    s = s.copy()
    for i, j in zip(comp[1:4], comp[2:5]):
        _, key, p = R.get_key(s, int(offs[j]))
        R.set_key(s, int(offs[i]), key=key, ddk_prop=(p & ~0xffff) | (R.get_key(s, int(offs[i]))[2] & 0xffff))
    assert oracle.stream_restamp(s)[0] == 0
    for frames in (False, True):
        _, st, bs = B._run(oracle, "verify", s, frames=frames, lzjb=True)
        _, want = R.block_check(oracle, s, R.VERIFY, lzjb=True, frames=frames)
        assert want["frame_miss"] == 3 and want["first_frame_miss"] == comp[1]
        B._same(bs, want)
        assert st["bad_record"] == R.NONE


def test_corrupted_then_restamped_records(oracle):
    """an lzjb- or zle-keyed record is a frame miss at its index, never an error"""
    s, dcs = _mixed(oracle, n=40)
    for dc in (R.DC_LZJB, R.DC_ZLE):
        idx = sorted(i for i, v in dcs.items() if v == dc)
        k = idx[len(idx) // 2]
        c = B._corrupt_restamped(oracle, s, k, byte=100)
        _, st, bs = B._run(oracle, "verify", c, batch_bytes=1 << 18, lzjb=True)
        _, want = R.block_check(oracle, c, R.VERIFY, lzjb=True)
        assert want["frame_miss"] == 1 and want["first_frame_miss"] == k
        B._same(bs, want)
        assert st["bad_record"] == R.NONE


@pytest.mark.parametrize("name", ["sha256", "sha512"])
def test_sha256_and_sha512_keys(oracle, name):
    s, dcs = _mixed(oracle, n=24)
    src = R.as_sha(oracle, s, name)
    for frames in (False, True):
        bs = _verify_matches_model(oracle, src, dcs, frames=frames, **{name: True})
        assert bs[name] == len(dcs) - (0 if frames else _count(dcs, R.DC_LZ4))
    # without the hash's flag the records stay skipped: nothing is encoded for them
    _, _, off = B._run(oracle, "verify", src, lzjb=True)
    assert off["lzjb_encoded"] == off["zle_encoded"] == 0 and off["skipped"] == len(dcs)


@pytest.mark.parametrize("mode", ["verify", "recompress"])
def test_send_c_stream_frames_checked_as_they_arrive(oracle, mode):
    s, dcs = _mixed(oracle)
    c = R.as_send_c(oracle, s)
    a, sa, ba = B._run(oracle, mode, c)
    b, sb, bb = B._run(oracle, mode, c, lzjb=True)
    assert np.array_equal(a, b)
    assert sa == sb
    ncomp = _count(dcs, R.DC_LZJB) + _count(dcs, R.DC_ZLE)
    assert bb["lzjb_encoded"] == bb["zle_encoded"] == 0
    assert bb["frame_ok"] == ba["frame_ok"] + ncomp and bb["skipped"] == ba["skipped"] - ncomp
    B._same(bb, B._want(oracle, mode, c, b, lzjb=True)[1])


def test_compress_and_decompress_are_unchanged(oracle):
    s, _ = _mixed(oracle)
    c, _, _ = B._run(oracle, "compress", s)
    for mode, src in (("compress", s), ("decompress", c), ("recompress", s)):
        a, sa, ba = B._run(oracle, mode, src, batch_bytes=1 << 18)
        b, sb, bb = B._run(oracle, mode, src, batch_bytes=1 << 18, lzjb=True)
        assert np.array_equal(a, b), mode
        assert sa == sb and ba == bb and bb["lzjb_encoded"] == bb["zle_encoded"] == 0, mode


@pytest.mark.parametrize("chunk", [4093, 1 << 20])
def test_ring_api(oracle, chunk):
    s, dcs = _mixed(oracle)
    _, want = R.block_check(oracle, s, R.VERIFY, lzjb=True)
    for kw in (dict(batch_bytes=1 << 18), {}):
        with B._stage("verify", lzjb=True, **kw) as g:
            out, err = B._pump(g, s.tobytes(), chunk)
            assert not err, err
            assert out == s.tobytes()
            B._same(g.block_stats(), want)
            assert want["lzjb_encoded"] == _count(dcs, R.DC_LZJB) > 0


def device_api_subbatched(oracle, mem, nrec):
    """VERIFY on the device API over more records than one frame sub-batch holds, a frame miss near
    the end, and a logical mismatch near the end"""
    from manatee_b200 import index_host
    from manatee_b200._native import MtzError, ECKSUM
    s, dcs = _mixed(oracle, n=nrec, recsize=4096)
    comp = sorted(i for i, v in dcs.items() if v in (R.DC_LZJB, R.DC_ZLE))
    raw = sorted(i for i, v in dcs.items() if v == R.DC_OFF)
    miss = B._corrupt_restamped(oracle, s, comp[-2], byte=100)
    bad = B._corrupt_restamped(oracle, s, raw[-2], byte=100)
    for src, fails in ((s, False), (miss, False), (bad, True)):
        recs, _ = index_host(src)
        d_in, p_in = mem.put(src)
        d_recs, p_recs = mem.put(recs.view(np.uint8))
        with B._stage("verify", lzjb=True) as g:
            g.dev_submit(p_in, src.size, p_recs, len(recs))
            if fails:
                with pytest.raises(MtzError) as ei:
                    g.dev_finish()
                assert ei.value.code == ECKSUM and g.stats()["bad_record"] == raw[-2]
            else:
                g.dev_finish()
                _, want = R.block_check(oracle, src, R.VERIFY, lzjb=True)
                assert want["lzjb_encoded"] + want["zle_encoded"] == len(comp)
                B._same(g.block_stats(), want)


def test_device_api_across_the_subbatch_edge(oracle):
    device_api_subbatched(oracle, B.TorchMem(), 66000)


def test_deferred_shards(oracle):
    from manatee_b200 import index_host
    from manatee_b200._native import FLAG_DEFER_VERIFY
    s, dcs = _mixed(oracle, n=60)
    comp = sorted(i for i, v in dcs.items() if v in (R.DC_LZJB, R.DC_ZLE))
    recs, _ = index_host(s)
    cut = int(recs["off"][31])
    late = [i for i in comp if i > 31][0]
    for miss in (None, late):
        src = s if miss is None else B._corrupt_restamped(oracle, s, miss, byte=100)
        _, want = R.block_check(oracle, src, R.VERIFY, lzjb=True)
        gs = [B._stage("verify", batch_bytes=1 << 18, flags=FLAG_DEFER_VERIFY, lzjb=True) for _ in range(2)]
        try:
            gs[0].process_host(src[:cut]); gs[1].process_host(src[cut:])
            a0 = gs[0].dev_aggregate()
            c1 = oracle.fletcher4_apply((0, 0, 0, 0), (a0[0] & ((1 << 63) - 1),) + a0[1:])
            gs[0].dev_finish(carry_in=(0, 0, 0, 0))
            gs[1].dev_finish(carry_in=c1)
            b0, b1 = gs[0].block_stats(), gs[1].block_stats()
            assert b0["lzjb_encoded"] + b1["lzjb_encoded"] + b0["zle_encoded"] + b1["zle_encoded"] == len(comp)
            assert b0["frame_ok"] + b1["frame_ok"] == want["frame_ok"]
            if miss is not None:
                assert b1["frame_miss"] == 1 and b1["first_frame_miss"] + 31 == miss
        finally:
            for g in gs:
                g.close()


def test_device_group(oracle):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    s, _ = _mixed(oracle)
    _, want = R.block_check(oracle, s, R.VERIFY, lzjb=True)
    _, _, bs = B._run(oracle, "verify", s, devices=[0, 1], batch_bytes=1 << 18, lzjb=True)
    B._same(bs, want)


def test_real_streams_with_lzjb_or_zle_keys(oracle):
    """a real stream from a pool with lzjb / zle blocks: every such frame matches the encoders"""
    paths = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "real", "*.zstream")))
    found = False
    for p in paths:
        s = np.fromfile(p, dtype=np.uint8)
        keyed = [i for i, (off, _, _, t) in enumerate(R.records(s))
                 if t == 3 and R.unprop(R.get_key(s, off)[2])[2] in (R.DC_LZJB, R.DC_ZLE)]
        if not keyed:
            continue
        found = True
        _, st, bs = B._run(oracle, "verify", s, sha256=True, sha512=True, lzjb=True)
        assert bs["frame_miss"] == 0, (p, bs)
    if not found:
        pytest.skip("no real stream with lzjb or zle keys under tests/golden/real")
