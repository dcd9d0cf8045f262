"""GPU: MTZ_FLAG_BLOCK_LOGICAL through the C ABI -- the re-encoding modes check keys from the logical
bytes they hold.  The invariant: a raw stream with a mix of keys counts the same in VERIFY (with
MTZ_FLAG_BLOCK_FRAMES, which gives VERIFY the frames COMPRESS has anyway) and, with the flag, in
COMPRESS on it, in DECOMPRESS on the COMPRESS output and in RECOMPRESS on its compressed form, for
every subset of the SHA and lzjb flags.  A raw-keyed record corrupted inside its LZ4 frame fails a
RECOMPRESS relay with the flag and travels on without it.  Covered on process_host, the ring API and
the device API (sub-batched and deferred shards).  Every counter is the reference model's
(tests/block_ref.py); the output bytes and the non-timing mtz_stats fields are those of the
flag off."""
import itertools

import numpy as np
import pytest

import block_ref as R
import test_gpu_block_cksum as B

pytestmark = pytest.mark.gpu

MODES = ("compress", "decompress", "recompress")
SUBSETS = [dict(zip(("sha256", "sha512", "lzjb"), v)) for v in itertools.product((False, True), repeat=3)]
ALL = dict(sha256=True, sha512=True, lzjb=True)
ON = dict(frames=True, logical=True, **ALL)         # every flag: the stage of the invariant
OFF = dict(frames=True, **ALL)                      # the same without MTZ_FLAG_BLOCK_LOGICAL


def _same_as_verify(bs, v):
    assert {k: bs[k] for k in R.TRANSFER} == {k: v[k] for k in R.TRANSFER}, (bs, v)


def _inputs(oracle, x):
    """the input of each stage of the invariant: COMPRESS takes x, DECOMPRESS the wire form of COMPRESS(x),
    RECOMPRESS the compressed form of x"""
    rc, wire, _ = oracle.stream_compress(x)
    assert rc == 0
    return {"compress": x, "decompress": np.ascontiguousarray(wire), "recompress": R.send_c_form(oracle, x)}


@pytest.mark.parametrize("flags", SUBSETS, ids=lambda f: "+".join(k for k in f if f[k]) or "fletcher4")
def test_the_compressed_wire_counts_what_verify_counts(oracle, flags):
    x, dcs = R.mixed_keys_stream(oracle, n=48)
    want = R.four_ways(oracle, x, frames=True, **flags)
    _, _, v = B._run(oracle, "verify", x, frames=True, **flags)
    B._same(v, want["verify"][1])
    assert v["skipped"] < len(dcs) and (not flags["lzjb"] or v["lzjb_encoded"] > 0 < v["zle_encoded"])
    for mode, src in _inputs(oracle, x).items():
        for kw in (dict(batch_bytes=1 << 18), {})[:2 if flags == ALL else 1]:
            a, sa, ba = B._run(oracle, mode, src, frames=True, **flags, **kw)
            b, sb, bb = B._run(oracle, mode, src, frames=True, logical=True, **flags, **kw)
            assert np.array_equal(a, b) and sa == sb, mode
            B._same(bb, want[mode][1])
            _same_as_verify(bb, v)
            assert ba["logical_checked"] == 0 and bb["frames_encoded"] == 0
            assert bb["logical_checked"] == ba["skipped"] - bb["skipped"], (mode, ba, bb)
        assert bb["logical_checked"] > 0 or mode != "recompress" and not flags["lzjb"], (mode, bb)


def test_without_the_flag_the_modes_count_what_they_did(oracle):
    x, _ = R.mixed_keys_stream(oracle, n=30)
    for mode, src in _inputs(oracle, x).items():
        out, _, bs = B._run(oracle, mode, src, **OFF)
        B._same(bs, B._want(oracle, mode, src, out, **OFF)[1])
        assert bs["logical_checked"] == 0


def test_verify_accepts_the_flag_and_does_not_change(oracle):
    x, _ = R.mixed_keys_stream(oracle, n=30)
    for src in (x, R.send_c_form(oracle, x)):
        a, sa, ba = B._run(oracle, "verify", src, **OFF)
        b, sb, bb = B._run(oracle, "verify", src, **ON)
        assert np.array_equal(a, b) and sa == sb and ba == bb and bb["logical_checked"] == 0


def test_the_flag_without_block_checksums_is_einval(oracle):
    from manatee_b200 import GpuSnapshotStage
    from manatee_b200._native import MtzError, EINVAL, FLAG_BLOCK_LOGICAL, FLAG_BLOCK_LZJB
    for mode in ("verify", "compress", "decompress", "recompress", "passthrough"):
        for kw in (dict(block_logical=True), dict(flags=FLAG_BLOCK_LOGICAL), dict(flags=FLAG_BLOCK_LOGICAL | FLAG_BLOCK_LZJB)):
            with pytest.raises(MtzError) as ei:
                GpuSnapshotStage(mode, **kw)
            assert ei.value.code == EINVAL, (mode, kw)


def _corrupt_a_literal(oracle, c, k):
    """flip a bit of the first literal byte of the LZ4 frame of record k (the frame still decodes to
    lsize: a literal is copied as it is), then re-stamp: every stream checksum holds again"""
    c = c.copy()
    _, offs = oracle.stream_index(c)
    o = int(offs[k])
    assert c[o + 50] == R.DC_LZ4
    p = o + 312 + 4                                  # the block's first token, after BE32(clen)
    assert c[p] >> 4 > 0
    q = p + 1
    if c[p] >> 4 == 15:
        while c[q] == 255:
            q += 1
        q += 1
    c[q] ^= 0x20
    assert oracle.stream_restamp(c)[0] == 0 and oracle.stream_verify(c)[0] == 0
    return c


@pytest.mark.parametrize("name", ["fletcher4", "sha256", "sha512"])
def test_a_corrupted_raw_keyed_lz4_record_fails_the_recompress_relay(oracle, name):
    """a compression=off dataset on the compressed wire: the relay's decoder output is not the block on
    disk, the stream checksums (re-stamped) all hold"""
    x = oracle.synth_stream(40, recsize=16384, kind=oracle.PAYLOAD_PGPAGE)
    if name != "fletcher4":
        x = R.as_sha(oracle, x, name)
    bad = _corrupt_a_literal(oracle, R.send_c_form(oracle, x), 17)
    _, want = R.block_check(oracle, bad, R.RECOMPRESS, oracle.stream_recompress(bad)[1], sha256=True, sha512=True,
                            logical=True)
    assert want["first_bad"] == 17
    _, _, off = B._run(oracle, "recompress", bad, **OFF)
    assert off["logical_ok"] == 0 and off["skipped"] == 40
    for kw in (dict(batch_bytes=1 << 18), {}):
        msg = B._fails("recompress", bad, 17, **ON, **kw)
        assert "block checksum" in msg and "object 8" in msg and "offset %d" % (15 * 16384) in msg, msg
        assert ("(%s key)" % name in msg) == (name != "fletcher4"), msg


@pytest.mark.parametrize("chunk", [4093, 1 << 20])
def test_ring_api(oracle, chunk):
    x, _ = R.mixed_keys_stream(oracle, n=40)
    want = R.four_ways(oracle, x, frames=True, **ALL)
    for mode, src in _inputs(oracle, x).items():
        for kw in (dict(batch_bytes=1 << 18), {}):
            with B._stage(mode, **ON, **kw) as g:
                out, err = B._pump(g, src.tobytes(), chunk)
                assert not err, err
                assert out == B._run(oracle, mode, src, **OFF)[0].tobytes()
                B._same(g.block_stats(), want[mode][1])


def _dev_run(mem, mode, src, recs=None, logical=True, flags=0, finish=True):
    """one device-API submit of the plain stream `src` -> (stage, device output, its capacity)"""
    from manatee_b200 import index_host
    if recs is None:
        recs, _ = index_host(src)
    d_in, p_in = mem.put(src)
    d_recs, p_recs = mem.put(recs.view(np.uint8))
    cap = int(recs["lsize"].sum()) + int(src.size) + (1 << 20)
    d_out, p_out = mem.zeros(cap)
    g = B._stage(mode, flags=flags, **(ON if logical else OFF))
    g.dev_submit(p_in, src.size, p_recs, len(recs), p_out, cap)
    g._keep = (d_in, d_recs, d_out)
    return g, d_out


def _raw_keyed_lz4_records(c):
    """the records of the compressed stream `c` that arrive LZ4 under a fletcher4 key over the logical block"""
    return [i for i, (off, _, _, t) in enumerate(R.records(c)) if t == 3 and c[off + 50] == R.DC_LZ4 and
            c[off + 48] == R.FLETCHER4 and R.unprop(R.get_key(c, off)[2])[2:] == (R.DC_OFF, 0)]


def compress_of_lz4_records(oracle, mem):
    """COMPRESS decodes nothing, and the device API hands it whatever records it is given: an lzjb- or
    zle-keyed record that arrives LZ4 has no logical bytes there, passes through and stays skipped, with
    the flag as without it"""
    x, dcs = R.as_on_disk(oracle, B._raw_stream(oracle, n=12), 9, lambda i: (R.DC_LZJB, R.DC_ZLE)[i % 2])
    c = R.send_c_form(oracle, x)
    lz4 = [i for i, (off, _, _, t) in enumerate(R.records(c)) if t == 3 and c[off + 50] == R.DC_LZ4]
    assert len(lz4) == 12 and R.DC_LZJB in dcs.values()
    got = []
    for logical in (False, True):
        g, d_out = _dev_run(mem, "compress", c, logical=logical)
        with g:
            ob, _, _ = g.dev_finish()
            got.append((mem.get(d_out, ob), g.block_stats()))
    assert np.array_equal(got[0][0], got[1][0]) and got[0][1] == got[1][1]
    _, want = R.block_check(oracle, c, R.COMPRESS, got[1][0], **ON)
    B._same(got[1][1], want)
    assert want["skipped"] == 12 and want["logical_checked"] == 0


def test_compress_leaves_an_lz4_record_it_cannot_decode_skipped(oracle):
    compress_of_lz4_records(oracle, B.TorchMem())


def device_api_subbatched(oracle, mem, nrec, modes=MODES, recsize=4096):
    """`modes` on the device API over more records than one codec sub-batch holds: the counters are the
    model's, the output that of the flag off; a raw-keyed record corrupted near the end fails the relay"""
    from manatee_b200._native import MtzError, ECKSUM
    x, _ = R.mixed_keys_stream(oracle, n=nrec, recsize=recsize)
    c = R.send_c_form(oracle, x)
    want = R.four_ways(oracle, x, frames=True, **ALL)
    for mode, src in (("compress", x), ("decompress", c), ("recompress", c)):
        if mode not in modes:
            continue
        outs = []
        for logical in (False, True):
            g, d_out = _dev_run(mem, mode, src, logical=logical)
            with g:
                ob, _, _ = g.dev_finish()
                outs.append(mem.get(d_out, ob))
                if logical:
                    B._same(g.block_stats(), want[mode][1])
        assert np.array_equal(outs[0], outs[1]), mode
    if "recompress" not in modes:
        return
    k = _raw_keyed_lz4_records(c)[-2]
    g, _ = _dev_run(mem, "recompress", _corrupt_a_literal(oracle, c, k))
    with g:
        with pytest.raises(MtzError) as ei:
            g.dev_finish()
        assert ei.value.code == ECKSUM and g.stats()["bad_record"] == k and "block checksum" in str(ei.value)


def test_device_api_across_the_subbatch_edge(oracle):
    device_api_subbatched(oracle, B.TorchMem(), 66000)


def deferred_shards(oracle, mem):
    """MTZ_FLAG_DEFER_VERIFY: two RECOMPRESS shards of one stream; the counters add up to the model's and a
    corrupted raw-keyed record of the second shard surfaces at its mtz_dev_finish"""
    from manatee_b200 import index_host
    from manatee_b200 import shard as SH
    from manatee_b200._native import FLAG_DEFER_VERIFY, MtzError, ECKSUM
    x, _ = R.mixed_keys_stream(oracle, n=60)
    c = R.send_c_form(oracle, x)
    raw_lz4 = _raw_keyed_lz4_records(c)
    cut = 31
    late = [i for i in raw_lz4 if i > cut][0]
    for bad in (None, late):
        src = c if bad is None else _corrupt_a_literal(oracle, c, bad)
        _, want = R.block_check(oracle, src, R.RECOMPRESS, oracle.stream_recompress(src)[1], **ON)
        recs, _ = index_host(src)
        cut_off = int(recs["off"][cut])
        parts = [(src[:cut_off], recs[:cut].copy()), (src[cut_off:], recs[cut:].copy())]
        parts[1][1]["off"] -= cut_off
        gs = [_dev_run(mem, "recompress", np.ascontiguousarray(p), r, flags=FLAG_DEFER_VERIFY)[0] for p, r in parts]
        try:
            aggs = [g.dev_aggregate() for g in gs]
            ob, _, co = gs[0].dev_finish(carry_in=SH.carry_before(0, aggs), carry_out_in=(0, 0, 0, 0))
            if bad is None:
                gs[1].dev_finish(carry_in=SH.carry_before(1, aggs), carry_out_in=co)
                b0, b1 = gs[0].block_stats(), gs[1].block_stats()
                for k in R.COUNTERS:
                    if k != "first_frame_miss":
                        assert b0[k] + b1[k] == want[k], (k, b0, b1, want)
            else:
                with pytest.raises(MtzError) as ei:
                    gs[1].dev_finish(carry_in=SH.carry_before(1, aggs), carry_out_in=co)
                assert ei.value.code == ECKSUM and gs[1].stats()["bad_record"] + cut == bad
        finally:
            for g in gs:
                g.close()


def test_deferred_codec_shards(oracle):
    deferred_shards(oracle, B.TorchMem())


def test_device_group(oracle):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    x, _ = R.mixed_keys_stream(oracle, n=40)
    want = R.four_ways(oracle, x, frames=True, **ALL)
    for mode, src in _inputs(oracle, x).items():
        _, _, bs = B._run(oracle, mode, src, devices=[0, 1], batch_bytes=1 << 18, **ON)
        B._same(bs, want[mode][1])
