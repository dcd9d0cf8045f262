"""GPU: COMPRESS with MTZ_FLAG_COMPRESSED_IN | MTZ_FLAG_GZIP_IN -- a `zfs send -c` stream of a gzip pool
in, the lz4-stage-v1 wire out.  gzip-1 .. gzip-9 records are inflated on the GPU (k_inflate) and encoded
like raw ones.  Every output byte and counter is the reference model's (tests/gzip_in_ref.py), a frame
zlib would not inflate to exactly drr_logical_size bytes is MTZ_ECODEC at the model's record, and a stock
DECOMPRESS turns the wire into plain(x): through mtz_process_host, the ring API, the device API, a device
group and two fan-out peers."""
import struct

import numpy as np
import pytest

import block_ref as B
import compressed_in_ref as M
import gzip_in_ref as G
import test_gpu_block_cksum as K
import test_gpu_compressed_in as S

pytestmark = pytest.mark.gpu

CODECS = {"gzip-1": G.DC_GZIP[1], "gzip-6": G.DC_GZIP[6], "gzip-9": G.DC_GZIP[9], "mixed": G.mixed_codecs}


def send_c_stream(oracle, codec="mixed", n=20, recsize=8192):
    """pg-page records with incompressible and all-zero ones mixed in, written with `codec` (CODECS) and
    sent with -c"""
    from test_gpu_codec import _mixed_stream
    return G.send_c(oracle, _mixed_stream(oracle, n=n, recsize=recsize), 9, CODECS[codec])


def _stage(mode="compress", **kw):
    from manatee_b200 import GpuSnapshotStage
    return GpuSnapshotStage(mode, **dict(dict(compressed_input=True, gzip_input=True), **kw))


def _run(x, mode="compress", **kw):
    """process_host -> (output, stats without the timing fields, compressed-in stats)"""
    out = np.zeros(x.size * 3 + (1 << 20), dtype=np.uint8)
    with _stage(mode, **kw) as g:
        n = g.process_host(x, None if mode in ("verify", "passthrough") else out)
        st = g.stats()
        for k in S.TIMING:
            st.pop(k)
        return (x if mode in ("verify", "passthrough") else out[:n].copy()), st, g.compressed_in_stats()


def _check_wire(oracle, x, out, st, cst, want=None):
    """`out` is the model's COMPRESS of x, the counters are the model's, and a stock DECOMPRESS gives
    plain(x)"""
    want = G.expected(oracle, x) if want is None else want
    assert out.size == want.size and np.array_equal(out, want)
    bad, cnt = G.verdict(oracle, x)
    assert bad is None and cst == cnt, (cst, cnt)
    assert st["lz4_encoded"] == M.encoded(oracle, out, x) and st["lz4_decoded"] == 0
    assert st["bad_record"] == B.NONE
    back, _, _ = S._run("decompress", out, cin=False)
    assert np.array_equal(back, G.plain(oracle, x))


@pytest.mark.parametrize("codec", sorted(CODECS))
@pytest.mark.parametrize("recsize", [8192, 131072, 1 << 20])
def test_inflated_output_equals_the_model(oracle, codec, recsize):
    x = send_c_stream(oracle, codec, n={8192: 30, 131072: 12, 1 << 20: 5}[recsize], recsize=recsize)
    out, st, cst = _run(x)
    _check_wire(oracle, x, out, st, cst)
    assert cst["gzip_decoded"] > 0


def test_with_the_high_ratio_encoder(oracle):
    """MTZ_FLAG_LZ4_HC: the inflated records are what K3h makes of the plain stream"""
    x = send_c_stream(oracle, "mixed", n=30)
    base, _, _ = S._run("compress", G.plain(oracle, x), cin=False, lz4_hc=True)
    out, st, cst = _run(x, lz4_hc=True)
    _check_wire(oracle, x, out, st, cst, want=M.splice(oracle, base, x))


def _fails(x, rec, **kw):
    from manatee_b200._native import MtzError, ECODEC
    with _stage(**kw) as g:
        with pytest.raises(MtzError) as ei:
            g.process_host(x, np.zeros(x.size * 3 + (1 << 20), dtype=np.uint8))
        assert ei.value.code == ECODEC
        assert g.stats()["bad_record"] == rec


def corrupted_streams(oracle):
    """(name, stream, failing record) of the model: a gzip frame with a flipped Adler-32 byte, one with a
    flipped bit in its deflate data, one cut inside its stream, one whose lsize is a sector short, and a
    zstd record"""
    x = send_c_stream(oracle, "mixed", n=20)
    gz = M.write_records(x, G.DC_GZIP[6])
    out = []

    def frame(k):
        i, off, po, pl = gz[k]
        return i, off, bytearray(x[po:po + pl].tobytes())

    def end(fr):
        """the length of the zlib stream at the front of fr"""
        import zlib
        d = zlib.decompressobj()
        d.decompress(bytes(fr))
        return len(fr) - len(d.unused_data)

    i, _, fr = frame(0)
    fr[end(fr) - 1] ^= 0x01
    out.append(("adler", M.replace_payload(oracle, x, i, fr), i))
    i, _, fr = frame(1)
    fr[end(fr) // 2] ^= 0x10
    out.append(("bitflip", M.replace_payload(oracle, x, i, fr), i))
    i, _, fr = frame(2)
    out.append(("truncated", M.replace_payload(oracle, x, i, fr[:(end(fr) - 8) & ~7]), i))
    i, off, fr = frame(3)
    s = np.array(M.replace_payload(oracle, x, i, fr), copy=True)
    ho = B.records(s)[i][0]
    lsize = int.from_bytes(s[ho + 32:ho + 40].tobytes(), "little")
    s[ho + 32:ho + 40] = np.frombuffer(struct.pack("<Q", lsize - 512), dtype=np.uint8)   # output too long
    B.set_key(s, ho, ddk_prop=0)
    assert oracle.stream_restamp(s)[0] == 0
    out.append(("lsize", s, i))
    i, off, po, pl = gz[4]
    out.append(("zstd", M.replace_payload(oracle, x, i, x[po:po + pl], comp=M.DC_ZSTD), i))
    for name, s, i in out:
        assert G.verdict(oracle, s)[0] == i, name
    return out


def test_corrupted_frames_and_zstd_are_ecodec(oracle):
    for name, s, i in corrupted_streams(oracle):
        _fails(s, i)


def test_gzip_input_needs_compressed_input(oracle):
    from manatee_b200._native import MtzError, EINVAL
    for mode in ("compress", "verify"):
        with pytest.raises(MtzError) as ei:
            _stage(mode, compressed_input=False)
        assert ei.value.code == EINVAL


def test_the_other_modes_do_not_change(oracle):
    x = send_c_stream(oracle, "mixed", n=20)
    p = G.plain(oracle, x)
    wire, _, _ = S._run("compress", p, cin=False)
    lz = B.as_send_c(oracle, B.as_on_disk(oracle, p, 9)[0])
    for mode, src in (("verify", x), ("recompress", lz), ("decompress", wire), ("passthrough", x)):
        a = S._run(mode, src, cin=False)
        b = _run(src, mode)
        assert np.array_equal(a[0], b[0]) and a[1] == b[1], mode
        assert all(v == 0 for v in b[2].values()), mode
    # COMPRESS of a plain stream: the same bytes, no counter
    a, b = S._run("compress", p, cin=False), _run(p)
    assert np.array_equal(a[0], b[0]) and a[1] == b[1] and all(v == 0 for v in b[2].values())


def sha256_keyed(oracle, x):
    """x with the keys of its gzip records turned into SHA-256 keys of their frames, the first one wrong"""
    s = np.array(x, copy=True)
    first = True
    for i, off, po, pl in M.write_records(s):
        h = B.header(s[off:off + 312].tobytes())
        if G.is_gzip(h.dc) and h.arrive == h.dc:
            key = B.sha256_key(s[po:po + pl].tobytes() + bytes(h.psize - pl))
            B.set_key(s, off, B.SHA256, (key[0] ^ 1,) + key[1:] if first else key)
            first = False
    assert oracle.stream_restamp(s)[0] == 0
    return s


@pytest.mark.parametrize("sha256,logical", [(False, False), (False, True), (True, False), (True, True)])
def test_gzip_block_counters(oracle, sha256, logical):
    """block checks: a record with a gzip-N key that arrives as that frame is compared as it is; the
    other rows are those of VERIFY"""
    x = send_c_stream(oracle, "mixed", n=30)
    if sha256:
        x = sha256_keyed(oracle, x)
    flags = dict(lzjb=True, logical=logical, sha256=sha256)
    out, st, bs = K._run(oracle, "compress", x, compressed_input=True, gzip_input=True, **flags)
    _check_wire(oracle, x, out, st, _run(x)[2])
    _, want = G.block_check(oracle, x, sha256=sha256)
    K._same(bs, want)
    assert bs["frame_ok"] > 0 and bs["frame_miss"] == (1 if sha256 else 0)
    # without MTZ_FLAG_GZIP_IN the gzip keys stay skipped (and the records fail: no decoder)
    assert want["skipped"] < B.block_check(oracle, x, B.VERIFY, lzjb=True, sha256=sha256)[1]["skipped"]


def ring_api(oracle, chunk, n=20):
    x = send_c_stream(oracle, "mixed", n=n)
    with _stage(batch_bytes=1 << 18) as g:
        out, err = K._pump(g, x.tobytes(), chunk)
        assert not err, err
        out = np.frombuffer(out, dtype=np.uint8)
        assert np.array_equal(out, G.expected(oracle, x))
        assert g.compressed_in_stats() == G.verdict(oracle, x)[1]
    back, _, _ = S._run("decompress", out, cin=False)
    assert np.array_equal(back, G.plain(oracle, x))
    from manatee_b200._native import MtzError, ECODEC
    name, bad, i = corrupted_streams(oracle)[1]
    with _stage(batch_bytes=1 << 16) as g:
        _, err = K._pump(g, bad.tobytes(), chunk)
        assert any(isinstance(e, MtzError) and e.code == ECODEC for e in err), err
        assert g.stats()["bad_record"] == i


@pytest.mark.parametrize("chunk", [4093, 1 << 20])
def test_ring_api(oracle, chunk):
    ring_api(oracle, chunk)


def device_api(oracle, mem, n=20):
    """the device API's COMPRESS output is the wire without preamble"""
    from manatee_b200 import index_host
    x = send_c_stream(oracle, "mixed", n=n)
    p = G.plain(oracle, x)
    recs, _ = index_host(x)
    d_in, p_in = mem.put(x)
    d_recs, p_recs = mem.put(recs.view(np.uint8))
    cap = p.size + (1 << 20)
    d_out, p_out = mem.zeros(cap)
    with _stage() as g:
        g.dev_submit(p_in, x.size, p_recs, len(recs), p_out, cap)
        ob, _, _ = g.dev_finish()
        out = mem.get(d_out, ob)
        assert np.array_equal(out, oracle.wire_strip(G.expected(oracle, x)))
        assert g.compressed_in_stats() == G.verdict(oracle, x)[1]
    from manatee_b200._native import MtzError, ECODEC
    name, bad, i = corrupted_streams(oracle)[0]
    rb, _ = index_host(bad)
    d_b, p_b = mem.put(bad)
    d_rb, p_rb = mem.put(rb.view(np.uint8))
    with _stage() as g:
        g.dev_submit(p_b, bad.size, p_rb, len(rb), p_out, cap)
        with pytest.raises(MtzError) as ei:
            g.dev_finish()
        assert ei.value.code == ECODEC and g.stats()["bad_record"] == i


def test_device_api(oracle):
    device_api(oracle, K.TorchMem())


def test_device_group(oracle):
    S._two_gpus()
    x = send_c_stream(oracle, "mixed", n=40)
    out, st, cst = _run(x, devices=[0, 1], batch_bytes=1 << 18)
    _check_wire(oracle, x, out, st, cst)


def test_fanout_of_two_peers(oracle):
    S._two_gpus()
    x = send_c_stream(oracle, "mixed", n=40)
    want = G.expected(oracle, x)
    with _stage(devices=[0, 1], batch_bytes=1 << 18) as g:
        for p in (0, 1):
            g.fanout_attach(p)
        g.write(x)
        g.flush()
        for p in (0, 1):
            got = []
            while True:
                b = g.read_peer(p, 1 << 20)
                if b is None:
                    break
                got.append(b)
            assert b"".join(got) == want.tobytes(), p
