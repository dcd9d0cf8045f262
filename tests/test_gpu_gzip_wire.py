"""GPU: MTZ_FLAG_GZIP_WIRE -- gzip frames on the compressed wire.  COMPRESS with MTZ_FLAG_COMPRESSED_IN
forwards the gzip-1 .. gzip-9 records of a `zfs send -c` stream as they arrive and marks every preamble
with WIRE_F_GZIP; DECOMPRESS with the flag inflates them on the GPU (k_inflate) and gives plain(x).  Every
output byte and counter is the reference model's (tests/gzip_wire_ref.py): through mtz_process_host, the
ring API, the device API, a device group and two fan-out peers.  A receiver without the flag refuses the
wire, and a receiver with it decodes an ordinary lz4-stage-v1 wire as before."""

import numpy as np
import pytest

import block_ref as B
import compressed_in_ref as M
import gzip_in_ref as G
import gzip_wire_ref as W
import test_gpu_block_cksum as K
import test_gpu_compressed_in as S
import test_gpu_gzip_in as GI

pytestmark = pytest.mark.gpu

SEND = dict(compressed_input=True, gzip_wire=True)
RECV = dict(gzip_wire=True)
send_c_stream = GI.send_c_stream


def _stage(mode, **kw):
    from manatee_b200 import GpuSnapshotStage
    return GpuSnapshotStage(mode, **kw)


def _run(mode, x, **kw):
    """process_host -> (output, stats without the timing fields, compressed-in stats)"""
    out = np.zeros(x.size * 4 + (1 << 20), dtype=np.uint8)
    with _stage(mode, **kw) as g:
        n = g.process_host(x, None if mode in ("verify", "passthrough") else out)
        st = g.stats()
        for k in S.TIMING:
            st.pop(k)
        return (x if mode in ("verify", "passthrough") else out[:n].copy()), st, g.compressed_in_stats()


def lz4_on_wire(oracle, wire):
    """DRR_WRITEs that are LZ4 on `wire`: what DECOMPRESS counts in lz4_decoded"""
    b = oracle.wire_strip(wire)
    return sum(1 for off, _, _, t in B.records(b) if t == 3 and b[off + 50] == M.DC_LZ4)


def check_round_trip(oracle, x, out, st, cst, want=None, **recv):
    """`out` is the model's COMPRESS of x with its counters, and DECOMPRESS with the flag gives plain(x)
    with the model's receiver counters"""
    want = W.expected(oracle, x) if want is None else want
    assert out.size == want.size and np.array_equal(out, want)
    bad, cnt = W.verdict(oracle, x)
    assert bad is None and cst == cnt, (cst, cnt)
    assert st["lz4_encoded"] == M.encoded(oracle, out, x) and st["lz4_decoded"] == 0
    assert st["bad_record"] == B.NONE
    back, rst, rcst = _run("decompress", out, **dict(RECV, **recv))
    assert np.array_equal(back, G.plain(oracle, x))
    assert rcst == W.receiver_verdict(oracle, out)[1]
    assert rst["lz4_decoded"] == lz4_on_wire(oracle, out) and rst["bad_record"] == B.NONE


@pytest.mark.parametrize("codec", sorted(GI.CODECS))
@pytest.mark.parametrize("recsize", [8192, 131072, 1 << 20])
def test_round_trip_equals_the_model(oracle, codec, recsize):
    x = send_c_stream(oracle, codec, n={512: 60, 8192: 30, 131072: 12, 1 << 20: 5}[recsize], recsize=recsize)
    out, st, cst = _run("compress", x, **SEND)
    check_round_trip(oracle, x, out, st, cst)
    assert W.pre_flags(oracle, out)[0] & W.WIRE_F_GZIP
    assert cst["gzip_passed"] > 0 or recsize == 512          # no 512-byte block saves a sector


def test_with_the_high_ratio_encoder(oracle):
    """MTZ_FLAG_LZ4_HC: gzip records are still forwarded; the others are what K3h makes of plain(x)"""
    x = send_c_stream(oracle, "mixed", n=30)
    base, _, _ = S._run("compress", G.plain(oracle, x), cin=False, lz4_hc=True)
    out, st, cst = _run("compress", x, lz4_hc=True, **SEND)
    check_round_trip(oracle, x, out, st, cst, want=W.splice(oracle, base, x))


def test_einval_combinations(oracle):
    from manatee_b200._native import MtzError, EINVAL
    bad = [("compress", dict(gzip_wire=True)),
           ("compress", dict(compressed_input=True, gzip_wire=True, gzip_input=True)),
           ("decompress", dict(compressed_input=True, gzip_wire=True, gzip_input=True)),
           ("verify", dict(gzip_wire=True, gzip_input=True))]
    for mode, kw in bad:
        with pytest.raises(MtzError) as ei:
            _stage(mode, **kw)
        assert ei.value.code == EINVAL, (mode, kw)
    for mode in ("decompress", "verify", "recompress", "passthrough"):
        _stage(mode, gzip_wire=True).close()


def test_a_receiver_without_the_flag_refuses_the_gzip_wire(oracle):
    from manatee_b200._native import MtzError, EFORMAT
    x = send_c_stream(oracle, "gzip-6", n=12)
    w, _, _ = _run("compress", x, **SEND)
    for kw in ({}, dict(compressed_input=True)):
        with _stage("decompress", **kw) as g:
            with pytest.raises(MtzError) as ei:
                g.process_host(w, np.zeros(w.size * 4 + (1 << 20), dtype=np.uint8))
            assert ei.value.code == EFORMAT
    # ... and one with the flag still refuses a capability bit nobody knows
    at = W.preambles(oracle, w)[0]
    unknown = w.copy()
    unknown[at + 13] = 0x80
    with _stage("decompress", **RECV) as g:
        with pytest.raises(MtzError) as ei:
            g.process_host(unknown, np.zeros(w.size * 4 + (1 << 20), dtype=np.uint8))
        assert ei.value.code == EFORMAT


def test_the_flag_changes_nothing_on_an_lz4_wire(oracle):
    """today's wire (COMPRESS with gzip_input) and a plain stream's wire: the same output and counters"""
    x = send_c_stream(oracle, "mixed", n=30)
    for w in (_run("compress", x, compressed_input=True, gzip_input=True)[0],
              _run("compress", G.plain(oracle, x))[0]):
        assert all(f & W.WIRE_F_GZIP == 0 for f in W.pre_flags(oracle, w))
        a, b = _run("decompress", w), _run("decompress", w, **RECV)
        assert np.array_equal(a[0], b[0]) and np.array_equal(b[0], G.plain(oracle, x)) and a[1] == b[1]
        assert all(v == 0 for v in b[2].values())


def test_the_other_modes_do_not_change(oracle):
    x = send_c_stream(oracle, "mixed", n=20)
    p = G.plain(oracle, x)
    lz = B.as_send_c(oracle, B.as_on_disk(oracle, p, 9)[0])
    for mode, src in (("verify", x), ("recompress", lz), ("passthrough", x)):
        a = _run(mode, src)
        b = _run(mode, src, **RECV)
        assert np.array_equal(a[0], b[0]) and a[1] == b[1], mode
        assert all(v == 0 for v in b[2].values()), mode
    # COMPRESS of a plain stream: the same bytes but for the preamble's bit
    a, b = _run("compress", p), _run("compress", p, **SEND)
    assert np.array_equal(W.set_pre_flags(oracle, a[0], on=W.WIRE_F_GZIP), b[0]) and a[1] == b[1]


def bad_wires(oracle):
    """(name, send -c stream with one corrupted gzip frame, its record, the wire the sender makes of it):
    GI.corrupted_streams' gzip cases; the sender forwards the frame and re-stamps the stream"""
    x = send_c_stream(oracle, "mixed", n=20)
    rc, lz, _ = oracle.stream_compress(G.plain(oracle, x))
    assert rc == 0
    out = []
    for name, s, i in GI.corrupted_streams(oracle):
        if name != "zstd":
            out.append((name, s, i, W.splice(oracle, lz, s)))
    return out


def test_a_corrupted_frame_is_ecodec_at_the_receiver(oracle):
    from manatee_b200._native import MtzError, ECODEC
    for name, s, i, want in bad_wires(oracle):
        w, _, cst = _run("compress", s, **SEND)
        assert np.array_equal(w, want), name
        assert W.receiver_verdict(oracle, w)[0] == i, name
        with _stage("decompress", **RECV) as g:
            with pytest.raises(MtzError) as ei:
                g.process_host(w, np.zeros(w.size * 4 + (1 << 20), dtype=np.uint8))
            assert ei.value.code == ECODEC and g.stats()["bad_record"] == i, name
    # zstd is no gzip: the sender still fails it
    name, s, i = GI.corrupted_streams(oracle)[-1]
    assert name == "zstd"
    with _stage("compress", **SEND) as g:
        with pytest.raises(MtzError) as ei:
            g.process_host(s, np.zeros(s.size * 4 + (1 << 20), dtype=np.uint8))
        assert ei.value.code == ECODEC and g.stats()["bad_record"] == i


def ring_api(oracle, chunk, n=20):
    x = send_c_stream(oracle, "mixed", n=n)
    with _stage("compress", batch_bytes=1 << 18, **SEND) as g:
        out, err = K._pump(g, x.tobytes(), chunk)
        assert not err, err
        out = np.frombuffer(out, dtype=np.uint8)
        assert np.array_equal(out, W.expected(oracle, x))
        assert g.compressed_in_stats() == W.verdict(oracle, x)[1]
    with _stage("decompress", batch_bytes=1 << 18, **RECV) as g:
        back, err = K._pump(g, out.tobytes(), chunk)
        assert not err, err
        assert np.array_equal(np.frombuffer(back, dtype=np.uint8), G.plain(oracle, x))
        assert g.compressed_in_stats() == W.receiver_verdict(oracle, out)[1]
    from manatee_b200._native import MtzError, ECODEC
    name, _, i, bad = bad_wires(oracle)[1]
    with _stage("decompress", batch_bytes=1 << 16, **RECV) as g:
        _, err = K._pump(g, bad.tobytes(), chunk)
        assert any(isinstance(e, MtzError) and e.code == ECODEC for e in err), err
        assert g.stats()["bad_record"] == i


@pytest.mark.parametrize("chunk", [4093, 1 << 20])
def test_ring_api(oracle, chunk):
    ring_api(oracle, chunk)


def _dev(mem, mode, src, cap, **kw):
    """(stage, output buffer) after dev_submit of the whole of `src` on the device API"""
    from manatee_b200 import index_host
    recs, _ = index_host(src)
    d_in, p_in = mem.put(src)
    d_recs, p_recs = mem.put(recs.view(np.uint8))
    d_out, p_out = mem.zeros(cap)
    g = _stage(mode, **kw)
    g.dev_submit(p_in, src.size, p_recs, len(recs), p_out, cap)
    g._keep = (d_in, d_recs)
    return g, d_out


def device_api(oracle, mem, n=20, recsize=8192, codec="mixed"):
    """COMPRESS on the device API gives the wire without preambles, and DECOMPRESS with the flag of that
    gives plain(x) (no preamble reaches the library there: the flag is the handle's); more records than
    one codec sub-batch holds take the second job table across the sub-batch edge"""
    x = send_c_stream(oracle, codec, n=n, recsize=recsize)
    p = G.plain(oracle, x)
    cap = max(p.size, x.size) + (1 << 20)
    wire = W.expected(oracle, x)
    cnt = W.verdict(oracle, x)[1]
    g, d_out = _dev(mem, "compress", x, cap, **SEND)
    with g:
        ob, _, _ = g.dev_finish()
        out = mem.get(d_out, ob)
        assert np.array_equal(out, oracle.wire_strip(wire))
        assert g.compressed_in_stats() == cnt
    g, d_back = _dev(mem, "decompress", out, cap, **RECV)
    with g:
        ob, _, _ = g.dev_finish()
        assert np.array_equal(mem.get(d_back, ob), p)
        assert g.compressed_in_stats()["gzip_decoded"] == cnt["gzip_passed"] > 0
        assert g.stats()["lz4_decoded"] == lz4_on_wire(oracle, wire)
    from manatee_b200._native import MtzError, ECODEC
    name, _, i, bad = bad_wires(oracle)[0]
    g, _ = _dev(mem, "decompress", oracle.wire_strip(bad), cap, **RECV)
    with g:
        with pytest.raises(MtzError) as ei:
            g.dev_finish()
        assert ei.value.code == ECODEC and g.stats()["bad_record"] == i


def test_device_api(oracle):
    device_api(oracle, K.TorchMem())


def test_device_api_across_the_subbatch_edge(oracle):
    device_api(oracle, K.TorchMem(), n=70000, recsize=1024, codec="gzip-6")


def test_device_group(oracle):
    S._two_gpus()
    x = send_c_stream(oracle, "mixed", n=40)
    out, st, cst = _run("compress", x, devices=[0, 1], batch_bytes=1 << 18, **SEND)
    check_round_trip(oracle, x, out, st, cst, devices=[0, 1], batch_bytes=1 << 18)


def test_fanout_of_two_peers(oracle):
    S._two_gpus()
    x = send_c_stream(oracle, "mixed", n=40)
    want = W.expected(oracle, x)
    with _stage("compress", devices=[0, 1], batch_bytes=1 << 18, **SEND) as g:
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


def keyed_stream(oracle, n=30, recsize=8192):
    """a `send -c` stream of gzip-6, LZ4 and raw-on-disk records whose keys are fletcher4, sha256 and
    sha512 in turn over the bytes on disk (the padded frame, or the logical bytes of a raw block)"""
    from test_gpu_codec import _mixed_stream
    s, _ = G.as_on_disk(oracle, _mixed_stream(oracle, n=n, recsize=recsize), 9,
                        lambda i: (G.DC_GZIP[6], B.DC_LZ4, B.DC_OFF)[i % 3])
    x = np.array(G.as_send_c(oracle, s), copy=True)
    for k, (i, off, po, pl) in enumerate(M.write_records(x)):
        h = B.header(x[off:off + 312].tobytes())
        if k % 3 == 0 or h.prop == 0:
            continue
        data = x[po:po + pl].tobytes() + bytes(max(0, h.psize - pl))
        if k % 3 == 1:
            B.set_key(x, off, B.SHA256, B.sha256_key(data))
        else:
            B.set_key(x, off, B.SHA512, B.sha512_key(data))
    assert oracle.stream_restamp(x)[0] == 0
    return x


def test_sender_and_receiver_count_the_same_blocks(oracle):
    """with fletcher4 / sha256 / sha512 keys over gzip, LZ4 and raw blocks, COMPRESS and the DECOMPRESS
    of its wire report equal block counters, and the sender's are the model's"""
    x = keyed_stream(oracle)
    out, st, bs = K._run(oracle, "compress", x, sha256=True, sha512=True, **SEND)
    assert np.array_equal(out, W.expected(oracle, x))
    back, _, rbs = K._run(oracle, "decompress", out, sha256=True, sha512=True, **RECV)
    assert np.array_equal(back, G.plain(oracle, x))
    K._same(bs, rbs)
    assert bs["first_frame_miss"] == rbs["first_frame_miss"]
    _, want = G.block_check(oracle, x, sha256=True, sha512=True)
    K._same(bs, want)
    assert bs["frame_ok"] > 0 and bs["sha256"] > 0 and bs["sha512"] > 0
