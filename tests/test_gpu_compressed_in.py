"""GPU: COMPRESS with MTZ_FLAG_COMPRESSED_IN -- a `zfs send -c` stream in, the lz4-stage-v1 wire out.
LZ4 records are forwarded as they arrive, lzjb / zle records decoded on the GPU (k_lzjb_decode,
k_zle_decode) and encoded like raw ones, any other compression is MTZ_ECODEC.  Every output byte and
counter is the reference model's (tests/compressed_in_ref.py), and a stock DECOMPRESS turns the wire
into plain(x), the stream `zfs send` without -c would have produced: through mtz_process_host, the ring
API, the device API, a device group and two fan-out peers."""
import numpy as np
import pytest

import block_ref as B
import compressed_in_ref as M
import test_gpu_block_cksum as K

pytestmark = pytest.mark.gpu

CODECS = {"lz4-9": (9, M.DC_LZ4), "lz4-12": (12, M.DC_LZ4), "lzjb": (9, M.DC_LZJB), "zle": (9, M.DC_ZLE),
          "mixed": (9, B.mixed_codecs)}
TIMING = ("gpu_ms", "k1_ms", "codec_ms", "k3_ms", "kernel_launches")


def send_c_stream(oracle, codec="mixed", n=20, recsize=8192):
    """pg-page records with incompressible and all-zero ones mixed in, written with `codec` (CODECS) and
    sent with -c"""
    from test_gpu_codec import _mixed_stream
    ashift, dc = CODECS[codec]
    return M.send_c(oracle, _mixed_stream(oracle, n=n, recsize=recsize), ashift, dc)


def _stage(mode, cin=True, **kw):
    from manatee_b200 import GpuSnapshotStage
    return GpuSnapshotStage(mode, compressed_input=cin, **kw)


def _run(mode, x, cin=True, **kw):
    """process_host -> (output, stats without the timing fields, compressed-in stats)"""
    out = np.zeros(x.size * 3 + (1 << 20), dtype=np.uint8)
    with _stage(mode, cin, **kw) as g:
        n = g.process_host(x, None if mode in ("verify", "passthrough") else out)
        st = g.stats()
        for k in TIMING:
            st.pop(k)
        return (x if mode in ("verify", "passthrough") else out[:n].copy()), st, g.compressed_in_stats()


def _check_wire(oracle, x, out, st, cst, want=None):
    """`out` is the model's COMPRESS of x, the counters are the model's, and a stock DECOMPRESS gives
    plain(x)"""
    want = M.expected(oracle, x) if want is None else want
    assert out.size == want.size and np.array_equal(out, want)
    bad, cnt = M.verdict(oracle, x)
    assert bad is None and cst == cnt, (cst, cnt)
    assert st["lz4_encoded"] == M.encoded(oracle, out, x) and st["lz4_decoded"] == 0
    assert st["bad_record"] == B.NONE
    back, _, _ = _run("decompress", out, cin=False)
    assert np.array_equal(back, M.plain(oracle, x))


@pytest.mark.parametrize("codec", sorted(CODECS))
@pytest.mark.parametrize("recsize", [8192, 131072])
def test_output_equals_the_model(oracle, codec, recsize):
    x = send_c_stream(oracle, codec, n=12 if recsize > 8192 else 30, recsize=recsize)
    out, st, cst = _run("compress", x)
    _check_wire(oracle, x, out, st, cst)
    if codec in ("lzjb", "zle"):
        assert cst[codec + "_decoded"] > 0


def test_lz4_payloads_are_forwarded_as_they_arrive(oracle):
    """trimmed frames (payload = the frame rounded up to 8 bytes, not PSIZE) travel byte for byte"""
    x = B.trim_frames(oracle, send_c_stream(oracle, "lz4-9", n=30), align=8)
    out, st, cst = _run("compress", x)
    _check_wire(oracle, x, out, st, cst)
    xb, ob = np.asarray(x), oracle.wire_strip(out)
    n = 0
    for (xo, xpo, xpl, t), (oo, opo, opl, _) in zip(B.records(xb), B.records(ob)):
        if t == 3 and xb[xo + 50] == M.DC_LZ4:
            # the header up to drr_checksum (re-stamped) and the payload
            assert np.array_equal(xb[xo:xo + 280], ob[oo:oo + 280])
            assert np.array_equal(xb[xpo:xpo + xpl], ob[opo:opo + opl])
            n += 1
    assert n == cst["lz4_passed"] > 0


@pytest.mark.parametrize("feat", [0, M.FEAT_EMBED_DATA])
@pytest.mark.parametrize("lz4", [False, True])
def test_the_preamble_says_what_plain_send_would_have_said(oracle, feat, lz4):
    x = send_c_stream(oracle, "mixed", n=10)
    x = M.set_features(oracle, x, on=feat | (M.FEAT_LZ4 if lz4 else 0), off=0 if lz4 else M.FEAT_LZ4)
    out, st, cst = _run("compress", x)
    flags = int.from_bytes(out[12:16].tobytes(), "little")
    assert flags == (1 if lz4 and feat else 0)
    _check_wire(oracle, x, out, st, cst)


def test_with_the_high_ratio_encoder(oracle):
    """MTZ_FLAG_LZ4_HC: the records that arrived LZ4 are still forwarded; the rest are what K3h makes
    of the plain stream"""
    x = send_c_stream(oracle, "mixed", n=30)
    base, _, _ = _run("compress", M.plain(oracle, x), cin=False, lz4_hc=True)
    out, st, cst = _run("compress", x, lz4_hc=True)
    _check_wire(oracle, x, out, st, cst, want=M.splice(oracle, base, x))


def _fails(x, rec, **kw):
    from manatee_b200._native import MtzError, ECODEC
    with _stage("compress", **kw) as g:
        with pytest.raises(MtzError) as ei:
            g.process_host(x, np.zeros(x.size * 3 + (1 << 20), dtype=np.uint8))
        assert ei.value.code == ECODEC
        assert g.stats()["bad_record"] == rec


def corrupted_streams(oracle):
    """(name, stream, failing record) of the model: an lzjb match reaching before the block, a
    truncated lzjb frame, a zle run past lsize, a gzip and a zstd record"""
    x = send_c_stream(oracle, "mixed", n=20)
    out = []
    lz = M.write_records(x, M.DC_LZJB)
    i, off, po, pl = lz[1]
    fr = bytearray(x[po:po + pl].tobytes())
    lsize = int.from_bytes(x[off + 32:off + 40].tobytes(), "little")
    pos, _, op = next(it for it in M.lzjb_items(fr, lsize) if it[1])
    fr[pos] = (fr[pos] & 0xfc) | 0x03
    fr[pos + 1] = 0xff                                         # offset 1023 > op
    assert op < 1023
    out.append(("lzjb-bad-offset", M.replace_payload(oracle, x, i, fr), i))
    i, off, po, pl = lz[-1]
    lsize = int.from_bytes(x[off + 32:off + 40].tobytes(), "little")
    end = max(p for p, _, _ in M.lzjb_items(x[po:po + pl], lsize)) + 1
    out.append(("lzjb-truncated", M.replace_payload(oracle, x, i, x[po:po + ((end - 1) & ~7)]), i))
    i, off, po, pl = M.write_records(x, M.DC_ZLE)[0]
    lsize = int.from_bytes(x[off + 32:off + 40].tobytes(), "little")
    fr = bytearray(x[po:po + pl].tobytes())
    tp, n, zero = M.zle_tokens(fr, lsize)[-1]
    fr[tp] = 255 if zero else 63                                # a longer last run: past lsize
    out.append(("zle-overrun", M.replace_payload(oracle, x, i, fr), i))
    for name, dc in (("gzip", M.DC_GZIP6), ("zstd", M.DC_ZSTD)):
        i, off, po, pl = M.write_records(x, M.DC_LZJB)[2]
        out.append((name, M.replace_payload(oracle, x, i, x[po:po + pl], comp=dc), i))
    for name, s, i in out:
        assert M.verdict(oracle, s)[0] == i, name
    return out


def test_corrupted_frames_and_unknown_compressions_are_ecodec(oracle):
    for name, s, i in corrupted_streams(oracle):
        _fails(s, i)


def test_the_other_modes_do_not_change(oracle):
    x = send_c_stream(oracle, "mixed", n=20)
    wire, _, _ = _run("compress", B.as_on_disk(oracle, M.plain(oracle, x), 9)[0], cin=False)
    for mode, src in (("verify", x), ("recompress", x), ("decompress", wire), ("passthrough", x)):
        a = _run(mode, src, cin=False)
        b = _run(mode, src, cin=True)
        assert np.array_equal(a[0], b[0]) and a[1] == b[1], mode
        assert all(v == 0 for v in b[2].values()), mode
    # COMPRESS of a plain stream: the same bytes, no counter
    p = M.plain(oracle, x)
    a, b = _run("compress", p, cin=False), _run("compress", p, cin=True)
    assert np.array_equal(a[0], b[0]) and a[1] == b[1] and all(v == 0 for v in b[2].values())


@pytest.mark.parametrize("logical", [False, True])
def test_block_counters_are_those_of_verify(oracle, logical):
    """block checks: a record that arrives as its disk frame is compared as it is, as VERIFY does"""
    x = send_c_stream(oracle, "mixed", n=30)
    flags = dict(lzjb=True, logical=logical)
    out, st, bs = K._run(oracle, "compress", x, compressed_input=True, **flags)
    _check_wire(oracle, x, out, st, _run("compress", x)[2])
    _, want = B.block_check(oracle, x, B.VERIFY, lzjb=True)
    K._same(bs, want)
    assert bs["frame_miss"] == 0 and bs["skipped"] == 0


def ring_api(oracle, chunk, n=20):
    x = send_c_stream(oracle, "mixed", n=n)
    with _stage("compress", batch_bytes=1 << 18) as g:
        out, err = K._pump(g, x.tobytes(), chunk)
        assert not err, err
        out = np.frombuffer(out, dtype=np.uint8)
        assert np.array_equal(out, M.expected(oracle, x))
        assert g.compressed_in_stats() == M.verdict(oracle, x)[1]
    back, _, _ = _run("decompress", out, cin=False)
    assert np.array_equal(back, M.plain(oracle, x))
    # a failure surfaces on the ring API at the model's record
    from manatee_b200._native import MtzError, ECODEC
    name, bad, i = corrupted_streams(oracle)[0]
    with _stage("compress", batch_bytes=1 << 16) as g:
        _, err = K._pump(g, bad.tobytes(), chunk)
        assert any(isinstance(e, MtzError) and e.code == ECODEC for e in err), err
        assert g.stats()["bad_record"] == i


@pytest.mark.parametrize("chunk", [4093, 1 << 20])
def test_ring_api(oracle, chunk):
    ring_api(oracle, chunk)


def device_api(oracle, mem, n=20):
    """the device API has no wire framing: its COMPRESS output is the wire without preamble, and its
    DECOMPRESS makes plain(x) of it"""
    from manatee_b200 import index_host
    x = send_c_stream(oracle, "mixed", n=n)
    p = M.plain(oracle, x)
    recs, _ = index_host(x)
    d_in, p_in = mem.put(x)
    d_recs, p_recs = mem.put(recs.view(np.uint8))
    cap = p.size + (1 << 20)
    d_out, p_out = mem.zeros(cap)
    with _stage("compress") as g:
        g.dev_submit(p_in, x.size, p_recs, len(recs), p_out, cap)
        ob, _, _ = g.dev_finish()
        out = mem.get(d_out, ob)
        assert np.array_equal(out, oracle.wire_strip(M.expected(oracle, x)))
        assert g.compressed_in_stats() == M.verdict(oracle, x)[1]
    r2, _ = index_host(out)
    d_c, p_c = mem.put(out)
    d_r2, p_r2 = mem.put(r2.view(np.uint8))
    d_o2, p_o2 = mem.zeros(cap)
    with _stage("decompress", cin=False) as g:
        g.dev_submit(p_c, out.size, p_r2, len(r2), p_o2, cap)
        ob2, _, _ = g.dev_finish()
        assert np.array_equal(mem.get(d_o2, ob2), p)
    from manatee_b200._native import MtzError, ECODEC
    name, bad, i = corrupted_streams(oracle)[3]
    rb, _ = index_host(bad)
    d_b, p_b = mem.put(bad)
    d_rb, p_rb = mem.put(rb.view(np.uint8))
    with _stage("compress") as g:
        g.dev_submit(p_b, bad.size, p_rb, len(rb), p_out, cap)
        with pytest.raises(MtzError) as ei:
            g.dev_finish()
        assert ei.value.code == ECODEC and g.stats()["bad_record"] == i


def test_device_api(oracle):
    device_api(oracle, K.TorchMem())


def _two_gpus():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")


def test_device_group(oracle):
    _two_gpus()
    x = send_c_stream(oracle, "mixed", n=40)
    out, st, cst = _run("compress", x, devices=[0, 1], batch_bytes=1 << 18)
    _check_wire(oracle, x, out, st, cst)


def test_fanout_of_two_peers(oracle):
    _two_gpus()
    x = send_c_stream(oracle, "mixed", n=40)
    want = M.expected(oracle, x)
    with _stage("compress", devices=[0, 1], batch_bytes=1 << 18) as g:
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
