"""CPU: the reference model of SHA-512 block keys (MTZ_FLAG_BLOCK_SHA512, tests/block_sha512_ref.py).
The key is checked against the FIPS 180-4 SHA-512/256 known answers and its byte order against the
sha256 key's; the re-keyed stream must be classified record by record as the fletcher4 model
classifies the original; without the flag the model must be tests/block_sha256_ref.py's, verdict for
verdict; and bytes at hand shorter than what the key covers are zero-extended, wherever in a
128-byte block they end."""
import hashlib
import struct

import numpy as np
import pytest

import block_cksum_ref as F
import block_sha256_ref as H
import block_sha512_ref as R

KAT = [
    (b"", "c672b8d1ef56ed28ab87c3622c5114069bdd3ad7b8f9737498d0c01ecef0967a"),
    (b"abc", "53048e2681941ef99b2e29b76b4c7dabe4c2d0c634fc6d46e0e2f13107e7af23"),
    (b"abcdefghbcdefghicdefghijdefghijkefghijklfghijklmghijklmnhijklmnoijklmnopjklmnopqklmnopqrlmnopqrs"
     b"mnopqrstnopqrstu", "3928e184fb8690f840da3988121d31be65cb9d3ef83ee6146feac861e19b563a"),
]


@pytest.mark.parametrize("msg,hexdigest", KAT)
def test_key_bytes_are_the_sha512_256_digest_in_order(msg, hexdigest):
    d = bytes.fromhex(hexdigest)
    assert hashlib.new("sha512_256", msg).digest() == d
    key = R.sha512_key(msg)
    h = np.zeros(312, dtype=np.uint8)
    R.set_key(h, 0, R.SHA512, key)
    assert bytes(h[56:88]) == d
    # a sha256 key packs each 8-byte group big endian: the same digest would land byte-reversed
    h256 = np.zeros(312, dtype=np.uint8)
    R.set_key(h256, 0, R.SHA256, struct.unpack(">4Q", d))
    assert all(bytes(h256[56 + 8 * i:64 + 8 * i]) == d[8 * i:8 * i + 8][::-1] for i in range(4))
    assert bytes(h256[56:88]) != d


def _runs(oracle, s):
    """(input, output, mode) of every mode over an as_lz4_on_disk()-style stream `s`"""
    c = R.as_send_c(oracle, s)
    rc, comp, _ = oracle.stream_compress(s)
    assert rc == 0
    return [(s, None, R.VERIFY), (s, oracle.stream_compress_plain(s)[1], R.COMPRESS),
            (c, None, R.VERIFY), (c, oracle.stream_recompress(c)[1], R.RECOMPRESS),
            (oracle.wire_strip(comp), s, R.DECOMPRESS)]


def _skippable(oracle, n=40):
    """an as_lz4_on_disk() stream with keys the check skips whatever their type, and one foreign
    frame key"""
    from test_gpu_codec import _mixed_stream
    s, dcs = R.as_lz4_on_disk(oracle, _mixed_stream(oracle, n=n, recsize=8192))
    s = s.copy()
    recs = R.records(s)
    lz4 = [i for i, v in dcs.items() if v == R.DC_LZ4]
    mutate = {lz4[0]: dict(ddk_prop=0), lz4[1]: dict(ddk_prop=R.prop(8192, 4096, R.DC_ZSTD)),
              lz4[2]: dict(ddk_prop=R.prop(8192, 8192, R.DC_OFF, crypt=1))}
    for i, m in mutate.items():
        R.set_key(s, recs[i][0], **m)
    assert oracle.stream_restamp(s)[0] == 0
    return s


def test_rekeyed_stream_is_classified_as_the_fletcher4_model_classifies_the_original(oracle):
    s = _skippable(oracle)
    h = R.as_sha512(oracle, s)
    assert oracle.stream_verify(h)[0] == 0
    nwrite = sum(1 for r in R.records(s) if r[3] == 3)
    assert sum(1 for off, _, _, t in R.records(h) if t == 3 and h[off + 48] == R.SHA512) == nwrite
    for (fi, fo, mode), (si, so, _) in zip(_runs(oracle, s), _runs(oracle, h)):
        fv, fst = F.block_check(fi, fo, mode)
        for sha256 in (False, True):
            sv, sst = R.block_check(si, so, mode, sha256=sha256, sha512=True)
            assert fv == sv, mode
            assert fst == {k: v for k, v in sst.items() if k not in ("sha256", "sha512")}
            assert sst["sha256"] == 0 and sst["sha512"] == sum(1 for v in sv.values() if v != R.SKIPPED) > 0
            # without the flag every sha512 key is skipped, whatever the sha256 flag says
            ov, ost = R.block_check(si, so, mode, sha256=sha256)
            assert set(ov.values()) == {R.SKIPPED} and ost["skipped"] == nwrite and ost["sha512"] == 0


def _three_types(oracle):
    """fletcher4, sha256 and sha512 keys, and the skipped classes, in one stream"""
    s = _skippable(oracle)
    a, b = R.as_sha256(oracle, s), R.as_sha512(oracle, s)
    out = s.copy()
    recs = R.records(s)
    w = [i for i, r in enumerate(recs) if r[3] == 3]
    for i in w[1::3]:
        out[recs[i][0] + 48:recs[i][0] + 88] = a[recs[i][0] + 48:recs[i][0] + 88]
    for i in w[2::3]:
        out[recs[i][0] + 48:recs[i][0] + 88] = b[recs[i][0] + 48:recs[i][0] + 88]
    assert oracle.stream_restamp(out)[0] == 0
    return out


def test_without_the_flag_the_model_is_the_sha256_model(oracle):
    s = _three_types(oracle)
    for fi, fo, mode in _runs(oracle, s):
        for sha256 in (False, True):
            v, st = R.block_check(fi, fo, mode, sha256=sha256)
            hv, hst = H.block_check(fi, fo, mode, sha256=sha256)
            assert v == hv and st == dict(hst, sha512=0), mode
        # with both flags every compared record is fletcher4, sha256 or sha512
        v, st = R.block_check(fi, fo, mode, sha256=True, sha512=True)
        assert st["sha256"] > 0 and st["sha512"] > 0
        assert st["logical_ok"] + st["frame_ok"] + st["frame_miss"] > st["sha256"] + st["sha512"]
        assert st["skipped"] == H.block_check(fi, fo, mode, sha256=True)[1]["skipped"] - st["sha512"]


def test_corrupted_and_relabelled_keys_are_mismatches(oracle):
    base = oracle.synth_stream(10, recsize=4096, kind=oracle.PAYLOAD_PCG)
    s = R.as_sha512(oracle, base)
    recs = R.records(s)
    s[recs[6][1] + 17] ^= 1
    assert oracle.stream_restamp(s)[0] == 0 and oracle.stream_verify(s)[0] == 0
    verdicts, st = R.block_check(s, None, R.VERIFY, sha512=True)
    assert st["first_bad"] == 6 and st["logical_ok"] == 9 and st["sha512"] == 10
    assert verdicts[6] == R.LOGICAL_BAD
    # a sha256 key labelled sha512, and a sha512 key labelled sha256: compared by the wrong hash
    a = R.as_sha256(oracle, base)
    R.set_key(a, recs[3][0], ctype=R.SHA512)
    b = R.as_sha512(oracle, base)
    R.set_key(b, recs[4][0], ctype=R.SHA256)
    for x, bad in ((a, 3), (b, 4)):
        assert R.block_check(x, None, R.VERIFY, sha256=True, sha512=True)[1]["first_bad"] == bad


@pytest.mark.parametrize("ashift", [9, 12])
@pytest.mark.parametrize("align", [8, 128])
def test_frames_shorter_than_psize_are_zero_extended(oracle, ashift, align):
    from test_gpu_codec import _mixed_stream
    s, dcs = R.as_lz4_on_disk(oracle, _mixed_stream(oracle, n=24, recsize=8192), ashift)
    c = R.trim_frames_to(oracle, R.as_send_c(oracle, R.as_sha512(oracle, s), ashift), align)
    assert oracle.stream_verify(c)[0] == 0
    ends = []
    for off, po, pl, t in R.records(c):
        if t == 3 and c[off + 50] == R.DC_LZ4:
            _, key, p = R.get_key(c, off)
            psize = R.unprop(p)[1]
            assert pl <= psize and pl % align == 0
            ends.append((pl, psize))
            assert key == R.sha512_key(c[po:po + pl].tobytes() + bytes(psize - pl))
    assert len(ends) == sum(1 for v in dcs.values() if v == R.DC_LZ4)
    short = [pl for pl, psize in ends if pl < psize]
    assert short and (all(pl % 128 == 0 for pl in short) if align == 128 else any(pl % 128 for pl in short))
    v, st = R.block_check(c, None, R.VERIFY, sha512=True)
    assert st["frame_ok"] == len(ends) and st["frame_miss"] == 0 and st["sha512"] == len(dcs)
    # the last byte at hand counts: flip it and the frame no longer matches
    off, po, pl, _ = next(r for r in R.records(c) if r[3] == 3 and c[r[0] + 50] == R.DC_LZ4 and
                          r[2] < R.unprop(R.get_key(c, r[0])[2])[1])
    bad = c.copy()
    bad[po + pl - 1] ^= 0x01
    assert oracle.stream_restamp(bad)[0] == 0
    assert R.block_check(bad, None, R.VERIFY, sha512=True)[1]["frame_miss"] == 1
