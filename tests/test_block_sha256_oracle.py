"""CPU: the reference model of SHA-256 block keys (MTZ_FLAG_BLOCK_SHA256, tests/block_sha256_ref.py).
Without SHA-256 keys it must be the fletcher4 model of tests/block_cksum_ref.py, verdict for verdict;
the key packing is checked against the FIPS 180-4 known answers, the re-keyed stream must be
classified record by record as the fletcher4 model classifies the original, and bytes at hand that
are shorter than what the key covers are zero-extended, wherever in a 64-byte block they end."""
import hashlib
import struct

import numpy as np
import pytest

import block_cksum_ref as F
import block_sha256_ref as R

KAT = [
    (b"", "e3b0c44298fc1c149afbf4c8996fb92427ae41e4649b934ca495991b7852b855"),
    (b"abc", "ba7816bf8f01cfea414140de5dae2223b00361a396177a9cb410ff61f20015ad"),
    (b"abcdbcdecdefdefgefghfghighijhijkijkljklmklmnlmnomnopnopq",
     "248d6a61d20638b8e5c026930c3e6039a33ce45964ff2167f6ecedd419db06c1"),
]


@pytest.mark.parametrize("msg,hexdigest", KAT)
def test_key_words_are_the_big_endian_u64s_of_the_digest(msg, hexdigest):
    d = bytes.fromhex(hexdigest)
    key = R.sha256_key(msg)
    assert key == tuple(int.from_bytes(d[8 * i:8 * i + 8], "big") for i in range(4))
    # in the header the words are native little endian: byte 56 + 8i + j is digest byte 8i + 7 - j
    h = np.zeros(312, dtype=np.uint8)
    R.set_key(h, 0, R.SHA256, key)
    assert all(bytes(h[56 + 8 * i:64 + 8 * i]) == d[8 * i:8 * i + 8][::-1] for i in range(4))
    assert struct.unpack("<4Q", bytes(h[56:88])) == struct.unpack(">4Q", hashlib.sha256(msg).digest())


def _runs(oracle, s):
    """(input, output, mode) of every mode over an as_lz4_on_disk()-style stream `s`"""
    c = R.as_send_c(oracle, s)
    rc, comp, _ = oracle.stream_compress(s)
    assert rc == 0
    return [(s, None, R.VERIFY), (s, oracle.stream_compress_plain(s)[1], R.COMPRESS),
            (c, None, R.VERIFY), (c, oracle.stream_recompress(c)[1], R.RECOMPRESS),
            (oracle.wire_strip(comp), s, R.DECOMPRESS)]


def test_rekeyed_stream_is_classified_as_the_fletcher4_model_classifies_the_original(oracle):
    from test_gpu_codec import _mixed_stream
    s, dcs = R.as_lz4_on_disk(oracle, _mixed_stream(oracle, n=40, recsize=8192))
    s = s.copy()
    recs = R.records(s)
    lz4 = [i for i, v in dcs.items() if v == R.DC_LZ4]
    # keys the check skips whatever their type, and one foreign frame key
    mutate = {lz4[0]: dict(ddk_prop=0), lz4[1]: dict(ddk_prop=R.prop(8192, 4096, R.DC_ZSTD)),
              lz4[2]: dict(ddk_prop=R.prop(8192, 8192, R.DC_OFF, crypt=1))}
    for i, m in mutate.items():
        R.set_key(s, recs[i][0], **m)
    assert oracle.stream_restamp(s)[0] == 0
    h = R.as_sha256(oracle, s)
    assert oracle.stream_verify(h)[0] == 0
    nwrite = sum(1 for r in recs if r[3] == 3)
    assert sum(1 for off, _, _, t in R.records(h) if t == 3 and h[off + 48] == R.SHA256) == nwrite
    for (fi, fo, mode), (si, so, _) in zip(_runs(oracle, s), _runs(oracle, h)):
        fv, fst = R.block_check(fi, fo, mode)
        sv, sst = R.block_check(si, so, mode, sha256=True)
        assert fv == sv, mode
        assert {k: v for k, v in fst.items() if k != "sha256"} == {k: v for k, v in sst.items() if k != "sha256"}
        assert fst["sha256"] == 0 and sst["sha256"] == sum(1 for v in sv.values() if v != R.SKIPPED) > 0
        # without the flag every sha256 key is skipped
        ov, ost = R.block_check(si, so, mode)
        assert set(ov.values()) == {R.SKIPPED} and ost["skipped"] == nwrite
        # on fletcher4 keys the model is block_cksum_ref's, with or without the flag
        for sha in (False, True):
            v, st = R.block_check(fi, fo, mode, sha256=sha)
            assert (v, {k: x for k, x in st.items() if k != "sha256"}) == F.block_check(fi, fo, mode)
            assert st["sha256"] == 0


def test_a_corrupted_block_is_a_logical_mismatch_after_restamping(oracle):
    s = R.as_sha256(oracle, oracle.synth_stream(10, recsize=4096, kind=oracle.PAYLOAD_PCG))
    recs = R.records(s)
    s[recs[6][1] + 17] ^= 1
    assert oracle.stream_restamp(s)[0] == 0 and oracle.stream_verify(s)[0] == 0
    verdicts, st = R.block_check(s, None, R.VERIFY, sha256=True)
    assert st["first_bad"] == 6 and st["logical_ok"] == 9 and st["sha256"] == 10
    assert verdicts[6] == R.LOGICAL_BAD
    # a fletcher4 key labelled sha256 is compared by SHA-256: a mismatch
    f = oracle.synth_stream(10, recsize=4096, kind=oracle.PAYLOAD_PCG).copy()
    R.set_key(f, R.records(f)[3][0], ctype=R.SHA256)
    assert R.block_check(f, None, R.VERIFY, sha256=True)[1]["first_bad"] == 3


@pytest.mark.parametrize("ashift", [9, 12])
def test_frames_shorter_than_psize_are_zero_extended(oracle, ashift):
    from test_gpu_codec import _mixed_stream
    s, dcs = R.as_lz4_on_disk(oracle, _mixed_stream(oracle, n=24, recsize=8192), ashift)
    c = R.trim_frames(oracle, R.as_send_c(oracle, R.as_sha256(oracle, s), ashift))
    assert oracle.stream_verify(c)[0] == 0
    ends = []
    for i, (off, po, pl, t) in enumerate(R.records(c)):
        if t == 3 and c[off + 50] == R.DC_LZ4:
            _, key, p = R.get_key(c, off)
            psize = R.unprop(p)[1]
            assert pl <= psize and pl % 8 == 0
            ends.append((pl, psize))
            frame = c[po:po + pl].tobytes()
            assert key == R.sha256_key(frame + bytes(psize - pl))
    assert len(ends) == sum(1 for v in dcs.values() if v == R.DC_LZ4)
    assert any(pl < psize for pl, psize in ends) and any(pl % 64 for pl, _ in ends)
    v, st = R.block_check(c, None, R.VERIFY, sha256=True)
    assert st["frame_ok"] == len(ends) and st["frame_miss"] == 0 and st["sha256"] == len(dcs)
    # the last byte at hand counts: flip it and the frame no longer matches
    off, po, pl, _ = next(r for r in R.records(c) if r[3] == 3 and c[r[0] + 50] == R.DC_LZ4 and r[2] % 64)
    bad = c.copy()
    bad[po + pl - 1] ^= 0x01
    assert oracle.stream_restamp(bad)[0] == 0
    assert R.block_check(bad, None, R.VERIFY, sha256=True)[1]["frame_miss"] == 1
