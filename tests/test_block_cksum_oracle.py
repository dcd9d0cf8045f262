"""CPU: the reference model of the block-checksum check (tests/block_cksum_ref.py) and its stream
rewrites.  The keys the "LZ4 on disk" rewrite writes must be the Fletcher-4 (the C oracle's, not the
model's numpy one) of a frame that decodes to the block, zero-padded to a PSIZE that is a whole
number of 2**ashift sectors -- or of the logical block where ZFS stores it raw; and the
classification must follow the table of MTZ_FLAG_BLOCK_CKSUM record by record."""
import struct

import numpy as np
import pytest

import block_cksum_ref as R


@pytest.mark.parametrize("ashift,recsize", [(9, 8192), (12, 8192), (9, 131072), (12, 131072)])
def test_lz4_on_disk_keys_are_the_fletcher4_of_the_disk_bytes(oracle, ashift, recsize):
    from test_gpu_codec import _mixed_stream
    raw = _mixed_stream(oracle, n=16, recsize=recsize)
    s, dcs = R.as_lz4_on_disk(oracle, raw, ashift)
    assert oracle.stream_verify(s)[0] == 0
    assert set(dcs.values()) == {R.DC_OFF, R.DC_LZ4}
    c = R.as_send_c(oracle, s, ashift)
    assert oracle.stream_verify(c)[0] == 0
    recs, crecs = R.records(s), R.records(c)
    for i, dc in dcs.items():
        off, po, pl, _ = recs[i]
        ctype, key, p = R.get_key(s, off)
        lsize, psize, pdc, crypt = R.unprop(p)
        assert (ctype, lsize, pdc, crypt) == (R.FLETCHER4, recsize, dc, 0)
        logical = s[po:po + pl]
        coff, cpo, cpl, _ = crecs[i]
        if dc == R.DC_OFF:
            assert psize == lsize and key == oracle.fletcher4(logical)
            assert c[coff + 50] == 0 and np.array_equal(c[cpo:cpo + cpl], logical)
            continue
        assert psize % (1 << ashift) == 0 and psize < lsize
        frame = c[cpo:cpo + cpl]                                  # the send -c payload
        assert c[coff + 50] == R.DC_LZ4 and cpl == psize
        assert struct.unpack_from("<Q", c[coff:coff + 312].tobytes(), 96)[0] == psize
        assert key == oracle.fletcher4(frame)
        clen = 4 + int.from_bytes(frame[:4].tobytes(), "big")
        assert not frame[clen:].any()
        rc, dec = oracle.zfs_lz4_decompress(frame, lsize)
        assert rc == 0 and np.array_equal(dec, logical)
        # the padding beyond the 512-byte frame is what ashift adds: the key covers it
        assert key == R.f4((0, 0, 0, 0), frame[:clen].tobytes() + bytes(psize - clen))


def _table(ctype, p, arrive, drr_lsize, mode):
    """MTZ_FLAG_BLOCK_CKSUM's table, restated: (what is compared, source) or None = skipped"""
    lsize, psize, dc, crypt = R.unprop(p)
    if ctype != R.FLETCHER4 or p == 0 or crypt or lsize != drr_lsize:
        return None
    if dc in (0, 2):
        if psize != lsize:
            return None
        if arrive == 0:
            return ("logical", "input")
        if arrive == 15 and mode == R.DECOMPRESS:
            return ("logical", "output")
        return None
    if dc == 15:
        if arrive == 15:
            return ("frame", "input")
        if arrive == 0 and mode in (R.COMPRESS, R.RECOMPRESS):
            return ("frame", "output")
    return None


def test_classification_follows_the_table(oracle):
    """Every key class in every mode: the model's verdict is the table's, and a checked block's
    verdict is OK exactly when its key is left as written."""
    from test_gpu_codec import _mixed_stream
    s, dcs = R.as_lz4_on_disk(oracle, _mixed_stream(oracle, n=40, recsize=8192))
    s = s.copy()
    recs = R.records(s)
    lz4 = [i for i, v in dcs.items() if v == R.DC_LZ4]
    # a compressible block stored raw (a dataset without compression): the stage compresses it
    off, po, pl, _ = recs[lz4[6]]
    R.set_key(s, off, key=oracle.fletcher4(s[po:po + pl]), ddk_prop=R.prop(pl, pl, 0))
    mutate = {lz4[0]: dict(ctype=R.SHA256), lz4[1]: dict(ddk_prop=0),
              lz4[2]: dict(ddk_prop=R.prop(8192, 4096, R.DC_ZSTD)),
              lz4[3]: dict(ddk_prop=R.prop(8192, 8192, R.DC_OFF, crypt=1)),
              lz4[4]: dict(ddk_prop=R.prop(4096, 4096, R.DC_OFF)),        # LSIZE != drr_logical_size
              lz4[5]: dict(key=(1, 2, 3, 4))}                             # a frame that is not this one
    for i, m in mutate.items():
        R.set_key(s, recs[i][0], **m)
    assert oracle.stream_restamp(s)[0] == 0
    c = R.as_send_c(oracle, s)
    rc, comp, _ = oracle.stream_compress(s)
    assert rc == 0
    runs = [(s, None, R.VERIFY), (s, oracle.stream_compress_plain(s)[1], R.COMPRESS),
            (c, None, R.VERIFY), (c, oracle.stream_recompress(c)[1], R.RECOMPRESS),
            (oracle.wire_strip(comp), s, R.DECOMPRESS)]
    seen = set()
    for inp, out, mode in runs:
        verdicts, st = R.block_check(inp, out, mode)
        b = inp.tobytes()
        for i, (off, po, pl, t) in enumerate(R.records(inp)):
            if t != 3:
                assert i not in verdicts
                continue
            h = b[off:off + 312]
            row = _table(h[48], struct.unpack_from("<Q", h, 88)[0], h[50],
                         struct.unpack_from("<Q", h, 32)[0], mode)
            v = verdicts[i]
            seen.add((mode, row, v))
            if row is None:
                assert v == R.SKIPPED, (mode, i)
            elif row[0] == "logical":
                assert v == (R.LOGICAL_BAD if i in mutate else R.LOGICAL_OK), (mode, i)
            else:
                assert v == (R.FRAME_MISS if i in mutate else R.FRAME_OK), (mode, i)
        assert st["first_bad"] == R.NONE
        # the one foreign key is compared wherever a frame is at hand: not in VERIFY of a raw stream
        assert st["frame_miss"] == (0 if (mode == R.VERIFY and inp is s) else 1)
    # every row of the table was reached
    rows = {(r[0], r[1]) if r else None for _, r, _ in seen}
    assert rows == {None, ("logical", "input"), ("logical", "output"), ("frame", "input"), ("frame", "output")}


def test_a_corrupted_block_is_a_logical_mismatch_after_restamping(oracle):
    s = oracle.synth_stream(10, recsize=4096, kind=oracle.PAYLOAD_PCG).copy()
    recs = R.records(s)
    s[recs[6][1] + 17] ^= 1
    assert oracle.stream_restamp(s)[0] == 0 and oracle.stream_verify(s)[0] == 0
    verdicts, st = R.block_check(s, None, R.VERIFY)
    assert st["first_bad"] == 6 and st["logical_ok"] == 9 and verdicts[6] == R.LOGICAL_BAD
