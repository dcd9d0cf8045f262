"""CPU: the reference model of the block-checksum check (tests/block_ref.py) and its stream rewrites.
The keys the "LZ4 on disk" rewrite writes must be the Fletcher-4 (the C oracle's, not the model's
numpy one) of a frame that decodes to the block, zero-padded to a PSIZE that is a whole number of
2**ashift sectors -- or of the logical block where ZFS stores it raw; and the classification must
follow a hand-written table of block_classify's rows, with every flag that adds rows, record by
record and counter by counter.  flag_off() holds the model to the same table one flag at a time."""
import itertools
import struct

import numpy as np
import pytest

import block_ref as R


@pytest.mark.parametrize("ashift,recsize", [(9, 8192), (12, 8192), (9, 131072), (12, 131072)])
def test_lz4_on_disk_keys_are_the_fletcher4_of_the_disk_bytes(oracle, ashift, recsize):
    from test_gpu_codec import _mixed_stream
    raw = _mixed_stream(oracle, n=16, recsize=recsize)
    s, dcs = R.as_on_disk(oracle, raw, ashift)
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


# block_classify's rows, restated by hand: (key covers, arrives as, modes, flags needed) -> (what is
# compared, source, a row of MTZ_FLAG_BLOCK_LOGICAL).  "raw": a raw-on-disk key (compression 0 or 2,
# PSIZE = LSIZE); "same": the record arrives as the frame its key covers.
V, C, D, RC = R.VERIFY, R.COMPRESS, R.DECOMPRESS, R.RECOMPRESS
ROWS = [
    ("raw", 0, (V, C, D, RC), (), ("logical", "input", False)),
    ("raw", 15, (D,), (), ("logical", "output", False)),
    ("raw", 15, (RC,), ("logical",), ("logical", "decoded", True)),
    ("lz4", 15, (V, C, D, RC), (), ("frame", "input", False)),
    ("lz4", 0, (C, RC), (), ("frame", "output", False)),
    ("lz4", 0, (V,), ("frames",), ("frame", "encoded", False)),
    ("lz4", 0, (D,), ("logical",), ("frame", "none", True)),
    ("lzjb/zle", "same", (V, RC), ("lzjb",), ("frame", "input", False)),
    ("lzjb/zle", 0, (V,), ("lzjb",), ("frame", "encoded", False)),
    ("lzjb/zle", 0, (C, D, RC), ("lzjb", "logical"), ("frame", "encoded", True)),
    ("lzjb/zle", 15, (D, RC), ("lzjb", "logical"), ("frame", "encoded", True)),
]
FLAG_COUNTERS = {"sha256": ("sha256",), "sha512": ("sha512",), "frames": ("frames_encoded",),
                 "lzjb": ("lzjb_encoded", "zle_encoded"), "logical": ("logical_checked",)}


def _table(h, mode, flags):
    """the index into ROWS of the WRITE header `h` in `mode` with `flags`, or None = skipped"""
    ctype, p, arrive = h[48], struct.unpack_from("<Q", h, 88)[0], h[50]
    lsize, psize, dc, crypt = R.unprop(p)
    hashed = {R.FLETCHER4} | {t for t, f in ((R.SHA256, "sha256"), (R.SHA512, "sha512")) if flags.get(f)}
    if ctype not in hashed or p == 0 or crypt or lsize != struct.unpack_from("<Q", h, 32)[0]:
        return None
    covers = "raw" if dc in (0, 2) and psize == lsize else "lz4" if dc == 15 else "lzjb/zle" if dc in (3, 14) else None
    for k, (c, a, modes, needs, _) in enumerate(ROWS):
        if c == covers and (a == arrive or a == "same" and arrive == dc) and mode in modes and \
                all(flags.get(f) for f in needs):
            return k
    return None


def table(inp, mode, flags):
    """{record index: (row index or None, header)} of every WRITE of the plain stream `inp`"""
    b = inp.tobytes()
    return {i: (_table(b[off:off + 312], mode, flags), b[off:off + 312])
            for i, (off, _, _, t) in enumerate(R.records(inp)) if t == 3}


def tally(rows, verdicts):
    """the counters of mtz_block_stats (and first_bad) of `verdicts`, classified by `rows` (table())"""
    st = {k: sum(1 for v in verdicts.values() if v == k) for k in ("logical_ok", "frame_ok", "frame_miss", "skipped")}
    st["first_frame_miss"] = min([i for i, v in verdicts.items() if v == R.FRAME_MISS], default=R.NONE)
    st["first_bad"] = min([i for i, v in verdicts.items() if v == R.LOGICAL_BAD], default=R.NONE)
    checked = [(ROWS[k][4], h) for k, h in rows.values() if k is not None]
    st["sha256"] = sum(1 for _, h in checked if h[48] == R.SHA256)
    st["sha512"] = sum(1 for _, h in checked if h[48] == R.SHA512)
    for name, dc in (("frames_encoded", 15), ("lzjb_encoded", 3), ("zle_encoded", 14)):
        st[name] = sum(1 for (what, src, _), h in checked
                       if what == "frame" and src == "encoded" and R.unprop(R.get_key(h, 0)[2])[2] == dc)
    st["logical_checked"] = sum(1 for (_, _, lg), _ in checked if lg)
    return st


def flag_off(oracle, inp, mode, out, flag, **flags):
    """Turning `flag` off turns exactly the records of its rows (the table's, with it on; for a SHA flag
    every compared key of its type) to skipped,
    zeroes its counters and changes no other verdict; with it on and off every counter is the table's
    tally of the verdicts.  Returns the number of records the flag adds."""
    on, off = dict(flags, **{flag: True}), dict(flags, **{flag: False})
    von, son = R.block_check(oracle, inp, mode, out, **on)
    voff, soff = R.block_check(oracle, inp, mode, out, **off)
    rows = table(inp, mode, on)
    ctype = {"sha256": R.SHA256, "sha512": R.SHA512}.get(flag)
    mine = {i for i, (k, h) in rows.items() if k is not None and (flag in ROWS[k][3] or h[48] == ctype)}
    assert {i for i in von if von[i] != voff[i]} == mine and all(voff[i] == R.SKIPPED for i in mine), (mode, flag)
    assert all(soff[k] == 0 for k in FLAG_COUNTERS[flag]), (mode, flag, soff)
    assert son == tally(rows, von) and soff == tally(table(inp, mode, off), voff), (mode, flag)
    return len(mine)


def _foreign_lz4_key(oracle, s, i):
    """record i (an incompressible block keyed raw) keyed as if another LZ4 encoder had stored it: the
    stage's encoder stores it raw, so it is a frame miss wherever it is compared (re-stamped)"""
    off = R.records(s)[i][0]
    lsize = R.unprop(R.get_key(s, off)[2])[0]
    R.set_key(s, off, ddk_prop=R.prop(lsize, lsize - 512, R.DC_LZ4))
    assert oracle.stream_restamp(s)[0] == 0


def test_classification_follows_the_table(oracle):
    """Every key class in every mode, with every subset of the flags that add rows: the model's verdict
    is the table's, a checked block's verdict is OK exactly when its key is left as written, every
    counter is the table's tally, and every row of the table is reached."""
    from test_gpu_codec import _mixed_stream
    s, dcs = R.as_on_disk(oracle, _mixed_stream(oracle, n=40, recsize=8192), 9, R.mixed_codecs)
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
    foreign = next(i for i, v in dcs.items() if v == R.DC_OFF and
                   oracle.zfs_lz4_compress(s[recs[i][1]:recs[i][1] + recs[i][2]])[1] is None)
    for x in (s, c):
        _foreign_lz4_key(oracle, x, foreign)
    bad = set(mutate) | {foreign}
    rc, comp, _ = oracle.stream_compress(s)
    assert rc == 0
    sc = R.send_c_form(oracle, s)
    runs = [(s, None, R.VERIFY), (s, oracle.stream_compress_plain(s)[1], R.COMPRESS),
            (c, None, R.VERIFY), (c, oracle.stream_recompress(c)[1], R.RECOMPRESS),
            (sc, oracle.stream_recompress(sc)[1], R.RECOMPRESS), (oracle.wire_strip(comp), s, R.DECOMPRESS)]
    seen = set()
    for inp, out, mode in runs:
        for v in itertools.product((False, True), repeat=4):
            flags = dict(zip(("sha256", "frames", "lzjb", "logical"), v))
            verdicts, st = R.block_check(oracle, inp, mode, out, **flags)
            rows = table(inp, mode, flags)
            assert set(verdicts) == set(rows)
            for i, (k, _) in rows.items():
                seen.add(k)
                if k is None:
                    assert verdicts[i] == R.SKIPPED, (mode, flags, i)
                elif ROWS[k][4][0] == "logical":
                    assert verdicts[i] == (R.LOGICAL_BAD if i in bad else R.LOGICAL_OK), (mode, flags, i)
                else:
                    assert verdicts[i] == (R.FRAME_MISS if i in bad else R.FRAME_OK), (mode, flags, i)
            assert st["first_bad"] == R.NONE
            assert st == tally(rows, verdicts), (mode, flags)
    assert seen == {None} | set(range(len(ROWS)))


def test_a_corrupted_block_is_a_logical_mismatch_after_restamping(oracle):
    s = oracle.synth_stream(10, recsize=4096, kind=oracle.PAYLOAD_PCG).copy()
    recs = R.records(s)
    s[recs[6][1] + 17] ^= 1
    assert oracle.stream_restamp(s)[0] == 0 and oracle.stream_verify(s)[0] == 0
    verdicts, st = R.block_check(oracle, s, R.VERIFY)
    assert st["first_bad"] == 6 and st["logical_ok"] == 9 and verdicts[6] == R.LOGICAL_BAD
