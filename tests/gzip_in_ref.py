"""Reference model of COMPRESS with MTZ_FLAG_COMPRESSED_IN | MTZ_FLAG_GZIP_IN: compressed_in_ref's model
with gzip-1 .. gzip-9 records (drr_compressiontype 5..13) inflated.  Test infrastructure, built on
compressed_in_ref, block_ref and Python's zlib.

ZFS's gzip-N ([EXTERNAL] gzip.c gzip_compress) is zlib's compress2 at level N into a buffer of
d_len = lsize - lsize/8 bytes: a stream that does not fit is stored raw.  zio pads the frame to a whole
sector, the block is stored raw when that does not save one at the ashift, and the key covers the padded
frame.  `zfs send -c` carries that frame (compressed_size = PSIZE).

The stage's acceptance rule is zlib's made strict on length: inflate of the whole payload reaches the
end of the stream (Adler-32 trailer checked) and yields exactly lsize bytes; the bytes after the
trailer are ignored.  inflate() below states it through zlib.decompressobj."""
import struct
import zlib

import numpy as np

import block_ref as B
import compressed_in_ref as M

GZIP_IN = 1024              # MTZ_FLAG_GZIP_IN
DC_GZIP = {n: 4 + n for n in range(1, 10)}      # gzip-N -> on-disk / stream compression 5..13
GZIP_DCS = tuple(DC_GZIP.values())


def is_gzip(dc):
    return dc in GZIP_DCS


def level(dc):
    return dc - 4


def inflate(frame, lsize):
    """the lsize bytes zlib inflates `frame` to, or None when the stage must fail the record"""
    d = zlib.decompressobj()
    try:
        out = d.decompress(bytes(frame))
    except zlib.error:
        return None
    return out if d.eof and len(out) == lsize else None


def gzip_frame(logical, dc):
    """what ZFS's gzip-N stores for `logical`: the zlib stream zero-padded to a 512-byte sector, or None
    when the block is stored raw (the stream exceeds d_len, or padding saves no sector)"""
    b = bytes(logical)
    c = zlib.compress(b, level(dc))
    if len(c) > len(b) - len(b) // 8:
        return None
    ps = -(-len(c) // 512) * 512
    return None if ps >= len(b) else c + bytes(ps - len(c))


def disk_frame(oracle, logical, ashift, codec):
    """block_ref.disk_frame extended to gzip-N"""
    if not is_gzip(codec):
        return B.disk_frame(oracle, logical, ashift, codec)
    fr = gzip_frame(logical, codec)
    if fr is None:
        return None
    psize = -(-len(fr) // (1 << ashift)) << ashift
    if psize >= len(logical):
        return None
    return np.frombuffer(fr + bytes(psize - len(fr)), dtype=np.uint8)


def as_on_disk(oracle, stream, ashift=9, codec=DC_GZIP[6]):
    """block_ref.as_on_disk with gzip-N codecs as well: every DRR_WRITE keyed with the Fletcher-4 of its
    disk frame, or of its logical bytes where ZFS stores it raw.  Returns (stream, {index: on-disk dc})."""
    pick = codec if callable(codec) else (lambda i: codec)
    s = np.array(stream, dtype=np.uint8, copy=True)
    dcs = {}
    for i, (off, po, pl, t) in enumerate(B.records(s)):
        if t != 3 or s[off + 50] != 0:
            continue
        logical = s[po:po + pl]
        dc = pick(i)
        fr = None if dc == B.DC_OFF else disk_frame(oracle, logical, ashift, dc)
        if fr is None:
            B.set_key(s, off, B.FLETCHER4, B.f4((0, 0, 0, 0), logical.tobytes()), B.prop(pl, pl, B.DC_OFF))
            dcs[i] = B.DC_OFF
        else:
            B.set_key(s, off, B.FLETCHER4, B.f4((0, 0, 0, 0), fr.tobytes()), B.prop(pl, fr.size, dc))
            dcs[i] = dc
    assert oracle.stream_restamp(s)[0] == 0
    return s, dcs


def as_send_c(oracle, stream, ashift=9):
    """block_ref.as_send_c with gzip-N blocks travelling as their disk frame too"""
    def rec(t, h, pay):
        if t == 0:
            vi = struct.unpack_from("<Q", h.tobytes(), 16)[0] | ((B.FEAT_COMPRESSED | B.FEAT_LZ4) << 2)
            h[16:24] = np.frombuffer(struct.pack("<Q", vi), dtype=np.uint8)
        if t == 3 and h[50] == 0:
            _, _, p = B.get_key(h, 0)
            lsize, psize, dc, _ = B.unprop(p)
            if dc in (B.DC_LZ4, B.DC_LZJB, B.DC_ZLE) or is_gzip(dc):
                fr = disk_frame(oracle, pay, ashift, dc)
                assert fr is not None and fr.size == psize
                h[50] = dc
                h[96:104] = np.frombuffer(struct.pack("<Q", psize), dtype=np.uint8)
                pay = fr
        return [h, pay]
    return B._rebuild(oracle, stream, rec)


def send_c(oracle, s, ashift=9, codec=DC_GZIP[6]):
    """the `zfs send -c` stream of the raw stream s written with compression=codec at this ashift"""
    return as_send_c(oracle, as_on_disk(oracle, s, ashift, codec)[0], ashift)


def mixed_codecs(i):
    """gzip-6, lz4, lzjb and (unchanged: logical) keys in turn"""
    return (DC_GZIP[6], B.DC_LZ4, DC_GZIP[6], B.DC_LZJB, B.DC_OFF)[i % 5]


# ---- the model --------------------------------------------------------------------------------------

def decode(oracle, comp, frame, lsize):
    """compressed_in_ref.decode with gzip-N inflated"""
    return inflate(frame, lsize) if is_gzip(comp) else M.decode(oracle, comp, frame, lsize)


def plain(oracle, x):
    """the stream `zfs send` without -c would have produced for the `send -c` stream x"""
    def rec(t, h, pay):
        if t == 0:
            vi = struct.unpack_from("<Q", h.tobytes(), 16)[0]
            feat = (vi >> 2) & ((1 << 30) - 1)
            if feat & M.FEAT_COMPRESSED:
                vi &= ~(M.FEAT_COMPRESSED << 2)
                if not feat & M.FEAT_EMBED_DATA:
                    vi &= ~(M.FEAT_LZ4 << 2)
                h[16:24] = np.frombuffer(struct.pack("<Q", vi), dtype=np.uint8)
        if t == 3 and h[50] != 0:
            d = decode(oracle, int(h[50]), pay, M._lsize(h))
            assert d is not None, "plain() of a stream the stage refuses"
            h[50] = 0
            h[96:104] = 0
            pay = np.frombuffer(d, dtype=np.uint8)
        return [h, pay]
    return B._rebuild(oracle, x, rec)


def verdict(oracle, x):
    """(first failing record or None, the counters of mtz_compressed_in_stats with gzip_decoded)"""
    st = {"lz4_passed": 0, "lzjb_decoded": 0, "zle_decoded": 0, "gzip_decoded": 0}
    b = np.asarray(x, dtype=np.uint8)
    for i, (off, po, pl, t) in enumerate(B.records(b)):
        if t != 3 or b[off + 50] == 0:
            continue
        c = int(b[off + 50])
        if c == M.DC_LZ4:
            st["lz4_passed"] += 1
            continue
        if decode(oracle, c, b[po:po + pl], M._lsize(b[off:off + 312])) is None:
            return i, st
        st["gzip_decoded" if is_gzip(c) else "lzjb_decoded" if c == M.DC_LZJB else "zle_decoded"] += 1
    return None, st


def expected(oracle, x):
    """COMPRESS with MTZ_FLAG_COMPRESSED_IN | MTZ_FLAG_GZIP_IN of x (a stream the stage accepts)"""
    rc, w, _ = oracle.stream_compress(plain(oracle, x))
    assert rc == 0
    return M.splice(oracle, w, x)


def block_check(oracle, x, **flags):
    """the block counters of COMPRESS with the flag over the send -c stream x: VERIFY's (block_ref with
    MTZ_FLAG_BLOCK_LZJB) plus the new row -- a record with a gzip-N key that arrives as that frame is
    compared as it is, frame_ok or frame_miss; without MTZ_FLAG_GZIP_IN it stays skipped"""
    verdicts, st = B.block_check(oracle, x, B.VERIFY, lzjb=True, **flags)
    hashes = {B.FLETCHER4: lambda d: B.f4((0, 0, 0, 0), d)}
    if flags.get("sha256"):
        hashes[B.SHA256] = B.sha256_key
    if flags.get("sha512"):
        hashes[B.SHA512] = B.sha512_key
    b = np.asarray(x, dtype=np.uint8).tobytes()
    for i, (off, po, pl, t) in enumerate(B.records(b)):
        if t != 3:
            continue
        h = B.header(b[off:off + 312])
        if not (is_gzip(h.dc) and h.arrive == h.dc and h.ctype in hashes and h.prop != 0 and not h.crypt
                and h.lsize == h.drr_lsize):
            continue
        assert verdicts[i] == B.SKIPPED
        data = b[po:po + pl]
        ok = len(data) <= h.psize and hashes[h.ctype](data + bytes(h.psize - len(data))) == h.key
        verdicts[i] = B.FRAME_OK if ok else B.FRAME_MISS
        st["skipped"] -= 1
        st[verdicts[i]] += 1
        if h.ctype in (B.SHA256, B.SHA512):
            st["sha256" if h.ctype == B.SHA256 else "sha512"] += 1
        if not ok:
            st["first_frame_miss"] = min(st["first_frame_miss"], i)
    return verdicts, st
