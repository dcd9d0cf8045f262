"""Reference model of COMPRESS with MTZ_FLAG_COMPRESSED_IN: a `zfs send -c` stream in, the lz4-stage-v1
wire out.  Test infrastructure: plain Python and numpy over whole records, built from the pieces the
repository already trusts -- the oracle's ZFS-LZ4 codec and stream re-stamp (oracle/), the lzjb / zle
decoders of tests/lzjb_ref.py (the pure-Python restatement, bounded by the frame: an IndexError is a
malformed frame; ZFS's C code of tests/lzjb_zfs.c as a second opinion wherever the first accepts) and
block_ref's stream rewrites.

  plain(x)     what `zfs send` without -c would have produced: every compressed DRR_WRITE replaced by
               its logical bytes (compression 0, compressed size 0), COMPRESSED cleared from BEGIN and
               LZ4 cleared unless EMBED_DATA is set; re-stamped.  DECOMPRESS(COMPRESS_flag(x)) == plain(x).
  expected(x)  COMPRESS_flag(x) byte for byte: COMPRESS of plain(x) with every record that arrived LZ4
               put back as it arrived; re-stamped, one preamble in front of each BEGIN.
  verdict(x)   the stage's verdict: (None, counters) or (index of the failing record, counters)."""
import struct

import numpy as np

import block_ref as B
import lzjb_ref as Z

COMPRESS_IN = 512           # MTZ_FLAG_COMPRESSED_IN
DC_LZJB, DC_ZLE, DC_LZ4, DC_GZIP6, DC_ZSTD = 3, 14, 15, 7, 16
FEAT_EMBED_DATA, FEAT_LZ4, FEAT_COMPRESSED = 1 << 16, 1 << 17, 1 << 22
WIRE_F_ORIG_LZ4 = 1


def features(h):
    return (struct.unpack_from("<Q", bytes(h[:312]), 16)[0] >> 2) & ((1 << 30) - 1)


def orig_lz4(feat):
    """the preamble's WIRE_F_ORIG_LZ4 for a BEGIN with these features: the stream `zfs send` without
    -c would have produced carries the LZ4 feature (-c alone sets it, without -c only -e does)"""
    return bool(feat & FEAT_LZ4) and (not feat & FEAT_COMPRESSED or bool(feat & FEAT_EMBED_DATA))


def decode(oracle, comp, frame, lsize):
    """the logical bytes of a DRR_WRITE payload stored with `comp`, or None when the stage must fail
    the record (a malformed frame, or a compression it has no decoder for)"""
    frame = bytes(frame)
    if comp == DC_LZ4:
        rc, d = oracle.zfs_lz4_decompress(np.frombuffer(frame, dtype=np.uint8), lsize)
        return d.tobytes() if rc == 0 else None
    if comp not in (DC_LZJB, DC_ZLE):
        return None
    py, zfs = (Z.py_lzjb_decompress, Z.zfs_lzjb_decompress) if comp == DC_LZJB else \
        (Z.py_zle_decompress, Z.zfs_zle_decompress)
    try:
        d = py(frame, lsize)
    except IndexError:                 # the decode would read at or past the end of the frame
        return None
    if d is not None:
        assert zfs(frame, lsize) == d, "the two restatements of ZFS's decoder disagree"
    return d


def _comp(h):
    return int(h[50])


def _lsize(h):
    return struct.unpack_from("<Q", bytes(h[:312]), 32)[0]


def plain(oracle, x):
    """the stream `zfs send` without -c would have produced for the `send -c` stream x"""
    def rec(t, h, pay):
        if t == 0:
            vi = struct.unpack_from("<Q", h.tobytes(), 16)[0]
            feat = (vi >> 2) & ((1 << 30) - 1)
            if feat & FEAT_COMPRESSED:
                vi &= ~(FEAT_COMPRESSED << 2)
                if not feat & FEAT_EMBED_DATA:
                    vi &= ~(FEAT_LZ4 << 2)
                h[16:24] = np.frombuffer(struct.pack("<Q", vi), dtype=np.uint8)
        if t == 3 and _comp(h) != 0:
            d = decode(oracle, _comp(h), pay, _lsize(h))
            assert d is not None, "plain() of a stream the stage refuses"
            h[50] = 0
            h[96:104] = 0
            pay = np.frombuffer(d, dtype=np.uint8)
        return [h, pay]
    return B._rebuild(oracle, x, rec)


def verdict(oracle, x):
    """(first failing record or None, the counters of mtz_compressed_in_stats)"""
    st = {"lz4_passed": 0, "lzjb_decoded": 0, "zle_decoded": 0}
    b = np.asarray(x, dtype=np.uint8)
    for i, (off, po, pl, t) in enumerate(B.records(b)):
        if t != 3 or b[off + 50] == 0:
            continue
        c = int(b[off + 50])
        if c == DC_LZ4:
            st["lz4_passed"] += 1
            continue
        if decode(oracle, c, b[po:po + pl], _lsize(b[off:off + 312])) is None:
            return i, st
        st["lzjb_decoded" if c == DC_LZJB else "zle_decoded"] += 1
    return None, st


def splice(oracle, wire, x):
    """`wire` (a COMPRESS output of plain(x), preambles included) with every record that arrived LZ4 in
    x put back as it arrived, re-stamped: what COMPRESS with the flag makes of x when its encoder makes
    `wire` of plain(x)"""
    w = np.asarray(wire, dtype=np.uint8)
    body = oracle.wire_strip(w)
    pres = [w[i:i + 32].copy() for i in range(w.size - 7) if w[i:i + 8].tobytes() == oracle.WIRE_MAGIC]
    xb = np.asarray(x, dtype=np.uint8)
    xr, wr = B.records(xb), B.records(body)
    assert len(xr) == len(wr)
    parts, k = [], 0
    for (xo, xpo, xpl, t), (wo, wpo, wpl, _) in zip(xr, wr):
        if t == 0:
            parts.append(pres[k])
            k += 1
        if t == 3 and xb[xo + 50] == DC_LZ4:
            parts.append(xb[xo:xpo + xpl])
        else:
            parts.append(body[wo:wpo + wpl])
    out = np.ascontiguousarray(np.concatenate(parts))
    # re-stamp the records between the preambles
    pos = [i for i in range(out.size - 7) if out[i:i + 8].tobytes() == oracle.WIRE_MAGIC] + [out.size]
    for a, e in zip(pos, pos[1:]):
        seg = np.ascontiguousarray(out[a + 32:e])
        assert oracle.stream_restamp(seg)[0] == 0
        out[a + 32:e] = seg
    return out


def expected(oracle, x):
    """COMPRESS with MTZ_FLAG_COMPRESSED_IN of x (a stream the stage accepts), with ZFS's LZ4 encoder"""
    rc, w, _ = oracle.stream_compress(plain(oracle, x))
    assert rc == 0
    return splice(oracle, w, x)


def encoded(oracle, wire, x):
    """mtz_stats.lz4_encoded of that COMPRESS: LZ4 records on the wire that did not arrive LZ4"""
    xb, wb = np.asarray(x, dtype=np.uint8), oracle.wire_strip(wire)
    n = 0
    for (xo, _, _, t), (wo, _, _, _) in zip(B.records(xb), B.records(wb)):
        n += t == 3 and wb[wo + 50] == DC_LZ4 and xb[xo + 50] != DC_LZ4
    return n


# ---- streams ----------------------------------------------------------------------------------------

def send_c(oracle, s, ashift=9, codec=DC_LZ4):
    """the `zfs send -c` stream of the raw stream s written with compression=codec at this ashift
    (codec as block_ref.as_on_disk takes it)"""
    return B.as_send_c(oracle, B.as_on_disk(oracle, s, ashift, codec)[0], ashift)


def set_features(oracle, x, on=0, off=0):
    """x with BEGIN features `on` set and `off` cleared; re-stamped"""
    s = np.array(x, dtype=np.uint8, copy=True)
    vi = struct.unpack_from("<Q", s[16:24].tobytes(), 0)[0]
    vi = (vi | (on << 2)) & ~(off << 2)
    s[16:24] = np.frombuffer(struct.pack("<Q", vi), dtype=np.uint8)
    assert oracle.stream_restamp(s)[0] == 0
    return s


def write_records(x, comp=None):
    """[(index, header offset, payload offset, payload length)] of x's DRR_WRITEs (of compression comp)"""
    b = np.asarray(x, dtype=np.uint8)
    return [(i, off, po, pl) for i, (off, po, pl, t) in enumerate(B.records(b))
            if t == 3 and (comp is None or b[off + 50] == comp)]


def replace_payload(oracle, x, index, payload, comp=None):
    """x with record `index`'s payload replaced (compressed_size follows; compression = comp if given);
    re-stamped"""
    seen = [-1]

    def rec(t, h, pay):
        seen[0] += 1
        if seen[0] == index:
            pay = np.frombuffer(bytes(payload), dtype=np.uint8)
            h[96:104] = np.frombuffer(struct.pack("<Q", pay.size), dtype=np.uint8)
            if comp is not None:
                h[50] = comp
        return [h, pay]
    return B._rebuild(oracle, x, rec)


def lzjb_items(frame, lsize):
    """[(frame position, is a match, output position)] of the items ZFS's decoder reads from an lzjb
    frame that decodes"""
    f, items, i, op, cm, bit = bytes(frame), [], 0, 0, 0, 0x80
    while op < lsize:
        bit <<= 1
        if bit == 0x100:
            cm, bit = f[i], 1
            i += 1
        if cm & bit:
            items.append((i, True, op))
            op += min((f[i] >> 2) + 3, lsize - op)
            i += 2
        else:
            items.append((i, False, op))
            op += 1
            i += 1
    return items


def zle_tokens(frame, lsize):
    """[(frame position, run bytes, a zero run)] of the tokens ZFS's zle decoder reads"""
    f, toks, i, op = bytes(frame), [], 0, 0
    while op < lsize:
        n = 1 + f[i]
        toks.append((i, n if n <= Z.ZLE_N else n - Z.ZLE_N, n > Z.ZLE_N))
        if n <= Z.ZLE_N:
            i += n
        else:
            n -= Z.ZLE_N
        i += 1
        op += n
    return toks
