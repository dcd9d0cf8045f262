"""Reference model of the block-checksum check (MTZ_FLAG_BLOCK_CKSUM) and the stream rewrites its
tests need.  Test infrastructure: plain Python and numpy over whole records, independent of the
library's closed form (K1 sums with the checksum-field words removed and zero words appended).

`zfs send` copies each block pointer's checksum into its DRR_WRITE record ([EXTERNAL] dmu_send.c
dump_write(); SURVEY.md App. A.1): drr_checksumtype at header byte 48, drr_key.ddk_cksum at 56..87,
drr_key.ddk_prop at 88..95 (LSIZE bits 0..15 and PSIZE bits 16..31 as size/512 - 1, on-disk
compression bits 32..38, crypt bit 39).  The checksum covers the PSIZE bytes on disk: the logical
block when it is stored raw, ZFS's LZ4 frame zero-padded to PSIZE when it is stored LZ4."""
import struct

import numpy as np

from test_real_streams import f4, payload_len

VERIFY, COMPRESS, DECOMPRESS, RECOMPRESS = 0, 1, 2, 3
FLETCHER4, SHA256 = 7, 8
DC_OFF, DC_LZ4, DC_ZSTD = 2, 15, 16
FEAT_LZ4, FEAT_COMPRESSED = 1 << 17, 1 << 22
NONE = (1 << 64) - 1

LOGICAL_OK, LOGICAL_BAD, FRAME_OK, FRAME_MISS, SKIPPED = "logical_ok", "logical_bad", "frame_ok", "frame_miss", "skipped"


def records(stream):
    """[(header offset, payload offset, payload length, drr_type)] of a plain send stream"""
    b = stream.tobytes() if isinstance(stream, np.ndarray) else bytes(stream)
    out, off = [], 0
    while off < len(b):
        h = b[off:off + 312]
        pl = payload_len(h)
        out.append((off, off + 312, pl, struct.unpack_from("<I", h, 0)[0]))
        off += 312 + pl
    return out


def prop(lsize, psize, dc, crypt=0):
    return ((lsize // 512 - 1) | ((psize // 512 - 1) << 16) | (dc << 32) | (crypt << 39)) & NONE


def unprop(p):
    return ((p & 0xffff) + 1) * 512, (((p >> 16) & 0xffff) + 1) * 512, (p >> 32) & 0x7f, (p >> 39) & 1


def set_key(s, off, ctype=None, key=None, ddk_prop=None):
    """rewrite the block-pointer fields of the WRITE header at `off` (in place, not re-stamped)"""
    if ctype is not None:
        s[off + 48] = ctype
    if key is not None:
        s[off + 56:off + 88] = np.frombuffer(struct.pack("<4Q", *key), dtype=np.uint8)
    if ddk_prop is not None:
        s[off + 88:off + 96] = np.frombuffer(struct.pack("<Q", ddk_prop), dtype=np.uint8)


def get_key(s, off):
    b = bytes(s[off:off + 96])
    return b[48], struct.unpack_from("<4Q", b, 56), struct.unpack_from("<Q", b, 88)[0]


def disk_frame(oracle, logical, ashift):
    """What ZFS with compression=lz4 writes for `logical`: the padded frame, or None when the block
    is stored raw (saves < 12.5 %, or no whole sector after rounding PSIZE up to 2**ashift)."""
    ps, frame = oracle.zfs_lz4_compress(logical)
    if frame is None:
        return None
    clen = 4 + int.from_bytes(frame[:4].tobytes(), "big")
    psize = -(-clen // (1 << ashift)) << ashift
    if psize >= len(logical):
        return None
    out = np.zeros(psize, dtype=np.uint8)
    out[:clen] = frame[:clen]
    return out


def as_lz4_on_disk(oracle, stream, ashift=9):
    """A raw stream whose keys say "written by ZFS with compression=lz4 at this ashift": each
    block's key is the Fletcher-4 of its disk frame, or of its logical bytes where ZFS would have
    stored it raw.  Re-stamped.  Returns (stream, {record index: on-disk compression})."""
    s = np.array(stream, dtype=np.uint8, copy=True)
    dcs = {}
    for i, (off, po, pl, t) in enumerate(records(s)):
        if t != 3 or s[off + 50] != 0:
            continue
        logical = s[po:po + pl]
        fr = disk_frame(oracle, logical, ashift)
        if fr is None:
            set_key(s, off, FLETCHER4, f4((0, 0, 0, 0), logical.tobytes()), prop(pl, pl, DC_OFF))
            dcs[i] = DC_OFF
        else:
            set_key(s, off, FLETCHER4, f4((0, 0, 0, 0), fr.tobytes()), prop(pl, fr.size, DC_LZ4))
            dcs[i] = DC_LZ4
    assert oracle.stream_restamp(s)[0] == 0
    return s, dcs


def as_send_c(oracle, stream, ashift=9):
    """The `zfs send -c` form of an as_lz4_on_disk() stream: every block stored LZ4 on disk travels
    as its disk frame (payload = the frame zero-padded to PSIZE, compression 15, compressed_size =
    PSIZE), the BEGIN announces compressed LZ4 records.  Re-stamped."""
    parts = []
    b = np.asarray(stream, dtype=np.uint8)
    for off, po, pl, t in records(b):
        h = b[off:off + 312].copy()
        pay = b[po:po + pl]
        if t == 0:
            vi = struct.unpack_from("<Q", h.tobytes(), 16)[0] | ((FEAT_COMPRESSED | FEAT_LZ4) << 2)
            h[16:24] = np.frombuffer(struct.pack("<Q", vi), dtype=np.uint8)
        if t == 3 and h[50] == 0:
            _, _, p = get_key(h, 0)
            lsize, psize, dc, _ = unprop(p)
            if dc == DC_LZ4:
                fr = disk_frame(oracle, pay, ashift)
                assert fr is not None and fr.size == psize
                h[50] = DC_LZ4
                h[96:104] = np.frombuffer(struct.pack("<Q", psize), dtype=np.uint8)
                pay = fr
        parts += [h, pay]
    s = np.ascontiguousarray(np.concatenate(parts))
    assert oracle.stream_restamp(s)[0] == 0
    return s


def block_check(inp, out, mode):
    """The classification of MTZ_FLAG_BLOCK_CKSUM, record by record.  `out` = the stage's output
    without wire preambles (None in VERIFY).  Returns ({record index: verdict}, counters) with the
    counters of mtz_block_stats plus first_bad (first LOGICAL_BAD, NONE if none)."""
    ib = inp.tobytes() if isinstance(inp, np.ndarray) else bytes(inp)
    irecs = records(inp)
    orecs = records(out) if out is not None else None
    ob = out.tobytes() if out is not None else None
    verdicts = {}
    for i, (off, po, pl, t) in enumerate(irecs):
        if t != 3:
            continue
        h = ib[off:off + 312]
        ctype = h[48]
        key = struct.unpack_from("<4Q", h, 56)
        p = struct.unpack_from("<Q", h, 88)[0]
        lsize, psize, dc, crypt = unprop(p)
        arrive = h[50]
        drr_lsize = struct.unpack_from("<Q", h, 32)[0]
        src = None                                   # (bytes at hand, what they are)
        if ctype == FLETCHER4 and p != 0 and not crypt and lsize == drr_lsize:
            if dc in (0, DC_OFF) and psize == lsize:
                if arrive == 0:
                    src = (ib[po:po + pl], "logical")
                elif arrive == DC_LZ4 and mode == DECOMPRESS:
                    _, opo, opl, _ = orecs[i]
                    src = (ob[opo:opo + opl], "logical")
            elif dc == DC_LZ4:
                if arrive == DC_LZ4:
                    src = (ib[po:po + pl], "frame")
                elif arrive == 0 and mode in (COMPRESS, RECOMPRESS):
                    ooff, opo, opl, _ = orecs[i]
                    # the stage stored the block raw where ZFS stored a frame: no frame to compare
                    src = (ob[opo:opo + opl] if ob[ooff + 50] == DC_LZ4 else None, "frame")
        if src is None:
            verdicts[i] = SKIPPED
            continue
        data, what = src
        cover = lsize if what == "logical" else psize
        ok = data is not None and len(data) <= cover and \
            f4((0, 0, 0, 0), data + bytes(cover - len(data))) == key
        if what == "logical":
            verdicts[i] = LOGICAL_OK if ok else LOGICAL_BAD
        else:
            verdicts[i] = FRAME_OK if ok else FRAME_MISS
    v = list(verdicts.items())
    st = {"logical_ok": sum(1 for _, x in v if x == LOGICAL_OK),
          "frame_ok": sum(1 for _, x in v if x == FRAME_OK),
          "frame_miss": sum(1 for _, x in v if x == FRAME_MISS),
          "skipped": sum(1 for _, x in v if x == SKIPPED),
          "first_frame_miss": min([i for i, x in v if x == FRAME_MISS], default=NONE),
          "first_bad": min([i for i, x in v if x == LOGICAL_BAD], default=NONE)}
    return verdicts, st
