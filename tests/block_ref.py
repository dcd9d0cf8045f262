"""Reference model of the block-checksum check (MTZ_FLAG_BLOCK_CKSUM and the flags that widen it) and
the stream rewrites its tests need.  Test infrastructure: plain Python, numpy and hashlib over whole
records, the oracle's LZ4 codec and tests/lzjb_ref.py's lzjb / zle encoders; independent of the
library's closed form (K1 sums with the checksum-field words removed and zero words appended).

`zfs send` copies each block pointer's checksum into its DRR_WRITE record ([EXTERNAL] dmu_send.c
dump_write(); SURVEY.md App. A.1): drr_checksumtype at header byte 48, drr_key.ddk_cksum at 56..87,
drr_key.ddk_prop at 88..95 (LSIZE bits 0..15 and PSIZE bits 16..31 as size/512 - 1, on-disk
compression bits 32..38, crypt bit 39).  The checksum covers the PSIZE bytes on disk: the logical
block when it is stored raw, ZFS's LZ4, lzjb or zle frame zero-padded to PSIZE when it is stored
compressed.  A fletcher4 key (type 7) is four native u64s.  A sha256 key (type 8) is the FIPS 180-4
digest's big-endian u64s ([EXTERNAL] OpenZFS zio_checksum_SHA256), stored as native words like every
other key.  A sha512 key (type 11) is SHA-512/256 (FIPS 180-4 5.3.6) with the 32 digest bytes in order,
no BE_64 per word ([EXTERNAL] OpenZFS abd_checksum_sha512_native).

block_check() classifies every record by the rows of block_classify (manatee_b200/csrc/kernels_block.cuh),
compares the bytes the row names with the key, and counts what mtz_block_stats counts."""
import collections
import hashlib
import struct
from concurrent.futures import ThreadPoolExecutor

import numpy as np

import lzjb_ref as Z
from test_real_streams import f4, payload_len

VERIFY, COMPRESS, DECOMPRESS, RECOMPRESS = 0, 1, 2, 3
FLETCHER4, SHA256, SHA512 = 7, 8, 11
CKSUM_SKEIN = 12            # a salted hash: never checkable
DC_OFF, DC_LZJB, DC_ZLE, DC_LZ4, DC_ZSTD = 2, Z.DC_LZJB, Z.DC_ZLE, 15, 16
FEAT_LZ4, FEAT_COMPRESSED = 1 << 17, 1 << 22
NONE = (1 << 64) - 1

LOGICAL_OK, LOGICAL_BAD, FRAME_OK, FRAME_MISS, SKIPPED = "logical_ok", "logical_bad", "frame_ok", "frame_miss", "skipped"
# the counters of mtz_block_stats; block_check's counters also hold first_bad (first LOGICAL_BAD, NONE if none)
COUNTERS = ("logical_ok", "frame_ok", "frame_miss", "skipped", "first_frame_miss", "sha256", "sha512",
            "frames_encoded", "lzjb_encoded", "zle_encoded", "logical_checked")
# what every stage of a transfer counts the same (four_ways): not which stage encoded or decoded for the check
TRANSFER = tuple(k for k in COUNTERS if k not in ("frames_encoded", "logical_checked"))
# block_classify's BLK_SRC_*: where the bytes a key is compared with are
IN, OUT, JOB, NOSRC = "input", "output", "job", "none"


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


def sha256_key(data):
    """the four ddk_cksum words of a SHA-256 key of `data`: BE_64 of the digest's 8-byte groups"""
    return struct.unpack(">4Q", hashlib.sha256(data).digest())


def sha512_key(data):
    """the four ddk_cksum words of a SHA-512 key of `data`: the SHA-512/256 digest read as
    little-endian u64s (the digest bytes in order)"""
    return struct.unpack("<4Q", hashlib.new("sha512_256", data).digest())


# ---- the check --------------------------------------------------------------------------------------

Header = collections.namedtuple("Header", "ctype key prop lsize psize dc crypt arrive drr_lsize")


def header(h):
    """the fields of the WRITE header `h` (312 bytes) the check reads"""
    p = struct.unpack_from("<Q", h, 88)[0]
    return Header(h[48], struct.unpack_from("<4Q", h, 56), p, *unprop(p), h[50], struct.unpack_from("<Q", h, 32)[0])


def classify(h, mode, have_out, hashes, frames, lzjb, logical):
    """block_classify's rows, in its order: (what, source, a row of MTZ_FLAG_BLOCK_LOGICAL) for the key of
    header `h`, or None = skipped.  `what` is "logical" or "frame"; the source is IN (the input payload),
    OUT (the output payload of a re-encoding mode), JOB (the check's own bytes: the logical bytes, or the
    frame the declared encoder makes of them) or NOSRC (a miss by rule).  `hashes`: the key types checked
    at all; `have_out`: the output is at hand (every mode but VERIFY)."""
    if h.ctype not in hashes or h.prop == 0 or h.crypt or h.lsize != h.drr_lsize:
        return None
    raw_in, lz4_in = h.arrive == 0, h.arrive == DC_LZ4
    encodes, decodes = mode in (COMPRESS, RECOMPRESS), mode in (DECOMPRESS, RECOMPRESS)
    # the logical bytes of a record that arrives LZ4 exist only where the stage decodes it: not in COMPRESS
    lg = logical and ((encodes or decodes) if raw_in else (lz4_in and decodes))
    if h.dc in (0, DC_OFF) and h.psize == h.lsize:
        if raw_in:
            return "logical", IN, False
        if lz4_in and mode == DECOMPRESS and have_out:
            return "logical", OUT, False
        if lz4_in and mode == RECOMPRESS and lg:
            return "logical", JOB, True
    elif h.dc == DC_LZ4:
        if lz4_in:
            return "frame", IN, False
        if raw_in and encodes and have_out:
            return "frame", OUT, False
        if raw_in and frames and mode == VERIFY:
            return "frame", JOB, False
        if raw_in and mode == DECOMPRESS and lg:
            return "frame", NOSRC, True
    elif lzjb and h.dc in (DC_LZJB, DC_ZLE):
        if h.arrive == h.dc and mode in (VERIFY, RECOMPRESS):
            return "frame", IN, False
        if raw_in and mode == VERIFY:
            return "frame", JOB, False
        if (raw_in or lz4_in) and lg:
            return "frame", JOB, True
    return None


def encoder_frame(oracle, codec, logical):
    """what the stage's encoder of `codec` (DC_LZ4, DC_LZJB or DC_ZLE) stores for `logical`: the frame
    zero-padded to its 512-byte PSIZE, or None when it stores the block raw.  LZ4: the oracle's
    zfs_lz4_compress, the declared encoder; lzjb / zle: ZFS's C code at phase 0 (tests/lzjb_ref.py)."""
    if codec == DC_LZ4:
        ps, frame = oracle.zfs_lz4_compress(logical)
        if frame is None:
            return None
        clen = 4 + int.from_bytes(frame[:4].tobytes(), "big")
        return frame[:clen].tobytes() + bytes(ps - clen)
    (_, fr), _ = Z.zfs_lzjb_compress(logical, 0) if codec == DC_LZJB else Z.zfs_zle_compress(logical)
    return fr


def block_check(oracle, inp, mode, out=None, *, sha256=False, sha512=False, frames=False, lzjb=False,
                logical=False):
    """The block check in `mode` on the plain stream `inp`, `out` = the stage's plain output (None in
    VERIFY), with MTZ_FLAG_BLOCK_SHA256 / _SHA512 / _FRAMES / _LZJB / _LOGICAL as the flags say.
    Returns ({record index: verdict}, counters): COUNTERS and first_bad."""
    hashes = {FLETCHER4: lambda b: f4((0, 0, 0, 0), b)}
    if sha256:
        hashes[SHA256] = sha256_key
    if sha512:
        hashes[SHA512] = sha512_key
    ib = inp.tobytes() if isinstance(inp, np.ndarray) else bytes(inp)
    ob = out.tobytes() if isinstance(out, np.ndarray) else out
    orecs = records(ob) if ob is not None else None
    verdicts, st = {}, dict.fromkeys(COUNTERS, 0)
    for i, (off, po, pl, t) in enumerate(records(ib)):
        if t != 3:
            continue
        h = header(ib[off:off + 312])
        row = classify(h, mode, ob is not None, hashes, frames, lzjb, logical)
        if row is None:
            verdicts[i] = SKIPPED
            continue
        what, src, lg = row
        data = None
        if src == IN:
            data = ib[po:po + pl]
        elif src == OUT:
            ooff, opo, opl, _ = orecs[i]
            # the stage stored the block raw where ZFS stored a frame: no frame to compare
            data = ob[opo:opo + opl] if what == "logical" or ob[ooff + 50] == DC_LZ4 else None
        elif src == JOB:
            data = ib[po:po + pl]
            if h.arrive == DC_LZ4:
                rc, d = oracle.zfs_lz4_decompress(np.frombuffer(data, dtype=np.uint8), h.lsize)
                assert rc == 0
                data = d.tobytes()
            if what == "frame":
                data = encoder_frame(oracle, h.dc, np.frombuffer(data, dtype=np.uint8))
                st[{DC_LZ4: "frames_encoded", DC_LZJB: "lzjb_encoded", DC_ZLE: "zle_encoded"}[h.dc]] += 1
        cover = h.lsize if what == "logical" else h.psize
        ok = data is not None and len(data) <= cover and hashes[h.ctype](data + bytes(cover - len(data))) == h.key
        if what == "logical":
            verdicts[i] = LOGICAL_OK if ok else LOGICAL_BAD
        else:
            verdicts[i] = FRAME_OK if ok else FRAME_MISS
        if h.ctype in (SHA256, SHA512):
            st["sha256" if h.ctype == SHA256 else "sha512"] += 1
        st["logical_checked"] += lg
    v = list(verdicts.items())
    for x in (LOGICAL_OK, FRAME_OK, FRAME_MISS, SKIPPED):
        st[x] = sum(1 for _, y in v if y == x)
    st["first_frame_miss"] = min([i for i, x in v if x == FRAME_MISS], default=NONE)
    st["first_bad"] = min([i for i, x in v if x == LOGICAL_BAD], default=NONE)
    return verdicts, st


# ---- streams ----------------------------------------------------------------------------------------

def disk_frame(oracle, logical, ashift, codec=DC_LZ4):
    """What ZFS with compression=`codec` (DC_LZ4, DC_LZJB or DC_ZLE) writes for `logical` at this ashift:
    the encoder's frame zero-padded to PSIZE, or None when the block is stored raw (no whole sector
    saved after rounding PSIZE up to 2**ashift)."""
    fr = encoder_frame(oracle, codec, logical)
    if fr is None:
        return None
    psize = -(-len(fr) // (1 << ashift)) << ashift
    if psize >= len(logical):
        return None
    return np.frombuffer(fr + bytes(psize - len(fr)), dtype=np.uint8)


def as_on_disk(oracle, stream, ashift=9, codec=DC_LZ4):
    """A raw stream whose keys say "written by ZFS with compression=codec at this ashift", `codec` one of
    DC_LZ4 / DC_LZJB / DC_ZLE / DC_OFF or a function of the record index that returns one: each block's
    key is the Fletcher-4 of its disk frame, or of its logical bytes where ZFS would have stored it raw.
    Re-stamped.  Returns (stream, {record index: on-disk compression})."""
    pick = codec if callable(codec) else (lambda i: codec)
    s = np.array(stream, dtype=np.uint8, copy=True)
    dcs = {}
    for i, (off, po, pl, t) in enumerate(records(s)):
        if t != 3 or s[off + 50] != 0:
            continue
        logical = s[po:po + pl]
        dc = pick(i)
        fr = None if dc == DC_OFF else disk_frame(oracle, logical, ashift, dc)
        if fr is None:
            set_key(s, off, FLETCHER4, f4((0, 0, 0, 0), logical.tobytes()), prop(pl, pl, DC_OFF))
            dcs[i] = DC_OFF
        else:
            set_key(s, off, FLETCHER4, f4((0, 0, 0, 0), fr.tobytes()), prop(pl, fr.size, dc))
            dcs[i] = dc
    assert oracle.stream_restamp(s)[0] == 0
    return s, dcs


def mixed_codecs(i):
    """lzjb, zle, lz4 and (unchanged: logical) keys in turn"""
    return (DC_LZJB, DC_ZLE, DC_LZ4, DC_LZJB, DC_OFF)[i % 5]


def _rebuild(oracle, stream, fn):
    """the stream with each record's (header copy, payload) replaced by fn(type, header, payload); re-stamped"""
    parts = []
    b = np.asarray(stream, dtype=np.uint8)
    for off, po, pl, t in records(b):
        parts += fn(t, b[off:off + 312].copy(), b[po:po + pl])
    s = np.ascontiguousarray(np.concatenate(parts))
    assert oracle.stream_restamp(s)[0] == 0
    return s


def as_send_c(oracle, stream, ashift=9):
    """The `zfs send -c` form of an as_on_disk() stream: every block stored compressed on disk travels
    as its disk frame (payload = the frame zero-padded to PSIZE, compression = the on-disk one,
    compressed_size = PSIZE), the BEGIN announces compressed records.  Re-stamped."""
    def rec(t, h, pay):
        if t == 0:
            vi = struct.unpack_from("<Q", h.tobytes(), 16)[0] | ((FEAT_COMPRESSED | FEAT_LZ4) << 2)
            h[16:24] = np.frombuffer(struct.pack("<Q", vi), dtype=np.uint8)
        if t == 3 and h[50] == 0:
            _, _, p = get_key(h, 0)
            lsize, psize, dc, _ = unprop(p)
            if dc in (DC_LZ4, DC_LZJB, DC_ZLE):
                fr = disk_frame(oracle, pay, ashift, dc)
                assert fr is not None and fr.size == psize
                h[50] = dc
                h[96:104] = np.frombuffer(struct.pack("<Q", psize), dtype=np.uint8)
                pay = fr
        return [h, pay]
    return _rebuild(oracle, stream, rec)


def trim_frames(oracle, stream, align=8):
    """A `send -c` stream whose LZ4 payloads stop at the frame's end rounded up to `align` bytes (a
    multiple of 8 that divides 512) instead of PSIZE (compressed_size follows; the keys, which cover
    PSIZE, stay): the bytes at hand are shorter than what the key covers.  With align=8 most end inside
    a 64- or 128-byte block, with align=128 every one ends on a 128-byte boundary.  Re-stamped."""
    def rec(t, h, pay):
        if t == 3 and h[50] == DC_LZ4:
            n = -(-(4 + int.from_bytes(pay[:4].tobytes(), "big")) // align) * align
            if n < pay.size:
                pay = pay[:n]
                h[96:104] = np.frombuffer(struct.pack("<Q", n), dtype=np.uint8)
        return [h, pay]
    return _rebuild(oracle, stream, rec)


def as_sha(oracle, stream, name, threads=1):
    """The same stream written to a dataset with checksum=`name` ("sha256" or "sha512"): every fletcher4
    key of a WRITE that arrives raw becomes the SHA-256 or SHA-512/256 key of the bytes it covers -- the
    logical block, or its disk frame zero-padded to PSIZE.  Re-stamped; composes with as_send_c and
    trim_frames.  `threads` hash in parallel (hashlib releases the GIL)."""
    hf, ct = (sha256_key, SHA256) if name == "sha256" else (sha512_key, SHA512)
    s = np.array(stream, dtype=np.uint8, copy=True)
    todo = [(off, po, pl) for off, po, pl, t in records(s)
            if t == 3 and s[off + 50] == 0 and s[off + 48] == FLETCHER4]

    def key(job):
        off, po, pl = job
        _, psize, dc, _ = unprop(get_key(s, off)[2])
        logical = s[po:po + pl]
        if dc not in (DC_LZ4, DC_LZJB, DC_ZLE):
            return hf(logical.tobytes())
        fr = disk_frame(oracle, logical, 9, dc).tobytes()
        return hf(fr[:psize] + bytes(max(0, psize - len(fr))))

    if threads > 1:
        with ThreadPoolExecutor(threads) as ex:
            keys = list(ex.map(key, todo, chunksize=64))
    else:
        keys = [key(j) for j in todo]
    for (off, _, _), k in zip(todo, keys):
        set_key(s, off, ct, k)
    assert oracle.stream_restamp(s)[0] == 0
    return s


def mixed_keys_stream(oracle, n=40, recsize=8192, seed=0):
    """A raw stream (`zfs send` without -c) whose records carry a seeded mix of keys: on-disk lzjb, zle,
    LZ4 and raw; fletcher4, sha256 and sha512; and every ninth or so one the stage cannot check (zstd on
    disk, encrypted, a salted hash).  pg-page records with incompressible and all-zero ones mixed in, so
    some compressed-on-disk picks end up stored raw, and some of those carry an LZ4 key that no frame of
    the stage can match.  Returns (stream, {record index: on-disk compression
    of the checkable ones})."""
    from test_gpu_codec import _mixed_stream
    rng = np.random.default_rng(seed)
    picks = rng.integers(0, 4, 2 * n + 8)
    s, dcs = as_on_disk(oracle, _mixed_stream(oracle, n=n, recsize=recsize), 9,
                        lambda i: (DC_LZJB, DC_ZLE, DC_LZ4, DC_OFF)[picks[i]])
    for i, (off, po, pl, t) in enumerate(records(s)):
        if i not in dcs:
            continue
        lsize, psize, dc, _ = unprop(get_key(s, off)[2])
        logical = s[po:po + pl]
        data = logical.tobytes() if dcs[i] == DC_OFF else disk_frame(oracle, logical, 9, dc).tobytes()
        if dcs[i] == DC_OFF and picks[i] != 3 and i % 2 == 0 and lsize > 512:
            # a block no declared encoder shrinks, keyed as if another LZ4 encoder had: a frame miss wherever
            # it is checked, and on the compressed wire a record that travels raw under an LZ4 key
            set_key(s, off, ddk_prop=prop(lsize, lsize - 512, DC_LZ4))
            dcs[i] = DC_LZ4
        how = int(rng.integers(0, 9))
        if how in (1, 2):
            set_key(s, off, SHA256, sha256_key(data))
        elif how in (3, 4):
            set_key(s, off, SHA512, sha512_key(data))
        elif how == 5:
            kind = int(rng.integers(0, 3))
            if kind == 0:
                set_key(s, off, ddk_prop=prop(lsize, psize, DC_ZSTD))
            elif kind == 1:
                set_key(s, off, ddk_prop=prop(lsize, psize, dc, crypt=1))
            else:
                set_key(s, off, ctype=CKSUM_SKEIN)
            del dcs[i]
    assert oracle.stream_restamp(s)[0] == 0
    return s, dcs


def send_c_form(oracle, x):
    """the compressed form of a raw stream the RECOMPRESS tests feed the stage: every record the oracle's
    encoder can store as an LZ4 frame travels as one, whatever its key says"""
    rc, c, _ = oracle.stream_compress_plain(x)
    assert rc == 0
    return np.ascontiguousarray(c)


def four_ways(oracle, x, **flags):
    """the model's counters of the four stages of a transfer of the raw stream `x` with
    MTZ_FLAG_BLOCK_LOGICAL, `flags` the other flags: VERIFY on x, COMPRESS on x, DECOMPRESS on
    COMPRESS(x), RECOMPRESS on the send-c form.  With frames=True they agree on TRANSFER."""
    c = send_c_form(oracle, x)
    rc, d, _ = oracle.stream_decompress(oracle.stream_compress(x)[1])
    rc2, r, _ = oracle.stream_recompress(c)
    assert rc == 0 and rc2 == 0 and np.array_equal(d, x)
    return {"verify": block_check(oracle, x, VERIFY, None, logical=True, **flags),
            "compress": block_check(oracle, x, COMPRESS, c, logical=True, **flags),
            "decompress": block_check(oracle, c, DECOMPRESS, x, logical=True, **flags),
            "recompress": block_check(oracle, c, RECOMPRESS, r, logical=True, **flags)}
