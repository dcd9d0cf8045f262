"""Payload families for the LZ4 kernels' parity tests (test infrastructure), the frames other encoders
make of them, and the certificate verdict RECOMPRESS must reach on each frame.

`payload(family, seed, size)` is deterministic in its three arguments.  Each family is aimed at code
in manatee_b200/csrc/kernels_lz4.cuh (K2 warp_lz4_decode, K3 warp_lz4_encode3, K3c warp_lz4_certify)
or at the oracle's decoder (oracle/lz4_zfs.c); the comment on each says which.  The size lists restate
the thresholds the kernels and the library switch on, and `check_thresholds` fails when one of them
moves, so that the sizes are moved with it instead of quietly testing one side only."""
import ctypes as C
import os
import re

import numpy as np

import lz4_frames as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# ---- thresholds (kernels_lz4.cuh, mtz_lib.cu all_compact_blocks, oracle/lz4_zfs.c) -------------------
LZ4_64KLIMIT = (1 << 16) + 11     # below: TabU16, no distance test; from here: TabU32 (or Tab17)
COMPACT_MAX = 131072              # Tab17 serves 64 KiB + 11 .. 128 KiB, and only in all-compact batches
MIN_COMPRESS = 1024               # zio_compress_data / warp_zfs_lz4_compress: smaller blocks stay raw
CERT_LIMIT = 1 << 24              # k3c refuses lsize >= 2^24 (24-bit positions in K2's parse table)
LZ4_MAXDIST = 65535
EXT = (15, 15 + 255, 15 + 2 * 255)    # token nibble saturates; 255-byte extension runs begin / continue

SIZES_SMALL = (1024, 4096, 16384, 65536)                 # TabU16
SIZES_64K_EDGE = (LZ4_64KLIMIT - 1, LZ4_64KLIMIT, LZ4_64KLIMIT + 1)   # 65546 / 65547 / 65548
STREAM_64K_EDGE = 65552                                  # the smallest 8-aligned lsize (a DRR_WRITE's) of that class
SIZES_COMPACT = (66048, 131072)                          # Tab17 in all-compact batches, else TabU32
SIZES_BIG = (262144, 1 << 20)                            # TabU32 only
SIZE_HUGE = 16 << 20                                     # the encoder compresses it, K3c may not certify it

PERIODS = tuple(range(1, 10)) + (15, 16, 17, 31, 32, 33, 63, 64, 65)
FAR = (LZ4_MAXDIST, LZ4_MAXDIST + 1, LZ4_MAXDIST + 2)   # 65535 reachable, 65536 / 65537 not

# K2 sequences made with lz4_frames.emit: one field at a time on either side of each encoding edge
LIT_LENS = (0, 14, 15, 16, 269, 270, 271, 524, 525)
MATCH_LENS = (4, 18, 19, 20, 273, 274, 275)
OFFSETS = tuple(range(1, 34)) + (63, 64, 65, LZ4_MAXDIST)
TAIL_LENS = (12, 5, 0)        # the last match ends 12, 5 or 0 bytes before the end of the block


def check_thresholds():
    """the constants above against the sources that define them"""
    k = open(os.path.join(ROOT, "manatee_b200", "csrc", "kernels_lz4.cuh")).read()
    lib = open(os.path.join(ROOT, "manatee_b200", "csrc", "mtz_lib.cu")).read()
    orc = open(os.path.join(ROOT, "oracle", "lz4_zfs.c")).read()
    assert "#define LZ4_64KLIMIT     ((1 << 16) + (LZ4_MFLIMIT - 1))" in k
    assert "#define LZ4_MFLIMIT      12" in k and "#define LZ4_MAXDIST      65535" in k
    assert "lsize < 1024u || lsize >= (1u << 24) || d_len < 4u" in k                # K3c's range
    assert "lsize < 1024u || lsize > (16u << 20) || d_len < 4u" in k                # K3's range
    assert "lsize < (uint32_t)LZ4_64KLIMIT || lsize > 131072u" in k                 # compact launch
    assert re.search(r"recs\[i\]\.lsize < \(uint32_t\)LZ4_64KLIMIT \|\| recs\[i\]\.lsize > 131072u", lib)
    assert "seq ? (job.lsize >> 3) : 0u" in k                                       # parse table: lsize / 8
    assert "#define LIMIT64K      ((1 << 16) + (MFLIMIT - 1))" in orc
    assert "lsize < 1024 || lsize > ((size_t)16 << 20)" in orc
    assert SIZES_64K_EDGE[1] == LZ4_64KLIMIT and STREAM_64K_EDGE == (LZ4_64KLIMIT + 7) & ~7 and SIZES_COMPACT[-1] == COMPACT_MAX
    assert SIZES_COMPACT[0] > LZ4_64KLIMIT and SIZES_SMALL[-1] < LZ4_64KLIMIT and SIZES_BIG[0] > COMPACT_MAX
    assert SIZES_SMALL[0] == MIN_COMPRESS and MIN_COMPRESS <= SIZE_HUGE <= 16 << 20 and SIZE_HUGE >= CERT_LIMIT


def flavours(lsize):
    """the certificate tables a record of lsize can meet: 0 TabU16, 1 TabU32, 2 Tab17"""
    if lsize < LZ4_64KLIMIT:
        return (0,)
    return (1, 2) if lsize <= COMPACT_MAX else (1,)


# ---- payload families ---------------------------------------------------------------------------------
_WORDS = (b"the of and to in is that it was for on are with as his they be at one have this from or had "
          b"by not word but what some we can out other were all there when up use your how said an each "
          b"she which do their time if will way about many then them write would like so these her long "
          b"make thing see him two has look more day could go come did number sound no most people my over "
          b"know water than call first who may down side been now find any new work part take get place "
          b"made live where after back little only round man year came show every good me give our under "
          b"zfs snapshot dataset manatee postgres backup stream record checksum").split()


def _rand(rng, n):
    return rng.integers(0, 256, n, dtype=np.uint8)


def _pgpage(seed, n):
    import oracle
    return oracle.gen_payload(oracle.PAYLOAD_PGPAGE, seed, n).copy()


def _sparse(rng, n):
    # zero runs and random islands whose lengths straddle 15 / 270 / 525: K2's and the encoder's
    # 255-extension edges for literal AND match lengths; a zero run is an offset-1 overlapping match
    edges = np.array([e + d for e in (4,) + EXT for d in (-2, -1, 0, 1, 2)] + [2000, 5000])
    edges = edges[edges > 0]
    out, pos = [], 0
    while pos < n:
        z = int(rng.choice(edges)) + 4
        isl = int(rng.choice(edges))
        out += [np.zeros(z, np.uint8), _rand(rng, isl)]
        pos += z + isl
    return np.concatenate(out)[:n]


def _periodic(rng, n):
    # segments of period 1..9, 15..17, 31..33, 63..65 between short random breaks: K2's overlap copy
    # (lane % off, 32 % off), the oracle's off < 8 / >= 8 branches, K3 / K3c follow-on runs
    out, pos = [], 0
    while pos < n:
        p = int(rng.choice(PERIODS))
        ln = int(rng.integers(40, 4000))
        out += [np.resize(_rand(rng, p), ln), _rand(rng, int(rng.integers(0, 24)))]
        pos += ln + out[-1].size
    return np.concatenate(out)[:n]


def _tiny(rng, n, seed):
    # 2..5 symbols: many lanes of one round hash to one slot -> the __match_any_sync path (K3, K3c).
    # Even seeds: i.i.d. symbols (more matches than K2's parse table holds: never certified); odd
    # seeds: slices of a tiny-alphabet base copied between fresh symbols, few enough matches to certify
    k = 2 + int(rng.integers(0, 4))
    if seed % 2 == 0:
        return rng.integers(0, k, n, dtype=np.uint8) + np.uint8(0x61)
    base = rng.integers(0, k, 8192, dtype=np.uint8) + np.uint8(0x61)
    out, pos = [], 0
    while pos < n:
        a = int(rng.integers(0, base.size - 400))
        out += [base[a:a + int(rng.integers(24, 400))], rng.integers(0, k, int(rng.integers(0, 12)), dtype=np.uint8) + np.uint8(0x61)]
        pos += out[-2].size + out[-1].size
    return np.concatenate(out)[:n]


def _text(rng, n):
    # words of a small dictionary: many 4..12-byte matches between short literal runs; every other
    # stretch repeats an earlier phrase, so that the parse stays within K2's table of lsize / 8
    w = rng.integers(0, len(_WORDS), n // 3 + 8)
    sep = rng.choice(np.frombuffer(b"      ,.\n", np.uint8), w.size)
    b = bytearray()
    i = 0
    while len(b) < n:
        if len(b) > 256 and rng.integers(2):
            a = int(rng.integers(0, len(b) - 64))
            b += b[a:a + int(rng.integers(32, 200))]
        else:
            for j in range(i, i + 6):
                b += _WORDS[int(w[j % w.size])] + bytes([int(sep[j % w.size])])
            i += 6
    return np.frombuffer(bytes(b[:n]), np.uint8).copy()


def _ints(rng, n):
    # u32 / u64 counters with strides: matches at offsets 4, 8 and 16
    out, pos = [], 0
    while pos < n:
        dt = np.uint32 if rng.integers(2) else np.uint64
        cnt = int(rng.integers(64, 2048))
        stride = int(rng.choice([1, 1, 2, 3, 8, 256, 4096]))
        a = (int(rng.integers(0, 1 << 31)) + stride * np.arange(cnt, dtype=np.uint64)).astype(dt)
        if rng.integers(3) == 0:
            a = np.repeat(a, 2)                                  # pairs: offset 2 * itemsize
        out.append(a.view(np.uint8))
        pos += out[-1].size
    return np.concatenate(out)[:n]


def _far(rng, n):
    # random segments in zeros, each repeated exactly 65535, 65536 or 65537 bytes later, and again after
    # a one-byte break inside the copy: LZ4_MAXDIST, K3c's DIST argument and deferred MISS check,
    # Tab17's bit 16.  Zeros around them insert almost nothing, so the segment's slots survive 64 KiB.
    a = np.zeros(n, np.uint8)
    seg = 300
    dists = FAR if n > FAR[-1] + 2 * seg else (n // 2 - 1, n // 2, n // 2 + 1)
    pos = 64
    for d in dists:
        if pos + d + seg + 16 >= n:
            break
        a[pos:pos + seg] = _rand(rng, seg)
        a[pos + d:pos + d + seg] = a[pos:pos + seg]
        a[pos + d + seg // 2] ^= 0x5a                             # the match breaks and resumes
        pos += seg + int(rng.integers(64, 512))
    return a


def _mixture(rng, n, seed):
    # a long random head (the search step (67+a)>>6 grows before the first hit) then a compressible
    # tail; odd seeds the other way round
    cut = int(n * (0.3 + 0.5 * rng.random()))
    comp = _text(rng, n) if seed % 4 < 2 else _pgpage(seed, n)
    a = comp.copy()
    if seed % 2 == 0:
        a[:cut] = _rand(rng, cut)
    else:
        a[cut:] = _rand(rng, n - cut)
    return a


FAMILIES = ("pgpage", "random", "zeros", "sparse", "periodic", "tiny", "text", "ints", "far", "mixture")


def payload(family, seed, size):
    rng = np.random.default_rng([FAMILIES.index(family), seed, size])
    if family == "pgpage":
        return _pgpage(seed, size)                   # baseline: what the certificate was built on
    if family == "random":
        return _rand(rng, size)                      # stored raw: the frame rule
    if family == "zeros":
        return np.zeros(size, np.uint8)              # one offset-1 match, 255-runs up to the end
    if family == "sparse":
        return _sparse(rng, size)
    if family == "periodic":
        return _periodic(rng, size)
    if family == "tiny":
        return _tiny(rng, size, seed)
    if family == "text":
        return _text(rng, size)
    if family == "ints":
        return _ints(rng, size)
    if family == "far":
        return _far(rng, size)
    if family == "mixture":
        return _mixture(rng, size, seed)
    raise ValueError(family)


# ---- frames -------------------------------------------------------------------------------------------
def frame_of(block):
    """ZFS frame of a raw LZ4 block: BE32 clen, the block, zero pad to 512 bytes"""
    m = len(block)
    pad = (-(m + 4)) % 512
    return np.frombuffer(m.to_bytes(4, "big") + bytes(block) + bytes(pad), np.uint8).copy()


def block_of(frame):
    clen = int.from_bytes(bytes(frame[:4]), "big")
    return bytes(frame[4:4 + clen])


_liblz4 = None


def _lz4():
    global _liblz4
    if _liblz4 is None:
        L = C.CDLL("liblz4.so.1")
        L.LZ4_compress_fast.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
        L.LZ4_compress_HC.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
        L.LZ4_compressBound.argtypes = [C.c_int]
        _liblz4 = L
    return _liblz4


def liblz4_block(data, fn, param):
    """a raw block from the installed liblz4: fn "fast" (param = acceleration) or "hc" (level)"""
    a = np.ascontiguousarray(data, dtype=np.uint8)
    L = _lz4()
    dst = np.empty(L.LZ4_compressBound(a.size) + 16, np.uint8)
    f = L.LZ4_compress_fast if fn == "fast" else L.LZ4_compress_HC
    m = f(a.ctypes.data, dst.ctypes.data, a.size, dst.size, param)
    assert m > 0
    return dst[:m].tobytes()


FOREIGN = (("fast", 1), ("fast", 4), ("fast", 17), ("fast", 64), ("hc", 3), ("hc", 9), ("hc", 12), ("ref_hc", 0))


def foreign_blocks(data):
    """[(name, raw block)] of the same bytes from other encoders"""
    import lz4hc_ref
    out = []
    for fn, p in FOREIGN:
        if fn == "ref_hc":
            b = lz4hc_ref.lz4hc_compress_block(data)
            if b is not None:
                out.append(("lz4hc_ref", b.tobytes()))
        else:
            out.append(("%s%d" % (fn, p), liblz4_block(data, fn, p)))
    return out


def mutated_blocks(block, rng, stacked=3):
    """[(name, block)]: every lz4_frames.MUTATIONS applied once, then `stacked` of them on one block"""
    out = []
    for kind in F.MUTATIONS:
        nb = F.mutate(block, kind, rng)
        if nb is not None and nb != block:
            out.append((kind, nb))
    nb = block
    for _ in range(stacked):
        t = F.mutate(nb, F.MUTATIONS[int(rng.integers(len(F.MUTATIONS)))], rng)
        nb = t if t is not None else nb
    if nb != block:
        out.append(("stacked", nb))
    return out


def expected_certified(frame, data):
    """The certificate's verdict on `frame` for the logical bytes `data`: certified exactly when the
    frame's block is the declared encoder's (oracle.zfs_lz4_compress) for these bytes, its parse fits
    K2's table of lsize / 8 matches, 1024 <= lsize < 2^24, and the frame is one zio_compress_data
    keeps (it saves 12.5 % and its sector-rounded size is below lsize).  The pad bytes after the
    block are not part of it: a certified frame is re-padded with zeros."""
    import oracle
    data = np.ascontiguousarray(data, dtype=np.uint8)
    lsize = data.size
    if not MIN_COMPRESS <= lsize < CERT_LIMIT:
        return False
    f = bytes(frame)
    if len(f) < 4:
        return False
    clen = int.from_bytes(f[:4], "big")
    d_len = lsize - (lsize >> 3)
    if clen + 4 > d_len or ((clen + 4 + 511) & ~511) >= lsize:
        return False
    ps, want = oracle.zfs_lz4_compress(data)
    if want is None or f[:4 + clen] != want[:4 + clen].tobytes() or int.from_bytes(want[:4].tobytes(), "big") != clen:
        return False
    seqs, _ = F.parse(f[4:4 + clen])
    return len(seqs) <= lsize // 8


# ---- synthesized K2 blocks and malformed frames --------------------------------------------------------
def synthesized_blocks(seed):
    """[(name, block, data)]: valid blocks with one field at each edge of its encoding -- literal
    length, match length, offset (overlapping for off < ml), closing literal count"""
    rng = np.random.default_rng(seed)
    out = []

    def one(name, lits, off, ml, tail):
        head = _rand(rng, max(64, off)).tobytes()
        seqs = [(head, 16, 20), (lits, off, ml), (_rand(rng, 3).tobytes(), 7, 9)]
        if tail == 0:
            seqs = seqs[:2]
        tl = _rand(rng, tail).tobytes()
        out.append((name, F.emit(seqs, tl), F.decode(seqs, tl)))

    for ll in LIT_LENS:
        one("ll%d" % ll, _rand(rng, ll).tobytes(), 7, 18, 12)
    for ml in MATCH_LENS:
        one("ml%d" % ml, b"xyz", 5, ml, 12)
    for off in OFFSETS:
        one("off%d" % off, b"q", off, 40, 12)
    for t in TAIL_LENS:
        one("tail%d" % t, b"ab", 3, 25, t)
    return out


def _ext_positions(block):
    """byte offsets inside `block` of 255-extension bytes"""
    b, ip, pos = bytes(block), 0, []
    while True:
        tok = b[ip]; ip += 1
        ll = tok >> 4
        if ll == 15:
            while True:
                pos.append(ip); s = b[ip]; ip += 1; ll += s
                if s != 255:
                    break
        ip += ll
        if ip >= len(b):
            return pos
        ip += 2
        if tok & 15 == 15:
            while True:
                pos.append(ip); s = b[ip]; ip += 1
                if s != 255:
                    break


def malformed(block, data):
    """[(name, frame, lsize)] of bad variants of a valid block whose decode is `data`"""
    lsize = len(data)
    fr = frame_of(block)
    clen = len(block)
    psize = fr.size
    out = []

    def with_clen(v):
        f = fr.copy()
        f[:4] = np.frombuffer(int(v).to_bytes(4, "big"), np.uint8)
        return f

    ext = _ext_positions(block)
    if ext:
        out.append(("trunc_in_ext", with_clen(ext[len(ext) // 2]), lsize))     # ends inside a 255 run
    seqs, tail = F.parse(block)
    if seqs:
        lits, off, ml = seqs[0]
        op = len(lits)
        if op + 1 <= 65535:
            out.append(("off_op_plus_1", frame_of(F.emit([(lits, op + 1, ml)] + seqs[1:], tail)), lsize))
        lits, off, ml = seqs[-1]
        longer = seqs[:-1] + [(lits, off, ml + len(tail) + 1)]
        out.append(("match_past_lsize", frame_of(F.emit(longer, b"")), lsize))
    out.append(("clen0", with_clen(0), lsize))
    out.append(("clen_psize_m3", with_clen(psize - 3), lsize))
    out.append(("clen_psize_m4", with_clen(psize - 4), lsize))
    for d in (-512, -1, 1, 512):
        if lsize + d > 0:
            out.append(("lsize%+d" % d, fr, lsize + d))
    return out
