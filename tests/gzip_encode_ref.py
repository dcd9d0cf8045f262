"""Reference model of MTZ_FLAG_GZIP_ENCODE: the stage's deflate re-coding of K3's LZ4 parse.  Test
infrastructure; it states the frame k_deflate_from_lz4 (manatee_b200/csrc/kernels_deflate.cuh) must write,
byte for byte.

  frame(data)           the zlib frame of the logical bytes `data`, zero-padded to a multiple of 512 bytes,
                        when K3 (oracle.zfs_lz4_compress) stores `data` as an LZ4 frame and the padded zlib
                        frame is smaller than `data`; None otherwise (mtz_k_gzip_encode's "store raw")
  stage_payload(data)   what COMPRESS with the flag sends for a raw DRR_WRITE: (comp, payload), the smallest
                        of K3's LZ4 frame (15), the zlib frame (5, only when strictly smaller than the LZ4
                        frame) and raw (0, when K3 stores it raw)
  expected(oracle, s)   COMPRESS with the flag of the raw stream s

The frame, from K3's LZ4 frame of `data`:
  symbols  K3's sequences in order.  Each literal is a literal symbol.  A match with offset > 32768 becomes
           the literal symbols of the bytes it covers.  Any other match of length L is cut into pieces of
           at most 258: while L > 258 the piece is 258 when L - 258 >= 3 and L - 3 otherwise (259 -> 256 + 3,
           260 -> 257 + 3, 261 -> 258 + 3).  The block ends with symbol 256.
  block    one, BFINAL = 1, BTYPE = 2.  Code lengths by huff_lengths: 15 bits for literal/length and
           distance, 7 for the code-length code.  A record without matches sends one distance code (0)
           of length 1.  HLIT / HDIST / HCLEN trimmed to the last non-zero length (at least 257 / 1 / 4).
           The literal/length and distance lengths are one sequence for the code-length code, run-coded
           by cl_symbols.
  zlib     CMF 0x78, FLG 0x01, the block, zero bits to the byte boundary, Adler-32 big endian, then zeros
           to the next multiple of 512 bytes."""
import zlib

import numpy as np

GZIP_ENCODE = 4096          # MTZ_FLAG_GZIP_ENCODE
DC_GZIP1 = 5
DC_LZ4 = 15
MAXDIST = 32768
CL_ORDER = (16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15)


def _len_table():
    base = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131,
            163, 195, 227, 258]
    extra = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
    code = np.zeros(259, dtype=np.int64)
    for c in range(29):
        code[base[c]:base[c + 1] if c < 28 else 259] = c
    return code, np.array(base, dtype=np.int64), np.array(extra, dtype=np.int64)


def _dist_table():
    base, extra = [], []
    for c in range(30):
        e = max(0, c // 2 - 1)
        base.append(1 + c if c < 4 else ((2 + (c & 1)) << e) + 1)
        extra.append(e)
    return np.array(base, dtype=np.int64), np.array(extra, dtype=np.int64)


LEN_CODE, LEN_BASE, LEN_EXTRA = _len_table()
DIST_BASE, DIST_EXTRA = _dist_table()


def dist_code(d):
    return np.searchsorted(DIST_BASE, d, side="right") - 1


def sequences(frame):
    """(literal count, match length, offset) of each sequence of the ZFS-LZ4 frame (BE32 clen + block);
    the last one has match length 0"""
    f = bytes(frame)
    clen = int.from_bytes(f[:4], "big")
    b, ip, end = f[4:4 + clen], 0, clen
    out = []
    while ip < end:
        tok = b[ip]
        ip += 1
        nl = tok >> 4
        if nl == 15:
            while True:
                c = b[ip]
                ip += 1
                nl += c
                if c != 255:
                    break
        ip += nl
        if ip >= end:
            out.append((nl, 0, 0))
            break
        off = b[ip] | (b[ip + 1] << 8)
        ip += 2
        ml = tok & 15
        if ml == 15:
            while True:
                c = b[ip]
                ip += 1
                ml += c
                if c != 255:
                    break
        out.append((nl, ml + 4, off))
    return out


def split(L):
    """the pieces of a match of length L (no piece longer than 258 or shorter than 3)"""
    out = []
    while L > 258:
        p = 258 if L - 258 >= 3 else L - 3
        out.append(p)
        L -= p
    out.append(L)
    return out


def tokens(data, frame):
    """the block's symbols: (literal/length symbol, length extra value, distance or 0) per token, as arrays
    (EOB not included)"""
    d = np.asarray(data, dtype=np.uint8)
    lit, ln, ds = [], [], []
    pos = 0
    for nl, ml, off in sequences(frame):
        if nl:
            lit.append(d[pos:pos + nl].astype(np.int64))
            ln.append(np.zeros(nl, dtype=np.int64))
            ds.append(np.zeros(nl, dtype=np.int64))
            pos += nl
        if ml == 0:
            continue
        if off > MAXDIST:
            lit.append(d[pos:pos + ml].astype(np.int64))
            ln.append(np.zeros(ml, dtype=np.int64))
            ds.append(np.zeros(ml, dtype=np.int64))
        else:
            ps = split(ml)
            lit.append(257 + LEN_CODE[ps])
            ln.append(np.array(ps, dtype=np.int64))
            ds.append(np.full(len(ps), off, dtype=np.int64))
        pos += ml
    assert pos == d.size
    cat = lambda xs: np.concatenate(xs) if xs else np.zeros(0, dtype=np.int64)  # noqa: E731
    return cat(lit), cat(ln), cat(ds)


def huff_lengths(freq, limit):
    """Code lengths of a length-limited Huffman code for `freq`.  No used symbol: all zero.  One: length 1.
    Otherwise the used symbols are sorted by (frequency, symbol) and merged by two queues (leaves, then
    internal nodes in the order they are made); the two smallest are taken each time, a leaf before an
    internal node of the same weight.  A leaf's length is its depth.  When the deepest leaf is deeper than
    `limit`, every used frequency f becomes (f + 1) // 2 and the code is built again."""
    f = [int(x) for x in freq]
    n = len(f)
    L = [0] * n
    used = [s for s in range(n) if f[s]]
    if not used:
        return L
    if len(used) == 1:
        L[used[0]] = 1
        return L
    while True:
        order = sorted(used, key=lambda s: (f[s], s))
        nl = len(order)
        lw = [f[s] for s in order]
        iw, ipar, lpar = [], [], [0] * nl
        i = j = 0
        for k in range(nl - 1):
            w = 0
            for _ in range(2):
                if i < nl and (j >= k or lw[i] <= iw[j]):
                    lpar[i] = k
                    w += lw[i]
                    i += 1
                else:
                    ipar[j] = k
                    w += iw[j]
                    j += 1
            iw.append(w)
            ipar.append(-1)
        depth = [0] * (nl - 1)
        for k in range(nl - 3, -1, -1):
            depth[k] = depth[ipar[k]] + 1
        ld = [depth[lpar[i]] + 1 for i in range(nl)]
        if max(ld) <= limit:
            for i, s in enumerate(order):
                L[s] = ld[i]
            return L
        f = [(x + 1) >> 1 for x in f]


def canonical(L):
    """the RFC 1951 canonical codes of lengths L, bit-reversed for LSB-first output"""
    mx = max(L) if L else 0
    cnt = [0] * (mx + 2)
    for x in L:
        if x:
            cnt[x] += 1
    nxt, code = [0] * (mx + 2), 0
    for b in range(1, mx + 1):
        code = (code + cnt[b - 1]) << 1
        nxt[b] = code
    out = [0] * len(L)
    for s, x in enumerate(L):
        if x:
            c = nxt[x]
            nxt[x] += 1
            out[s] = int(format(c, "0%db" % x)[::-1], 2)
    return out


def cl_symbols(lens):
    """the code-length code's symbols of the length sequence: (symbol, extra value).  At a run of r equal
    lengths v: v == 0 and r >= 3 -> 18 (r >= 11) or 17 over min(r, 138); else v once, and for v != 0
    the rest of the run as 16s of min(rest, 6) while at least 3 are left"""
    out, i, n = [], 0, len(lens)
    while i < n:
        v, r = lens[i], 1
        while i + r < n and lens[i + r] == v:
            r += 1
        if v == 0 and r >= 3:
            k = min(r, 138)
            out.append((18, k - 11) if k >= 11 else (17, k - 3))
            i += k
            continue
        out.append((v, 0))
        i += 1
        r -= 1
        while v != 0 and r >= 3:
            k = min(r, 6)
            out.append((16, k - 3))
            i += k
            r -= k
    return out


CL_EXTRA = {16: 2, 17: 3, 18: 7}


def _pack(vals, nbits):
    """LSB-first bit packing of (value, width) items into bytes, the last one zero-filled"""
    vals = np.asarray(vals, dtype=np.uint64)
    nb = np.asarray(nbits, dtype=np.int64)
    tot = int(nb.sum())
    idx = np.repeat(np.arange(nb.size), nb)
    start = np.repeat(np.cumsum(nb) - nb, nb)
    sh = (np.arange(tot, dtype=np.int64) - start).astype(np.uint64)
    bits = ((vals[idx] >> sh) & np.uint64(1)).astype(np.uint8)
    return np.packbits(bits, bitorder="little")


def deflate(data, frame):
    """the unpadded zlib stream of `data` re-coded from K3's LZ4 frame `frame`"""
    d = np.asarray(data, dtype=np.uint8)
    ll, ln, ds = tokens(d, frame)
    lf = np.bincount(ll, minlength=286)
    lf[256] += 1
    m = ll >= 257
    dc = dist_code(ds[m]).astype(np.int64)
    df = np.bincount(dc, minlength=30)
    Ll = huff_lengths(lf, 15)
    Ld = huff_lengths(df, 15) if dc.size else [1] + [0] * 29
    hlit = max(257, max(s for s in range(286) if Ll[s]) + 1)
    hdist = max(1, max(s for s in range(30) if Ld[s]) + 1)
    cls = cl_symbols(Ll[:hlit] + Ld[:hdist])
    cf = np.bincount([s for s, _ in cls], minlength=19)
    Lc = huff_lengths(cf, 7)
    hclen = max(4, max(i for i in range(19) if Lc[CL_ORDER[i]]) + 1)
    Cl, Cd, Cc = canonical(Ll), canonical(Ld), canonical(Lc)
    V, N = [1 | (2 << 1), hlit - 257, hdist - 1, hclen - 4], [3, 5, 5, 4]
    for i in range(hclen):
        V.append(Lc[CL_ORDER[i]])
        N.append(3)
    for s, x in cls:
        V.append(Cc[s] | (x << Lc[s]))
        N.append(Lc[s] + CL_EXTRA.get(s, 0))
    # data tokens: code | length extra | distance code | distance extra, at most 48 bits each
    Cl_a, Ll_a = np.array(Cl, dtype=np.uint64), np.array(Ll, dtype=np.int64)
    v = Cl_a[ll].copy()
    nb = Ll_a[ll].copy()
    if dc.size:
        lc = ll[m] - 257
        lx = (ln[m] - LEN_BASE[lc]).astype(np.uint64)
        lxn = LEN_EXTRA[lc]
        dxv = (ds[m] - DIST_BASE[dc]).astype(np.uint64)
        dxn = DIST_EXTRA[dc]
        Cd_a, Ld_a = np.array(Cd, dtype=np.uint64), np.array(Ld, dtype=np.int64)
        vm, nm = v[m], nb[m]
        vm |= lx << nm.astype(np.uint64)
        nm = nm + lxn
        vm |= Cd_a[dc] << nm.astype(np.uint64)
        nm = nm + Ld_a[dc]
        vm |= dxv << nm.astype(np.uint64)
        nm = nm + dxn
        v[m], nb[m] = vm, nm
    vals = np.concatenate([np.array(V, dtype=np.uint64), v, np.array([Cl[256]], dtype=np.uint64)])
    nbits = np.concatenate([np.array(N, dtype=np.int64), nb, np.array([Ll[256]], dtype=np.int64)])
    body = _pack(vals, nbits)
    return b"\x78\x01" + body.tobytes() + zlib.adler32(d.tobytes()).to_bytes(4, "big")


def pad512(b):
    return b + bytes((-len(b)) % 512)


def frame(oracle, data, limit=None):
    """the padded zlib frame of `data` when K3 makes an LZ4 frame of it and the padded zlib frame is
    smaller than `limit` (default: len(data)); None otherwise"""
    d = np.asarray(data, dtype=np.uint8)
    ps, lz = oracle.zfs_lz4_compress(d)
    if lz is None:
        return None
    z = pad512(deflate(d, lz))
    return z if len(z) < (d.size if limit is None else limit) else None


def stage_payload(oracle, data):
    """(drr_compressiontype, payload) COMPRESS with the flag sends for the raw logical bytes `data`"""
    d = np.asarray(data, dtype=np.uint8)
    ps, lz = oracle.zfs_lz4_compress(d)
    if lz is None:
        return 0, d.copy()
    z = pad512(deflate(d, lz))
    if len(z) < ps:
        return DC_GZIP1, np.frombuffer(z, dtype=np.uint8).copy()
    return DC_LZ4, lz


def splice(oracle, wire, x):
    """`wire` (a COMPRESS output of the raw-or-decoded records of x, preambles included) with every DRR_WRITE
    that left as K3's LZ4 frame replaced by the zlib frame where that is smaller (header bytes 50 and
    96..103 rewritten), re-stamped, and WIRE_F_GZIP set in every preamble.  The records of x that
    arrived LZ4 or gzip (forwarded) are left alone: those are recognised as not being K3's frame of the
    logical bytes (a gzip record of x is never LZ4 on the wire)."""
    import block_ref as B
    import gzip_wire_ref as W
    w = np.asarray(wire, dtype=np.uint8)
    body = oracle.wire_strip(w)
    pres = [w[i:i + W.PRE_BYTES].copy() for i in W.preambles(oracle, w)]
    xb = np.asarray(x, dtype=np.uint8)
    parts, k = [], 0
    for (xo, xpo, xpl, t), (wo, wpo, wpl, _) in zip(B.records(xb), B.records(body)):
        if t == 0:
            parts.append(pres[k])
            k += 1
        rec = body[wo:wpo + wpl]
        if t == 3 and body[wo + 50] == DC_LZ4 and int(xb[xo + 50]) != DC_LZ4:
            logical = _logical(oracle, xb[xo:xpo + xpl])
            comp, pay = stage_payload(oracle, logical)
            if comp == DC_GZIP1:
                h = rec[:312].copy()
                h[50] = DC_GZIP1
                h[96:104] = np.frombuffer(int(pay.size).to_bytes(8, "little"), dtype=np.uint8)
                rec = np.concatenate([h, pay])
        parts.append(rec)
    out = np.ascontiguousarray(np.concatenate(parts))
    pos = W.preambles(oracle, out) + [out.size]
    for a, e in zip(pos, pos[1:]):
        seg = np.ascontiguousarray(out[a + W.PRE_BYTES:e])
        assert oracle.stream_restamp(seg)[0] == 0
        out[a + W.PRE_BYTES:e] = seg
    return W.set_pre_flags(oracle, out, on=W.WIRE_F_GZIP)


def _logical(oracle, rec):
    """the logical bytes of one DRR_WRITE record (raw, lzjb or zle on arrival)"""
    import compressed_in_ref as M
    h = rec[:312]
    comp, lsize = int(h[50]), M._lsize(h)
    pay = rec[312:]
    if comp == 0:
        return pay[:lsize]
    out = M.decode(oracle, comp, pay, lsize)
    assert out is not None
    return np.frombuffer(bytes(out), dtype=np.uint8)


def expected(oracle, x, compressed_in=False):
    """COMPRESS with the flag (and MTZ_FLAG_COMPRESSED_IN when `compressed_in`) of x"""
    if compressed_in:
        import compressed_in_ref as M
        return splice(oracle, M.expected(oracle, x), x)
    rc, w, _ = oracle.stream_compress(x)
    assert rc == 0
    return splice(oracle, w, x)


def counts(oracle, wire):
    """(LZ4 records, gzip-1 records) on `wire`"""
    import block_ref as B
    b = oracle.wire_strip(np.asarray(wire, dtype=np.uint8))
    n4 = ng = 0
    for off, _, _, t in B.records(b):
        if t == 3:
            n4 += b[off + 50] == DC_LZ4
            ng += b[off + 50] == DC_GZIP1
    return int(n4), int(ng)
