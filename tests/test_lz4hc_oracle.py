"""The high-ratio LZ4 encoder of MTZ_FLAG_LZ4_HC on the CPU: its executable statement (spec_block below)
equals the C restatement (tests/lz4hc_ref.c) on crafted blocks, every block decodes to its input under
liblz4 and the oracle's decoder, the frame rule is ZFS's, the HC frames of the pg-page model are smaller
than ZFS's, and COMPRESS with it round-trips through the oracle's DECOMPRESS."""
import ctypes as C

import numpy as np
import pytest

import lz4hc_ref as R

MINMATCH, MFLIMIT, LASTLITERALS, MAXOFF, HB, W, CAP = 4, 12, 5, 65535, 12, 16, 64


def _le32(b, p):
    return b[p] | (b[p + 1] << 8) | (b[p + 2] << 16) | (b[p + 3] << 24)


def _lenext(out, v):
    while v >= 255:
        out.append(255)
        v -= 255
    out.append(v)


def _seq(out, lits, off=0, ml=0):
    mc = ml - MINMATCH if ml else 0
    out.append((min(len(lits), 15) << 4) | min(mc, 15))
    if len(lits) >= 15:
        _lenext(out, len(lits) - 15)
    out += lits
    if ml:
        out += bytes((off & 255, off >> 8))
        if mc >= 15:
            _lenext(out, mc - 15)


def spec_block(src):
    """The encoder as specified: 4096 buckets of the last 16 positions, every position below p inserted
    before p is searched, candidates with p-c <= 65535 and equal LE32, the longest capped (64-byte)
    comparison wins with ties to the larger c, then only the winner is extended; greedy parse."""
    b = bytes(src)
    n = len(b)
    mflimit, matchlimit = n - MFLIMIT, n - LASTLITERALS
    buckets = [[] for _ in range(1 << HB)]
    h = lambda p: ((_le32(b, p) * 2654435761) & 0xFFFFFFFF) >> (32 - HB)  # noqa: E731
    out, p, anchor, ins = bytearray(), 0, 0, 0
    while p < mflimit:
        for q in range(ins, p):
            bk = buckets[h(q)]
            bk.append(q)
            if len(bk) > W:
                bk.pop(0)
        ins = p
        v, lim, best, bc = _le32(b, p), min(CAP, matchlimit - p), 0, -1
        for c in buckets[h(p)]:
            if p - c > MAXOFF or _le32(b, c) != v:
                continue
            n_eq = 0
            while n_eq < lim and b[c + n_eq] == b[p + n_eq]:
                n_eq += 1
            if n_eq > best or (n_eq == best and c > bc):
                best, bc = n_eq, c
        if bc < 0:
            p += 1
            continue
        ml = best
        if ml == CAP:
            while p + ml < matchlimit and b[bc + ml] == b[p + ml]:
                ml += 1
        _seq(out, b[anchor:p], p - bc, ml)
        p += ml
        anchor = p
    _seq(out, b[anchor:])
    return bytes(out)


def _pcg(n, seed=1):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)


def _crafted():
    rng = np.random.default_rng(5)
    cases = {"zero": np.zeros(4096, np.uint8), "pcg": _pcg(4096)}
    for per in (1, 2, 3, 7):
        cases["period%d" % per] = np.tile(rng.integers(0, 256, per, dtype=np.uint8), 4096 // per + 1)[:4096]
    # a 200-byte pattern seen again exactly 65535 bytes later (taken) and one seen 65536 later (not);
    # zeros in between keep the pattern's buckets from overflowing
    for name, d in (("offset65535", 65535), ("offset65536", 65536)):
        a = np.zeros(d + 300, np.uint8)
        a[:300] = _pcg(300, d)
        a[d:d + 200] = a[0:200]
        a[d + 200:] = _pcg(100, d + 1)
        cases[name] = a
    # 20 positions with one 4-byte value (same hash), each followed by a shorter run of the same bytes:
    # the bucket overflows, and the oldest (longest) copies are evicted before the last one is searched
    c = np.zeros(8192, np.uint8)
    for i in range(20):
        c[200 * i:200 * i + 4] = [9, 8, 7, 6]
        c[200 * i + 4:200 * i + 4 + (40 - i)] = 1 + (np.arange(40 - i) % 200).astype(np.uint8)
    c[6000:6004] = [9, 8, 7, 6]
    c[6004:6044] = 1 + (np.arange(40) % 200).astype(np.uint8)
    cases["bucket_overflow"] = c
    # ties: three earlier copies of the same 24 bytes; the newest must win
    d = _pcg(4096, 5)
    for o in (100, 600, 1100, 3000):
        d[o:o + 24] = np.arange(24, dtype=np.uint8) + 50
    cases["ties"] = d
    # a match that runs into matchlimit
    e = _pcg(2048, 6)
    e[1024:] = e[:1024]
    cases["to_matchlimit"] = e
    cases["long_zero_run"] = np.concatenate([_pcg(500, 7), np.zeros(3000, np.uint8), _pcg(600, 8)])
    return cases


def _offsets(blk):
    """(offset, match length) of every sequence of a raw block"""
    b, ip, out = bytes(blk), 0, []
    while True:
        tok = b[ip]; ip += 1
        ll = tok >> 4
        if ll == 15:
            while True:
                s = b[ip]; ip += 1; ll += s
                if s != 255:
                    break
        ip += ll
        if ip == len(b):
            return out
        off = b[ip] | (b[ip + 1] << 8); ip += 2
        ml = tok & 15
        if ml == 15:
            while True:
                s = b[ip]; ip += 1; ml += s
                if s != 255:
                    break
        out.append((off, ml + 4))


def _liblz4_decode(blk, n):
    lz = C.CDLL("liblz4.so.1")
    dst = C.create_string_buffer(n + 16)
    got = lz.LZ4_decompress_safe(bytes(blk), dst, len(blk), n + 16)
    return dst.raw[:got] if got >= 0 else None


def _check_block(oracle, src):
    src = np.ascontiguousarray(src, dtype=np.uint8)
    blk = R.lz4hc_compress_block(src)
    assert blk is not None
    assert _liblz4_decode(blk.tobytes(), src.size) == src.tobytes()
    rc, dec = oracle.lz4_decompress_block(blk, src.size)
    assert rc == src.size and np.array_equal(dec, src)
    return blk


@pytest.mark.parametrize("name", sorted(_crafted()))
def test_the_spec_equals_the_c_restatement_on_crafted_blocks(oracle, name):
    src = _crafted()[name]
    blk = _check_block(oracle, src)
    assert spec_block(src) == blk.tobytes()
    offs = _offsets(blk)
    if name == "offset65535":
        assert any(o == 65535 and ml >= 200 for o, ml in offs)
    if name == "offset65536":
        assert not any(o > 60000 and ml >= 100 for o, ml in offs)
    if name == "ties":
        assert (3000 - 1100, 24) in offs                 # the newest copy at equal length
    if name == "bucket_overflow":
        assert (6000 - 200 * 4, 36 + 4) in offs          # copies 0..3 (longer) are out of the bucket
    if name == "to_matchlimit":
        assert offs[-1] == (1024, 1024 - LASTLITERALS)


@pytest.mark.parametrize("n", [1024, 4096, 65536 - 512, 65536 + 512, 131072])
def test_the_spec_equals_the_c_restatement_on_pg_pages(oracle, n):
    src = oracle.gen_payload(oracle.PAYLOAD_PGPAGE, n, n)
    assert spec_block(src) == _check_block(oracle, src).tobytes()


@pytest.mark.parametrize("n", [0, 1, 5, 12, 13, 17, 100])
def test_tiny_blocks(oracle, n):
    src = _pcg(n, n) if n else np.zeros(0, np.uint8)
    blk = R.lz4hc_compress_block(src)
    assert blk is not None and spec_block(src) == blk.tobytes()
    if n:
        assert _liblz4_decode(blk.tobytes(), n) == src.tobytes()


def test_every_payload_kind_decodes(oracle):
    for kind in (oracle.PAYLOAD_PCG, oracle.PAYLOAD_PGPAGE, oracle.PAYLOAD_ZERO):
        for r, n in enumerate((1024, 8192, 65535, 131072, 1 << 20)):
            _check_block(oracle, oracle.gen_payload(kind, r, n))


def test_the_frame_rule_is_zfs(oracle):
    pg = oracle.gen_payload(oracle.PAYLOAD_PGPAGE, 1, 131072)
    assert R.zfs_lz4hc_compress(pg[:1023]) == (1023, None)              # below 1024 bytes: raw
    assert R.zfs_lz4hc_compress(_pcg(4096))[0] == 4096                  # saves under 12.5 %: raw
    # compresses to 4 + clen <= lsize - lsize/8 but rounds up to a psize >= lsize: raw
    x = np.concatenate([np.zeros(300, np.uint8), _pcg(724, 9)])
    blk = R.lz4hc_compress_block(x)
    assert 4 + blk.size <= 1024 - 128 and R.zfs_lz4hc_compress(x) == (1024, None)
    ps, fr = R.zfs_lz4hc_compress(pg)
    blk = R.lz4hc_compress_block(pg)
    assert ps == (4 + blk.size + 511) & ~511 and fr.size == ps
    assert int.from_bytes(fr[:4].tobytes(), "big") == blk.size
    assert np.array_equal(fr[4:4 + blk.size], blk) and not fr[4 + blk.size:].any()
    rc, dec = oracle.zfs_lz4_decompress(fr, pg.size)
    assert rc == 0 and np.array_equal(dec, pg)


def test_pg_pages_compress_better_than_zfs(oracle):
    logical = zfs = hc = 0
    for r in range(64):
        p = oracle.gen_payload(oracle.PAYLOAD_PGPAGE, r, 131072)
        logical += p.size
        zfs += oracle.zfs_lz4_compress(p)[0]
        hc += R.zfs_lz4hc_compress(p)[0]
    print("pg-page records 0..63: logical/frames ZFS %.3f, HC %.3f" % (logical / zfs, logical / hc))
    assert hc < zfs and logical / hc > 2.7


def _streams(oracle):
    pg = lambda n, rs, first=0: oracle.synth_stream(n, recsize=rs, kind=oracle.PAYLOAD_PGPAGE,  # noqa: E731
                                                    first_rec=first)
    yield "pg-128k", pg(20, 131072)
    yield "pg-4k", pg(40, 4096)
    yield "pcg", oracle.synth_stream(6, recsize=65536, kind=oracle.PAYLOAD_PCG)
    yield "zero", oracle.synth_stream(6, recsize=131072, kind=oracle.PAYLOAD_ZERO)
    yield "sub-streams", np.concatenate([pg(5, 8192), oracle.synth_stream(3, recsize=131072,
                                         kind=oracle.PAYLOAD_PCG), pg(4, 1024, 7), pg(3, 1 << 20, 9)])


def test_stream_compress_hc_round_trips(oracle):
    for name, s in _streams(oracle):
        rc, c, st = R.stream_compress(s, hc=True)
        assert rc == 0, name
        rc0, c0, st0 = oracle.stream_compress(s)
        assert st.records == st0.records and st.write_records == st0.write_records
        rc, d, _ = oracle.stream_decompress(c)
        assert rc == 0 and np.array_equal(d, s), name
        if name.startswith("pg"):
            assert c.size <= c0.size and (name != "pg-128k" or c.size < c0.size), name
        if name == "pcg":
            assert np.array_equal(c, c0)                  # incompressible records stay raw either way
