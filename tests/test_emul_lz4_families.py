"""K3c (warp_lz4_certify), K2 (warp_lz4_decode) on the SIMT emulator, over every payload family of
tests/lz4_payloads.py and every table flavour a record size can meet.

The certificate must say "certified" exactly when lz4_payloads.expected_certified does -- for the
declared encoder's frame, for every parse mutation of lz4_frames, for several mutations stacked on one
block, and for frames of the same bytes from liblz4 (LZ4_compress_fast, LZ4_compress_HC) and from
tests/lz4hc_ref.  A false certificate breaks RECOMPRESS's bit-exactness; a missed one costs speed only,
and no output comparison would notice it.  Records of 65547..131072 bytes are certified under Tab17 in
all-compact batches and under TabU32 otherwise, so both are asked.

K2 must agree with the oracle's safe decoder on accept / reject and on the bytes, for the same frames,
for blocks synthesized at each edge of the sequence encoding, and for malformed variants of them --
inside guard pages, so that a read or write past the frame or the output is a crash here."""
import numpy as np
import pytest

import lz4_frames as F
import lz4_payloads as P
from test_emul_device_code import ECODEC, Guarded, emu  # noqa: F401  (emu: module fixture)


def _certify(emu, frame, data, flavour):
    src = Guarded(emu, data.size, slack=16, data=data)       # the product's scratch is padded by 16 too
    fr = np.ascontiguousarray(frame, dtype=np.uint8)
    v = emu.emu_lz4_certify(fr.ctypes.data, fr.size, src.ptr, data.size, flavour)
    src.free()
    assert v in (0, 1), (v, data.size, flavour)
    return bool(v)


def _frames(data, rng, foreign=True, mutations=True):
    """[(name, frame)] for these bytes: the encoder's, its mutations, other encoders'"""
    import oracle
    out = []
    ps, fr = oracle.zfs_lz4_compress(data)
    if fr is not None:
        out.append(("oracle", fr))
        if mutations:
            out += [(n, P.frame_of(b)) for n, b in P.mutated_blocks(P.block_of(fr), rng)]
    if foreign:
        out += [(n, P.frame_of(b)) for n, b in P.foreign_blocks(data)]
    return out


def _agree(emu, cases, misses):
    n = 0
    for tag, data, frames in cases:
        for fl in P.flavours(data.size):
            for name, fr in frames:
                want = P.expected_certified(fr, data)
                got = _certify(emu, fr, data, fl)
                if got != want:
                    misses.append((tag, data.size, fl, name, "got", got, "want", want))
                n += 1
    return n


def test_thresholds_are_the_kernels():
    P.check_thresholds()
    assert P.flavours(P.SIZES_64K_EDGE[0]) == (0,) and P.flavours(P.SIZES_64K_EDGE[1]) == (1, 2)
    assert P.flavours(P.SIZES_COMPACT[0]) == (1, 2) and P.flavours(P.SIZES_BIG[0]) == (1,)


def test_payload_families_are_deterministic_and_distinct():
    for fam in P.FAMILIES:
        a = P.payload(fam, 3, 4096)
        assert a.dtype == np.uint8 and a.size == 4096, fam
        assert np.array_equal(a, P.payload(fam, 3, 4096)), fam
        if fam != "zeros":
            assert not np.array_equal(a, P.payload(fam, 4, 4096)), fam


def test_certificate_verdicts_on_small_records(emu):
    """volume: every family, four seeds, TabU16 sizes, every frame variant"""
    rng = np.random.default_rng(31)
    cases, certified = [], 0
    for fam in P.FAMILIES:
        for seed in (1, 2, 3, 4):
            for n in P.SIZES_SMALL[:3]:
                d = P.payload(fam, seed, n)
                fr = _frames(d, rng)
                certified += P.expected_certified(fr[0][1], d) if fr[0][0] == "oracle" else 0
                cases.append(("%s/%d" % (fam, seed), d, fr))
    misses = []
    n = _agree(emu, cases, misses)
    assert not misses, misses[:20]
    assert n > 1500 and certified > 60, (n, certified)


@pytest.mark.parametrize("sizes", [P.SIZES_SMALL[3:] + P.SIZES_64K_EDGE, P.SIZES_COMPACT])
def test_certificate_verdicts_at_the_table_edges(emu, sizes):
    """one record per family and size, both tables for 65547..131072: the encoder's frame, two parse
    mutations and one foreign frame.  (ints: TabU16 sizes only; its 128 KiB replay is slow here and
    runs on the GPU.)"""
    rng = np.random.default_rng(sizes[0])
    cases = []
    for fam in P.FAMILIES:
        for n in sizes:
            if fam == "ints" and n >= P.LZ4_64KLIMIT:
                continue
            d = P.payload(fam, 5, n)
            fr = _frames(d, rng, foreign=False)
            fr = fr[:3] + [(nm, P.frame_of(b)) for nm, b in P.foreign_blocks(d)[:1]]
            cases.append((fam, d, fr))
    misses = []
    _agree(emu, cases, misses)
    assert not misses, misses[:20]


def test_far_repeats_under_both_tables(emu):
    """copies at 65535 (reachable), 65536 and 65537 (refused by the distance test, but their bytes
    match): certified under TabU32 and Tab17, and a frame that takes a 65535 match as literals is not"""
    import oracle
    for n in (P.SIZES_COMPACT[-1], P.SIZES_BIG[0]):
        d = P.payload("far", 1, n)
        ps, fr = oracle.zfs_lz4_compress(d)
        assert fr is not None
        seqs, tail = F.parse(P.block_of(fr))
        offs = [o for _, o, _ in seqs]
        assert P.LZ4_MAXDIST in offs, "the 65535 copy is not a match"
        assert P.expected_certified(fr, d)
        for fl in P.flavours(n):
            assert _certify(emu, fr, d, fl), (n, fl)
        # the 65535 match given as literals: valid LZ4 of the same bytes, not the encoder's parse
        i = offs.index(P.LZ4_MAXDIST)
        body = seqs[i][0] + d[sum(len(l) + m for l, _, m in seqs[:i]) + len(seqs[i][0]):][:seqs[i][2]].tobytes()
        nxt = seqs[i + 1] if i + 1 < len(seqs) else None
        alt = seqs[:i] + ([(body + nxt[0], nxt[1], nxt[2])] + seqs[i + 2:] if nxt else [])
        blk = F.emit(alt, tail if nxt else body + tail)
        assert F.decode(*F.parse(blk)) == d.tobytes()
        for fl in P.flavours(n):
            assert not _certify(emu, P.frame_of(blk), d, fl), (n, fl)


def _decode(emu, frame, lsize):
    fr = np.ascontiguousarray(frame, dtype=np.uint8)
    src = Guarded(emu, fr.size, slack=0, data=fr)
    dst = Guarded(emu, lsize, slack=0)
    dst.a[:] = 0xEE
    rc = emu.emu_zfs_lz4_decode(src.ptr, fr.size, dst.ptr, lsize)
    out = dst.a.copy()
    src.free()
    dst.free()
    return rc, out


def _decode_agrees(emu, frame, lsize, what):
    import oracle
    rc, got = _decode(emu, frame, lsize)
    orc, want = oracle.zfs_lz4_decompress(frame, lsize)
    assert rc in (0, ECODEC), (what, rc)
    assert (rc == 0) == (orc == 0), (what, rc, orc)
    if rc == 0:
        assert np.array_equal(got, want), what
    return rc == 0


def test_k2_on_family_and_foreign_frames(emu):
    rng = np.random.default_rng(77)
    ok = bad = 0
    for fam in P.FAMILIES:
        for n in (4096, 16384, P.SIZES_64K_EDGE[1]):
            d = P.payload(fam, 9, n)
            for name, fr in _frames(d, rng):
                assert _decode_agrees(emu, fr, n, (fam, n, name))
                ok += 1
                for mname, mf, ls in P.malformed(P.block_of(fr), d)[:4] if name in ("oracle", "fast1") else ():
                    bad += not _decode_agrees(emu, mf, ls, (fam, n, name, mname))
    assert ok > 300 and bad > 20, (ok, bad)


def test_k2_on_synthesized_sequences_and_their_malformed_variants(emu):
    ok = rejected = 0
    for name, blk, data in P.synthesized_blocks(3):
        d = np.frombuffer(data, np.uint8)
        assert _decode_agrees(emu, P.frame_of(blk), d.size, name)
        ok += 1
        for mname, mf, ls in P.malformed(blk, data):
            rejected += not _decode_agrees(emu, mf, ls, (name, mname))
    # every malformed variant but clen = psize - 4 (the pad is read as sequences) must be refused
    assert ok == len(P.LIT_LENS) + len(P.MATCH_LENS) + len(P.OFFSETS) + len(P.TAIL_LENS)
    assert rejected >= ok * 8, (ok, rejected)
