"""CPU: the reference model of MTZ_FLAG_GZIP_ENCODE (tests/gzip_encode_ref.py) -- every frame inflates with zlib to
its logical bytes and passes gzip_in_ref's acceptance rule, no record gets larger than without the flag, pg-page
records get at least 15 % fewer wire bytes, and the hand-built cases the frame definition names: all-zero
records, matches of 259 / 260 / 261 bytes, offsets of 32768 / 32769, records without matches or with one
literal value, the 15-bit limit, and records up to 1 MiB."""
import os
import zlib

import numpy as np
import pytest

import gzip_encode_ref as E
import gzip_in_ref as G
import lz4_payloads as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def check_frame(data, frame):
    """`frame` (a padded zlib frame) inflates to `data` by zlib and by the stage's acceptance rule"""
    z = np.frombuffer(frame, dtype=np.uint8)
    assert z.size % 512 == 0 and z[0] == 0x78 and z[1] == 0x01
    assert zlib.decompressobj().decompress(frame) == np.asarray(data, dtype=np.uint8).tobytes()
    assert G.inflate(z, len(data)) is not None


@pytest.mark.parametrize("family", P.FAMILIES)
@pytest.mark.parametrize("size", [512, 4096, 131072])
def test_every_frame_inflates_to_its_record(oracle, family, size):
    d = P.payload(family, 7, size)
    comp, pay = E.stage_payload(oracle, d)
    ps, lz = oracle.zfs_lz4_compress(d)
    if lz is None:
        assert comp == 0 and np.array_equal(pay, d)
        return
    check_frame(d, E.pad512(E.deflate(d, lz)))
    assert pay.size <= ps                     # never larger than the LZ4 frame
    if comp == E.DC_GZIP1:
        check_frame(d, pay.tobytes())
        assert pay.size < ps


def test_pg_pages_save_at_least_15_percent(oracle):
    lz = gz = 0
    for r in range(64):
        d = oracle.gen_payload(oracle.PAYLOAD_PGPAGE, r, 131072)
        ps, _ = oracle.zfs_lz4_compress(d)
        _, pay = E.stage_payload(oracle, d)
        assert pay.size <= ps
        lz += ps
        gz += pay.size
    assert gz <= 0.85 * lz, (lz, gz)


def test_match_pieces():
    assert E.split(258) == [258]
    assert E.split(259) == [256, 3]
    assert E.split(260) == [257, 3]
    assert E.split(261) == [258, 3]
    assert E.split(516) == [258, 258]
    assert E.split(517) == [258, 256, 3]
    for L in range(3, 2000):
        p = E.split(L)
        assert sum(p) == L and all(3 <= x <= 258 for x in p)


def test_an_all_zero_record_splits_long_offset_one_matches(oracle):
    d = np.zeros(131072, dtype=np.uint8)
    ps, lz = oracle.zfs_lz4_compress(d)
    seqs = E.sequences(lz)
    assert any(ml > 258 and off == 1 for _, ml, off in seqs)
    ll, ln, ds = E.tokens(d, lz)
    assert (ln[ll >= 257] <= 258).all() and (ds[ll >= 257] == 1).all()
    check_frame(d, E.pad512(E.deflate(d, lz)))


def _hand(seqs, n):
    """(data, ZFS-LZ4 frame) of sequences (literals, match length, offset) over random literal bytes"""
    rng = np.random.default_rng(n)
    out, blk = bytearray(), bytearray()

    def ext(v):
        while v >= 255:
            blk.append(255)
            v -= 255
        blk.append(v)
    for nl, ml, off in seqs:
        lits = rng.integers(0, 256, nl, dtype=np.uint8).tobytes()
        tok = (min(nl, 15) << 4) | (min(ml - 4, 15) if ml else 0)
        blk.append(tok)
        if nl >= 15:
            ext(nl - 15)
        blk += lits
        out += lits
        if ml == 0:
            break
        blk += off.to_bytes(2, "little")
        if ml - 4 >= 15:
            ext(ml - 4 - 15)
        for _ in range(ml):
            out.append(out[-off])
    return np.frombuffer(bytes(out), dtype=np.uint8), len(blk).to_bytes(4, "big") + bytes(blk)


@pytest.mark.parametrize("ml", [259, 260, 261])
def test_matches_of_259_to_261_bytes(ml):
    d, lz = _hand([(40, ml, 7), (20, 0, 0)], ml)
    ll, ln, _ = E.tokens(d, lz)
    assert list(ln[ll >= 257]) == E.split(ml)
    check_frame(d, E.pad512(E.deflate(d, lz)))


@pytest.mark.parametrize("off,far", [(32768, False), (32769, True)])
def test_offsets_of_32768_and_32769(off, far):
    d, lz = _hand([(off + 10, 50, off), (20, 0, 0)], off)
    ll, _, ds = E.tokens(d, lz)
    assert (ll >= 257).sum() == (0 if far else 1)
    assert ll.size == (off + 10 + 50 + 20 if far else off + 10 + 1 + 20)
    check_frame(d, E.pad512(E.deflate(d, lz)))


def test_a_record_without_matches_and_one_with_one_literal_value():
    d, lz = _hand([(5000, 0, 0)], 1)
    ll, _, _ = E.tokens(d, lz)
    assert (ll < 256).all()
    check_frame(d, E.pad512(E.deflate(d, lz)))
    d = np.full(3000, 0x41, dtype=np.uint8)
    blk = bytes([0xf0]) + b"\xff" * 11 + bytes([3000 - 15 - 255 * 11]) + d.tobytes()
    lz = len(blk).to_bytes(4, "big") + blk
    assert E.sequences(lz) == [(3000, 0, 0)]
    check_frame(d, E.pad512(E.deflate(d, lz)))


def test_the_15_bit_limit():
    fib = [1, 1]
    while len(fib) < 30:
        fib.append(fib[-1] + fib[-2])
    freq = fib + [0] * (286 - len(fib))
    L = E.huff_lengths(freq, 15)
    assert max(L) == 15
    assert sum(2.0 ** -x for x in L if x) == 1.0
    assert all((a == 0) == (b == 0) for a, b in zip(L, freq))
    L7 = E.huff_lengths(fib[:19], 7)
    assert max(L7) <= 7 and sum(2.0 ** -x for x in L7 if x) == 1.0
    # unlimited it would be deeper
    assert max(E.huff_lengths(freq, 64)) > 15


def test_large_records(oracle):
    for n in (262144, 1 << 20):
        d = oracle.gen_payload(oracle.PAYLOAD_PGPAGE, 3, n)
        z = E.frame(oracle, d)
        assert z is not None
        check_frame(d, z)


def test_the_flag_cost_workload_is_listed():
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import flag_cost
    assert "gzip_encode" in flag_cost.WORKLOADS
