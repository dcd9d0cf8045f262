"""CPU: the reference model of MTZ_FLAG_GZIP_IN (tests/gzip_in_ref.py) -- plain() undoes `send -c` for
every gzip level and a mixed pool, the model's wire DECOMPRESSes to plain(x), its acceptance rule says no
to one hand-built frame per rejection rule (and yes to zlib's single-code and empty-distance-code
cases), and tools/flag_cost.py's gzip_in defaults and its refusal without a GPU."""
import os
import sys
import zlib

import numpy as np
import pytest

import block_ref as B
import gzip_in_ref as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- hand-built zlib streams ------------------------------------------------------------------------

class Bits(object):
    """an RFC 1951 bit writer: fields LSB first, Huffman codes MSB first"""

    def __init__(self):
        self.v, self.n = 0, 0

    def put(self, value, nbits):
        self.v |= (value & ((1 << nbits) - 1)) << self.n
        self.n += nbits
        return self

    def code(self, code, nbits):
        return self.put(int(format(code, "0%db" % nbits)[::-1], 2) if nbits else 0, nbits)

    def align(self):
        self.n += -self.n % 8
        return self

    def bytes(self):
        return self.v.to_bytes((self.n + 7) // 8, "little")


def canonical(lens):
    """{symbol: (code, length)} of the canonical code of lens"""
    out, code = {}, 0
    for L in range(1, 16):
        for s, ls in enumerate(lens):
            if ls == L:
                out[s] = (code, L)
                code += 1
        code <<= 1
    return out


def zwrap(body, data=None, cmf=0x78, flg=None, adler=None):
    """a zlib stream around the deflate bytes `body`; the trailer is data's Adler-32 unless given"""
    if flg is None:
        flg = (31 - (cmf * 256) % 31) % 31
    a = zlib.adler32(data or b"") if adler is None else adler
    return bytes([cmf, flg]) + body + a.to_bytes(4, "big")


CL_LENS = [4] * 13 + [5] * 6                          # a complete code-length code over 0..18
CL_ORDER = (16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15)


def dynamic(w, lit, dist, symbols, final=1, cl=CL_LENS, nlit=None, ndist=None, cl_syms=None):
    """a dynamic block of the literal/length lengths `lit` and distance lengths `dist`, then `symbols`
    ([("lit", s)] or [("len", s, extra bits, nbits), ("dist", s, extra, nbits)]); `cl_syms` replaces the
    code-length symbols ([(symbol, extra, nbits)])"""
    nlit = len(lit) if nlit is None else nlit
    ndist = len(dist) if ndist is None else ndist
    w.put(final, 1).put(2, 2).put(nlit - 257, 5).put(ndist - 1, 5).put(19 - 4, 4)
    for s in CL_ORDER:
        w.put(cl[s], 3)
    cc = canonical(cl)
    for s, extra, nb in (cl_syms if cl_syms is not None else [(x, 0, 0) for x in list(lit) + list(dist)]):
        w.code(*cc[s]).put(extra, nb)
    lc, dc = canonical(lit), canonical(dist)
    for sym in symbols:
        if sym[0] == "dist":
            w.code(*dc[sym[1]]).put(sym[2], sym[3])
        else:
            w.code(*lc[sym[1]])
            if sym[0] == "len":
                w.put(sym[2], sym[3])
    return w


def lit_lens(pairs, n=259):
    lens = [0] * n
    for s, L in pairs.items():
        lens[s] = L
    return lens


# "A", a match of 3 at distance 1, end of block: "AAAA"
GOOD_LIT = lit_lens({65: 2, 256: 2, 257: 2, 258: 2})
GOOD_DIST = [1, 1]
GOOD_SYMS = [("lit", 65), ("len", 257, 0, 0), ("dist", 0, 0, 0), ("lit", 256)]


def good_frame():
    return zwrap(dynamic(Bits(), GOOD_LIT, GOOD_DIST, GOOD_SYMS).bytes(), b"AAAA")


def fixed(syms):
    """a final fixed-Huffman block: [("lit", s)] / [("dist", s, extra, nbits)] / [("raw", code, nbits)]"""
    w = Bits().put(1, 1).put(1, 2)
    for sym in syms:
        if sym[0] == "dist":
            w.code(sym[1], 5).put(sym[2], sym[3])
            continue
        s = sym[1]
        if s < 144:
            w.code(0x30 + s, 8)
        elif s < 256:
            w.code(0x190 + s - 144, 9)
        elif s < 280:
            w.code(s - 256, 7)
        else:
            w.code(0xc0 + s - 280, 8)
    return w.bytes()


def malformed_frames():
    """[(rule, frame, lsize)] -- one zlib stream per way the stage's acceptance rule refuses one"""
    out = []
    ok = good_frame()
    assert G.inflate(ok, 4) == b"AAAA"

    def add(name, frame, lsize=4):
        out.append((name, bytes(frame), lsize))

    body = ok[2:-4]
    add("cm-not-8", zwrap(body, b"AAAA", cmf=0x77))
    add("cinfo-over-7", zwrap(body, b"AAAA", cmf=0x88))
    add("fcheck", bytes([0x78, 0x9d]) + ok[2:])
    add("fdict", zwrap(body, b"AAAA", flg=0x20 + (31 - (0x7820 % 31)) % 31))
    add("block-type-3", zwrap(Bits().put(1, 1).put(3, 2).bytes(), b""))
    add("stored-len-nlen", zwrap(Bits().put(1, 1).put(0, 2).align().put(4, 16).put(0xfffa, 16).bytes() + b"AAAA",
                                 b"AAAA"))
    add("hlit-over-286", zwrap(dynamic(Bits(), GOOD_LIT, GOOD_DIST, GOOD_SYMS, nlit=287).bytes(), b"AAAA"))
    add("hdist-over-30", zwrap(dynamic(Bits(), GOOD_LIT, GOOD_DIST, GOOD_SYMS, ndist=31).bytes(), b"AAAA"))
    over = lit_lens({65: 2, 66: 2, 256: 2, 257: 2, 258: 2})
    add("lit-over-subscribed", zwrap(dynamic(Bits(), over, GOOD_DIST, GOOD_SYMS).bytes(), b"AAAA"))
    inc = lit_lens({65: 2, 256: 2, 257: 2})
    add("lit-incomplete", zwrap(dynamic(Bits(), inc, GOOD_DIST, GOOD_SYMS).bytes(), b"AAAA"))
    add("dist-over-subscribed", zwrap(dynamic(Bits(), GOOD_LIT, [1, 1, 1], GOOD_SYMS).bytes(), b"AAAA"))
    add("dist-incomplete", zwrap(dynamic(Bits(), GOOD_LIT, [2, 2, 2], GOOD_SYMS).bytes(), b"AAAA"))
    cl = list(CL_LENS)
    cl[18] = 0
    add("cl-incomplete", zwrap(dynamic(Bits(), GOOD_LIT, GOOD_DIST, GOOD_SYMS, cl=cl).bytes(), b"AAAA"))
    cl = list(CL_LENS)
    cl[0] = 3
    add("cl-over-subscribed", zwrap(dynamic(Bits(), GOOD_LIT, GOOD_DIST, GOOD_SYMS, cl=cl).bytes(), b"AAAA"))
    lens = GOOD_LIT + GOOD_DIST
    add("repeat-16-first", zwrap(dynamic(Bits(), GOOD_LIT, GOOD_DIST, GOOD_SYMS,
                                         cl_syms=[(16, 0, 2)] + [(x, 0, 0) for x in lens[3:]]).bytes(), b"AAAA"))
    add("repeat-past-end", zwrap(dynamic(Bits(), GOOD_LIT, GOOD_DIST, GOOD_SYMS,
                                         cl_syms=[(x, 0, 0) for x in lens[:-2]] + [(18, 0, 7)]).bytes(), b"AAAA"))
    noeob = lit_lens({65: 2, 255: 2, 257: 2, 258: 2})
    add("no-end-of-block", zwrap(dynamic(Bits(), noeob, GOOD_DIST,
                                         [("lit", 65), ("len", 257, 0, 0), ("dist", 0, 0, 0)]).bytes(), b"AAAA"))
    add("length-286", zwrap(fixed([("lit", 65), ("lit", 286)]), b"A"), 1)
    add("length-287", zwrap(fixed([("lit", 65), ("lit", 287)]), b"A"), 1)
    add("distance-30", zwrap(fixed([("lit", 65), ("lit", 257), ("dist", 30, 0, 0)]), b"AAAA"))
    add("distance-31", zwrap(fixed([("lit", 65), ("lit", 257), ("dist", 31, 0, 0)]), b"AAAA"))
    add("distance-before-start", zwrap(fixed([("lit", 65), ("lit", 257), ("dist", 1, 0, 0), ("lit", 256)]), b"AAAA"))
    add("output-past-lsize", ok, 3)
    add("output-short-of-lsize", ok, 5)
    add("read-past-end", ok[:len(ok) - 1])
    add("stream-cut", ok[:len(ok) - 6])
    add("adler", zwrap(body, adler=zlib.adler32(b"AAAA") ^ 1))
    return out


def test_every_rule_refuses_its_frame():
    rules = malformed_frames()
    assert len({r for r, _, _ in rules}) == len(rules) >= 20
    for name, frame, lsize in rules:
        assert G.inflate(frame, lsize) is None, name


def test_zlib_accepts_what_the_rule_accepts():
    """a single code of length 1 (lit/len and distance), a distance code with no code at all, padding
    after the trailer, and no padding"""
    stored = Bits().put(0, 1).put(0, 2).align().put(2, 16).put(0xfffd, 16).bytes() + b"hi"
    only_eob = dynamic(Bits(), lit_lens({256: 1}, 257), [0], [("lit", 256)]).bytes()
    f = zwrap(stored + only_eob, b"hi")
    assert G.inflate(f, 2) == b"hi"
    assert G.inflate(f + bytes(13), 2) == b"hi"
    f = zwrap(dynamic(Bits(), lit_lens({65: 1, 256: 1}, 257), [1], [("lit", 65), ("lit", 256)]).bytes(), b"A")
    assert G.inflate(f, 1) == b"A"


@pytest.mark.parametrize("level", range(1, 10))
def test_gzip_frames_follow_zfs(oracle, level):
    s = oracle.synth_stream(12, recsize=16384, kind=oracle.PAYLOAD_PGPAGE)
    keyed = G.as_on_disk(oracle, s, 9, G.DC_GZIP[level])[0]
    x = G.as_send_c(oracle, keyed, 9)
    assert G.plain(oracle, x).tobytes() == keyed.tobytes()
    bad, st = G.verdict(oracle, x)
    assert bad is None and st["gzip_decoded"] > 0
    for i, off, po, pl in __import__("compressed_in_ref").write_records(x, G.DC_GZIP[level]):
        lsize = int.from_bytes(x[off + 32:off + 40].tobytes(), "little")
        assert pl % 512 == 0 and pl <= lsize - lsize // 8 + 511 and pl < lsize
        assert G.inflate(x[po:po + pl], lsize) == zlib.decompress(x[po:po + pl].tobytes())


def test_mixed_pool_and_its_wire(oracle):
    s = oracle.synth_stream(20, recsize=8192, kind=oracle.PAYLOAD_PGPAGE)
    s = G.as_on_disk(oracle, s, 9, G.mixed_codecs)[0]
    x = G.as_send_c(oracle, s, 9)
    comps = {int(x[off + 50]) for _, off, _, _ in __import__("compressed_in_ref").write_records(x)}
    assert {G.DC_GZIP[6], B.DC_LZ4, B.DC_LZJB} <= comps
    assert G.plain(oracle, x).tobytes() == s.tobytes()
    w = G.expected(oracle, x)
    rc, back, _ = oracle.stream_decompress(w)
    assert rc == 0 and back.tobytes() == s.tobytes()


def _flag_cost():
    sys.path.append(os.path.join(ROOT, "tools"))
    import flag_cost
    return flag_cost


def test_flag_cost_defaults():
    fc = _flag_cost()
    a = vars(fc.parse_args(["gzip_in"]))
    assert a.pop("workload") == "gzip_in" and a.pop("out") is None
    assert a == dict(gib=0.5, steps=5, warmup=1, host_steps=3, ring_steps=3, profile_steps=2)


def test_flag_cost_needs_a_gpu(monkeypatch):
    import torch
    fc = _flag_cost()
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(SystemExit) as e:
        fc.main(["gzip_in"])
    assert e.value.code == "flag_cost.py gzip_in measures device time: it needs a GPU"


def test_keyed_builds_the_model_gzip_pool(oracle):
    fc = _flag_cost()
    s = oracle.synth_stream(12, recsize=16384, kind=oracle.PAYLOAD_PGPAGE)
    for codec in (G.DC_GZIP[1], G.mixed_codecs):
        assert fc.keyed(oracle, s, 4, codec).tobytes() == G.as_on_disk(oracle, s, 9, codec)[0].tobytes()
    assert np.array_equal(G.as_send_c(oracle, s), B.as_send_c(oracle, s))
