"""CPU: the reference model of MTZ_FLAG_GZIP_WIRE (tests/gzip_wire_ref.py) -- the gzip wire undoes to
plain(x), carries WIRE_F_GZIP in every preamble, is exactly the `send -c` size plus one preamble per BEGIN
for a pool whose every block is stored compressed, and is smaller than today's inflated and re-encoded
wire on gzip-1 / 6 / 9 pools; and tools/flag_cost.py's gzip_wire workload."""
import os
import sys

import numpy as np
import pytest

import block_ref as B
import compressed_in_ref as M
import gzip_in_ref as G
import gzip_wire_ref as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CODECS = {"gzip-1": G.DC_GZIP[1], "gzip-6": G.DC_GZIP[6], "gzip-9": G.DC_GZIP[9], "mixed": G.mixed_codecs}


def mixed_stream(oracle, n, recsize):
    from test_gpu_codec import _mixed_stream
    return _mixed_stream(oracle, n=n, recsize=recsize)


def pg_pool(oracle, codec, n=16, recsize=131072):
    """pg-page records only: every block of a gzip pool is stored as its gzip frame"""
    return G.send_c(oracle, oracle.synth_stream(n, recsize=recsize, kind=oracle.PAYLOAD_PGPAGE).copy(), 9,
                    CODECS[codec])


@pytest.mark.parametrize("codec", sorted(CODECS))
@pytest.mark.parametrize("recsize", [512, 8192, 131072])
def test_the_wire_undoes_to_plain(oracle, codec, recsize):
    x = G.send_c(oracle, mixed_stream(oracle, {512: 60, 8192: 30, 131072: 8}[recsize], recsize), 9, CODECS[codec])
    w = W.expected(oracle, x)
    # the records between the preambles are a `send -c`-like stream: its plain form is x's
    assert np.array_equal(G.plain(oracle, oracle.wire_strip(w)), G.plain(oracle, x))
    feat = M.features(x)
    assert W.pre_flags(oracle, w) == [W.WIRE_F_GZIP | (M.WIRE_F_ORIG_LZ4 if M.orig_lz4(feat) else 0)]
    bad, st = W.verdict(oracle, x)
    assert bad is None
    assert st["gzip_passed"] == sum(G.is_gzip(int(x[off + 50])) for _, off, _, _ in M.write_records(x))
    assert st["gzip_passed"] > 0 or recsize == 512          # no 512-byte block saves a sector
    assert st["gzip_decoded"] == 0
    assert W.receiver_verdict(oracle, w) == (None, dict(W.verdict(oracle, x)[1], lz4_passed=0, lzjb_decoded=0,
                                                        zle_decoded=0, gzip_passed=0,
                                                        gzip_decoded=st["gzip_passed"]))


def test_gzip_and_lz4_records_travel_as_they_arrived(oracle):
    x = G.send_c(oracle, mixed_stream(oracle, 30, 8192), 9, G.mixed_codecs)
    xb, wb = np.asarray(x), oracle.wire_strip(W.expected(oracle, x))
    n = 0
    for (xo, xpo, xpl, t), (wo, wpo, wpl, _) in zip(B.records(xb), B.records(wb)):
        if t == 3 and W.forwarded(int(xb[xo + 50])):
            assert np.array_equal(xb[xo:xo + 280], wb[wo:wo + 280])
            assert np.array_equal(xb[xpo:xpo + xpl], wb[wpo:wpo + wpl])
            n += 1
    assert n > 0


@pytest.mark.parametrize("codec", ["gzip-1", "gzip-6", "gzip-9"])
def test_a_gzip_pool_is_its_send_c_size_and_smaller_than_the_lz4_wire(oracle, codec):
    x = pg_pool(oracle, codec)
    w = W.expected(oracle, x)
    assert w.size == W.wire_size(oracle, x) == x.size + W.PRE_BYTES
    lz4_wire = G.expected(oracle, x)
    assert w.size < lz4_wire.size, (w.size, lz4_wire.size)


def test_a_corrupted_frame_fails_at_the_receiver(oracle):
    """the sender forwards what it does not decode; the receiver's rule is gzip_in_ref's"""
    x = G.send_c(oracle, mixed_stream(oracle, 20, 8192), 9, G.DC_GZIP[6])
    i, _, po, pl = M.write_records(x, G.DC_GZIP[6])[2]
    fr = bytearray(x[po:po + pl].tobytes())
    fr[4] ^= 0x10
    bad = M.replace_payload(oracle, x, i, fr)
    assert W.verdict(oracle, bad)[0] is None
    rc, lz, _ = oracle.stream_compress(G.plain(oracle, x))
    assert rc == 0
    assert W.receiver_verdict(oracle, W.splice(oracle, lz, bad))[0] == i


def _flag_cost():
    sys.path.append(os.path.join(ROOT, "tools"))
    import flag_cost
    return flag_cost


def test_flag_cost_defaults():
    a = vars(_flag_cost().parse_args(["gzip_wire"]))
    assert a.pop("workload") == "gzip_wire" and a.pop("out") is None
    assert a == dict(gib=0.5, steps=5, warmup=1, host_steps=3, ring_steps=3, profile_steps=2,
                     pools="gzip1,gzip6,gzip9,mixed_gzip6_lz4_lzjb_raw")


def test_flag_cost_needs_a_gpu(monkeypatch):
    import torch
    fc = _flag_cost()
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(SystemExit) as e:
        fc.main(["gzip_wire"])
    assert e.value.code == "flag_cost.py gzip_wire measures device time: it needs a GPU"
