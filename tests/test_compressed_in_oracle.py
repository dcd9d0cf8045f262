"""CPU: the reference model of COMPRESS with MTZ_FLAG_COMPRESSED_IN (tests/compressed_in_ref.py) against
the oracle -- its wire decodes to plain(x) through the DECOMPRESS that ships, plain() undoes `zfs send -c`,
the wire preamble's rule over the four COMPRESSED / EMBED_DATA combinations -- and the compressed_in
subcommand of tools/flag_cost.py (its defaults, its refusal to run without a GPU)."""
import os
import sys

import numpy as np
import pytest

import block_ref as B
import compressed_in_ref as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.append(os.path.join(ROOT, "tools"))


def _raw(oracle, n=20, recsize=8192):
    from test_gpu_codec import _mixed_stream
    return _mixed_stream(oracle, n=n, recsize=recsize)


@pytest.mark.parametrize("codec", [M.DC_LZ4, M.DC_LZJB, M.DC_ZLE, B.mixed_codecs])
@pytest.mark.parametrize("ashift", [9, 12])
def test_plain_undoes_send_c(oracle, codec, ashift):
    s, dcs = B.as_on_disk(oracle, _raw(oracle), ashift, codec)
    x = B.as_send_c(oracle, s, ashift)
    assert any(x[off + 50] != 0 for _, off, _, _ in M.write_records(x))
    assert M.plain(oracle, x).tobytes() == s.tobytes()


@pytest.mark.parametrize("codec", [M.DC_LZ4, M.DC_LZJB, M.DC_ZLE, B.mixed_codecs])
def test_the_model_wire_decompresses_to_plain(oracle, codec):
    x = M.send_c(oracle, _raw(oracle), 9, codec)
    w = M.expected(oracle, x)
    rc, d, _ = oracle.stream_decompress(w)
    assert rc == 0 and d.tobytes() == M.plain(oracle, x).tobytes()
    bad, st = M.verdict(oracle, x)
    assert bad is None
    assert st["lz4_passed"] == len(M.write_records(x, M.DC_LZ4))
    assert st["lzjb_decoded"] == len(M.write_records(x, M.DC_LZJB))
    assert st["zle_decoded"] == len(M.write_records(x, M.DC_ZLE))
    # the records that arrived LZ4 are on the wire byte for byte
    xb, wb = np.asarray(x), oracle.wire_strip(w)
    for (xo, xpo, xpl, t), (wo, wpo, wpl, _) in zip(B.records(xb), B.records(wb)):
        if t == 3 and xb[xo + 50] == M.DC_LZ4:
            # the header up to drr_checksum (re-stamped) and the payload
            assert xb[xo:xo + 280].tobytes() == wb[wo:wo + 280].tobytes()
            assert xb[xpo:xpo + xpl].tobytes() == wb[wpo:wpo + wpl].tobytes()


@pytest.mark.parametrize("embed", [False, True])
@pytest.mark.parametrize("compressed", [False, True])
def test_the_preamble_rule(oracle, compressed, embed):
    """WIRE_F_ORIG_LZ4 = LZ4 && (!COMPRESSED || EMBED_DATA): a stock DECOMPRESS then gives the BEGIN plain
    `zfs send` would have written"""
    s = _raw(oracle, n=6)
    x = M.send_c(oracle, s, 9, M.DC_LZJB) if compressed else s
    x = M.set_features(oracle, x, on=M.FEAT_LZ4 | (M.FEAT_EMBED_DATA if embed else 0))
    assert M.orig_lz4(M.features(x[:312])) == (embed or not compressed)
    w = M.expected(oracle, x)
    assert int.from_bytes(w[12:16].tobytes(), "little") == (1 if embed or not compressed else 0)
    rc, d, _ = oracle.stream_decompress(w)
    p = M.plain(oracle, x)
    assert rc == 0 and d.tobytes() == p.tobytes()
    assert bool(M.features(p[:312]) & M.FEAT_LZ4) == (embed or not compressed)
    assert not M.features(p[:312]) & M.FEAT_COMPRESSED


def test_malformed_frames_and_other_compressions_fail_the_record(oracle):
    x = M.send_c(oracle, _raw(oracle), 9, B.mixed_codecs)
    i, off, po, pl = M.write_records(x, M.DC_LZJB)[0]
    lsize = int.from_bytes(x[off + 32:off + 40].tobytes(), "little")
    cut = M.replace_payload(oracle, x, i, x[po:po + 8])
    assert M.verdict(oracle, cut)[0] == i
    for dc in (M.DC_GZIP6, M.DC_ZSTD, 99):
        assert M.verdict(oracle, M.replace_payload(oracle, x, i, x[po:po + pl], comp=dc))[0] == i
    assert M.decode(oracle, M.DC_LZJB, x[po:po + pl], lsize) is not None


def test_flag_cost_defaults():
    import flag_cost
    a = vars(flag_cost.parse_args(["compressed_in"]))
    assert a.pop("workload") == "compressed_in" and a.pop("out") is None
    assert a == dict(gib=0.5, steps=5, warmup=1, host_steps=3, ring_steps=3, profile_steps=2)


def test_flag_cost_needs_a_gpu(monkeypatch):
    import torch
    import flag_cost
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(SystemExit) as e:
        flag_cost.main(["compressed_in"])
    assert e.value.code == "flag_cost.py compressed_in measures device time: it needs a GPU"
