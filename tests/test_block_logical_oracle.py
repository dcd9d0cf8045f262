"""CPU: the model of MTZ_FLAG_BLOCK_LOGICAL (tests/block_ref.py). Turning the flag off skips exactly the
records it adds and changes no other verdict, in every mode (none in VERIFY); with it the four stages of
a transfer count the same on a stream with a mix of keys, for every subset of the SHA and lzjb flags; a
raw-keyed record corrupted inside its LZ4 frame is a logical mismatch at its index in RECOMPRESS."""
import numpy as np
import pytest

import block_ref as R
import test_block_cksum_oracle as T
import test_gpu_block_logical as G


def test_the_mixed_stream_has_every_kind_of_key(oracle):
    x, dcs = R.mixed_keys_stream(oracle, n=48)
    assert oracle.stream_verify(x)[0] == 0
    assert {R.DC_LZJB, R.DC_ZLE, R.DC_LZ4, R.DC_OFF} == set(dcs.values())
    types = {int(x[off + 48]) for off, _, _, t in R.records(x) if t == 3}
    assert {R.FLETCHER4, R.SHA256, R.SHA512, R.CKSUM_SKEIN} <= types
    writes = sum(1 for _, _, _, t in R.records(x) if t == 3)
    assert len(dcs) < writes
    assert not np.array_equal(x, R.mixed_keys_stream(oracle, n=48, seed=1)[0])


def test_the_model_without_the_flag_is_the_existing_one(oracle):
    x, _ = R.mixed_keys_stream(oracle, n=30)
    c = R.send_c_form(oracle, x)
    r = oracle.stream_recompress(c)[1]
    for mode, inp, out in ((R.VERIFY, x, None), (R.COMPRESS, x, c), (R.DECOMPRESS, c, x), (R.RECOMPRESS, c, r)):
        for lzjb in (False, True):
            n = T.flag_off(oracle, inp, mode, out, "logical", lzjb=lzjb, sha256=True)
            # VERIFY does not change with the flag
            assert (n > 0) == (mode != R.VERIFY and (lzjb or mode != R.COMPRESS)), (mode, lzjb)


@pytest.mark.parametrize("flags", G.SUBSETS, ids=lambda f: "+".join(k for k in f if f[k]) or "fletcher4")
@pytest.mark.parametrize("seed", [0, 1])
def test_the_four_stages_count_the_same(oracle, flags, seed):
    x, dcs = R.mixed_keys_stream(oracle, n=48, seed=seed)
    w = R.four_ways(oracle, x, frames=True, **flags)
    v = w["verify"][1]
    for mode in G.MODES:
        assert {k: w[mode][1][k] for k in R.TRANSFER} == {k: v[k] for k in R.TRANSFER}, mode
        assert w[mode][1]["first_bad"] == R.NONE
    assert w["recompress"][1]["logical_checked"] > 0
    assert (w["compress"][1]["logical_checked"] > 0) == flags["lzjb"]
    if flags["sha256"] and flags["sha512"]:
        # the blocks the stage's LZ4 encoder stores raw under an LZ4 key: a miss at both ends of the wire
        assert v["frame_miss"] == w["decompress"][1]["frame_miss"] > 0
        assert w["decompress"][1]["logical_checked"] > 0


def test_compress_has_no_logical_bytes_of_an_lz4_record(oracle):
    """COMPRESS decodes nothing: lzjb / zle keys of records that arrive LZ4 stay skipped there, while
    DECOMPRESS and RECOMPRESS, which decode them, check them"""
    x, dcs = R.as_on_disk(oracle, oracle.synth_stream(12, recsize=8192, kind=oracle.PAYLOAD_PGPAGE), 9, R.DC_LZJB)
    c = R.send_c_form(oracle, x)
    assert all(c[off + 50] == R.DC_LZ4 for off, _, _, t in R.records(c) if t == 3) and len(dcs) == 12
    on = R.block_check(oracle, c, R.COMPRESS, c, lzjb=True, logical=True)
    assert on == R.block_check(oracle, c, R.COMPRESS, c, lzjb=True)
    assert on[1]["skipped"] == 12 and on[1]["logical_checked"] == 0
    for mode, out in ((R.DECOMPRESS, x), (R.RECOMPRESS, oracle.stream_recompress(c)[1])):
        st = R.block_check(oracle, c, mode, out, lzjb=True, logical=True)[1]
        assert st["frame_ok"] == st["lzjb_encoded"] == st["logical_checked"] == 12


def test_a_corrupted_raw_keyed_lz4_record_is_a_logical_mismatch(oracle):
    x = oracle.synth_stream(24, recsize=16384, kind=oracle.PAYLOAD_PGPAGE)
    bad = G._corrupt_a_literal(oracle, R.send_c_form(oracle, x), 9)
    rc, r, _ = oracle.stream_recompress(bad)
    assert rc == 0
    off, po, pl, _ = R.records(bad)[9]
    rc, d = oracle.zfs_lz4_decompress(bad[po:po + pl], 16384)
    xo = R.records(x)[9][1]
    assert rc == 0 and not np.array_equal(d, x[xo:xo + 16384])
    assert R.block_check(oracle, bad, R.RECOMPRESS, r)[1]["first_bad"] == R.NONE
    v, st = R.block_check(oracle, bad, R.RECOMPRESS, r, logical=True)
    assert st["first_bad"] == 9 and v[9] == R.LOGICAL_BAD and st["logical_ok"] == 23 and st["logical_checked"] == 24
