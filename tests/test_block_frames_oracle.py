"""CPU: the reference model of VERIFY with MTZ_FLAG_BLOCK_FRAMES (tests/block_ref.py).  Its verdicts
must be those of COMPRESS on the same stream (the stage's encoder output compared by the COMPRESS
rules); on a stream without LZ4-on-disk keys that arrive raw the flag must add no record, verdict for
verdict; on an as_on_disk() stream it must turn exactly the LZ4-keyed records from
skipped into frame_ok; and a key taken from another record's frame must be a miss."""
import pytest

import block_ref as R
import test_block_cksum_oracle as T

CMP = R.TRANSFER + ("first_bad",)


def _mixed(oracle, n=40, recsize=8192, ashift=9):
    from test_gpu_codec import _mixed_stream
    return R.as_on_disk(oracle, _mixed_stream(oracle, n=n, recsize=recsize), ashift)


def _compress_model(oracle, s, sha256=False, sha512=False):
    rc, out, _ = oracle.stream_compress_plain(s)
    assert rc == 0
    return R.block_check(oracle, s, R.COMPRESS, out, sha256=sha256, sha512=sha512)


@pytest.mark.parametrize("ashift", [9, 12])
@pytest.mark.parametrize("key", ["fletcher4", "sha256", "sha512"])
def test_the_model_is_compress_on_the_same_stream(oracle, ashift, key):
    s, dcs = _mixed(oracle, ashift=ashift)
    kw = {}
    if key == "sha256":
        s, kw = R.as_sha(oracle, s, "sha256"), dict(sha256=True)
    elif key == "sha512":
        s, kw = R.as_sha(oracle, s, "sha512"), dict(sha512=True)
    v, st = R.block_check(oracle, s, R.VERIFY, frames=True, **kw)
    cv, cst = _compress_model(oracle, s, **kw)
    assert v == cv
    assert {k: st[k] for k in CMP} == {k: cst[k] for k in CMP}
    assert st["frames_encoded"] == sum(1 for x in dcs.values() if x == R.DC_LZ4)


@pytest.mark.parametrize("ashift", [9, 12])
def test_exactly_the_raw_lz4_keyed_records_turn_from_skipped_to_frame_ok(oracle, ashift):
    s, dcs = _mixed(oracle, ashift=ashift)
    lz4 = {i for i, x in dcs.items() if x == R.DC_LZ4}
    assert 0 < len(lz4) < len(dcs)
    vv, vst = R.block_check(oracle, s, R.VERIFY)
    fv, fst = R.block_check(oracle, s, R.VERIFY, frames=True)
    assert {i for i in vv if vv[i] != fv[i]} == lz4
    assert all(vv[i] == R.SKIPPED and fv[i] == R.FRAME_OK for i in lz4)
    assert vst["skipped"] == len(lz4) and fst["skipped"] == 0
    assert fst["frame_ok"] == fst["frames_encoded"] == len(lz4) and fst["frame_miss"] == 0
    assert fst["logical_ok"] == vst["logical_ok"] == len(dcs) - len(lz4)


def test_the_model_is_the_verify_model_without_raw_lz4_keys(oracle):
    """streams the generator writes (every key logical), their sha256 / sha512 forms, the `send -c`
    form of an lz4 dataset (its LZ4 blocks arrive as frames), and keys the check cannot read"""
    from test_gpu_codec import _mixed_stream
    raw = oracle.synth_stream(24, recsize=8192, kind=oracle.PAYLOAD_PGPAGE)
    s, dcs = _mixed(oracle)
    c = R.as_send_c(oracle, s)
    unread = s.copy()
    recs = R.records(unread)
    for i in [i for i, x in dcs.items() if x == R.DC_LZ4][:3]:
        R.set_key(unread, recs[i][0], ctype=12)                # skein: salted, never checked
    lz4_unflagged = R.as_sha(oracle, s, "sha256")              # sha256 keys without BLOCK_SHA256
    assert oracle.stream_restamp(unread)[0] == 0
    cases = [(raw, {}), (R.as_sha(oracle, raw, "sha256"), dict(sha256=True)),
             (R.as_sha(oracle, raw, "sha512"), dict(sha512=True)), (c, {}), (c, dict(sha256=True, sha512=True)),
             (lz4_unflagged, {}), (_mixed_stream(oracle, n=20), {})]
    for src, kw in cases:
        assert T.flag_off(oracle, src, R.VERIFY, None, "frames", **kw) == 0
    assert T.flag_off(oracle, unread, R.VERIFY, None, "frames") == sum(1 for x in dcs.values() if x == R.DC_LZ4) - 3


def test_a_key_copied_from_another_frame_is_a_miss(oracle):
    s, dcs = _mixed(oracle)
    lz4 = sorted(i for i, x in dcs.items() if x == R.DC_LZ4)
    recs = R.records(s)
    s = s.copy()
    for i, j in zip(lz4[1:4], lz4[2:5]):
        _, key, p = R.get_key(s, recs[j][0])
        R.set_key(s, recs[i][0], key=key, ddk_prop=(p & ~0xffff) | (R.get_key(s, recs[i][0])[2] & 0xffff))
    assert oracle.stream_restamp(s)[0] == 0
    v, st = R.block_check(oracle, s, R.VERIFY, frames=True)
    assert [i for i in lz4 if v[i] == R.FRAME_MISS] == lz4[1:4]
    assert st["frame_miss"] == 3 and st["first_frame_miss"] == lz4[1]
    assert st["frames_encoded"] == len(lz4) and st["frame_ok"] == len(lz4) - 3
    cv, cst = _compress_model(oracle, s)
    assert v == cv and {k: st[k] for k in CMP} == {k: cst[k] for k in CMP}
