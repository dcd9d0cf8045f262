"""GPU: gpu.blockLzjb in the host pipeline on a fake `zfs` (tests/test_host_pipeline.py's harness).
A dataset written with compression=lzjb and sent without -c: with gpu.blockChecksums and
gpu.blockLzjb, a VERIFY stage on either side compares every block ZFS stored lzjb with its encoder
frame, and job.gpu.blocks / gpuRecv.blocks count them as frame_ok and lzjb_encoded (zle likewise as
zle_encoded).  The restore is byte for byte what `zfs send` produced.  Without gpu.blockLzjb those
blocks are skipped."""
import hashlib

import pytest

import block_lzjb_ref as R
from test_host_pipeline import _run_restore, fakezfs  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("codec", [R.DC_LZJB, R.DC_ZLE])
def test_lzjb_and_zle_keys_in_verify_on_both_sides(fakezfs, tmp_path, oracle, codec):  # noqa: F811
    s, dcs = R.as_on_disk(oracle, fakezfs["stream"], 9, codec)
    ncomp = sum(1 for v in dcs.values() if v == codec)
    assert 0 < ncomp <= len(dcs)
    p = tmp_path / "lzjb.bin"
    s.tofile(str(p))
    env = {"FAKE_ZFS_STREAM": str(p)}
    cfg = {"batchBytes": 4 << 20, "ringBytes": 32 << 20, "blockChecksums": True}
    counter, other = ("lzjb_encoded", "zle_encoded") if codec == R.DC_LZJB else ("zle_encoded", "lzjb_encoded")
    for sender_mode, lzjb in (("verify", True), ("compress", True), ("verify", False)):
        c = dict(cfg, blockLzjb=True) if lzjb else cfg
        res, cli, events = _run_restore(fakezfs, sender_gpu=dict(c, mode=sender_mode),
                                        recv_gpu=dict(c, mode="verify"), env_extra=env)
        assert res["err"] is None, res
        digest, n = open(fakezfs["recv_out"]).read().split()
        assert int(n) == s.size and digest == hashlib.sha256(s.tobytes()).hexdigest()
        job = cli._restoreObject
        assert job.get("wire") != "lz4-stage-v1"
        for side in ("gpu", "gpuRecv"):
            b = job[side]["blocks"]
            assert b["logical_ok"] == len(dcs) - ncomp, (side, b)
            assert b[other] == 0 and b["frames_encoded"] == 0, (side, b)
            if lzjb:
                assert b["frame_ok"] == b[counter] == ncomp and b["skipped"] == 0, (side, b)
            else:
                assert b["frame_ok"] == b[counter] == 0 and b["skipped"] == ncomp, (side, b)
