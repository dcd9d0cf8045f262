"""GPU: gpu.blockFrames in the host pipeline on a fake `zfs` (tests/test_host_pipeline.py's harness).
A dataset written with compression=lz4 and sent without -c: with gpu.blockChecksums and
gpu.blockFrames, a VERIFY stage on either side compares every block ZFS stored LZ4 with its encoder
frame, and job.gpu.blocks / gpuRecv.blocks count them as frame_ok and frames_encoded.  The same holds
for a sender configured to compress whose requester asked for the plain wire (it runs VERIFY), and
the restore is byte for byte what `zfs send` produced.  Without gpu.blockFrames those blocks are
skipped."""
import hashlib

import pytest

import block_ref as R
from test_host_pipeline import _run_restore, fakezfs  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


def test_lz4_on_disk_keys_in_verify_on_both_sides(fakezfs, tmp_path, oracle):  # noqa: F811
    s, dcs = R.as_on_disk(oracle, fakezfs["stream"])
    nlz4 = sum(1 for v in dcs.values() if v == R.DC_LZ4)
    assert 0 < nlz4 <= len(dcs)
    p = tmp_path / "lz4.bin"
    s.tofile(str(p))
    env = {"FAKE_ZFS_STREAM": str(p)}
    cfg = {"batchBytes": 4 << 20, "ringBytes": 32 << 20, "blockChecksums": True}
    for sender_mode, frames in (("verify", True), ("compress", True), ("verify", False)):
        c = dict(cfg, blockFrames=True) if frames else cfg
        res, cli, events = _run_restore(fakezfs, sender_gpu=dict(c, mode=sender_mode),
                                        recv_gpu=dict(c, mode="verify"), env_extra=env)
        assert res["err"] is None, res
        digest, n = open(fakezfs["recv_out"]).read().split()
        assert int(n) == s.size and digest == hashlib.sha256(s.tobytes()).hexdigest()
        job = cli._restoreObject
        assert job.get("wire") != "lz4-stage-v1"
        assert job["gpu"]["lz4_encoded"] == 0             # the sender ran VERIFY
        for side in ("gpu", "gpuRecv"):
            b = job[side]["blocks"]
            assert b["logical_ok"] == len(dcs) - nlz4, (side, b)
            if frames:
                assert b["frame_ok"] == b["frames_encoded"] == nlz4 and b["skipped"] == 0, (side, b)
            else:
                assert b["frame_ok"] == b["frames_encoded"] == 0 and b["skipped"] == nlz4, (side, b)
