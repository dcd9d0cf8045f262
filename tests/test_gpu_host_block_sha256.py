"""GPU: gpu.blockSha256 in the host pipeline on a fake `zfs` (tests/test_host_pipeline.py's harness).
A dataset written with checksum=sha256: with gpu.blockChecksums and gpu.blockSha256 on both sides,
job.gpu.blocks / gpuRecv.blocks count every block as compared by SHA-256, and the restore is byte
for byte what `zfs send` produced.  With gpu.blockChecksums alone the same blocks are skipped."""
import hashlib

import pytest

import block_sha256_ref as R
from test_host_pipeline import _run_restore, fakezfs  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


def test_sha256_keys_on_the_compressed_wire(fakezfs, tmp_path, oracle):  # noqa: F811
    s = R.as_sha256(oracle, fakezfs["stream"])
    p = tmp_path / "sha256.bin"
    s.tofile(str(p))
    env = {"FAKE_ZFS_STREAM": str(p)}
    cfg = {"batchBytes": 4 << 20, "ringBytes": 32 << 20, "outRingBytes": 32 << 20, "blockChecksums": True}
    for sha in (True, False):
        c = dict(cfg, blockSha256=True) if sha else cfg
        res, cli, events = _run_restore(fakezfs, sender_gpu=dict(c, mode="compress"),
                                        recv_gpu=dict(c, mode="decompress"), env_extra=env)
        assert res["err"] is None, res
        digest, n = open(fakezfs["recv_out"]).read().split()
        assert int(n) == s.size and digest == hashlib.sha256(s.tobytes()).hexdigest()
        job = cli._restoreObject
        assert job["wire"] == "lz4-stage-v1"
        for side in ("gpu", "gpuRecv"):
            b = job[side]["blocks"]
            if sha:
                assert b["sha256"] == b["logical_ok"] == 24 and b["skipped"] == 0, (side, b)
            else:
                assert b["sha256"] == b["logical_ok"] == 0 and b["skipped"] == 24, (side, b)
