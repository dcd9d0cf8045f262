"""GPU: gpu.blockLogical in the host pipeline on a fake `zfs` (tests/test_host_pipeline.py's harness).
A dataset written with compression=lzjb (or zle), sent without -c over the compressed wire: COMPRESS
on the sender, DECOMPRESS on the receiver.  With gpu.blockChecksums, gpu.blockLzjb and
gpu.blockLogical both stages compare every block ZFS stored compressed with their encoder frame of
its logical bytes, and job.gpu.blocks / gpuRecv.blocks agree; without gpu.blockLogical those blocks
are skipped at both ends.  The restore is byte for byte what `zfs send` produced."""
import hashlib

import pytest

import block_ref as R
from test_host_pipeline import _run_restore, fakezfs  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("codec", [R.DC_LZJB, R.DC_ZLE])
def test_lzjb_and_zle_keys_on_the_compressed_wire(fakezfs, tmp_path, oracle, codec):  # noqa: F811
    s, dcs = R.as_on_disk(oracle, fakezfs["stream"], 9, codec)
    ncomp = sum(1 for v in dcs.values() if v == codec)
    assert 0 < ncomp <= len(dcs)
    p = tmp_path / "logical.bin"
    s.tofile(str(p))
    env = {"FAKE_ZFS_STREAM": str(p)}
    cfg = {"batchBytes": 4 << 20, "ringBytes": 32 << 20, "blockChecksums": True, "blockLzjb": True}
    counter = "lzjb_encoded" if codec == R.DC_LZJB else "zle_encoded"
    for logical in (True, False):
        c = dict(cfg, blockLogical=True) if logical else cfg
        res, cli, events = _run_restore(fakezfs, sender_gpu=dict(c, mode="compress"),
                                        recv_gpu=dict(c, mode="decompress"), env_extra=env)
        assert res["err"] is None, res
        digest, n = open(fakezfs["recv_out"]).read().split()
        assert int(n) == s.size and digest == hashlib.sha256(s.tobytes()).hexdigest()
        job = cli._restoreObject
        assert job.get("wire") == "lz4-stage-v1"
        for side in ("gpu", "gpuRecv"):
            b = job[side]["blocks"]
            assert b["logical_ok"] == len(dcs) - ncomp, (side, b)
            if logical:
                assert b["frame_ok"] == b[counter] == b["logical_checked"] == ncomp and b["skipped"] == 0, (side, b)
            else:
                assert b["frame_ok"] == b[counter] == b["logical_checked"] == 0 and b["skipped"] == ncomp, (side, b)
        assert job["gpu"]["blocks"] == job["gpuRecv"]["blocks"]
