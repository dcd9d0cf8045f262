"""GPU, host mirror: gpu.sendCompressed on a `compress` sender.  A job on the stage wire spawns
`zfs send -c -v -P <snap>` and opens COMPRESS with MTZ_FLAG_COMPRESSED_IN; a stock `decompress`
receiver hands `zfs recv` the stream `zfs send` without -c would have produced.  A requester that
does not accept the stage wire gets the raw stream from the reference command.  tools/fake_zfs.py
serves the -c form from $FAKE_ZFS_STREAM_C and records every send's arguments."""
import hashlib
import json

import pytest

import block_ref as B
import compressed_in_ref as M
from test_host_pipeline import _run_restore, fakezfs  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


@pytest.fixture()
def sendc(fakezfs, tmp_path, oracle):  # noqa: F811
    s = fakezfs["stream"]
    keyed, _ = B.as_on_disk(oracle, s, 9, B.mixed_codecs)
    x = B.as_send_c(oracle, keyed, 9)
    xp = tmp_path / "stream_c.bin"
    x.tofile(str(xp))
    args = tmp_path / "send_args.jsonl"
    env = {"FAKE_ZFS_STREAM_C": str(xp), "FAKE_ZFS_SEND_ARGS": str(args)}
    return dict(fakezfs, x=x, keyed=keyed, env_extra=env, args=str(args))


def _sends(path):
    return [json.loads(line) for line in open(path)]


def test_compress_sender_with_send_compressed_to_a_stock_receiver(sendc, oracle):
    x = sendc["x"]
    p = M.plain(oracle, x)
    assert p.tobytes() == sendc["keyed"].tobytes()          # the stream the same pool sends without -c
    res, cli, _ = _run_restore(sendc, sender_gpu={"mode": "compress", "sendCompressed": True},
                               recv_gpu={"mode": "decompress"}, env_extra=sendc["env_extra"])
    assert res["err"] is None, res
    digest, n = open(sendc["recv_out"]).read().split()
    assert int(n) == p.size and digest == hashlib.sha256(p.tobytes()).hexdigest()
    assert [a[:2] for a in _sends(sendc["args"])] == [["send", "-c"]]
    job = cli._restoreObject
    assert job.get("wire") == "lz4-stage-v1"
    assert job["gpu"]["compressed_in"] == M.verdict(oracle, x)[1]


def test_a_requester_without_accept_gets_the_reference_command(sendc, oracle):
    s = sendc["stream"]
    res, cli, _ = _run_restore(sendc, sender_gpu={"mode": "compress", "sendCompressed": True},
                               recv_gpu=None, env_extra=sendc["env_extra"])
    assert res["err"] is None, res
    digest, n = open(sendc["recv_out"]).read().split()
    assert int(n) == s.size and digest == hashlib.sha256(s.tobytes()).hexdigest()
    assert [a[:2] for a in _sends(sendc["args"])] == [["send", "-v"]]
    job = cli._restoreObject
    assert job.get("wire") == "raw"
