"""GPU, host mirror: gpu.sendCompressed + gpu.sendGzip on a `compress` sender.  A job on the stage wire
spawns `zfs send -c -v -P <snap>` of a gzip pool and opens COMPRESS with MTZ_FLAG_COMPRESSED_IN |
MTZ_FLAG_GZIP_IN; a stock `decompress` receiver hands `zfs recv` the stream `zfs send` without -c would
have produced.  A requester that does not accept the stage wire gets the raw stream from the reference
command, through a VERIFY stage opened without the gzip flag."""
import hashlib
import json

import pytest

import gzip_in_ref as G
from test_host_pipeline import _run_restore, fakezfs  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

SENDER = {"mode": "compress", "sendCompressed": True, "sendGzip": True}


@pytest.fixture()
def sendc(fakezfs, tmp_path, oracle):  # noqa: F811
    keyed, _ = G.as_on_disk(oracle, fakezfs["stream"], 9, G.mixed_codecs)
    x = G.as_send_c(oracle, keyed, 9)
    xp = tmp_path / "stream_c.bin"
    x.tofile(str(xp))
    args = tmp_path / "send_args.jsonl"
    env = {"FAKE_ZFS_STREAM_C": str(xp), "FAKE_ZFS_SEND_ARGS": str(args)}
    return dict(fakezfs, x=x, keyed=keyed, env_extra=env, args=str(args))


def _sends(path):
    return [json.loads(line) for line in open(path)]


def test_gzip_pool_through_send_c_to_a_stock_receiver(sendc, oracle):
    x = sendc["x"]
    p = G.plain(oracle, x)
    assert p.tobytes() == sendc["keyed"].tobytes()
    res, cli, _ = _run_restore(sendc, sender_gpu=SENDER, recv_gpu={"mode": "decompress"},
                               env_extra=sendc["env_extra"])
    assert res["err"] is None, res
    digest, n = open(sendc["recv_out"]).read().split()
    assert int(n) == p.size and digest == hashlib.sha256(p.tobytes()).hexdigest()
    assert [a[:2] for a in _sends(sendc["args"])] == [["send", "-c"]]
    cin = cli._restoreObject["gpu"]["compressed_in"]
    assert cin == G.verdict(oracle, x)[1] and cin["gzip_decoded"] > 0


def test_a_requester_without_accept_gets_the_reference_command(sendc, oracle):
    s = sendc["stream"]
    res, cli, _ = _run_restore(sendc, sender_gpu=SENDER, recv_gpu=None, env_extra=sendc["env_extra"])
    assert res["err"] is None, res
    digest, n = open(sendc["recv_out"]).read().split()
    assert int(n) == s.size and digest == hashlib.sha256(s.tobytes()).hexdigest()
    assert [a[:2] for a in _sends(sendc["args"])] == [["send", "-v"]]
    assert cli._restoreObject.get("wire") == "raw"
