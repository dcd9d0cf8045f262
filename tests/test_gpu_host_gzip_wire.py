"""GPU, host mirror: gzip frames on the compressed wire.  A `decompress` receiver with gpu.acceptGzip posts
`acceptGzip: true`; a `compress` sender with gpu.sendCompressed whose every requester of a send did so sets
job.wireGzip, spawns `zfs send -c` and opens COMPRESS with MTZ_FLAG_COMPRESSED_IN | MTZ_FLAG_GZIP_WIRE; the
receiver's DECOMPRESS, opened with MTZ_FLAG_GZIP_WIRE, inflates the gzip records and hands `zfs recv` the
stream `zfs send` without -c would have produced.  One requester without acceptGzip in a coalesced send
puts every requester back on the inflated, re-encoded wire."""
import hashlib
import threading

import pytest

import gzip_in_ref as G
import gzip_wire_ref as W
from test_gpu_host_gzip_in import _sends, sendc  # noqa: F401  (fixture)
from test_host_pipeline import _free_port, _run_restore, fakezfs  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

SENDER = {"mode": "compress", "sendCompressed": True, "sendGzip": True}
RECEIVER = {"mode": "decompress", "acceptGzip": True}


def _digest(path):
    digest, n = open(path).read().split()
    return digest, int(n)


def test_gzip_frames_travel_to_an_accepting_receiver(sendc, oracle):  # noqa: F811
    x = sendc["x"]
    p = G.plain(oracle, x)
    res, cli, _ = _run_restore(sendc, sender_gpu=SENDER, recv_gpu=RECEIVER, env_extra=sendc["env_extra"])
    assert res["err"] is None, res
    assert _digest(sendc["recv_out"]) == (hashlib.sha256(p.tobytes()).hexdigest(), p.size)
    assert [a[:2] for a in _sends(sendc["args"])] == [["send", "-c"]]
    job = cli._restoreObject
    assert job["acceptGzip"] is True and job["wireGzip"] is True
    cin = job["gpu"]["compressed_in"]
    assert cin == W.verdict(oracle, x)[1] and cin["gzip_passed"] > 0 and cin["gzip_decoded"] == 0


def test_one_requester_without_accept_gzip_inflates_for_all(sendc, tmp_path, oracle):  # noqa: F811
    """a coalesced send: the receiver that did not opt in would refuse the gzip wire, so nobody gets it"""
    from manatee_b200.host import BackupSender, BackupServer, ZfsClient
    x = sendc["x"]
    p = G.plain(oracle, x)
    env = dict(sendc["env"], **sendc["env_extra"])
    srv = BackupServer.start({"log": None, "port": 0, "host": "127.0.0.1"})
    sender = BackupSender.start({"log": None, "dataset": "zones/x/data/manatee", "zfsPath": sendc["zfs"],
                                 "queue": srv.getQueue(), "env": env, "coalesceMs": 300, "gpu": SENDER})
    outs, results, threads = [], [], []
    for k, recv_gpu in enumerate((RECEIVER, {"mode": "decompress"})):
        e2 = dict(env, FAKE_ZFS_RECV_OUT=str(tmp_path / ("recv%d.out" % k)))
        outs.append(e2["FAKE_ZFS_RECV_OUT"])
        cli = ZfsClient({"log": None, "dataset": "zones/y%d/data/manatee" % k, "dbUser": "postgres",
                         "mountpoint": "/manatee/pg", "pollInterval": 50, "zfsHost": "127.0.0.1",
                         "zfsPath": sendc["zfs"], "zfsPort": _free_port(), "env": e2, "gpu": recv_gpu,
                         "zfsBin": sendc["zfs"], "zfsEnv": e2})
        res = {}
        results.append((res, cli))
        t = threading.Thread(target=cli.restore, args=("http://127.0.0.1:%d" % srv.port,
                                                       lambda err, old, res=res: res.update(err=err)))
        threads.append(t)
        t.start()
    for t in threads:
        t.join(60)
    sender.join(10)
    srv.close()
    want = (hashlib.sha256(p.tobytes()).hexdigest(), p.size)
    for (res, cli), o in zip(results, outs):
        assert res.get("err") is None, res
        assert _digest(o) == want
        job = cli._restoreObject
        assert job["wire"] == "lz4-stage-v1" and job["wireGzip"] is False
        assert job["gpu"]["compressed_in"]["gzip_decoded"] > 0
    assert [a[:2] for a in _sends(sendc["args"])] == [["send", "-c"]]
