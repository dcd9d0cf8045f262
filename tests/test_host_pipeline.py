"""Host logic of the peer-bootstrap path (mirror of lib/backupServer.js,
lib/backupQueue.js, lib/backupSender.js, lib/zfsClient.js) with a fake `zfs`
selected through the reference's own zfsPath knob.  CPU tests run the legacy
identity pipe (gpu off == reference behaviour); the gpu-marked ones put the stage
in the pipe: VERIFY on both sides, and COMPRESS on the sender / DECOMPRESS on the
receiver with transport identity end to end."""
import hashlib
import json
import os
import socket
import stat
import sys
import threading
import time
import urllib.error
import urllib.request

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.fixture()
def fakezfs(tmp_path, oracle):
    """dir with an executable `zfs`, a seeded stream file and the env to use them"""
    z = tmp_path / "bin"
    z.mkdir()
    zfs = z / "zfs"
    zfs.write_text("#!/bin/sh\nexec %s %s \"$@\"\n" % (sys.executable, os.path.join(ROOT, "tools", "fake_zfs.py")))
    zfs.chmod(zfs.stat().st_mode | stat.S_IEXEC)
    stream = oracle.synth_stream(24, recsize=131072, kind=oracle.PAYLOAD_PGPAGE)
    sp = tmp_path / "stream.bin"
    stream.tofile(str(sp))
    env = dict(os.environ)
    env["PATH"] = str(z) + os.pathsep + env.get("PATH", "")
    env["FAKE_ZFS_STREAM"] = str(sp)
    env["FAKE_ZFS_RECV_OUT"] = str(tmp_path / "recv.out")
    env["FAKE_ZFS_STATE"] = str(tmp_path / "pool.json")      # dataset lifecycle model (8f f3/f4)
    return {"zfs": str(zfs), "env": env, "stream": stream, "recv_out": str(tmp_path / "recv.out"),
            "state": str(tmp_path / "pool.json")}


def _run_restore(fakezfs, sender_gpu=None, recv_gpu=None, env_extra=None):
    from manatee_b200.host import BackupSender, BackupServer, ZfsClient
    env = dict(fakezfs["env"])
    env.update(env_extra or {})
    srv = BackupServer.start({"log": None, "port": 0, "host": "127.0.0.1"})
    sender = BackupSender.start({"log": None, "dataset": "zones/x/data/manatee", "zfsPath": fakezfs["zfs"],
                                 "queue": srv.getQueue(), "gpu": sender_gpu, "env": env})
    events = []
    sender.on("err", lambda e: events.append(("err", e)))
    sender.on("done", lambda j: events.append(("done", j)))
    cli = ZfsClient({"log": None, "dataset": "zones/y/data/manatee", "dbUser": "postgres",
                     "mountpoint": "/manatee/pg", "pollInterval": 50, "zfsHost": "127.0.0.1",
                     "zfsPath": fakezfs["zfs"], "zfsPort": _free_port(), "gpu": recv_gpu, "env": env,
                     "zfsBin": fakezfs["zfs"], "zfsEnv": env})
    res = {}
    cli.restore("http://127.0.0.1:%d" % srv.port, lambda err, old: res.update(err=err, old=old))
    sender.join(10)
    srv.close()
    return res, cli, events


def test_rest_surface(fakezfs):
    from manatee_b200.host import BackupServer
    srv = BackupServer.start({"log": None, "port": 0, "host": "127.0.0.1"})
    base = "http://127.0.0.1:%d" % srv.port
    try:
        pushed = []
        srv.getQueue().on("push", pushed.append)
        req = urllib.request.Request(base + "/backup/", data=json.dumps(
            {"host": "10.0.0.9", "port": 1234, "dataset": "zones/a/b"}).encode(),
            headers={"Content-Type": "application/json"})
        obj = json.loads(urllib.request.urlopen(req).read())
        assert set(obj) == {"jobid", "jobPath"} and obj["jobPath"] == "/backup/" + obj["jobid"]
        time.sleep(0.05)
        assert pushed and pushed[0]["done"] is False and pushed[0]["dataset"] == "zones/a/b"
        job = json.loads(urllib.request.urlopen(base + obj["jobPath"]).read())
        assert job["uuid"] == obj["jobid"] and job["host"] == "10.0.0.9" and job["port"] == 1234
        # missing parameter -> 409 MissingParameter (lib/backupServer.js:135-138)
        bad = urllib.request.Request(base + "/backup/", data=json.dumps({"host": "h", "port": 1}).encode(),
                                     headers={"Content-Type": "application/json"})
        with pytest.raises(urllib.error.HTTPError) as ei:
            urllib.request.urlopen(bad)
        assert ei.value.code == 409 and json.loads(ei.value.read())["code"] == "MissingParameter"
        with pytest.raises(urllib.error.HTTPError) as ei:
            urllib.request.urlopen(base + "/backup/00000000-0000-0000-0000-000000000000")
        assert ei.value.code == 404
        # job.err -> 500 InternalError; the sender mutates the same object the server serialises
        pushed[0]["err"] = RuntimeError("zfs send: boom 1")
        with pytest.raises(urllib.error.HTTPError) as ei:
            urllib.request.urlopen(base + obj["jobPath"])
        assert ei.value.code == 500 and "boom" in json.loads(ei.value.read())["message"]
    finally:
        srv.close()


def test_queue_never_evicts():
    from manatee_b200.host import BackupQueue
    q = BackupQueue({"log": None})
    seen = []
    q.on("push", seen.append)
    for i in range(3):
        q.push({"uuid": "u%d" % i})
    assert [j["uuid"] for j in seen] == ["u0", "u1", "u2"]
    assert q.get("u1", lambda j: j)["uuid"] == "u1"
    assert q.get("nope", lambda j: j) is None
    assert q.get("u0", lambda j: j) is not None          # still there: pop() is never called


def test_legacy_identity_pipe_end_to_end(fakezfs):
    """gpu off == the reference: bytes into `zfs recv` == bytes out of `zfs send`."""
    res, cli, events = _run_restore(fakezfs)
    assert res["err"] is None, res
    digest, n = open(fakezfs["recv_out"]).read().split()
    s = fakezfs["stream"]
    assert int(n) == s.size and digest == hashlib.sha256(s.tobytes()).hexdigest()
    job = cli._restoreObject
    assert job["done"] is True
    assert job["size"] == str(s.size) and job["completed"] == str(s.size)     # strings, like the regex captures
    assert events and events[0][0] == "done"


def test_latest_snapshot_selection_and_failures(fakezfs):
    from manatee_b200.host import BackupQueue, BackupSender
    snd = BackupSender.start({"log": None, "dataset": "zones/x/data/manatee", "zfsPath": fakezfs["zfs"],
                              "queue": BackupQueue({}), "env": fakezfs["env"]})
    assert snd._getLatestSnapshot() == "zones/x/data/manatee@1405378955344"   # 13 digits, operator snapshot skipped
    env = dict(fakezfs["env"]); env["FAKE_ZFS_NO_SNAPSHOTS"] = "1"
    snd2 = BackupSender.start({"log": None, "dataset": "d", "zfsPath": fakezfs["zfs"],
                               "queue": BackupQueue({}), "env": env})
    with pytest.raises(RuntimeError, match="no snapshots found"):
        snd2._getLatestSnapshot()
    # zfs send exiting non-zero => job.done == 'failed', 'err' event, receiver errors out
    res, cli, events = _run_restore(fakezfs, env_extra={"FAKE_ZFS_SEND_FAIL_AT": str(3 << 20)})
    assert res["err"] is not None
    assert events and events[0][0] == "err"


@pytest.mark.gpu
def test_gpu_verify_stage_in_both_pipes(fakezfs):
    res, cli, events = _run_restore(fakezfs, sender_gpu={"mode": "verify", "batchBytes": 2 << 20, "ringBytes": 16 << 20},
                                    recv_gpu={"mode": "verify", "batchBytes": 2 << 20, "ringBytes": 16 << 20})
    assert res["err"] is None, res
    digest, n = open(fakezfs["recv_out"]).read().split()
    s = fakezfs["stream"]
    assert int(n) == s.size and digest == hashlib.sha256(s.tobytes()).hexdigest()
    assert cli._restoreObject["done"] is True
    nrec = 3 + 24                                        # BEGIN, OBJECT, 24 x WRITE, END
    assert cli._restoreObject["gpu"]["records"] == nrec and cli._gpuStats["records"] == nrec


@pytest.mark.gpu
def test_gpu_compress_on_the_wire_identity_at_zfs_recv(fakezfs):
    """COMPRESS in the sender, DECOMPRESS in the receiver: fewer bytes on the TCP leg,
    `zfs recv` sees exactly the bytes `zfs send` produced."""
    cfg = {"batchBytes": 4 << 20, "ringBytes": 32 << 20, "outRingBytes": 32 << 20}
    res, cli, events = _run_restore(fakezfs, sender_gpu=dict(cfg, mode="compress"),
                                    recv_gpu=dict(cfg, mode="decompress"))
    assert res["err"] is None, res
    digest, n = open(fakezfs["recv_out"]).read().split()
    s = fakezfs["stream"]
    assert int(n) == s.size and digest == hashlib.sha256(s.tobytes()).hexdigest()
    g = cli._restoreObject["gpu"]
    assert g["lz4_encoded"] == 24 and g["bytes_out"] < g["bytes_in"] // 2
    assert cli._gpuStats["lz4_decoded"] == 24


@pytest.mark.gpu
def test_gpu_corrupt_stream_fails_the_job(fakezfs, tmp_path):
    s = fakezfs["stream"].copy()
    s[2_000_000] ^= 1
    p = tmp_path / "bad.bin"
    s.tofile(str(p))
    res, cli, events = _run_restore(fakezfs, sender_gpu={"mode": "verify", "batchBytes": 1 << 20, "ringBytes": 8 << 20},
                                    env_extra={"FAKE_ZFS_STREAM": str(p)})
    assert res["err"] is not None                    # receiver's poll sees done == 'failed' / 500
    assert events and events[0][0] == "err" and "checksum" in str(events[0][1])


def _big_stream(oracle, tmp_path, nwrites=96, corrupt_at=None):
    """a stream several times larger than the pipe + the rings the failure tests configure"""
    s = oracle.synth_stream(nwrites, recsize=131072, kind=oracle.PAYLOAD_PCG).copy()
    if corrupt_at is not None:
        s[corrupt_at] ^= 0x04
    p = tmp_path / "big.bin"
    s.tofile(str(p))
    return s, str(p)


@pytest.mark.gpu
def test_gpu_corruption_in_the_first_batch_does_not_hang_the_sender(fakezfs, tmp_path, oracle):
    """ADVICE r1 (high, a): the stage fails on the FIRST batch while `zfs send` still has megabytes
    to write.  The sender must kill the child instead of wait()ing on it forever: job.done ==
    'failed', 'err' emitted, and the restore returns within seconds."""
    s, path = _big_stream(oracle, tmp_path, corrupt_at=400_000)
    t0 = time.time()
    res, cli, events = _run_restore(fakezfs, sender_gpu={"mode": "verify", "batchBytes": 1 << 20, "ringBytes": 2 << 20},
                                    env_extra={"FAKE_ZFS_STREAM": path})
    assert time.time() - t0 < 30
    assert res["err"] is not None
    assert events and events[0][0] == "err" and "checksum" in str(events[0][1])
    assert cli._restoreObject is None or cli._restoreObject.get("done") in ("failed", 0, False)


@pytest.mark.gpu
def test_gpu_receiver_disconnect_mid_transfer_fails_the_job(fakezfs, tmp_path, oracle):
    """ADVICE r1 (high, b): the receiver closes its socket mid-transfer.  The drain thread's send
    error must cancel the stage so that the producer blocked on the full ring wakes up, the child
    is killed and the job ends 'failed' -- not a writer spinning in mtz_write forever."""
    from manatee_b200.host import BackupSender, BackupQueue
    s, path = _big_stream(oracle, tmp_path)
    env = dict(fakezfs["env"], FAKE_ZFS_STREAM=path)
    q = BackupQueue({"log": None})
    sender = BackupSender.start({"log": None, "dataset": "zones/x/data/manatee", "zfsPath": fakezfs["zfs"],
                                 "queue": q, "env": env,
                                 "gpu": {"mode": "verify", "batchBytes": 1 << 20, "ringBytes": 2 << 20}})
    events = []
    sender.on("err", lambda e: events.append(("err", e)))
    sender.on("done", lambda j: events.append(("done", j)))
    lsock = socket.socket()
    lsock.bind(("127.0.0.1", 0))
    lsock.listen(1)

    def rude_receiver():
        c, _ = lsock.accept()
        got = 0
        while got < (1 << 20):                       # take the first MiB, then hang up
            b = c.recv(1 << 16)
            if not b:
                break
            got += len(b)
        c.setsockopt(socket.SOL_SOCKET, socket.SO_LINGER, b"\x01\x00\x00\x00\x00\x00\x00\x00")
        c.close()
    t = threading.Thread(target=rude_receiver, daemon=True)
    t.start()
    job = {"uuid": "u-1", "host": "127.0.0.1", "port": lsock.getsockname()[1], "dataset": "x", "done": False}
    t0 = time.time()
    q.push(job)
    sender.join(30)
    assert time.time() - t0 < 30, "the sender hung"
    assert job["done"] == "failed" and events and events[0][0] == "err"
    lsock.close()


def test_coalesced_restores_share_one_send(fakezfs, tmp_path):
    """SURVEY.md 8f f1: two peers asking within the window get the same bytes from ONE
    `zfs send` (the reference would run two).  Default (coalesceMs absent) stays per-job."""
    _coalesced(fakezfs, tmp_path, None, None)


@pytest.mark.gpu
def test_gpu_coalesced_restores_fan_out_of_one_stage_pass(fakezfs, tmp_path):
    """f1 joined to the library's fan-out: the coalesced sender runs ONE zfs send through ONE stage
    (COMPRESS on the wire) with both requesters attached as fan-out peers (mtz_fanout_attach: one
    pinned ring per peer); each receiver decompresses and hands `zfs recv` the original bytes."""
    results = _coalesced(fakezfs, tmp_path, {"mode": "compress", "batchBytes": 1 << 20, "ringBytes": 4 << 20,
                                             "outRingBytes": 2 << 20}, {"mode": "decompress"})
    for res, cli in results:
        job = cli._restoreObject
        assert job["wire"] == "lz4-stage-v1" and job["gpu"]["lz4_encoded"] > 0
        assert job["gpuRecv"]["lz4_decoded"] == job["gpu"]["lz4_encoded"]


def _coalesced(fakezfs, tmp_path, sender_gpu, recv_gpu):
    from manatee_b200.host import BackupSender, BackupServer, ZfsClient
    env = dict(fakezfs["env"])
    counter = tmp_path / "sends"
    env["FAKE_ZFS_SEND_COUNT"] = str(counter)
    srv = BackupServer.start({"log": None, "port": 0, "host": "127.0.0.1"})
    sender = BackupSender.start({"log": None, "dataset": "zones/x/data/manatee", "zfsPath": fakezfs["zfs"],
                                 "queue": srv.getQueue(), "env": env, "coalesceMs": 300, "gpu": sender_gpu})
    outs, results, threads = [], [], []
    for k in range(2):
        e2 = dict(env); e2["FAKE_ZFS_RECV_OUT"] = str(tmp_path / ("recv%d.out" % k))
        outs.append(e2["FAKE_ZFS_RECV_OUT"])
        cli = ZfsClient({"log": None, "dataset": "zones/y%d/data/manatee" % k, "dbUser": "postgres",
                         "mountpoint": "/manatee/pg", "pollInterval": 50, "zfsHost": "127.0.0.1",
                         "zfsPath": fakezfs["zfs"], "zfsPort": _free_port(), "env": e2, "gpu": recv_gpu,
                         "zfsBin": fakezfs["zfs"], "zfsEnv": e2})
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
    want = hashlib.sha256(fakezfs["stream"].tobytes()).hexdigest()
    for (res, cli), o in zip(results, outs):
        assert res.get("err") is None, res
        digest, n = open(o).read().split()
        assert digest == want and int(n) == fakezfs["stream"].size
        assert cli._restoreObject["done"] is True
    assert open(str(counter)).read().count("send") == 1, "coalesced requests must share one zfs send"
    return results


class _IdentityStageDouble(object):
    """TEST DOUBLE with GpuSnapshotStage's streaming surface (write/flush/read/stats/close).
    It only lets the CPU suite walk the host threading around a stage (drain threads, job
    fields, negotiation); the product has no such thing -- the real stage needs an H100."""
    made = []

    def __init__(self, mode="verify", **kw):
        import collections
        self.mode, self.q, self.cv, self.eof, self.n = mode, collections.deque(), threading.Condition(), False, 0
        _IdentityStageDouble.made.append(self)

    def write(self, chunk, block=True):
        with self.cv:
            self.q.append(bytes(chunk)); self.n += len(chunk); self.cv.notify_all()

    def flush(self):
        with self.cv:
            self.eof = True; self.cv.notify_all()

    def read(self, cap=1 << 20, block=True):
        with self.cv:
            while not self.q and not self.eof:
                self.cv.wait(0.05)
            if self.q:
                b = self.q.popleft()
                if len(b) > cap:
                    self.q.appendleft(b[cap:]); b = b[:cap]
                return b
            return None

    def stats(self):
        return {"bytes_in": self.n, "bytes_out": self.n, "lz4_encoded": 0, "mode": self.mode}

    def close(self):
        pass


def test_host_threading_around_a_stage_cpu(fakezfs, monkeypatch):
    """The host code paths the gpu-marked tests take (stage in both pipes, job.gpu / gpuRecv,
    wire negotiation, a second restore isolating the first one's dataset), with the stage
    replaced by an identity double so that they also run where there is no GPU."""
    import manatee_b200.stage as stage_mod
    monkeypatch.setattr(stage_mod, "GpuSnapshotStage", _IdentityStageDouble)
    _IdentityStageDouble.made = []
    s = fakezfs["stream"]
    want = hashlib.sha256(s.tobytes()).hexdigest()
    res, cli, events = _run_restore(fakezfs, sender_gpu={"mode": "verify"}, recv_gpu={"mode": "verify"})
    assert res["err"] is None and res["old"] is None, res
    digest, n = open(fakezfs["recv_out"]).read().split()
    assert digest == want and int(n) == s.size
    assert [m.mode for m in _IdentityStageDouble.made] == ["verify", "verify"]
    job = cli._restoreObject
    assert job["done"] is True and job["wire"] == "raw"
    assert job["gpu"]["bytes_in"] == s.size and job["gpuRecv"]["bytes_out"] == s.size
    assert events and events[-1][0] == "done"
    # compress sender + plain receiver -> the sender's stage is opened in verify mode
    _IdentityStageDouble.made = []
    res, cli, events = _run_restore(fakezfs, sender_gpu={"mode": "compress"}, recv_gpu=None)
    assert res["err"] is None and res["old"].startswith("zones/y/data/isolated/autorebuild-")
    assert [m.mode for m in _IdentityStageDouble.made] == ["verify"] and cli._restoreObject["wire"] == "raw"
    assert "gpuRecv" not in cli._restoreObject
    # negotiated
    _IdentityStageDouble.made = []
    res, cli, events = _run_restore(fakezfs, sender_gpu={"mode": "compress"}, recv_gpu={"mode": "decompress"})
    assert res["err"] is None
    assert sorted(m.mode for m in _IdentityStageDouble.made) == ["compress", "decompress"]
    assert cli._restoreObject["wire"] == "lz4-stage-v1"
    # mixed versions, the other way round: a reference sender (no stage, no `wire` field) and a
    # receiver configured to decompress -> the raw stream is verified, not rejected
    _IdentityStageDouble.made = []
    res, cli, events = _run_restore(fakezfs, sender_gpu=None, recv_gpu={"mode": "decompress"})
    assert res["err"] is None, res
    assert [m.mode for m in _IdentityStageDouble.made] == ["verify"]
    assert "wire" not in cli._restoreObject and cli._restoreObject["gpuRecv"]["bytes_in"] == s.size
    # a verifying (non-compressing) GPU sender and a decompress receiver
    _IdentityStageDouble.made = []
    res, cli, events = _run_restore(fakezfs, sender_gpu={"mode": "verify"}, recv_gpu={"mode": "decompress"})
    assert res["err"] is None and cli._restoreObject["wire"] == "raw"
    assert [m.mode for m in _IdentityStageDouble.made] == ["verify", "verify"]


@pytest.mark.gpu
def test_gpu_sender_compress_falls_back_for_plain_receiver(fakezfs):
    """Mixed versions (f2): a receiver that did not ask for the compressed wire gets the raw,
    verified stream even from a sender configured to compress."""
    cfg = {"batchBytes": 4 << 20, "ringBytes": 32 << 20, "outRingBytes": 32 << 20}
    res, cli, events = _run_restore(fakezfs, sender_gpu=dict(cfg, mode="compress"), recv_gpu=None)
    assert res["err"] is None, res
    digest, n = open(fakezfs["recv_out"]).read().split()
    s = fakezfs["stream"]
    assert int(n) == s.size and digest == hashlib.sha256(s.tobytes()).hexdigest()
    assert cli._restoreObject["wire"] == "raw" and cli._restoreObject["gpu"]["lz4_encoded"] == 0
    # and the negotiated case advertises it in the job object
    res, cli, events = _run_restore(fakezfs, sender_gpu=dict(cfg, mode="compress"),
                                    recv_gpu=dict(cfg, mode="decompress"))
    assert res["err"] is None and cli._restoreObject["wire"] == "lz4-stage-v1"


@pytest.mark.gpu
def test_gpu_decompress_receiver_with_reference_sender(fakezfs):
    """Mixed versions (f2), other direction: the sender is the reference (identity pipe, no
    `wire` in the job); a receiver configured to decompress must verify the raw stream and
    hand it to zfs recv unchanged instead of failing on the missing stage marker."""
    cfg = {"batchBytes": 4 << 20, "ringBytes": 32 << 20, "outRingBytes": 32 << 20}
    res, cli, events = _run_restore(fakezfs, sender_gpu=None, recv_gpu=dict(cfg, mode="decompress"))
    assert res["err"] is None, res
    digest, n = open(fakezfs["recv_out"]).read().split()
    s = fakezfs["stream"]
    assert int(n) == s.size and digest == hashlib.sha256(s.tobytes()).hexdigest()
    assert "wire" not in cli._restoreObject
    assert cli._restoreObject["gpuRecv"]["lz4_decoded"] == 0 and cli._restoreObject["gpuRecv"]["records"] > 0


@pytest.mark.gpu
def test_verify_process_host_copy_out(oracle):
    """VERIFY with a separate output buffer: the bytes come back from HBM (D2H), identical."""
    from manatee_b200 import GpuSnapshotStage
    s = oracle.synth_stream(20, recsize=65536, kind=oracle.PAYLOAD_PCG)
    out = np.zeros(s.size + 100, dtype=np.uint8)
    with GpuSnapshotStage("verify", batch_bytes=1 << 20) as g:
        n = g.process_host(s, out)
        assert n == s.size and np.array_equal(out[:n], s)
