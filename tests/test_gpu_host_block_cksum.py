"""GPU: gpu.blockChecksums in the host pipeline on a fake `zfs` (tests/test_host_pipeline.py's
harness).  With the key set, job.gpu / gpuRecv carry a `blocks` object and the restore is byte for
byte what `zfs send` produced; a stream that was corrupted and then re-stamped -- every stream
checksum valid -- fails the job.  Without the key the job object is as before."""
import hashlib
import socket
import threading
import time

import pytest

from test_host_pipeline import _run_restore, fakezfs  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


def test_block_checksums_on_the_compressed_wire(fakezfs):  # noqa: F811
    cfg = {"batchBytes": 4 << 20, "ringBytes": 32 << 20, "outRingBytes": 32 << 20, "blockChecksums": True}
    res, cli, events = _run_restore(fakezfs, sender_gpu=dict(cfg, mode="compress"),
                                    recv_gpu=dict(cfg, mode="decompress"))
    assert res["err"] is None, res
    digest, n = open(fakezfs["recv_out"]).read().split()
    s = fakezfs["stream"]
    assert int(n) == s.size and digest == hashlib.sha256(s.tobytes()).hexdigest()
    job = cli._restoreObject
    assert job["wire"] == "lz4-stage-v1"
    assert job["gpu"]["blocks"]["logical_ok"] == 24 and job["gpuRecv"]["blocks"]["logical_ok"] == 24
    # without the key: no `blocks`
    res, cli, events = _run_restore(fakezfs, sender_gpu={"mode": "verify"}, recv_gpu={"mode": "verify"})
    assert res["err"] is None and "blocks" not in cli._restoreObject["gpu"]
    assert "blocks" not in cli._restoreObject["gpuRecv"]


def test_corrupted_and_restamped_stream_fails_the_job(fakezfs, tmp_path, oracle):  # noqa: F811
    from manatee_b200.host import BackupSender, BackupQueue
    s = fakezfs["stream"].copy()
    _, offs = oracle.stream_index(s)
    s[int(offs[9]) + 312 + 777] ^= 0x20
    assert oracle.stream_restamp(s)[0] == 0 and oracle.stream_verify(s)[0] == 0
    p = tmp_path / "restamped.bin"
    s.tofile(str(p))
    q = BackupQueue({"log": None})
    sender = BackupSender.start({"log": None, "dataset": "zones/x/data/manatee", "zfsPath": fakezfs["zfs"],
                                 "queue": q, "env": dict(fakezfs["env"], FAKE_ZFS_STREAM=str(p)),
                                 "gpu": {"mode": "verify", "batchBytes": 1 << 20, "ringBytes": 8 << 20,
                                         "blockChecksums": True}})
    events = []
    sender.on("err", lambda e: events.append(("err", e)))
    sender.on("done", lambda j: events.append(("done", j)))
    lsock = socket.socket()
    lsock.bind(("127.0.0.1", 0))
    lsock.listen(1)
    got = []

    def receiver():
        c, _ = lsock.accept()
        while True:
            b = c.recv(1 << 16)
            if not b:
                break
            got.append(len(b))
        c.close()
    t = threading.Thread(target=receiver, daemon=True)
    t.start()
    job = {"uuid": "u-1", "host": "127.0.0.1", "port": lsock.getsockname()[1], "dataset": "x", "done": False}
    t0 = time.time()
    q.push(job)
    sender.join(30)
    assert time.time() - t0 < 30, "the sender hung"
    assert job["done"] == "failed" and events and events[0][0] == "err"
    assert "block checksum" in str(events[0][1])
    assert sum(got) <= int(offs[9])                  # nothing of the failing batch was sent
    t.join(5)
    lsock.close()
