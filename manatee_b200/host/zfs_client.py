"""ZfsClient (receive half) -- mirror of lib/zfsClient.js:_receive and helpers.

Reference data path (lib/zfsClient.js:793-794, 823-832):
    zfsRecv = spawn(zfsPath, ['recv', '-v', '-u', dataset])
    server = net.createServer(); server.on('connection', socket.pipe(zfsRecv.stdin))
    server.listen(zfsPort, zfsHost, 1)
Here:  socket -> GpuSnapshotStage(mode) -> zfsRecv.stdin.

Kept: POST {host, port, dataset} to <serverUrl>/backup (:638-668); poll the job
every pollInterval ms, `done === true` ends it, `done === 'failed'` or any HTTP
error is an error, anything else (false, 0) means in progress (:685-754); the last
polled job is kept in _restoreObject for the status server (:722); on any error
the `zfs recv` child is SIGKILLed (:867-876); restore(serverUrl, cb(err, oldDataset)).

Dataset lifecycle around the receive (SURVEY.md 8f f4), same order and same
zfs(1M) invocations as the reference:
    restore()         :115-207  isolateDataset('autorebuild') -> _receive ->
                                canmount=noauto -> mountpoint -> inherit snapdir ->
                                mount -> snapshotDataset; callback(err, oldDataset)
                                (oldDataset is reported on failure too)
    isolateDataset()  :514-624  exists? -> canmount=off -> mounted must be "no" ->
                                inherit mountpoint -> rename -p to
                                <parent>/isolated/<prefix>-<ISO time>
    snapshotDataset() :214-221  <dataset>@<epoch ms>
Additive (never read by the reference): _restoreObject['gpuRecv'] = receiver stage stats
(the sender's are the job's own 'gpu' field).
"""
import datetime
import json
import os
import socket
import subprocess
import threading
import time
import urllib.error
import urllib.request

from . import zfs_cmd

CHUNK = 1 << 20


class ZfsClient(object):
    def __init__(self, options):
        assert isinstance(options, dict), "options (object) is required"
        for k, t in (("dataset", str), ("dbUser", str), ("mountpoint", str), ("pollInterval", int),
                     ("zfsHost", str), ("zfsPath", str), ("zfsPort", int)):
            assert isinstance(options.get(k), t), "options.%s (%s) is required" % (k, t.__name__)
        self._dataset = options["dataset"]
        self._parentDataset = os.path.dirname(self._dataset)      # lib/zfsClient.js:75
        self._mountpoint = options["mountpoint"]
        self._dbUser = options["dbUser"]
        self._pollInterval = options["pollInterval"]
        self._restoreObject = None
        self._zfsHost = options["zfsHost"]
        self._zfsPort = options["zfsPort"]
        self._zfsPath = options["zfsPath"]
        self._gpu = options.get("gpu") or None
        self._env = options.get("env")
        self._gpuStats = None
        # metadata commands: the reference hard-codes /sbin/zfs with an empty environment
        # (lib/common.js:156-157); `zfsBin`/`zfsEnv` exist so tests can point at a fake
        self._zfsBin = options.get("zfsBin") or zfs_cmd.ZFS_BIN
        self._zfsEnv = options.get("zfsEnv") or {}

    def _z(self, **kw):
        kw["zfs"] = self._zfsBin
        kw["env"] = self._zfsEnv
        return kw

    # -- lib/zfsClient.js:115-207
    def restore(self, serverUrl, callback):
        oldDataset = None
        try:
            # move the existing dataset (if any) out of the way, keep its new name
            oldDataset = self.isolateDataset({"prefix": "autorebuild"})
            self._receive(self._dataset, serverUrl, self._pollInterval)
            # manatee mounts/unmounts the dataset itself
            zfs_cmd.zfsSet(self._z(dataset=self._dataset, property="canmount", value="noauto"))
            zfs_cmd.zfsSet(self._z(dataset=self._dataset, property="mountpoint", value=self._mountpoint))
            zfs_cmd.zfsInherit(self._z(dataset=self._dataset, property="snapdir"))
            zfs_cmd.zfsMount(self._z(dataset=self._dataset))
            self.snapshotDataset()
        except Exception as e:                                # noqa: BLE001
            err = RuntimeError('receiving snapshot from "%s": %s' % (serverUrl, e))
            err.__cause__ = e
            return callback(err, oldDataset)
        return callback(None, oldDataset)

    # -- lib/zfsClient.js:214-221
    def snapshotDataset(self):
        zfs_cmd.zfsSnapshot(self._z(dataset=self._dataset, snapshot=str(int(time.time() * 1000))))

    # -- lib/zfsClient.js:514-624 -> isolated name, or None when there was nothing to isolate
    def isolateDataset(self, opts):
        assert isinstance(opts, dict) and isinstance(opts.get("prefix"), str), "opts.prefix (string) is required"
        dataset = self._dataset
        now = datetime.datetime.now(datetime.timezone.utc)
        iso = now.strftime("%Y-%m-%dT%H:%M:%S.") + "%03dZ" % (now.microsecond // 1000)   # Date#toISOString
        isolatedName = "/".join([self._parentDataset, "isolated", opts["prefix"] + "-" + iso])
        try:
            if not zfs_cmd.zfsExists(self._z(dataset=dataset)):
                return None
            # canmount=off implicitly unmounts; fails if the dataset is busy
            zfs_cmd.zfsSet(self._z(dataset=dataset, property="canmount", value="off"))
            value = zfs_cmd.zfsGet(self._z(dataset=dataset, property="mounted"))
            if value != "no":
                raise zfs_cmd.ZfsError('wanted "no" but found "%s" for property "mounted"' % value)
            zfs_cmd.zfsInherit(self._z(dataset=dataset, property="mountpoint"))
            zfs_cmd.zfsRename(self._z(dataset=dataset, target=isolatedName, parents=True))
        except zfs_cmd.ZfsError as e:
            raise zfs_cmd.ZfsError('preserving dataset "%s": %s' % (dataset, e), cause=e)
        return isolatedName

    def _make_stage(self, mode=None):
        if not self._gpu or self._gpu.get("mode", "off") == "off":
            return None
        from ..stage import GpuSnapshotStage
        g = self._gpu
        return GpuSnapshotStage(mode or g["mode"], device=g.get("device", 0),
                                ring_bytes=g.get("ringBytes", 0), batch_bytes=g.get("batchBytes", 0),
                                out_ring_bytes=g.get("outRingBytes", 0), n_slots=g.get("slots", 0),
                                block_checksums=bool(g.get("blockChecksums")),
                                block_sha256=bool(g.get("blockSha256")),
                                block_sha512=bool(g.get("blockSha512")),
                                block_frames=bool(g.get("blockFrames")),
                                block_lzjb=bool(g.get("blockLzjb")),
                                block_logical=bool(g.get("blockLogical")))

    def _wire_mode(self, serverUrl, jobPath):
        """Which stage to put in the pipe for THIS job (SURVEY.md 8f f2).  A receiver configured
        to `decompress` only does so when the sender committed to the stage-compressed wire
        (`job.wire == "lz4-stage-v1"`, set before it connects); a reference sender, or a GPU
        sender that is not compressing, ships a raw stream and the stage just verifies it."""
        mode = self._gpu["mode"]
        if mode != "decompress":
            return mode
        try:
            with urllib.request.urlopen(serverUrl.rstrip("/") + jobPath, timeout=30) as r:
                obj = json.loads(r.read().decode())
        except (urllib.error.URLError, OSError, ValueError):
            obj = {}
        return "decompress" if obj.get("wire") == "lz4-stage-v1" else "verify"

    # -- lib/zfsClient.js:638-668
    def _postRestoreRequest(self, serverUrl):
        req_body = {"host": self._zfsHost, "port": self._zfsPort, "dataset": self._dataset}
        # SURVEY.md 8f f2 (additive): advertise what this receiver's stage can undo.  A
        # reference backupserver ignores unknown fields (lib/backupServer.js:134-146), a
        # reference receiver never sends this, so mixed-version shards stay on the raw wire.
        if self._gpu and self._gpu.get("mode") == "decompress":
            req_body["accept"] = "lz4-stage-v1"
        body = json.dumps(req_body).encode()
        req = urllib.request.Request(serverUrl.rstrip("/") + "/backup", data=body,
                                     headers={"Content-Type": "application/json"})
        try:
            with urllib.request.urlopen(req, timeout=30) as r:
                obj = json.loads(r.read().decode())
        except (urllib.error.URLError, OSError) as e:
            raise RuntimeError("Posting restore request failed: %s" % e)
        return obj.get("jobPath")

    # -- lib/zfsClient.js:685-754
    def _pollRestoreCompletion(self, serverUrl, pollInterval, jobPath, abort):
        while True:
            time.sleep(pollInterval / 1000.0)
            if abort.is_set():
                raise RuntimeError("receive pipe failed")
            try:
                with urllib.request.urlopen(serverUrl.rstrip("/") + jobPath, timeout=30) as r:
                    obj = json.loads(r.read().decode())
            except urllib.error.HTTPError as e:
                raise RuntimeError("error getting restore job status: %d %s" % (e.code, e.read().decode()))
            except (urllib.error.URLError, OSError) as e:
                raise RuntimeError("error getting restore job status: %s" % e)
            self._restoreObject = obj
            if obj.get("done") is True:
                return obj
            if obj.get("done") == "failed":
                raise RuntimeError("restore job failed")

    # -- lib/zfsClient.js:765-886
    def _receive(self, dataset, serverUrl, pollInterval):
        zfsRecv = subprocess.Popen([self._zfsPath, "recv", "-v", "-u", dataset],
                                   stdin=subprocess.PIPE, stdout=subprocess.PIPE,
                                   stderr=subprocess.PIPE, env=self._env)
        server = socket.socket(socket.AF_INET, socket.SOCK_STREAM)
        server.setsockopt(socket.SOL_SOCKET, socket.SO_REUSEADDR, 1)
        abort = threading.Event()
        pipe_err = []
        stage_box = []
        job_box = []
        posted = threading.Event()

        def serve():
            conn = None
            stage = None
            try:
                conn, _ = server.accept()
                if self._gpu and self._gpu.get("mode", "off") != "off":
                    # the sender connects only after our POST was queued; wait for its answer
                    if not posted.wait(30):
                        raise RuntimeError("no jobPath for the incoming connection")
                    stage = self._make_stage(self._wire_mode(serverUrl, job_box[0]))
                stage_box.append(stage)
                if stage is None:
                    while True:                               # socket.pipe(zfsRecv.stdin)
                        buf = conn.recv(CHUNK)
                        if not buf:
                            break
                        zfsRecv.stdin.write(buf)
                else:
                    def drain():
                        try:
                            while True:
                                b = stage.read(CHUNK)
                                if b is None:
                                    break
                                zfsRecv.stdin.write(b)
                        except Exception as e:                # noqa: BLE001
                            pipe_err.append(e)
                    td = threading.Thread(target=drain, daemon=True)
                    td.start()
                    try:
                        while True:
                            buf = conn.recv(CHUNK)
                            if not buf:
                                break
                            stage.write(buf)
                        stage.flush()
                    except Exception as e:                    # noqa: BLE001
                        pipe_err.append(e)
                    td.join()
                zfsRecv.stdin.close()
            except Exception as e:                            # noqa: BLE001
                pipe_err.append(e)
            finally:
                if pipe_err:
                    abort.set()
                if stage is not None:
                    self._gpuStats = stage.stats()
                    if self._gpu.get("blockChecksums"):
                        self._gpuStats["blocks"] = stage.block_stats()
                    stage.close()
                if conn is not None:
                    conn.close()

        try:
            server.bind((self._zfsHost, self._zfsPort))
            server.listen(1)                                  # backlog 1, lib/zfsClient.js:832
            ts = threading.Thread(target=serve, daemon=True)
            ts.start()
            jobPath = self._postRestoreRequest(serverUrl)
            job_box.append(jobPath)
            posted.set()
            self._pollRestoreCompletion(serverUrl, pollInterval, jobPath, abort)
            ts.join(60)
            if self._gpuStats is not None and isinstance(self._restoreObject, dict):
                self._restoreObject["gpuRecv"] = self._gpuStats   # additive field (SURVEY 8f f4)
            if pipe_err:
                raise pipe_err[0]
            code = zfsRecv.wait(60)
            if code != 0:
                raise RuntimeError("zfs recv: %s %d" % (zfsRecv.stderr.read().decode(errors="replace"), code))
        except Exception:
            try:
                zfsRecv.kill()                                # SIGKILL, lib/zfsClient.js:873
            except OSError:
                pass
            raise
        finally:
            try:
                server.close()
            except OSError:
                pass
