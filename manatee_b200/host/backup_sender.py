"""BackupSender -- mirror of lib/backupSender.js with the GPU stage in the pipe.

Reference data path (lib/backupSender.js:172-179):
    socket = net.connect(job.port, job.host)
    zfsSend = spawn(zfsPath, ['send', '-v', '-P', snapshot])
    zfsSend.stdout.pipe(socket)
Here:  zfsSend.stdout -> GpuSnapshotStage(mode) -> socket   (gpu cfg absent/off:
the legacy identity pipe, byte for byte).

Kept verbatim: one _send per 'push' (no coalescing, :72-73); job.done goes
false -> 0 -> True | 'failed' (:196, :218, :224); job.size / job.completed are the
decimal STRINGS captured by the two stderr regexes (:125, :136, :197-212); a
failure emits 'err' (not 'error') and sets job.err (:74-88); the POSTed `dataset`
is ignored, the sender ships its own configured dataset (:66, :253);
_getLatestSnapshot takes the first name matching /^\\d{13}$/ from
`zfs list -t snapshot -H -d 1 -S name -o name <ds>` (:244-288).
Not replicated: the crash when the socket errors before 'connect'
(zfsSend undefined, :230-233) -- guarded instead.
"""
import re
import socket
import subprocess
import threading

from .backup_queue import BackupQueue

ZFS_PROGRESS_HEADER = re.compile(r"^full\s+\S+\s+(\d+)\n.*\n*$")
ZFS_PROGRESS_REGEX = re.compile(r"^\d\d:\d\d:\d\d\t(\d+)\t\S+\n$")
CHUNK = 1 << 20


class BackupSender(object):
    def __init__(self, options):
        assert isinstance(options, dict), "options (object) is required"
        assert isinstance(options.get("dataset"), str), "options.dataset (string) is required"
        assert isinstance(options.get("queue"), BackupQueue), "options.queue (object) is required"
        assert isinstance(options.get("zfsPath"), str), "options.zfsPath (string) is required"
        self._zfsPath = options["zfsPath"]
        self._dataset = options["dataset"]
        self._queue = options["queue"]
        self._gpu = options.get("gpu") or None     # {'mode': 'verify'|'compress', 'device': 0, ...}
        self._env = options.get("env")
        # SURVEY.md 8f f1 (additive, default off == reference behaviour): requests that
        # arrive within coalesceMs of each other share ONE zfs send + ONE stage pass,
        # the processed stream is teed to every requester's socket.
        self._coalesceMs = int(options.get("coalesceMs", 0) or 0)
        self._pending = []
        self._pend_lock = threading.Lock()
        self._listeners = {}
        self._threads = []
        self._queue.on("push", self._on_push)

    @staticmethod
    def start(cfg):
        return BackupSender(cfg)

    def on(self, event, fn):
        self._listeners.setdefault(event, []).append(fn)
        return self

    def emit(self, event, *args):
        for fn in list(self._listeners.get(event, [])):
            fn(*args)

    def join(self, timeout=None):
        for t in list(self._threads):
            t.join(timeout)

    def _job_cb(self, backupJob):
        def cb(err):
            if err:
                backupJob["err"] = err
                self.emit("err", err)
            else:
                self.emit("done", backupJob)
        return cb

    def _on_push(self, backupJob):
        if self._coalesceMs <= 0:
            t = threading.Thread(target=self._send, args=(backupJob, self._job_cb(backupJob)),
                                 daemon=True)
            self._threads.append(t)
            t.start()
            return
        with self._pend_lock:
            self._pending.append(backupJob)
            first = len(self._pending) == 1
        if first:
            def fire():
                import time
                time.sleep(self._coalesceMs / 1000.0)
                with self._pend_lock:
                    jobs, self._pending = self._pending, []
                self._send_group(jobs)
            t = threading.Thread(target=fire, daemon=True)
            self._threads.append(t)
            t.start()

    # -- lib/backupSender.js:244-288
    def _getLatestSnapshot(self):
        cmd = "zfs list -t snapshot -H -d 1 -S name -o name " + self._dataset
        p = subprocess.run(cmd, shell=True, capture_output=True, text=True, env=self._env)
        if p.returncode != 0:
            raise RuntimeError("Command failed: %s\n%s" % (cmd, p.stderr))
        for line in p.stdout.split("\n"):
            parts = line.split("@")
            if len(parts) > 1 and re.match(r"^\d{13}$", parts[1]):
                return line
        raise RuntimeError("no snapshots found")

    def _decide_wire(self, jobs):
        """Capability negotiation (SURVEY.md 8f f2), settled BEFORE any socket is opened so a
        receiver that looks at the job on connect sees it: the stage-compressed wire is used
        only when this sender compresses AND every requester of this send advertised
        `accept: "lz4-stage-v1"`; everybody else gets the raw (verified) stream.  With the gpu
        stage off the job object is left exactly as the reference has it (no `wire` field).
        On the stage wire with gpu.sendCompressed, `wireGzip` says whether gzip records travel as
        their disk frames (MTZ_FLAG_GZIP_WIRE): only when every requester also advertised
        `acceptGzip: true`, since the receiver's stage then inflates them.  With gpu.gzipEncode the
        same condition, with or without gpu.sendCompressed, also makes COMPRESS deflate the records it
        encodes (MTZ_FLAG_GZIP_ENCODE)."""
        if not self._gpu or self._gpu.get("mode", "off") == "off":
            return
        compress = self._gpu["mode"] == "compress" and \
            all(j.get("accept") == "lz4-stage-v1" for j in jobs)
        gzip_capable = bool(self._gpu.get("sendCompressed") or self._gpu.get("gzipEncode"))
        gzip_wire = compress and gzip_capable and all(j.get("acceptGzip") is True for j in jobs)
        for j in jobs:
            j["wire"] = "lz4-stage-v1" if compress else "raw"
            if compress and gzip_capable:
                j["wireGzip"] = gzip_wire

    def _send_compressed(self, backupJob):
        """`zfs send -c` for this job: gpu.sendCompressed is set and _decide_wire chose the stage wire"""
        return bool(self._gpu and self._gpu.get("mode") == "compress" and self._gpu.get("sendCompressed")
                    and backupJob is not None and backupJob.get("wire") == "lz4-stage-v1")

    def _make_stage(self, backupJob=None):
        if not self._gpu or self._gpu.get("mode", "off") == "off":
            return None
        from ..stage import GpuSnapshotStage          # the product: fails loudly without the .so/GPU
        g = dict(self._gpu)
        if g["mode"] == "compress" and (backupJob is None or backupJob.get("wire") != "lz4-stage-v1"):
            g["mode"] = "verify"
        return GpuSnapshotStage(g["mode"], device=g.get("device", 0), devices=g.get("devices"),
                                ring_bytes=g.get("ringBytes", 0), batch_bytes=g.get("batchBytes", 0),
                                out_ring_bytes=g.get("outRingBytes", 0), n_slots=g.get("slots", 0),
                                block_checksums=bool(g.get("blockChecksums")),
                                block_sha256=bool(g.get("blockSha256")),
                                block_sha512=bool(g.get("blockSha512")),
                                block_frames=bool(g.get("blockFrames")),
                                block_lzjb=bool(g.get("blockLzjb")),
                                block_logical=bool(g.get("blockLogical")),
                                lz4_hc=bool(g.get("lz4Hc")),
                                compressed_input=self._send_compressed(backupJob),
                                gzip_input=self._send_compressed(backupJob) and bool(g.get("sendGzip"))
                                and not backupJob.get("wireGzip"),
                                gzip_wire=self._send_compressed(backupJob) and bool(backupJob.get("wireGzip")),
                                gzip_encode=g["mode"] == "compress" and bool(g.get("gzipEncode"))
                                and bool(backupJob.get("wireGzip")))

    def _stage_stats(self, stage):
        """job.gpu: the stage counters, plus `blocks` (block-checksum counters) with
        gpu.blockChecksums set and `compressed_in` (mtz_get_compressed_in_stats) with gpu.sendCompressed,
        gzip_decoded included with gpu.sendGzip, gzip_passed on a `wireGzip` job; with gpu.gzipEncode
        `compressed_in` too, gzip_encoded included on a `wireGzip` job"""
        st = stage.stats()
        if self._gpu.get("blockChecksums"):
            st["blocks"] = stage.block_stats()
        if self._gpu.get("sendCompressed") or self._gpu.get("gzipEncode"):
            st["compressed_in"] = stage.compressed_in_stats()
        return st

    def _send_group(self, jobs):
        """One zfs send + one stage pass teed to every job's socket (coalesced restore)."""
        class Tee(object):
            def __init__(self, socks):
                self.socks = socks

            def sendall(self, b):
                for j, s_ in list(self.socks.items()):
                    try:
                        s_.sendall(b)
                    except OSError as e:
                        jobs_by_id[j]["done"] = "failed"
                        self_cb[j](e)
                        del self.socks[j]
                if not self.socks:
                    raise OSError("every coalesced receiver went away")

            def shutdown(self, how):
                for s_ in self.socks.values():
                    try:
                        s_.shutdown(how)
                    except OSError:
                        pass

            def close(self):
                for s_ in self.socks.values():
                    s_.close()

        jobs_by_id = {id(j): j for j in jobs}
        self_cb = {id(j): self._job_cb(j) for j in jobs}
        self._decide_wire(jobs)
        socks = {}
        for j in jobs:
            try:
                socks[id(j)] = socket.create_connection((j["host"], int(j["port"])))
            except OSError as e:
                j["done"] = "failed"
                self_cb[id(j)](e)
        if not socks:
            return
        live = [jobs_by_id[k] for k in socks]
        lead = dict(live[0])                       # progress fields are mirrored to every job

        class Shared(dict):
            def __setitem__(self_, k, v):
                dict.__setitem__(self_, k, v)
                for j in live:
                    if j.get("done") != "failed" or k != "done":
                        j[k] = v
        shared = Shared(lead)

        def cb(err):
            for j in live:
                if j.get("done") == "failed" and not err:
                    continue
                self_cb[id(j)](err)
        if self._gpu and self._gpu.get("mode", "off") != "off":
            # ONE zfs send, ONE pass of the stage, every requester attached as a fan-out peer of
            # the library (mtz_fanout_attach): each peer drains its own pinned ring, fed from
            # its egress GPU -- the NCCL broadcast replaces N independent sends
            # (lib/backupSender.js:72-73).  A peer whose socket dies keeps being drained (and
            # discarded) so that it never back-pressures the others.
            def peer_failed(k, e):
                j = jobs_by_id[k]
                j["done"] = "failed"
                self_cb[k](e)
            self._send(shared, cb, sock=None, peer_socks=[(k, socks[k]) for k in socks],
                       peer_failed=peer_failed)
        else:
            self._send(shared, cb, sock=Tee(socks))

    # -- lib/backupSender.js:154-242
    def _send(self, backupJob, callback, sock=None, peer_socks=None, peer_failed=None):
        zfsSend = stage = None
        try:
            snapshot = self._getLatestSnapshot()
            if sock is None and peer_socks is None:
                self._decide_wire([backupJob])
                sock = socket.create_connection((backupJob["host"], int(backupJob["port"])))
            # gpu.sendCompressed: a compressed-wire job takes the disk frames (`zfs send -c`), which the
            # COMPRESS stage forwards (LZ4, and gzip on a `wireGzip` job) or decodes and re-encodes
            # (lzjb / zle, and gzip with gpu.sendGzip); every other job
            # spawns the reference's command
            flags = ["-c"] if self._send_compressed(backupJob) else []
            zfsSend = subprocess.Popen([self._zfsPath, "send"] + flags + ["-v", "-P", snapshot],
                                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=self._env)
            backupJob["size"] = None
            backupJob["done"] = 0
            last_msg = [""]

            def stderr_reader():
                for raw in iter(zfsSend.stderr.readline, b""):
                    data = raw.decode(errors="replace")
                    # zfs prints "full ...\nsize ...\n" as one write; mimic that grouping
                    if data.startswith("full") and not ZFS_PROGRESS_HEADER.match(data):
                        nxt = zfsSend.stderr.readline().decode(errors="replace")
                        data += nxt
                    m = ZFS_PROGRESS_HEADER.match(data)
                    if m:
                        backupJob["size"] = m.group(1)
                    else:
                        m = ZFS_PROGRESS_REGEX.match(data)
                        if m:
                            backupJob["completed"] = m.group(1)
                    last_msg[0] = data
            te = threading.Thread(target=stderr_reader, daemon=True)
            te.start()

            stage = self._make_stage(backupJob)
            pump_err = []
            if peer_socks is not None:
                assert stage is not None
                dead = {}
                for p, _ in enumerate(peer_socks):
                    stage.fanout_attach(p)

                def drain_peer(p, key, so):
                    try:
                        while True:
                            b = stage.read_peer(p, CHUNK)
                            if b is None:
                                break
                            if key in dead:
                                continue              # keep the ring moving for the others
                            try:
                                so.sendall(b)
                            except OSError as e:
                                dead[key] = e
                                peer_failed(key, e)
                        if key not in dead:
                            so.shutdown(socket.SHUT_WR)
                    except Exception as e:                    # noqa: BLE001  (stage failure)
                        pump_err.append(e)
                        stage.cancel()
                tds = [threading.Thread(target=drain_peer, args=(p, k, so), daemon=True)
                       for p, (k, so) in enumerate(peer_socks)]
                for t_ in tds:
                    t_.start()
                try:
                    while True:                               # stdout.pipe(stage)
                        buf = zfsSend.stdout.read(CHUNK)
                        if not buf:
                            break
                        stage.write(buf)
                    stage.flush()
                except Exception as e:                        # noqa: BLE001
                    pump_err.append(e)
                    stage.cancel()
                if pump_err and zfsSend.poll() is None:
                    zfsSend.terminate()
                for t_ in tds:
                    t_.join()
                backupJob["gpu"] = self._stage_stats(stage)
                if len(dead) == len(peer_socks) and not pump_err:
                    pump_err.append(OSError("every coalesced receiver went away"))
            elif stage is None:
                while True:                                   # stdout.pipe(socket)
                    buf = zfsSend.stdout.read(CHUNK)
                    if not buf:
                        break
                    sock.sendall(buf)
            else:
                def drain():
                    try:
                        while True:
                            b = stage.read(CHUNK)
                            if b is None:
                                break
                            sock.sendall(b)
                    except Exception as e:                    # noqa: BLE001
                        pump_err.append(e)
                        # the receiver went away (or the stage failed): nobody will empty the
                        # ring any more, so a producer blocked in stage.write() must be woken
                        stage.cancel()
                td = threading.Thread(target=drain, daemon=True)
                td.start()
                try:
                    while True:                               # stdout.pipe(stage)
                        buf = zfsSend.stdout.read(CHUNK)
                        if not buf:
                            break
                        stage.write(buf)
                    stage.flush()
                except Exception as e:                        # noqa: BLE001
                    pump_err.append(e)
                    stage.cancel()                            # a drain thread waiting for output
                if pump_err and zfsSend.poll() is None:
                    # nobody reads zfsSend.stdout any more: the child sits in write(2) on a full
                    # pipe and would never exit.  Kill it like the reference does on a socket
                    # error (lib/backupSender.js:230-233) BEFORE waiting for it.
                    zfsSend.terminate()
                td.join()
                backupJob["gpu"] = self._stage_stats(stage)   # additive field (SURVEY 8f f4)
            code = zfsSend.wait()
            te.join(2)
            if pump_err:
                raise pump_err[0]
            if code != 0:
                backupJob["done"] = "failed"
                raise RuntimeError("zfs send: %s %d" % (last_msg[0], code))
            if sock is not None:
                sock.shutdown(socket.SHUT_WR)
            backupJob["done"] = True
            callback(None)
        except Exception as e:                                # noqa: BLE001
            backupJob["done"] = "failed"
            if zfsSend is not None and zfsSend.poll() is None:
                zfsSend.terminate()                           # SIGTERM, lib/backupSender.js:233
            callback(e)
        finally:
            if stage is not None:
                stage.close()
            if sock is not None:
                sock.close()
            for _k, so in (peer_socks or []):
                so.close()
