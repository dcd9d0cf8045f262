#!/usr/bin/env python
"""Regenerates js/patches/*.patch as REAL unified diffs against a manatee checkout.

    python js/patches/make_patches.py [/path/to/manatee]      (default /root/reference)

Each edit is an (anchor text -> replacement) pair applied to the maintainer's file; the
script fails loudly if an anchor is missing or ambiguous (i.e. if upstream moved), then
writes `diff -u` output with a/ b/ prefixes, so that in a manatee checkout
    patch -p1 < js/patches/backupSender.js.patch
applies as is.  tests/test_js_patches.py checks them against tests/golden/js_patch_targets.json
(line digests of the upstream files; regenerate it with tests/golden/make_js_patch_golden.py
after regenerating the patches).  Only the three edited files are read; nothing of the
reference is stored here beyond the context lines a unified diff carries.

What the edits do (INTEGRATION.md):
  lib/backupSender.js   `gpu` option; wire format settled before net.connect(); the one
                        data-path line `zfsSend.stdout.pipe(socket)` gains the stage; the
                        job is `done` when the stage has handed its last byte to the socket
                        (not when the child exits); additive `job.gpu` / `job.wire`; guard
                        for the latent `zfsSend` undefined crash in the socket error handler
  lib/zfsClient.js      `gpu` option; `accept` in the POST body; the job path is remembered;
                        the one data-path line `socket.pipe(zfsRecv.stdin)` gains the stage,
                        whose mode follows `job.wire`; _receive completes only after the
                        stage has handed its last byte to `zfs recv`; additive `gpuRecv`
  lib/backupServer.js   the receiver's `accept` is carried on the job object
"""
import difflib
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))

EDITS = {
    "lib/backupSender.js": [
        ("""    assert.string(options.zfsPath, 'options.zfsPath');

    EventEmitter.call(this);
""", """    assert.string(options.zfsPath, 'options.zfsPath');
    assert.optionalObject(options.gpu, 'options.gpu');

    EventEmitter.call(this);

    /** @type {object} GPU stage config {mode, device, ringBytes, ...}; absent == off */
    this._gpu = options.gpu || { mode: 'off' };
    /**
     * @type {number} Requests for the latest snapshot that arrive within this
     * many ms of each other share ONE zfs send and ONE pass of the GPU stage
     * (fan-out to one pinned ring per peer).  0 == one send per request, as
     * before.
     */
    this._coalesceMs = this._gpu.coalesceMs || 0;
    this._waiting = [];
"""),
        ("""    self._queue.on('push', function (backupJob) {
        self._send(backupJob, function (err) {
""", """    var jobDone = function (backupJob, err) {
        if (err) {
            self._log.error({ backupJob: backupJob, err: err },
                            'unable to send backup');
            self.emit('err', err);
            backupJob.err = err;
        } else {
            self._log.info({ backupJob: backupJob },
                           'successfully sent backup');
            self.emit('done', backupJob);
        }
    };

    self._queue.on('push', function (backupJob) {
        if (self._coalesceMs > 0 && self._gpu.mode &&
            self._gpu.mode !== 'off') {
            /*
             * The first request opens the window; everybody who asks before
             * it closes rides the same send.
             */
            self._waiting.push(backupJob);
            if (self._waiting.length === 1) {
                setTimeout(function () {
                    var jobs = self._waiting;
                    self._waiting = [];
                    self._sendGroup(jobs, jobDone);
                }, self._coalesceMs);
            }
            return;
        }
        self._send(backupJob, function (err) {
"""),
        ("""            log.info({port: backupJob.port, host: backupJob.host},
                     'BackupSender._send: creating socket for zfs send');
            socket = net.connect(backupJob.port, backupJob.host);
            var zfsSend;
""", """            log.info({port: backupJob.port, host: backupJob.host},
                     'BackupSender._send: creating socket for zfs send');
            var gpuOn = (self._gpu.mode && self._gpu.mode !== 'off');
            if (gpuOn) {
                /*
                 * Settle the wire format BEFORE connecting, so that a receiver
                 * which reads the job when the connection arrives sees it: only
                 * a receiver that asked for the stage-compressed wire gets it.
                 */
                backupJob.wire = (self._gpu.mode === 'compress' &&
                    backupJob.accept === 'lz4-stage-v1') ? 'lz4-stage-v1' : 'raw';
            }
            socket = net.connect(backupJob.port, backupJob.host);
            var zfsSend;
            var stage = null;
            var stageEnded = false;
"""),
        ("""                zfsSend.stdout.pipe(socket);

                var msg = '';
""", """                if (gpuOn) {
                    var GpuSnapshotStage =
                        require('manatee-gpu/lib/gpuSnapshotStage');
                    var gpuCfg = JSON.parse(JSON.stringify(self._gpu));
                    if (gpuCfg.mode === 'compress' &&
                        backupJob.wire !== 'lz4-stage-v1') {
                        gpuCfg.mode = 'verify';
                    }
                    stage = new GpuSnapshotStage(gpuCfg);
                    stage.on('error', function (serr) {
                        log.error({err: serr},
                                  'BackupSender._send: gpu stage error');
                        backupJob.done = 'failed';
                        if (zfsSend) {
                            zfsSend.kill('SIGTERM');
                        }
                        socket.destroy();
                        return _cb(serr);
                    });
                    stage.on('end', function () {
                        stageEnded = true;
                        backupJob.gpu = stage.stats;
                    });
                    zfsSend.stdout.pipe(stage).pipe(socket);
                } else {
                    zfsSend.stdout.pipe(socket);
                }

                var msg = '';
"""),
        ("""                    backupJob.done = true;
                    log.info({backupJob: backupJob}, 'completed backup job');
                    return _cb();
                });
""", """                    var finish = function () {
                        backupJob.done = true;
                        log.info({backupJob: backupJob},
                                 'completed backup job');
                        return _cb();
                    };
                    /*
                     * With a stage in the pipe the tail of the stream (one GPU
                     * batch) is still on its way when the child exits: the job
                     * is done when the stage has handed over its last byte.
                     */
                    if (stage && !stageEnded) {
                        stage.once('end', finish);
                        return (undefined);
                    }
                    return finish();
                });
"""),
        ("""                backupJob.done = 'failed';
                zfsSend.kill('SIGTERM');
                return _cb(err);
""", """                backupJob.done = 'failed';
                if (zfsSend) {
                    zfsSend.kill('SIGTERM');
                }
                if (stage) {
                    /* frees the pinned rings, GPU slots and native threads */
                    stage.destroy();
                }
                return _cb(err);
"""),
        ("""/**
 * @callback BackupSender-cb
""", """/**
 * One `zfs send`, one pass of the GPU stage, N receivers (SURVEY 8f f1).  Every
 * job gets its own socket and its own output ring of the stage
 * (gpuFanoutStage: mtz_fanout_attach / mtz_out_peek_peer); progress fields are
 * mirrored into every job object, and a receiver that goes away only fails its
 * own job.
 *
 * @param {object[]} jobs The coalesced backup jobs.
 * @param {function} jobDone Called once per job with (job, err).
 */
BackupSender.prototype._sendGroup = function (jobs, jobDone) {
    var self = this;
    var log = self._log;
    var finished = {};
    var finish = function (job, err) {
        if (finished[job.uuid]) {
            return;
        }
        finished[job.uuid] = true;
        job.done = err ? 'failed' : true;
        jobDone(job, err);
    };
    var failAll = function (err) {
        jobs.forEach(function (job) { finish(job, err); });
    };

    self._getLatestSnapshot(function (err, snapshot) {
        if (err) {
            return failAll(err);
        }
        var compress = (self._gpu.mode === 'compress' &&
            jobs.every(function (j) { return j.accept === 'lz4-stage-v1'; }));
        jobs.forEach(function (j) {
            j.wire = compress ? 'lz4-stage-v1' : 'raw';
            j.size = null;
            j.done = 0;
        });
        var GpuFanoutStage = require('manatee-gpu/lib/gpuFanoutStage');
        var gpuCfg = JSON.parse(JSON.stringify(self._gpu));
        if (gpuCfg.mode === 'compress' && !compress) {
            gpuCfg.mode = 'verify';
        }
        gpuCfg.peers = jobs.length;
        var fan;
        try {
            fan = new GpuFanoutStage(gpuCfg);
        } catch (e) {
            return failAll(e);
        }
        var zfsSend = spawn(self._zfsPath, ['send', '-v', '-P', snapshot]);
        var left = jobs.length;
        jobs.forEach(function (job, i) {
            var socket = net.connect(job.port, job.host);
            socket.on('error', function (serr) {
                log.error({err: serr, job: job}, 'coalesced receiver failed');
                fan.peer(i).destroy();      /* keeps draining, discards */
                finish(job, serr);
            });
            fan.peer(i).on('end', function () {
                job.gpu = fan.stats;
                finish(job);
                if (--left === 0) {
                    log.info('coalesced backup jobs completed');
                }
            });
            fan.peer(i).pipe(socket);
        });
        fan.on('error', function (ferr) {
            zfsSend.kill('SIGTERM');
            failAll(ferr);
        });
        var msg = '';
        zfsSend.stderr.on('data', function (data) {
            var dataStr = data.toString();
            var m;
            if ((m = ZFS_PROGRESS_HEADER.exec(dataStr)) !== null) {
                jobs.forEach(function (j) { j.size = m[1]; });
            } else if ((m = ZFS_PROGRESS_REGEX.exec(dataStr)) !== null) {
                jobs.forEach(function (j) { j.completed = m[1]; });
            }
            msg = dataStr;
        });
        zfsSend.on('exit', function (code) {
            if (code !== 0) {
                fan.destroy();
                failAll(new verror.VError('zfs send: ' + msg + ' ' + code));
            }
        });
        zfsSend.stdout.pipe(fan);
        return (undefined);
    });
};

/**
 * @callback BackupSender-cb
"""),
    ],
    "lib/zfsClient.js": [
        ("""    assert.number(options.zfsPort, 'options.zfsPort');

    var self = this;
""", """    assert.number(options.zfsPort, 'options.zfsPort');
    assert.optionalObject(options.gpu, 'options.gpu');

    var self = this;

    /** GPU stage config {mode, device, ringBytes, ...}; absent == off */
    this._gpu = options.gpu || { mode: 'off' };
    this._jobPath = null;
"""),
        ("""        port: self._zfsPort,
        dataset: self._dataset
    };

    log.info({
        zfsHost: request.host,
""", """        port: self._zfsPort,
        dataset: self._dataset
    };
    if (self._gpu.mode === 'decompress') {
        /* ignored by a reference backupserver (unknown fields are dropped) */
        request.accept = 'lz4-stage-v1';
    }

    log.info({
        zfsHost: request.host,
"""),
        ("""        }, 'ZfsClient.postRestoreRequest: exiting');
        callback(err, obj ? obj.jobPath : null);
""", """        }, 'ZfsClient.postRestoreRequest: exiting');
        self._jobPath = obj ? obj.jobPath : null;
        callback(err, obj ? obj.jobPath : null);
"""),
        ("""    var restoreIntervalId;
    var server;
    var zfsRecv;
""", """    var restoreIntervalId;
    var server;
    var zfsRecv;
    var stage = null;
    var stageEnded = false;
    self._jobPath = null;       /* learnt from this restore's own POST */
"""),
        ("""                log.info('ZFSClient._receive: got socket, piping to zfs recv');
                socket.pipe(zfsRecv.stdin);
                cb();
""", """                log.info('ZFSClient._receive: got socket, piping to zfs recv');
                if (!self._gpu.mode || self._gpu.mode === 'off') {
                    socket.pipe(zfsRecv.stdin);
                    cb();
                    return;
                }
                /*
                 * A receiver configured to decompress only does so when the
                 * sender committed to the stage-compressed wire (job.wire, set
                 * before it connected).  A reference sender, or a GPU sender
                 * that is not compressing, ships a raw stream: verify it.
                 */
                socket.pause();
                var startPipe = function (wire) {
                    var GpuSnapshotStage =
                        require('manatee-gpu/lib/gpuSnapshotStage');
                    var gpuCfg = JSON.parse(JSON.stringify(self._gpu));
                    if (gpuCfg.mode === 'decompress' &&
                        wire !== 'lz4-stage-v1') {
                        gpuCfg.mode = 'verify';
                    }
                    stage = new GpuSnapshotStage(gpuCfg);
                    stage.on('error', function (serr) {
                        /*
                         * Same exit as a failed `zfs recv`.  Dropping the
                         * socket fails the sender's job, which ends the poll.
                         */
                        socket.destroy();
                        zfsRecv.kill('SIGKILL');
                        callback(new verror.VError(serr, 'gpu stage failed'));
                    });
                    stage.on('end', function () {
                        stageEnded = true;
                        if (self._restoreObject) {
                            self._restoreObject.gpuRecv = stage.stats;
                        }
                    });
                    socket.pipe(stage).pipe(zfsRecv.stdin);
                    socket.resume();
                };
                var lookup = function (tries) {
                    if (self._gpu.mode !== 'decompress') {
                        startPipe(undefined);
                    } else if (self._jobPath === null && tries > 0) {
                        /* the connection raced our own POST response */
                        setTimeout(lookup, 20, tries - 1);
                    } else if (self._jobPath === null) {
                        startPipe(undefined);
                    } else {
                        self._client.get(self._jobPath,
                            function (werr, wreq, wres, wobj) {
                            startPipe((!werr && wobj) ? wobj.wire : undefined);
                        });
                    }
                };
                lookup(500);
                cb();
"""),
        ("""        log.info({
            dataset: dataset,
            serverUrl: serverUrl,
            pollInterval: pollInterval
        }, 'successfully received zfs dataset');
        callback();
""", """        var complete = function () {
            log.info({
                dataset: dataset,
                serverUrl: serverUrl,
                pollInterval: pollInterval
            }, 'successfully received zfs dataset');
            callback();
        };
        /*
         * The sender reports done when its last byte is on the socket; with a
         * stage in this pipe that byte still has to come out of the GPU.
         */
        if (stage && !stageEnded) {
            stage.once('end', complete);
            return;
        }
        complete();
"""),
    ],
    "lib/backupServer.js": [
        ("""            dataset: params.dataset,
            done: false
        };

        self._queue.push(backupJob);
""", """            dataset: params.dataset,
            done: false
        };
        if (params.accept) {
            /* wire capability of the receiver's stage; additive */
            backupJob.accept = params.accept;
        }

        self._queue.push(backupJob);
"""),
    ],
}


def patched(text, edits, name):
    for old, new in edits:
        n = text.count(old)
        if n != 1:
            raise SystemExit("%s: anchor found %d times (upstream moved?):\n%s" % (name, n, old))
        text = text.replace(old, new)
    return text


def main():
    ref = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
    for rel, edits in EDITS.items():
        with open(os.path.join(ref, rel)) as f:
            a = f.read()
        b = patched(a, edits, rel)
        diff = difflib.unified_diff(a.splitlines(True), b.splitlines(True), "a/" + rel, "b/" + rel, n=3)
        out = os.path.join(HERE, os.path.basename(rel) + ".patch")
        with open(out, "w") as f:
            f.writelines(diff)
        print("wrote", out)


if __name__ == "__main__":
    main()
