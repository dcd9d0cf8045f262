/*
 * gpuSnapshotStage.js -- the stream.Transform that is spliced into manatee's
 * two pipes:
 *
 *     zfsSend.stdout.pipe(stage).pipe(socket)      // lib/backupSender.js:179
 *     socket.pipe(stage).pipe(zfsRecv.stdin)       // lib/zfsClient.js:826
 *
 * All work happens in libmanatee_gpu.so on the GPU; this file only moves Buffers
 * between Node's stream machinery and the library's pinned rings.  There is no
 * JS/CPU fallback: if the addon cannot be loaded or no H100 is present, creating
 * a stage throws, and the caller's `gpu.mode` must be 'off' to get the legacy
 * identity pipe.
 *
 * Written against the N-API addon in ../src/binding.cc.  Not executed in this
 * repository (no Node.js in the build image); manatee_b200/stage.py is the
 * mirror that the test-suite runs.
 */
var stream = require('stream');
var util = require('util');

var MODES = { verify: 0, compress: 1, decompress: 2, recompress: 3, passthrough: 4 };
var BLOCK_CKSUM = 4;        // MTZ_FLAG_BLOCK_CKSUM
var BLOCK_SHA256 = 8;       // MTZ_FLAG_BLOCK_SHA256 (with BLOCK_CKSUM only)
var BLOCK_SHA512 = 16;      // MTZ_FLAG_BLOCK_SHA512 (with BLOCK_CKSUM only)
var BLOCK_FRAMES = 32;      // MTZ_FLAG_BLOCK_FRAMES (with BLOCK_CKSUM only)
var BLOCK_LZJB = 64;        // MTZ_FLAG_BLOCK_LZJB (with BLOCK_CKSUM only)
var BLOCK_LOGICAL = 128;    // MTZ_FLAG_BLOCK_LOGICAL (with BLOCK_CKSUM only)

function GpuSnapshotStage(options) {
    if (!(this instanceof GpuSnapshotStage)) {
        return (new GpuSnapshotStage(options));
    }
    options = options || {};
    stream.Transform.call(this, { highWaterMark: options.highWaterMark || (4 << 20) });
    this._addon = require('../build/Release/manatee_gpu.node');
    this._h = this._addon.open({
        mode: MODES[options.mode || 'verify'],
        device: options.device || 0,
        deviceMask: options.deviceMask || 0,    // device group: bit i = CUDA device i
        ringBytes: options.ringBytes || 0,
        outRingBytes: options.outRingBytes || 0,
        batchBytes: options.batchBytes || 0,
        slots: options.slots || 0,
        flags: (options.blockChecksums ? BLOCK_CKSUM : 0) |   // gpu.blockChecksums
            (options.blockSha256 ? BLOCK_SHA256 : 0) |       // gpu.blockSha256
            (options.blockSha512 ? BLOCK_SHA512 : 0) |       // gpu.blockSha512
            (options.blockFrames ? BLOCK_FRAMES : 0) |       // gpu.blockFrames
            (options.blockLzjb ? BLOCK_LZJB : 0) |           // gpu.blockLzjb
            (options.blockLogical ? BLOCK_LOGICAL : 0)       // gpu.blockLogical
    });
    this._blockChecksums = !!options.blockChecksums;
    this._pending = null;      // {chunk, off, cb} waiting for ring space
    this._flushCb = null;
    this._wantMore = true;     // cleared when push() returns false, set again by _read()
    this._closed = false;
    var self = this;
    // wake-up source: the addon poll(2)s the library's eventfd on a native thread and calls
    // this function on the event loop (napi_threadsafe_function) whenever output, EOF or an
    // error is pending -- the loop neither blocks nor busy-polls.
    this._watch = this._addon.watch(this._h, function () { self._drain(); });
}
util.inherits(GpuSnapshotStage, stream.Transform);

GpuSnapshotStage.prototype._fail = function (err) {
    // sticky failure -> destroy(err) -> sender: job.done='failed', emit 'err'
    // (lib/backupSender.js:74-88, 218); receiver: _receive cb(err) -> SIGKILL zfs recv
    // (lib/zfsClient.js:867-876)
    this._cleanup();
    this.destroy(err);
};

/*
 * destroy() from outside (socket 'error', pipeline teardown): without this the native handle --
 * pinned rings, GPU slots, the engine and watcher threads -- would leak on every failed restore
 * of a long-lived daemon.  cancel() first: a chunk parked in _pending is waiting for ring space
 * that will never come.
 */
GpuSnapshotStage.prototype._destroy = function (err, cb) {
    if (!this._closed) {
        try { this._addon.cancel(this._h); } catch (e) {}
    }
    this._pending = null;
    this._cleanup();
    cb(err);
};

GpuSnapshotStage.prototype._cleanup = function () {
    if (this._closed) { return; }
    this._closed = true;
    try { this._addon.unwatch(this._watch); } catch (e) {}   // joins the poll thread first
    try { this._addon.close(this._h); } catch (e) {}
};

GpuSnapshotStage.prototype._feed = function () {
    var p = this._pending;
    if (!p) { return; }
    try {
        while (p.off < p.chunk.length) {
            var n = this._addon.write(this._h, p.chunk.slice(p.off));
            if (n === 0) { return; }            // ring full: retried from _drain()
            p.off += n;
        }
    } catch (e) { return (this._fail(e)); }
    this._pending = null;
    p.cb();
};

GpuSnapshotStage.prototype._transform = function (chunk, enc, cb) {
    this._pending = { chunk: chunk, off: 0, cb: cb };
    this._feed();
    this._drain();
};

GpuSnapshotStage.prototype._drain = function () {
    if (this._closed) { return; }
    try {
        // readable-side backpressure: stop pulling from the pinned output ring as soon as
        // push() says the consumer (socket / zfs recv stdin) is behind.  The ring then fills,
        // the engine stalls, the input ring fills, write() returns 0 and _transform's callback
        // is withheld -- the whole chain slows to the slowest consumer instead of buffering a
        // multi-GiB stream in the Node heap.  _read() re-arms it.
        while (this._wantMore) {
            var ab = this._addon.peek(this._h);
            if (ab === null) { break; }
            if (ab === 'eof') {
                var fcb = this._flushCb;
                this._flushCb = null;
                this.stats = this._addon.stats(this._h);
                if (this._blockChecksums) {
                    this.stats.blocks = this._addon.blockStats(this._h);
                }
                this._cleanup();
                if (fcb) { fcb(); }
                return;
            }
            // copy out of the pinned ring before releasing the slice
            var buf = Buffer.from(Buffer.from(ab));
            this._addon.consume(this._h, buf.length);
            if (!this.push(buf)) { this._wantMore = false; }
        }
    } catch (e) { return (this._fail(e)); }
    this._feed();
};

GpuSnapshotStage.prototype._read = function (n) {
    this._wantMore = true;
    this._drain();
    stream.Transform.prototype._read.call(this, n);
};

GpuSnapshotStage.prototype._flush = function (cb) {
    this._flushCb = cb;
    try { this._addon.flush(this._h); } catch (e) { return (this._fail(e)); }
    this._drain();
};

module.exports = GpuSnapshotStage;
