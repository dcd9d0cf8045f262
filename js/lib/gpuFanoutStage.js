/*
 * gpuFanoutStage.js -- ONE pass of the GPU stage feeding SEVERAL peers (SURVEY.md 8f f1).
 *
 * The reference starts one `zfs send` per requesting peer (one _send per 'push',
 * lib/backupSender.js:72-73).  When several peers ask for the same snapshot within the
 * coalescing window, the patched BackupSender spawns ONE `zfs send`, writes it into ONE of these
 * and pipes `fan.peer(i)` into each peer's socket:
 *
 *     zfsSend.stdout.pipe(fan);   fan.peer(0).pipe(socketA);   fan.peer(1).pipe(socketB); ...
 *
 * Underneath: mtz_fanout_attach(h, i) for every peer before the first byte; the library
 * processes the stream once on its device group, broadcasts each processed batch over NVLink
 * (NCCL, library-owned) to the peers' egress GPUs and fills one pinned ring per peer
 * (mtz_out_peek_peer / mtz_out_consume_peer).  A peer whose socket dies keeps being drained and
 * discarded here, so it never back-pressures the others.
 *
 * Same addon as gpuSnapshotStage.js; not executed in this repository (no Node.js in the build
 * image) -- manatee_b200/host/backup_sender.py::_send_group is the mirror the test-suite runs.
 */
var stream = require('stream');
var util = require('util');

var MODES = { verify: 0, compress: 1, decompress: 2, recompress: 3, passthrough: 4 };

function PeerReadable(fan, id) {
    stream.Readable.call(this, { highWaterMark: 4 << 20 });
    this._fan = fan;
    this._id = id;
    this.wantMore = false;
    this.ended = false;
    this.dead = false;         // socket gone: keep consuming, discard
}
util.inherits(PeerReadable, stream.Readable);
PeerReadable.prototype._read = function () {
    this.wantMore = true;
    this._fan._drain();
};
PeerReadable.prototype._destroy = function (err, cb) {
    this.dead = true;
    this._fan._drain();
    cb(err);
};

function GpuFanoutStage(options) {
    options = options || {};
    stream.Writable.call(this, { highWaterMark: 4 << 20 });
    this._addon = require('../build/Release/manatee_gpu.node');
    this._h = this._addon.open({
        mode: MODES[options.mode || 'verify'],
        device: options.device || 0,
        deviceMask: options.deviceMask || 0,
        ringBytes: options.ringBytes || 0,
        outRingBytes: options.outRingBytes || 0,
        batchBytes: options.batchBytes || 0,
        slots: options.slots || 0,
        flags: (options.blockChecksums ? 4 : 0) |   // gpu.blockChecksums: MTZ_FLAG_BLOCK_CKSUM
            (options.blockSha256 ? 8 : 0) |        // gpu.blockSha256: MTZ_FLAG_BLOCK_SHA256
            (options.blockSha512 ? 16 : 0) |       // gpu.blockSha512: MTZ_FLAG_BLOCK_SHA512
            (options.blockFrames ? 32 : 0) |       // gpu.blockFrames: MTZ_FLAG_BLOCK_FRAMES
            (options.blockLzjb ? 64 : 0) |         // gpu.blockLzjb: MTZ_FLAG_BLOCK_LZJB
            (options.blockLogical ? 128 : 0)       // gpu.blockLogical: MTZ_FLAG_BLOCK_LOGICAL
    });
    this._blockChecksums = !!options.blockChecksums;
    this._peers = [];
    for (var i = 0; i < (options.peers || 1); i++) {
        this._addon.attach(this._h, i);
        this._peers.push(new PeerReadable(this, i));
    }
    this._pending = null;
    this._finalCb = null;
    this._closed = false;
    var self = this;
    this._watch = this._addon.watch(this._h, function () { self._drain(); });
}
util.inherits(GpuFanoutStage, stream.Writable);

GpuFanoutStage.prototype.peer = function (i) { return (this._peers[i]); };

GpuFanoutStage.prototype._cleanup = function () {
    if (this._closed) { return; }
    this._closed = true;
    try { this._addon.unwatch(this._watch); } catch (e) {}
    try { this._addon.close(this._h); } catch (e) {}
};

GpuFanoutStage.prototype._fail = function (err) {
    this._cleanup();
    this._peers.forEach(function (p) { p.destroy(err); });
    this.destroy(err);
};

GpuFanoutStage.prototype._destroy = function (err, cb) {
    if (!this._closed) {
        try { this._addon.cancel(this._h); } catch (e) {}
    }
    this._pending = null;
    this._cleanup();
    cb(err);
};

GpuFanoutStage.prototype._feed = function () {
    var p = this._pending;
    if (!p) { return; }
    try {
        while (p.off < p.chunk.length) {
            var n = this._addon.write(this._h, p.chunk.slice(p.off));
            if (n === 0) { return; }
            p.off += n;
        }
    } catch (e) { return (this._fail(e)); }
    this._pending = null;
    p.cb();
};

GpuFanoutStage.prototype._write = function (chunk, enc, cb) {
    this._pending = { chunk: chunk, off: 0, cb: cb };
    this._feed();
    this._drain();
};

GpuFanoutStage.prototype._final = function (cb) {
    this._finalCb = cb;
    try { this._addon.flush(this._h); } catch (e) { return (this._fail(e)); }
    this._drain();
};

GpuFanoutStage.prototype._drain = function () {
    if (this._closed) { return; }
    var live = 0;
    try {
        for (var i = 0; i < this._peers.length; i++) {
            var p = this._peers[i];
            while (!p.ended && (p.wantMore || p.dead)) {
                var ab = this._addon.peek(this._h, i);
                if (ab === null) { break; }
                if (ab === 'eof') {
                    p.ended = true;
                    if (!p.dead) { p.push(null); }
                    break;
                }
                var buf = Buffer.from(Buffer.from(ab));
                this._addon.consume(this._h, buf.length, i);
                if (!p.dead && !p.push(buf)) { p.wantMore = false; }
            }
            if (!p.ended) { live++; }
        }
    } catch (e) { return (this._fail(e)); }
    if (live === 0 && this._finalCb) {
        var fcb = this._finalCb;
        this._finalCb = null;
        this.stats = this._addon.stats(this._h);
        if (this._blockChecksums) {
            this.stats.blocks = this._addon.blockStats(this._h);
        }
        this._cleanup();
        return (fcb());
    }
    this._feed();
};

module.exports = GpuFanoutStage;
