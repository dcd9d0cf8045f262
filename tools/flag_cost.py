#!/usr/bin/env python
"""What a flag of GpuSnapshotStage costs on the GPU, one subcommand per workload.  Every measurement
runs the same stream through two handles, the baseline leg and the flag leg, alternating step by step so
that both see the same machine, and prints one JSON line (and writes it to --out) with the GPU name,
power limit and max SM clock the numbers were taken on.

  block_cksum    MTZ_FLAG_BLOCK_CKSUM off / on: resident VERIFY of 16 GiB of uncompressed 128 KiB
                 records, resident RECOMPRESS of the `zfs send -c` form of 1 GiB with "LZ4 on disk" keys
  block_sha256   MTZ_FLAG_BLOCK_SHA256 against MTZ_FLAG_BLOCK_CKSUM alone on streams with SHA-256 keys:
                 resident VERIFY (with k_block_sha256's device time and the bytes it hashes per second),
                 mtz_process_host VERIFY with 128 KiB and 1 MiB records (SHA-256 is serial per record, so
                 1 MiB records give the kernel few threads and show the latency of one hash), resident
                 RECOMPRESS of the `send -c` form
  block_sha512   the same for MTZ_FLAG_BLOCK_SHA512 on streams with SHA-512 keys
  block_frames   MTZ_FLAG_BLOCK_FRAMES against MTZ_FLAG_BLOCK_CKSUM alone on pg-page records keyed as ZFS
                 with compression=lz4 at ashift 9 writes them, sent without -c: resident VERIFY, host
                 VERIFY with 128 KiB and 1 MiB records at 32 MiB and 256 MiB batches, and the ring API
                 (acquire + commit, bench.py's ring_run) at each leg's default batch size
  block_lzjb     the same for MTZ_FLAG_BLOCK_LZJB on lzjb-keyed records, plus resident VERIFY of
                 zle-keyed ones
  block_logical  MTZ_FLAG_BLOCK_LOGICAL against the same flags without it: resident COMPRESS and
                 DECOMPRESS of lzjb-keyed records (at --gib and at --large-gib), resident RECOMPRESS of
                 the compressed form of raw-keyed records (fletcher4 and sha256 keys), host COMPRESS
  lz4hc          MTZ_FLAG_LZ4_HC against COMPRESS without it: wire bytes, ratio and time, resident and host
  compressed_in  MTZ_FLAG_COMPRESSED_IN: COMPRESS of the `zfs send -c` stream x with the flag against COMPRESS
                 of plain(x), the stream today's sender pipes, for pg-page 128 KiB records written with lz4
                 at ashift 9 and 12, lzjb, zle and block_ref.mixed_codecs: resident step, mtz_process_host
                 and the ring API fed through a pipe (bench.py's ring_run, producer "pipe"), in GB/s of
                 logical bytes; input and wire bytes, the counters, and the decoders' device time
  gzip_in        MTZ_FLAG_GZIP_IN: the same legs, the flag leg with compressed_input + gzip_input, for
                 pg-page 128 KiB records written with gzip-1, gzip-6, gzip-9 and a gzip-6 / lz4 / lzjb /
                 raw pool; plus k_inflate's device time and single-thread zlib.decompress of the records
  gzip_wire      MTZ_FLAG_GZIP_WIRE on the pools of gzip_in.  Sender: COMPRESS of x with compressed_input +
                 gzip_input (today's wire) against compressed_input + gzip_wire: wire bytes, resident step,
                 mtz_process_host and the ring API through a pipe.  Receiver: DECOMPRESS of today's wire
                 against DECOMPRESS with gzip_wire of the gzip wire, and DECOMPRESS with gzip_wire of today's
                 wire (no gzip record on it): resident step, mtz_process_host, k_inflate and K2 device time;
                 every DECOMPRESS output is checked against plain(x); --pools picks some of the pools
  gzip_encode    MTZ_FLAG_GZIP_ENCODE: COMPRESS against COMPRESS with gzip_encode of pg-page 128 KiB records,
                 raw and (--mixed-gib of them) as a `send -c` stream of block_ref.mixed_codecs with
                 compressed_input: wire bytes, resident step with K3's and k_deflate_from_lz4's device time,
                 mtz_process_host, the ring API through a pipe, and the receiver's DECOMPRESS (with
                 gzip_wire on the new wire) with k_inflate's and K2's device time

A resident step is timed with CUDA events around dev_submit + dev_finish on a side stream, a host pass
with the host clock around mtz_process_host; kernel device times come from torch.profiler in a pass of
their own.  Every counter is one pass's: resident legs dev_reset before every step (outside the timed
window), host legs divide by the passes the handle ran; the first_* indices are reported as read.
usage: tools/flag_cost.py WORKLOAD [options] [--out F]    (tools/flag_cost.py WORKLOAD -h lists them)"""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor
from contextlib import ExitStack, contextmanager
from functools import partial

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import block_ref as R  # noqa: E402
import compressed_in_ref as CI  # noqa: E402
import gzip_in_ref as GZ  # noqa: E402
import gzip_wire_ref as GW  # noqa: E402
import oracle as O  # noqa: E402

RECSIZE = 131072
NTH = os.cpu_count() or 1
# the hash kernel of each SHA flag and its compression block: a 128 KiB record hashes 128 KiB + one
# padding block
HASHES = {"sha256": ("k_block_sha256", 64), "sha512": ("k_block_sha512", 128)}


def gpu_info():
    import torch
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip().splitlines()[0] if q.stdout.strip() else None
    except (OSError, subprocess.SubprocessError):
        info["power_limit_and_max_sm_clock"] = None
    return info


def pair(base, flag, **shared):
    """a leg pair: the baseline leg and the flag leg, each (name, GpuSnapshotStage keyword arguments),
    and the keyword arguments both legs share -> {name: keyword arguments}, the baseline first"""
    return {name: {**shared, **kw} for name, kw in (base, flag)}


@contextmanager
def stages(mode, legs):
    from manatee_b200 import GpuSnapshotStage
    with ExitStack() as es:
        yield {name: es.enter_context(GpuSnapshotStage(mode, **kw)) for name, kw in legs.items()}


def alternate(legs, passes):
    """(pass, leg name) for `passes` passes of every leg, the order swapped every pass"""
    names = list(legs)
    for i in range(passes):
        for name in (names if i % 2 == 0 else names[::-1]):
            yield i, name


def summary(legs, ms, nbytes=0, rate="gbps"):
    """the step times of a leg pair; with `nbytes` also each leg's <leg>_<rate> in GB/s"""
    base, flag = legs
    res = {}
    for name in legs:
        v = sorted(ms[name])
        res.update({name + "_ms_mean": sum(v) / len(v), name + "_ms_median": v[len(v) // 2],
                    name + "_ms_min": v[0], name + "_ms_max": v[-1]})
        if nbytes:
            res[name + "_" + rate] = nbytes / (res[name + "_ms_mean"] * 1e6)
    res["diff_ms_mean"] = res[flag + "_ms_mean"] - res[base + "_ms_mean"]
    res["diff_pct_mean"] = 100.0 * res["diff_ms_mean"] / res[base + "_ms_mean"]
    return res


def leg_fields(gs, counters, passes, fields, out_bytes):
    """the block counters of the legs named in `counters` (None: the flag leg) per pass, the flag leg's
    as block_stats and a baseline's as <leg>_block_stats, and fields(name, stage, output bytes) of
    every leg"""
    flag = list(gs)[1]
    res = {}
    for name in ((flag,) if counters is None else counters):
        st = gs[name].block_stats()
        res["block_stats" if name == flag else name + "_block_stats"] = {
            k: v if k.startswith("first_") else v // passes for k, v in st.items()}
    for name, g in gs.items():
        res.update(fields(name, g, out_bytes[name]) if fields else {})
    return res


def kernel_times(fn, n, kernels):
    """device ms and launches per step of each of `kernels` over n calls of fn (torch.profiler, CUDA
    activities)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    res = {}
    for kern in kernels:
        us, calls = 0.0, 0
        for e in prof.key_averages():
            if kern in e.key:
                us += getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                calls += e.count
        res[kern + "_ms_per_step"] = us / 1000.0 / n
        res[kern + "_launches_per_step"] = calls / n
    return res


def resident(a, mode, s, legs, kernels=(), counters=None, fields=None, rate=None, same_output=True):
    """ms per resident step of `mode` over the plain stream `s` held in HBM, on both legs of `legs`;
    then the device time of `kernels` on the flag leg over --profile-steps steps.  When the mode writes
    an output and both legs must write the same bytes, outputs_equal compares their last steps'."""
    import numpy as np
    import torch
    from manatee_b200 import index_host
    recs, used = index_host(s)
    assert used == s.size
    d_in = torch.empty(s.size + 512, dtype=torch.uint8, device="cuda")
    d_in[:s.size].copy_(torch.from_numpy(s))
    d_recs = torch.from_numpy(recs.view(np.uint8).copy()).cuda()
    # the re-encoding modes' worst case (mtz_dev_submit's check) and a margin
    cap = 0 if mode == "verify" else int(np.maximum(recs["lsize"], recs["payload"]).sum()) + 312 * len(recs) + (1 << 20)
    d_out = torch.empty(cap, dtype=torch.uint8, device="cuda") if cap else None
    st = torch.cuda.Stream()
    ms, outs = {name: [] for name in legs}, {}
    with stages(mode, legs) as gs:
        def step(g):
            g.dev_reset()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            g.dev_submit(d_in.data_ptr(), s.size, d_recs.data_ptr(), len(recs),
                         d_out.data_ptr() if cap else 0, cap, cuda_stream=st.cuda_stream)
            ob = g.dev_finish()[0]
            e1.record(st)
            torch.cuda.synchronize()
            return e0.elapsed_time(e1), ob

        for i, name in alternate(legs, a.warmup + a.steps):
            t, ob = step(gs[name])
            if i >= a.warmup:
                ms[name].append(t)
            if i == a.warmup + a.steps - 1:
                # records are 8-byte aligned
                outs[name] = (ob, d_out[:ob].view(torch.int64).sum().item() if cap else 0)
        res = summary(legs, ms, s.size if rate else 0, rate)
        res.update(leg_fields(gs, counters, 1, fields, {name: o[0] for name, o in outs.items()}))
        res["records"] = int(len(recs))
        res["stream_bytes"] = int(s.size)
        base, flag = legs
        if cap and same_output:
            res["outputs_equal"] = outs[base] == outs[flag]
        if kernels and a.profile_steps:
            res.update(kernel_times(partial(step, gs[flag]), a.profile_steps, kernels))
            res["profile_steps"] = a.profile_steps
        return res


def host(a, mode, s, legs, counters=None, fields=None, rate="gbps"):
    """wall ms per mtz_process_host pass of the whole stream `s`, 1 warm-up and --host-steps timed
    passes of both legs"""
    import numpy as np
    out = None if mode == "verify" else np.zeros(s.size + (64 << 20), dtype=np.uint8)
    ms, obs = {name: [] for name in legs}, {}
    with stages(mode, legs) as gs:
        for i, name in alternate(legs, 1 + a.host_steps):
            t0 = time.perf_counter()
            obs[name] = gs[name].process_host(s, out)
            dt = (time.perf_counter() - t0) * 1e3
            assert out is not None or obs[name] == s.size
            if i >= 1:
                ms[name].append(dt)
        res = summary(legs, ms, s.size, rate)
        res.update(leg_fields(gs, counters, 1 + a.host_steps, fields, obs))
        res["stream_bytes"] = int(s.size)
        return res


def ring(a, s, legs):
    """GB/s of VERIFY through the ring API, acquire + commit (bench.py's ring_run with its native
    producer), each pass of each leg on a fresh handle at its default batch size"""
    import bench
    from manatee_b200 import GpuSnapshotStage
    base, flag = legs
    secs, stats = {name: [] for name in legs}, {}
    for _, name in alternate(legs, a.ring_steps):
        with GpuSnapshotStage("verify", **legs[name]) as g:
            dt, ok, detail = bench.ring_run(g, s, producer="acquire", nthreads=bench.pump_threads())
            assert ok, detail
            secs[name].append(dt)
            stats[name] = g.block_stats()
    res = {}
    for name in legs:
        v = sorted(secs[name])
        res.update({name + "_gbps_mean": s.size / (sum(v) / len(v)) / 1e9, name + "_gbps_min": s.size / v[-1] / 1e9,
                    name + "_gbps_max": s.size / v[0] / 1e9})
    res["diff_pct_mean"] = 100.0 * (res[flag + "_gbps_mean"] / res[base + "_gbps_mean"] - 1.0)
    res["block_stats"] = stats[flag]
    res["stream_bytes"] = int(s.size)
    res["steps"] = a.ring_steps
    return res


def synth(gib, kind, rs=RECSIZE):
    """the generator's stream of about `gib` GiB of `rs`-byte records"""
    return O.synth_stream(max(1, int(gib * (1 << 30)) // (rs + 312)), rs, kind, nthreads=NTH)


def keyed(O, s, threads, codec, ashift=9):
    """block_ref.as_on_disk(O, s, ashift, codec)[0] for codec DC_LZ4, DC_LZJB, DC_ZLE or gzip-N (or a
    function of the record index that returns one), with the frames and their Fletcher-4 taken on
    `threads` threads (the C encoders, zlib and checksum release the GIL)"""
    import numpy as np
    s = np.array(s, dtype=np.uint8, copy=True)
    pick = codec if callable(codec) else (lambda i: codec)
    todo = [(i, off, po, pl) for i, (off, po, pl, t) in enumerate(R.records(s)) if t == 3 and s[off + 50] == 0]

    def key(job):
        i, _, po, pl = job
        logical = s[po:po + pl]
        dc = pick(i)
        fr = None if dc == R.DC_OFF else GZ.disk_frame(O, logical, ashift, dc)
        if fr is None:
            return O.fletcher4(logical), R.prop(pl, pl, R.DC_OFF)
        return O.fletcher4(np.ascontiguousarray(fr)), R.prop(pl, fr.size, dc)

    with ThreadPoolExecutor(threads) as ex:
        keys = list(ex.map(key, todo, chunksize=256))
    for (_, off, _, _), (k, p) in zip(todo, keys):
        R.set_key(s, off, R.FLETCHER4, k, p)
    assert O.stream_restamp(s)[0] == 0
    return s


# ---- the workloads ------------------------------------------------------------------------------------

def block_cksum(a):
    legs = pair(("off", {}), ("on", {"block_checksums": True}))
    c = R.as_send_c(O, keyed(O, synth(a.recompress_gib, O.PAYLOAD_PGPAGE), NTH, R.DC_LZ4))
    return {"verify": resident(a, "verify", synth(a.verify_gib, O.PAYLOAD_PCG), legs),
            "recompress": resident(a, "recompress", c, legs)}


def block_sha(a, hash_name):
    kern, blk = HASHES[hash_name]
    legs = pair(("cksum", {}), (hash_name, {"block_" + hash_name: True}), block_checksums=True)

    def sha_keyed(s):
        return R.as_sha(O, s, hash_name, threads=NTH)

    v = resident(a, "verify", sha_keyed(synth(a.verify_gib, O.PAYLOAD_PCG)), legs, (kern,))
    v["hashed_bytes_per_step"] = v["block_stats"][hash_name] * (RECSIZE + blk)
    if v.get(kern + "_ms_per_step"):
        v[kern + "_gbps"] = v["hashed_bytes_per_step"] / (v[kern + "_ms_per_step"] * 1e6)
    res = {"verify": v, "host": {}}
    for rs in (RECSIZE, 1 << 20):
        res["host"]["recsize_%d" % rs] = host(a, "verify", sha_keyed(synth(a.host_gib, O.PAYLOAD_PCG, rs)), legs)
    c = R.as_send_c(O, sha_keyed(keyed(O, synth(a.recompress_gib, O.PAYLOAD_PGPAGE), NTH, R.DC_LZ4)))
    res["recompress"] = resident(a, "recompress", c, legs, (kern,))
    return res


def frame_legs(a, legs, codec, kernels):
    """resident VERIFY, host VERIFY and the ring API over pg-page records keyed for `codec`"""
    def stream(gib, rs=RECSIZE):
        return keyed(O, synth(gib, O.PAYLOAD_PGPAGE, rs), NTH, codec)

    res = {"verify": resident(a, "verify", stream(a.verify_gib), legs, kernels, counters=tuple(legs)), "host": {}}
    for rs in (RECSIZE, 1 << 20):
        s = stream(a.host_gib, rs)
        for bb in (32 << 20, 256 << 20):
            r = host(a, "verify", s, {name: dict(kw, batch_bytes=bb) for name, kw in legs.items()})
            res["host"]["recsize_%d_batch_%dMiB" % (rs, bb >> 20)] = dict(r, batch_bytes=bb)
        del s
    res["ring"] = ring(a, stream(a.ring_gib), legs)
    return res


def block_frames(a):
    return frame_legs(a, pair(("cksum", {}), ("frames", {"block_frames": True}), block_checksums=True), R.DC_LZ4,
                      ("k3_lz4_encode", "k_frame_sums", "k_frame_plan"))


def block_lzjb(a):
    # the flag leg keeps block_frames' leg name, "frames"
    legs = pair(("cksum", {}), ("frames", {"block_lzjb": True}), block_checksums=True)
    kernels = ("k_lzjb_encode", "k_zle_encode", "k_frame_sums", "k_frame_plan")
    res = frame_legs(a, legs, R.DC_LZJB, kernels)
    zle = keyed(O, synth(a.zle_gib, O.PAYLOAD_PGPAGE), NTH, R.DC_ZLE)
    res["zle"] = resident(a, "verify", zle, legs, kernels, counters=tuple(legs))
    return res


def block_logical(a):
    import numpy as np
    from manatee_b200 import index_host
    kernels = ("k_logical_plan", "k_lzjb_encode", "k_zle_encode", "k_frame_sums", "k_block_check", "k_block_sha256",
               "k3_lz4_encode", "k2_lz4_decode")

    def with_flags(**shared):
        return pair(("base", {}), ("logical", {"block_logical": True}), block_checksums=True, **shared)

    def run(mode, s, legs):
        r = resident(a, mode, s, legs, kernels, counters=tuple(legs))
        return dict(r, logical_bytes=int(index_host(s)[0]["lsize"].sum()))

    lzjb = with_flags(block_lzjb=True)
    res = {}
    for gib in (a.gib, a.large_gib):
        s = keyed(O, synth(gib, O.PAYLOAD_PGPAGE), NTH, R.DC_LZJB)
        res["compress_lzjb_%gGiB" % gib] = run("compress", s, lzjb)
        res["decompress_lzjb_%gGiB" % gib] = run("decompress", R.send_c_form(O, s), lzjb)
        del s
    x = np.ascontiguousarray(synth(a.gib, O.PAYLOAD_PGPAGE))
    res["recompress_raw_keys_fletcher4"] = run("recompress", R.send_c_form(O, x), with_flags())
    x = R.as_sha(O, x, "sha256", NTH)
    res["recompress_raw_keys_sha256"] = run("recompress", R.send_c_form(O, x), with_flags(block_sha256=True))
    del x
    s = keyed(O, synth(a.host_gib, O.PAYLOAD_PGPAGE), NTH, R.DC_LZJB)
    res["host_compress_lzjb"] = host(a, "compress", s, lzjb)
    return res


def lz4hc(a):
    # the two encoders write different frames by design: no outputs_equal, the wire bytes of each instead
    # (payload frames + headers; the host legs' with their wire preambles)
    legs = pair(("zfs", {}), ("hc", {"lz4_hc": True}))

    def wire(name, ob, nbytes):
        return {name + "_wire_bytes": int(ob), name + "_ratio": nbytes / ob}

    res = {"payload": "pg-page 128 KiB records (oracle.gen_payload(PAYLOAD_PGPAGE, r, 131072))"}
    s = synth(a.gib, O.PAYLOAD_PGPAGE)
    res["resident_compress_%gGiB" % a.gib] = resident(
        a, "compress", s, legs, ("k3h_lz4hc_encode", "k3_lz4_encode"), counters=(), rate="input_gbps",
        same_output=False,
        fields=lambda name, g, ob: dict(wire(name, ob, s.size), **{name + "_lz4_encoded": g.stats()["lz4_encoded"]}))
    h = synth(a.host_gib, O.PAYLOAD_PGPAGE)
    res["host_compress_%gGiB" % a.host_gib] = host(a, "compress", h, legs, counters=(), rate="input_gbps",
                                                   fields=lambda name, g, ob: wire(name, ob, h.size))
    return res


CIN_STREAMS = (("lz4_ashift9", R.DC_LZ4, 9), ("lz4_ashift12", R.DC_LZ4, 12), ("lzjb", R.DC_LZJB, 9),
               ("zle", R.DC_ZLE, 9), ("mixed_codecs", R.mixed_codecs, 9))


def compressed_in(a):
    """each leg COMPRESSes its own form of the same data: "plain" the stream today's sender pipes (plain(x),
    which for these streams is the keyed stream itself), "send_c" the `zfs send -c` stream x with the flag.
    Both wires decode to the same plain stream; the check here is that the "send_c" wire DECOMPRESSes
    to the "plain" leg's input."""
    return send_c_legs(a, CIN_STREAMS, {"compressed_input": True}, ("k_lzjb_decode", "k_zle_decode", "k3_lz4_encode"))


def send_c_legs(a, streams, flag_kw, kernels, fields=None):
    """compressed_in's legs over each of `streams` (name, codec, ashift), the "send_c" leg opened with
    `flag_kw`; `fields(r, p, x)` adds a stream's own fields"""
    import numpy as np
    import torch
    import bench
    from manatee_b200 import GpuSnapshotStage, index_host
    names = ("plain", "send_c")
    kw = {"plain": {}, "send_c": flag_kw}
    res = {"payload": "pg-page 128 KiB records (oracle.gen_payload(PAYLOAD_PGPAGE, r, 131072))"}
    for sname, codec, ashift in streams:
        p = keyed(O, synth(a.gib, O.PAYLOAD_PGPAGE), NTH, codec, ashift)
        x = GZ.as_send_c(O, p, ashift)
        src = {"plain": p, "send_c": x}
        logical = int(index_host(p)[0]["lsize"].sum())
        r = {"logical_bytes": logical, "plain_bytes": int(p.size), "send_c_bytes": int(x.size)}
        # resident steps, alternating
        bufs = {}
        for n in names:
            recs, _ = index_host(src[n])
            d_in = torch.from_numpy(src[n]).cuda()
            d_recs = torch.from_numpy(recs.view(np.uint8).copy()).cuda()
            cap = int(np.maximum(recs["lsize"], recs["payload"]).sum()) + 312 * len(recs) + (1 << 20)
            bufs[n] = (d_in, d_recs, len(recs), torch.empty(cap, dtype=torch.uint8, device="cuda"), cap)
        st = torch.cuda.Stream()
        ms, wire = {n: [] for n in names}, {}
        with ExitStack() as es:
            gs = {n: es.enter_context(GpuSnapshotStage("compress", **kw[n])) for n in names}

            def step(n):
                g, (d_in, d_recs, nrec, d_out, cap) = gs[n], bufs[n]
                g.dev_reset()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                g.dev_submit(d_in.data_ptr(), d_in.numel(), d_recs.data_ptr(), nrec, d_out.data_ptr(), cap,
                             cuda_stream=st.cuda_stream)
                ob = g.dev_finish()[0]
                e1.record(st)
                torch.cuda.synchronize()
                return e0.elapsed_time(e1), ob

            for i, n in alternate(kw, a.warmup + a.steps):
                t, ob = step(n)
                if i >= a.warmup:
                    ms[n].append(t)
                wire[n] = ob
            r["resident"] = summary(names, ms, logical, "logical_gbps")
            for n in names:
                r["resident"][n + "_wire_bytes"] = int(wire[n])
                r["resident"][n + "_lz4_encoded"] = gs[n].stats()["lz4_encoded"]
            r["compressed_in_stats"] = gs["send_c"].compressed_in_stats()
            if a.profile_steps:
                r["resident"].update(kernel_times(partial(step, "send_c"), a.profile_steps, kernels))
        del bufs
        torch.cuda.empty_cache()
        # mtz_process_host, alternating; the send_c wire must decode to the plain stream
        out = np.zeros(p.size + (64 << 20), dtype=np.uint8)
        hms = {n: [] for n in names}
        with ExitStack() as es:
            gs = {n: es.enter_context(GpuSnapshotStage("compress", **kw[n])) for n in names}
            for i, n in alternate(kw, 1 + a.host_steps):
                t0 = time.perf_counter()
                ob = gs[n].process_host(src[n], out)
                if i >= 1:
                    hms[n].append((time.perf_counter() - t0) * 1e3)
                r[n + "_host_wire_bytes"] = int(ob)
            with GpuSnapshotStage("decompress") as d:
                back = np.zeros(p.size + (1 << 20), dtype=np.uint8)
                nb = d.process_host(out[:ob], back)
                r["decompressed_equals_plain"] = bool(nb == p.size and np.array_equal(back[:nb], p))
        r["host"] = summary(names, hms, logical, "logical_gbps")
        del out
        # the ring API fed through a pipe: the shape of zfsSend.stdout
        secs = {n: [] for n in names}
        for _, n in alternate(kw, a.ring_steps):
            with GpuSnapshotStage("compress", **kw[n]) as g:
                dt, ok, detail = bench.ring_run(g, src[n], producer="pipe")
                assert ok, detail
                secs[n].append(dt)
        r["ring_pipe"] = {n + "_logical_gbps_mean": logical / (sum(v) / len(v)) / 1e9 for n, v in secs.items()}
        r["ring_pipe"].update({n + "_input_gbps_mean": src[n].size / (sum(v) / len(v)) / 1e9
                               for n, v in secs.items()})
        if fields is not None:
            fields(r, p, x)
        res[sname] = r
        del p, x, src
    return res


GZIP_STREAMS = (("gzip1", GZ.DC_GZIP[1], 9), ("gzip6", GZ.DC_GZIP[6], 9), ("gzip9", GZ.DC_GZIP[9], 9),
                ("mixed_gzip6_lz4_lzjb_raw", lambda i: (GZ.DC_GZIP[6], R.DC_LZ4, R.DC_LZJB, R.DC_OFF)[i % 4], 9))


def gzip_in(a):
    """compressed_in's legs over gzip pools, the "send_c" leg with compressed_input + gzip_input; plus
    the single-thread zlib.decompress rate of the same gzip records, as context for what the sending
    host's CPU spends on them without -c"""
    import zlib

    def zlib_rate(r, p, x):
        frames = [x[po:po + pl].tobytes() for _, off, po, pl in CI.write_records(x) if GZ.is_gzip(int(x[off + 50]))]
        if not frames:
            return
        t0 = time.perf_counter()
        n = sum(len(zlib.decompress(f)) for f in frames)
        r["zlib_decompress_1thread_logical_gbps"] = n / (time.perf_counter() - t0) / 1e9
        r["gzip_records"] = len(frames)

    return send_c_legs(a, GZIP_STREAMS, {"compressed_input": True, "gzip_input": True},
                       ("k_inflate", "k_lzjb_decode", "k3_lz4_encode"), zlib_rate)


def dev_legs(a, legs, logical, profile=None, kernels=()):
    """resident steps of `legs` {name: (mode, GpuSnapshotStage keyword arguments, input stream)}, alternating:
    ms per dev_submit + dev_finish (CUDA events on a side stream), output bytes and the output of the last
    step per leg; with `profile` that leg's `kernels` device time (a pass of its own)"""
    import numpy as np
    import torch
    from manatee_b200 import GpuSnapshotStage, index_host
    bufs = {}
    for n, (_, _, src) in legs.items():
        recs, _ = index_host(src)
        cap = int(np.maximum(recs["lsize"], recs["payload"]).sum()) + 312 * len(recs) + (1 << 20)
        bufs[n] = (torch.from_numpy(src).cuda(), torch.from_numpy(recs.view(np.uint8).copy()).cuda(), len(recs),
                   torch.empty(cap, dtype=torch.uint8, device="cuda"), cap)
    st = torch.cuda.Stream()
    ms, nout, outs = {n: [] for n in legs}, {}, {}
    with ExitStack() as es:
        gs = {n: es.enter_context(GpuSnapshotStage(mode, **kw)) for n, (mode, kw, _) in legs.items()}

        def step(n):
            g, (d_in, d_recs, nrec, d_out, cap) = gs[n], bufs[n]
            g.dev_reset()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            g.dev_submit(d_in.data_ptr(), d_in.numel(), d_recs.data_ptr(), nrec, d_out.data_ptr(), cap,
                         cuda_stream=st.cuda_stream)
            ob = g.dev_finish()[0]
            e1.record(st)
            torch.cuda.synchronize()
            return e0.elapsed_time(e1), ob

        for i, n in alternate(legs, a.warmup + a.steps):
            t, ob = step(n)
            if i >= a.warmup:
                ms[n].append(t)
            nout[n] = int(ob)
        for n in legs:
            outs[n] = bufs[n][3][:nout[n]].cpu().numpy()
        names = list(legs)
        res = {}
        for k in range(1, len(names)):
            res.update(summary((names[0], names[k]), ms, logical, "logical_gbps"))
            res[names[k] + "_diff_ms_mean"] = res.pop("diff_ms_mean")
            res[names[k] + "_diff_pct_mean"] = res.pop("diff_pct_mean")
        res.update({n + "_out_bytes": nout[n] for n in names})
        res["compressed_in_stats"] = {n: gs[n].compressed_in_stats() for n in names}
        res["lz4_decoded"] = {n: gs[n].stats()["lz4_decoded"] for n in names}
        if profile is not None and a.profile_steps:
            res[profile + "_kernels"] = kernel_times(partial(step, profile), a.profile_steps, kernels)
    del bufs
    torch.cuda.empty_cache()
    return res, outs


def host_legs(a, legs, logical):
    """wall ms per mtz_process_host pass of `legs` (as dev_legs), 1 warm-up and --host-steps timed,
    alternating; the output of each leg's last pass"""
    import numpy as np
    from manatee_b200 import GpuSnapshotStage
    hms, outs = {n: [] for n in legs}, {}
    with ExitStack() as es:
        gs = {n: es.enter_context(GpuSnapshotStage(mode, **kw)) for n, (mode, kw, _) in legs.items()}
        for i, n in alternate(legs, 1 + a.host_steps):
            src = legs[n][2]
            out = np.zeros(src.size * 4 + (64 << 20), dtype=np.uint8)
            t0 = time.perf_counter()
            ob = gs[n].process_host(src, out)
            if i >= 1:
                hms[n].append((time.perf_counter() - t0) * 1e3)
            outs[n] = out[:ob].copy()
            del out
    names = list(legs)
    res = {}
    for k in range(1, len(names)):
        res.update(summary((names[0], names[k]), hms, logical, "logical_gbps"))
        res[names[k] + "_diff_ms_mean"] = res.pop("diff_ms_mean")
        res[names[k] + "_diff_pct_mean"] = res.pop("diff_pct_mean")
    return res, outs


def gzip_wire(a):
    """the sender and the receiver of MTZ_FLAG_GZIP_WIRE on the pools of gzip_in (module docstring)"""
    import numpy as np
    import bench
    from manatee_b200 import GpuSnapshotStage, index_host
    today = {"compressed_input": True, "gzip_input": True}
    flag = {"compressed_input": True, "gzip_wire": True}
    res = {"payload": "pg-page 128 KiB records (oracle.gen_payload(PAYLOAD_PGPAGE, r, 131072))"}
    for sname, codec, ashift in GZIP_STREAMS:
        if sname not in a.pools.split(","):
            continue
        p = keyed(O, synth(a.gib, O.PAYLOAD_PGPAGE), NTH, codec, ashift)
        x = GZ.as_send_c(O, p, ashift)
        logical = int(index_host(p)[0]["lsize"].sum())
        r = {"logical_bytes": logical, "plain_bytes": int(p.size), "send_c_bytes": int(x.size),
             "gzip_records": sum(1 for _, off, _, _ in CI.write_records(x) if GZ.is_gzip(int(x[off + 50])))}
        send = {"lz4_wire": ("compress", today, x), "gzip_wire": ("compress", flag, x)}
        r["sender_resident"], _ = dev_legs(a, send, logical)
        r["sender_host"], wires = host_legs(a, send, logical)
        r["lz4_wire_bytes"], r["gzip_wire_bytes"] = int(wires["lz4_wire"].size), int(wires["gzip_wire"].size)
        r["wire_saving_pct"] = 100.0 * (1 - r["gzip_wire_bytes"] / r["lz4_wire_bytes"])
        r["gzip_wire_equals_the_model"] = bool(np.array_equal(wires["gzip_wire"], GW.splice(O, wires["lz4_wire"], x)))
        secs = {n: [] for n in send}
        for _, n in alternate(send, a.ring_steps):
            with GpuSnapshotStage("compress", **send[n][1]) as g:
                dt, ok, detail = bench.ring_run(g, x, producer="pipe")
                assert ok, detail
                secs[n].append(dt)
        r["sender_ring_pipe"] = {n + "_logical_gbps_mean": logical / (sum(v) / len(v)) / 1e9 for n, v in secs.items()}
        # the receiver: the device API takes the wire without its preambles
        want = GZ.plain(O, x)
        lzw, gzw = wires["lz4_wire"], wires["gzip_wire"]
        recv = {"lz4_wire": ("decompress", {}, O.wire_strip(lzw)), "gzip_wire": ("decompress", {"gzip_wire": True},
                O.wire_strip(gzw)), "flag_on_lz4_wire": ("decompress", {"gzip_wire": True}, O.wire_strip(lzw))}
        r["receiver_resident"], outs = dev_legs(a, recv, logical, "gzip_wire", ("k_inflate", "k2_lz4_decode"))
        recv_host = {n: (m, kw, {"lz4_wire": lzw, "gzip_wire": gzw, "flag_on_lz4_wire": lzw}[n])
                     for n, (m, kw, _) in recv.items()}
        r["receiver_host"], houts = host_legs(a, recv_host, logical)
        r["decompressed_equals_plain"] = {n: bool(np.array_equal(houts[n], want)) for n in recv}
        r["resident_decompressed_equals_plain"] = {n: bool(np.array_equal(outs[n], want)) for n in recv}
        res[sname] = r
        del p, x, wires, outs, houts
    return res


def gzip_encode(a):
    """MTZ_FLAG_GZIP_ENCODE (module docstring): a raw pg-page stream, and a `send -c` stream of the
    block_ref.mixed_codecs pool with compressed_input"""
    import numpy as np
    import bench
    import gzip_encode_ref as GE
    from manatee_b200 import GpuSnapshotStage, index_host
    res = {"payload": "pg-page 128 KiB records (oracle.gen_payload(PAYLOAD_PGPAGE, r, 131072))"}
    p = synth(a.gib, O.PAYLOAD_PGPAGE)
    m = synth(a.mixed_gib, O.PAYLOAD_PGPAGE)
    for sname, x, kw in (("pgpage", p, {}), ("mixed_codecs_send_c", CI.send_c(O, m, 9, R.mixed_codecs),
                                            {"compressed_input": True})):
        logical = int(index_host(CI.plain(O, x) if kw else x)[0]["lsize"].sum())
        r = {"logical_bytes": logical, "input_bytes": int(x.size)}
        send = {"lz4_wire": ("compress", kw, x), "gzip_encode": ("compress", dict(kw, gzip_encode=True), x)}
        r["sender_resident"], _ = dev_legs(a, send, logical, "gzip_encode", ("k3_lz4_encode", "k_deflate_from_lz4"))
        r["sender_host"], wires = host_legs(a, send, logical)
        r["lz4_wire_bytes"], r["gzip_wire_bytes"] = int(wires["lz4_wire"].size), int(wires["gzip_encode"].size)
        r["wire_saving_pct"] = 100.0 * (1 - r["gzip_wire_bytes"] / r["lz4_wire_bytes"])
        r["wire_records_lz4_gzip"] = GE.counts(O, wires["gzip_encode"])
        secs = {n: [] for n in send}
        for _, n in alternate(send, a.ring_steps):
            with GpuSnapshotStage("compress", **send[n][1]) as g:
                dt, ok, detail = bench.ring_run(g, x, producer="pipe")
                assert ok, detail
                secs[n].append(dt)
        r["sender_ring_pipe"] = {n + "_logical_gbps_mean": logical / (sum(v) / len(v)) / 1e9 for n, v in secs.items()}
        lzw, gzw = wires["lz4_wire"], wires["gzip_encode"]
        want = CI.plain(O, x) if kw else x
        recv = {"lz4_wire": ("decompress", {}, O.wire_strip(lzw)),
                "gzip_encode": ("decompress", {"gzip_wire": True}, O.wire_strip(gzw))}
        r["receiver_resident"], outs = dev_legs(a, recv, logical, "gzip_encode", ("k_inflate", "k2_lz4_decode"))
        r["resident_decompressed_equals_input"] = {n: bool(np.array_equal(outs[n], want)) for n in recv}
        res[sname] = r
        del x, wires, outs
    return res


SHA_OPTIONS = dict(verify_gib=16.0, host_gib=2.0, recompress_gib=1.0, steps=10, warmup=2, host_steps=4,
                   profile_steps=3)
FRAME_OPTIONS = dict(verify_gib=16.0, host_gib=2.0, ring_gib=8.0, steps=10, warmup=2, host_steps=4, ring_steps=3,
                     profile_steps=3)
# subcommand -> (workload, its options and their defaults)
WORKLOADS = {
    "block_cksum": (block_cksum, dict(verify_gib=16.0, recompress_gib=1.0, steps=10, warmup=2)),
    "block_sha256": (partial(block_sha, hash_name="sha256"), SHA_OPTIONS),
    "block_sha512": (partial(block_sha, hash_name="sha512"), SHA_OPTIONS),
    "block_frames": (block_frames, FRAME_OPTIONS),
    "block_lzjb": (block_lzjb, dict(FRAME_OPTIONS, zle_gib=4.0)),
    "block_logical": (block_logical, dict(gib=1.0, large_gib=4.0, host_gib=2.0, steps=10, warmup=2, host_steps=4,
                                          profile_steps=3)),
    "lz4hc": (lz4hc, dict(gib=1.0, host_gib=1.0, steps=5, warmup=1, host_steps=3, profile_steps=2)),
    "compressed_in": (compressed_in, dict(gib=0.5, steps=5, warmup=1, host_steps=3, ring_steps=3, profile_steps=2)),
    "gzip_in": (gzip_in, dict(gib=0.5, steps=5, warmup=1, host_steps=3, ring_steps=3, profile_steps=2)),
    "gzip_wire": (gzip_wire, dict(gib=0.5, steps=5, warmup=1, host_steps=3, ring_steps=3, profile_steps=2,
                                  pools=",".join(s[0] for s in GZIP_STREAMS))),
    "gzip_encode": (gzip_encode, dict(gib=0.5, mixed_gib=0.125, steps=5, warmup=1, host_steps=3, ring_steps=3, profile_steps=2)),
}


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="cost of a GpuSnapshotStage flag on the GPU")
    sub = ap.add_subparsers(dest="workload", required=True)
    for name, (_, options) in WORKLOADS.items():
        sp = sub.add_parser(name)
        for k, v in options.items():
            sp.add_argument("--" + k.replace("_", "-"), type=type(v), default=v)
        sp.add_argument("--out", default=None)
    return ap.parse_args(argv)


def main(argv=None):
    a = parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        sys.exit("flag_cost.py %s measures device time: it needs a GPU" % a.workload)
    O.build()
    result = {"tool": a.workload + "_cost", **gpu_info(), "steps": a.steps, "warmup": a.warmup,
              **WORKLOADS[a.workload][0](a)}
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
