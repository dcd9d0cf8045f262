#!/usr/bin/env python
"""Cost of MTZ_FLAG_BLOCK_FRAMES (VERIFY encodes a frame for every raw block whose key covers an LZ4
frame on disk: k_frame_plan, K3, k_frame_sums, kernels_frames.cuh), each leg against
MTZ_FLAG_BLOCK_CKSUM alone on the same stream, the two handles alternating step by step so that both
see the same machine.  Every stream is the generator's pg-page records re-keyed by as_on_disk()
(ashift 9): what `zfs send` without -c carries for a dataset with compression=lz4.

  verify  a resident 16 GiB stream of 128 KiB records (device API, CUDA events): step time, and the
          device time of K3 and of k_frame_sums per step (torch.profiler, in a pass of its own)
  host    mtz_process_host VERIFY with 128 KiB and 1 MiB records, at 32 MiB and at 256 MiB batches
          (host clock around the synchronous call)
  ring    the ring API, acquire + commit (tools/ringpump.c's native producer, bench.py's ring_run), at
          the default batch size of each leg (32 MiB without the flag, 256 MiB with it)

Prints one JSON line (and writes it to --out) with the GPU name, power limit and max SM clock.
usage: tools/block_frames_cost.py [--verify-gib 16] [--host-gib 2] [--ring-gib 8] [--steps 10]
                                  [--warmup 2] [--out F]"""
import argparse
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import block_sha256_cost as H  # noqa: E402
from block_cksum_cost import gpu_info  # noqa: E402

LEGS = ("cksum", "frames")
H.LEGS = LEGS                  # the legs block_sha256_cost._summary reports
KERNELS = ("k3_lz4_encode", "k_frame_sums", "k_frame_plan")


def _stage(mode, leg, **kw):
    from manatee_b200 import GpuSnapshotStage
    return GpuSnapshotStage(mode, block_checksums=True, block_frames=(leg == "frames"), **kw)


def lz4_keyed(O, s, threads):
    """as_on_disk(O, s) with the frames and their Fletcher-4 taken on `threads` threads"""
    import numpy as np
    import block_ref as R
    s = np.array(s, dtype=np.uint8, copy=True)
    todo = [(off, po, pl) for off, po, pl, t in R.records(s) if t == 3 and s[off + 50] == 0]

    def key(job):
        _, po, pl = job
        logical = s[po:po + pl]
        fr = R.disk_frame(O, logical, 9)
        if fr is None:
            return O.fletcher4(logical), R.prop(pl, pl, R.DC_OFF)
        return O.fletcher4(fr), R.prop(pl, fr.size, R.DC_LZ4)

    with ThreadPoolExecutor(threads) as ex:
        keys = list(ex.map(key, todo, chunksize=256))
    for (off, _, _), (k, p) in zip(todo, keys):
        R.set_key(s, off, R.FLETCHER4, k, p)
    assert O.stream_restamp(s)[0] == 0
    return s


def kernel_times(fn, n, kernels=None):
    """device ms per step of `kernels` (default KERNELS, the frame kernels; torch.profiler, CUDA
    activities), over n steps"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    res = {}
    for kern in kernels or KERNELS:
        us, calls = 0.0, 0
        for e in prof.key_averages():
            if kern in e.key:
                us += getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                calls += e.count
        res[kern + "_ms_per_step"] = us / 1000.0 / n
        res[kern + "_launches_per_step"] = calls / n
    return res


def resident_legs(s, steps, warm, profile_steps):
    import numpy as np
    import torch
    from manatee_b200 import index_host
    recs, used = index_host(s)
    assert used == s.size
    d_in = torch.empty(s.size + 512, dtype=torch.uint8, device="cuda")
    d_in[:s.size].copy_(torch.from_numpy(s))
    d_recs = torch.from_numpy(recs.view(np.uint8).copy()).cuda()
    st = torch.cuda.Stream()
    legs = {name: _stage("verify", name) for name in LEGS}
    ms = {name: [] for name in LEGS}

    def step(g):
        g.dev_submit(d_in.data_ptr(), s.size, d_recs.data_ptr(), len(recs), cuda_stream=st.cuda_stream)
        return g.dev_finish(carry_in=(0, 0, 0, 0))

    try:
        for i in range(warm + steps):
            for name in (LEGS if i % 2 == 0 else LEGS[::-1]):
                e0 = torch.cuda.Event(enable_timing=True)
                e1 = torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record(st)
                step(legs[name])
                e1.record(st)
                torch.cuda.synchronize()
                if i >= warm:
                    ms[name].append(e0.elapsed_time(e1))
        res = H._summary(ms)
        res["block_stats"] = legs["frames"].block_stats()
        res["cksum_block_stats"] = legs["cksum"].block_stats()
        res["records"] = int(len(recs))
        res["stream_bytes"] = int(s.size)
        if profile_steps:
            res.update(kernel_times(lambda: step(legs["frames"]), profile_steps))
            res["profile_steps"] = profile_steps
        return res
    finally:
        for g in legs.values():
            g.close()


def host_legs(s, steps, warm, batch_bytes):
    legs = {name: _stage("verify", name, batch_bytes=batch_bytes) for name in LEGS}
    ms = {name: [] for name in LEGS}
    try:
        for i in range(warm + steps):
            for name in (LEGS if i % 2 == 0 else LEGS[::-1]):
                t0 = time.perf_counter()
                n = legs[name].process_host(s)
                dt = (time.perf_counter() - t0) * 1e3
                assert n == s.size
                if i >= warm:
                    ms[name].append(dt)
        res = H._summary(ms)
        for name in LEGS:
            res[name + "_gbps"] = s.size / (res[name + "_ms_mean"] * 1e6)
        res["block_stats"] = legs["frames"].block_stats()
        res["batch_bytes"] = batch_bytes
        res["stream_bytes"] = int(s.size)
        return res
    finally:
        for g in legs.values():
            g.close()


def ring_legs(src, steps):
    """GB/s of the ring API, acquire + commit, each leg on a fresh handle at its default batch size"""
    import bench
    secs = {name: [] for name in LEGS}
    stats = {}
    for i in range(steps):
        for name in (LEGS if i % 2 == 0 else LEGS[::-1]):
            g = _stage("verify", name)
            try:
                dt, ok, detail = bench.ring_run(g, src, producer="acquire", nthreads=bench.pump_threads())
                assert ok, detail
                secs[name].append(dt)
                stats[name] = g.block_stats()
            finally:
                g.close()
    res = {}
    for name in LEGS:
        v = sorted(secs[name])
        res[name + "_gbps_mean"] = src.size / (sum(v) / len(v)) / 1e9
        res[name + "_gbps_min"] = src.size / v[-1] / 1e9
        res[name + "_gbps_max"] = src.size / v[0] / 1e9
    res["diff_pct_mean"] = 100.0 * (res["frames_gbps_mean"] / res["cksum_gbps_mean"] - 1.0)
    res["block_stats"] = stats["frames"]
    res["stream_bytes"] = int(src.size)
    res["steps"] = steps
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--verify-gib", type=float, default=16.0)
    ap.add_argument("--host-gib", type=float, default=2.0)
    ap.add_argument("--ring-gib", type=float, default=8.0)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--host-steps", type=int, default=4)
    ap.add_argument("--ring-steps", type=int, default=3)
    ap.add_argument("--profile-steps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("block_frames_cost.py measures device time: it needs a GPU")
    import oracle as O
    O.build()
    nth = os.cpu_count() or 1
    result = {"tool": "block_frames_cost", **gpu_info(), "steps": args.steps, "warmup": args.warmup}

    rs = 131072
    n = max(1, int(args.verify_gib * (1 << 30)) // (rs + 312))
    s = lz4_keyed(O, O.synth_stream(n, rs, O.PAYLOAD_PGPAGE, nthreads=nth), nth)
    result["verify"] = resident_legs(s, args.steps, args.warmup, args.profile_steps)
    del s

    result["host"] = {}
    for rs in (131072, 1 << 20):
        n = max(1, int(args.host_gib * (1 << 30)) // (rs + 312))
        s = lz4_keyed(O, O.synth_stream(n, rs, O.PAYLOAD_PGPAGE, nthreads=nth), nth)
        for bb in (32 << 20, 256 << 20):
            result["host"]["recsize_%d_batch_%dMiB" % (rs, bb >> 20)] = host_legs(s, args.host_steps, 1, bb)
        del s

    rs = 131072
    n = max(1, int(args.ring_gib * (1 << 30)) // (rs + 312))
    s = lz4_keyed(O, O.synth_stream(n, rs, O.PAYLOAD_PGPAGE, nthreads=nth), nth)
    result["ring"] = ring_legs(s, args.ring_steps)
    del s
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
