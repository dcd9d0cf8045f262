#!/usr/bin/env python
"""Cost of MTZ_FLAG_BLOCK_LOGICAL (the re-encoding modes check keys from the logical bytes they hold:
k_logical_plan, k_lzjb_encode / k_zle_encode, k_frame_sums on the post stream of every sub-batch), each
leg against the same flags without it on the same stream, the two handles alternating step by step.

  compress    resident COMPRESS (device API, CUDA events) over pg-page 128 KiB records keyed as ZFS with
              compression=lzjb writes them, sent without -c: every record gets an lzjb frame for the check
  decompress  resident DECOMPRESS over the COMPRESS output of the same stream
              (both at --gib and at --large-gib, with MTZ_FLAG_BLOCK_LZJB on both handles)
  recompress  resident RECOMPRESS over the compressed form of a stream whose keys cover the logical
              blocks (a compression=off dataset), fletcher4 keys and sha256 keys: the flag adds one pass
              of Fletcher-4 or SHA-256 over K2's output
  host        mtz_process_host COMPRESS of the lzjb-keyed stream at the default batch size
Each resident leg also reports the device time of the check's kernels per step (torch.profiler, in a
pass of its own).  Prints one JSON line (and writes it to --out) with the GPU name, power limit and
max SM clock.
usage: tools/block_logical_cost.py [--gib 1] [--large-gib 4] [--host-gib 2] [--steps 10] [--warmup 2] [--out F]"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import block_frames_cost as F  # noqa: E402
from block_cksum_cost import gpu_info  # noqa: E402
from block_lzjb_cost import keyed  # noqa: E402

LEGS = ("base", "logical")
KERNELS = ("k_logical_plan", "k_lzjb_encode", "k_zle_encode", "k_frame_sums", "k_block_check", "k_block_sha256",
             "k3_lz4_encode", "k2_lz4_decode")


def _stage(mode, leg, **kw):
    from manatee_b200 import GpuSnapshotStage
    return GpuSnapshotStage(mode, block_checksums=True, block_logical=(leg == "logical"), **kw)


def _summary(ms):
    res = {}
    for name in LEGS:
        v = sorted(ms[name])
        res[name + "_ms_mean"] = sum(v) / len(v)
        res[name + "_ms_median"] = v[len(v) // 2]
        res[name + "_ms_min"] = v[0]
        res[name + "_ms_max"] = v[-1]
    res["diff_ms_mean"] = res["logical_ms_mean"] - res["base_ms_mean"]
    res["diff_pct_mean"] = 100.0 * res["diff_ms_mean"] / res["base_ms_mean"]
    return res


def resident_legs(mode, s, steps, warm, profile_steps, **kw):
    """ms per resident step of `mode` over the plain stream `s`, with and without the flag"""
    import numpy as np
    import torch
    from manatee_b200 import index_host
    recs, used = index_host(s)
    assert used == s.size
    d_in = torch.empty(s.size + 512, dtype=torch.uint8, device="cuda")
    d_in[:s.size].copy_(torch.from_numpy(s))
    d_recs = torch.from_numpy(recs.view(np.uint8).copy()).cuda()
    cap = int(np.maximum(recs["lsize"], recs["payload"]).sum()) + 312 * len(recs) + (1 << 20)
    d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
    st = torch.cuda.Stream()
    legs = {name: _stage(mode, name, **kw) for name in LEGS}
    ms = {name: [] for name in LEGS}

    def step(g):
        g.dev_submit(d_in.data_ptr(), s.size, d_recs.data_ptr(), len(recs), d_out.data_ptr(), cap,
                     cuda_stream=st.cuda_stream)
        return g.dev_finish()

    try:
        for i in range(warm + steps):
            for name in (LEGS if i % 2 == 0 else LEGS[::-1]):
                e0 = torch.cuda.Event(enable_timing=True)
                e1 = torch.cuda.Event(enable_timing=True)
                legs[name].dev_reset()
                torch.cuda.synchronize()
                e0.record(st)
                step(legs[name])
                e1.record(st)
                torch.cuda.synchronize()
                if i >= warm:
                    ms[name].append(e0.elapsed_time(e1))
        res = _summary(ms)
        res["block_stats"] = legs["logical"].block_stats()
        res["base_block_stats"] = legs["base"].block_stats()
        res["records"] = int(len(recs))
        res["stream_bytes"] = int(s.size)
        res["logical_bytes"] = int(recs["lsize"].sum())
        if profile_steps:
            res.update(F.kernel_times(lambda: (legs["logical"].dev_reset(), step(legs["logical"])), profile_steps,
                                      KERNELS))
            res["profile_steps"] = profile_steps
        return res
    finally:
        for g in legs.values():
            g.close()


def host_legs(s, steps, warm):
    import numpy as np
    out = np.zeros(s.size + (64 << 20), dtype=np.uint8)
    legs = {name: _stage("compress", name, block_lzjb=True) for name in LEGS}
    ms = {name: [] for name in LEGS}
    try:
        for i in range(warm + steps):
            for name in (LEGS if i % 2 == 0 else LEGS[::-1]):
                t0 = time.perf_counter()
                legs[name].process_host(s, out)
                dt = (time.perf_counter() - t0) * 1e3
                if i >= warm:
                    ms[name].append(dt)
        res = _summary(ms)
        for name in LEGS:
            res[name + "_gbps"] = s.size / (res[name + "_ms_mean"] * 1e6)
        res["block_stats"] = legs["logical"].block_stats()
        res["stream_bytes"] = int(s.size)
        return res
    finally:
        for g in legs.values():
            g.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=1.0)
    ap.add_argument("--large-gib", type=float, default=4.0)
    ap.add_argument("--host-gib", type=float, default=2.0)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--host-steps", type=int, default=4)
    ap.add_argument("--profile-steps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("block_logical_cost.py measures device time: it needs a GPU")
    import numpy as np
    import oracle as O
    import block_ref as R
    O.build()
    nth = os.cpu_count() or 1
    result = {"tool": "block_logical_cost", **gpu_info(), "steps": args.steps, "warmup": args.warmup}

    def raw(gib):
        n = max(1, int(gib * (1 << 30)) // (131072 + 312))
        return O.synth_stream(n, 131072, O.PAYLOAD_PGPAGE, nthreads=nth)

    for tag, gib in (("%gGiB" % args.gib, args.gib), ("%gGiB" % args.large_gib, args.large_gib)):
        s = keyed(O, raw(gib), nth, R.DC_LZJB)
        result["compress_lzjb_" + tag] = resident_legs("compress", s, args.steps, args.warmup, args.profile_steps,
                                                       block_lzjb=True)
        c = R.send_c_form(O, s)
        del s
        result["decompress_lzjb_" + tag] = resident_legs("decompress", c, args.steps, args.warmup,
                                                         args.profile_steps, block_lzjb=True)
        del c
    x = np.ascontiguousarray(raw(args.gib))
    result["recompress_raw_keys_fletcher4"] = resident_legs("recompress", R.send_c_form(O, x), args.steps,
                                                            args.warmup, args.profile_steps)
    x = R.as_sha(O, x, "sha256", nth)
    result["recompress_raw_keys_sha256"] = resident_legs("recompress", R.send_c_form(O, x), args.steps, args.warmup,
                                                         args.profile_steps, block_sha256=True)
    del x
    s = keyed(O, raw(args.host_gib), nth, R.DC_LZJB)
    result["host_compress_lzjb"] = host_legs(s, args.host_steps, 1)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
