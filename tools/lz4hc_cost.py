#!/usr/bin/env python
"""Wire size and cost of MTZ_FLAG_LZ4_HC (COMPRESS with the high-ratio LZ4 encoder K3h instead of K3) on
the pg-page payload model, each leg against a handle without the flag on the same stream, the two
handles alternating step by step.

  resident  COMPRESS over the device API (dev_submit + dev_finish, CUDA events) of --gib of pg-page
            128 KiB records resident in HBM; the HC step's kernel times come from torch.profiler in a
            pass of its own
  host      mtz_process_host COMPRESS of --host-gib at the default batch size (host clock)
Each leg reports the wire bytes (payload frames + headers; the host leg with its wire preambles), the
ratio stream bytes / wire bytes, ms per step and the input rate.  Prints one JSON line (and writes it to
--out) with the GPU name, power limit and max SM clock.
usage: tools/lz4hc_cost.py [--gib 1] [--host-gib 1] [--steps 5] [--warmup 1] [--out F]"""
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

LEGS = ("zfs", "hc")
KERNELS = ("k3h_lz4hc_encode", "k3_lz4_encode")


def _stage(leg, **kw):
    from manatee_b200 import GpuSnapshotStage
    return GpuSnapshotStage("compress", lz4_hc=(leg == "hc"), **kw)


def _summary(ms, nbytes):
    res = {}
    for name in LEGS:
        v = sorted(ms[name])
        res[name + "_ms_mean"] = sum(v) / len(v)
        res[name + "_ms_median"] = v[len(v) // 2]
        res[name + "_ms_min"] = v[0]
        res[name + "_ms_max"] = v[-1]
        res[name + "_input_gbps"] = nbytes / (res[name + "_ms_mean"] * 1e6)
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
    cap = s.size + (1 << 20)
    d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
    st = torch.cuda.Stream()
    legs = {name: _stage(name) for name in LEGS}
    ms = {name: [] for name in LEGS}
    wire = {}

    def step(g):
        g.dev_submit(d_in.data_ptr(), s.size, d_recs.data_ptr(), len(recs), d_out.data_ptr(), cap,
                     cuda_stream=st.cuda_stream)
        return g.dev_finish()[0]

    try:
        for i in range(warm + steps):
            for name in (LEGS if i % 2 == 0 else LEGS[::-1]):
                e0 = torch.cuda.Event(enable_timing=True)
                e1 = torch.cuda.Event(enable_timing=True)
                legs[name].dev_reset()
                torch.cuda.synchronize()
                e0.record(st)
                wire[name] = int(step(legs[name]))
                e1.record(st)
                torch.cuda.synchronize()
                if i >= warm:
                    ms[name].append(e0.elapsed_time(e1))
        res = _summary(ms, s.size)
        res["records"] = int(len(recs))
        res["stream_bytes"] = int(s.size)
        for name in LEGS:
            res[name + "_wire_bytes"] = wire[name]
            res[name + "_ratio"] = s.size / wire[name]
            res[name + "_lz4_encoded"] = legs[name].stats()["lz4_encoded"] // (warm + steps)
        if profile_steps:
            res.update(F.kernel_times(lambda: (legs["hc"].dev_reset(), step(legs["hc"])), profile_steps, KERNELS))
            res["profile_steps"] = profile_steps
        return res
    finally:
        for g in legs.values():
            g.close()


def host_legs(s, steps, warm):
    import numpy as np
    out = np.zeros(s.size + (64 << 20), dtype=np.uint8)
    legs = {name: _stage(name) for name in LEGS}
    ms = {name: [] for name in LEGS}
    wire = {}
    try:
        for i in range(warm + steps):
            for name in (LEGS if i % 2 == 0 else LEGS[::-1]):
                t0 = time.perf_counter()
                wire[name] = int(legs[name].process_host(s, out))
                dt = (time.perf_counter() - t0) * 1e3
                if i >= warm:
                    ms[name].append(dt)
        res = _summary(ms, s.size)
        res["stream_bytes"] = int(s.size)
        for name in LEGS:
            res[name + "_wire_bytes"] = wire[name]
            res[name + "_ratio"] = s.size / wire[name]
        return res
    finally:
        for g in legs.values():
            g.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=1.0)
    ap.add_argument("--host-gib", type=float, default=1.0)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--host-steps", type=int, default=3)
    ap.add_argument("--profile-steps", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("lz4hc_cost.py measures device time: it needs a GPU")
    import oracle as O
    O.build()
    nth = os.cpu_count() or 1
    result = {"tool": "lz4hc_cost", **gpu_info(), "steps": args.steps, "warmup": args.warmup,
              "payload": "pg-page 128 KiB records (oracle.gen_payload(PAYLOAD_PGPAGE, r, 131072))"}

    def raw(gib):
        n = max(1, int(gib * (1 << 30)) // (131072 + 312))
        return O.synth_stream(n, 131072, O.PAYLOAD_PGPAGE, nthreads=nth)

    result["resident_compress_%gGiB" % args.gib] = resident_legs(raw(args.gib), args.steps, args.warmup,
                                                                 args.profile_steps)
    result["host_compress_%gGiB" % args.host_gib] = host_legs(raw(args.host_gib), args.host_steps, 1)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
