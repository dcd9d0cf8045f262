#!/usr/bin/env python
"""Device-time cost of MTZ_FLAG_BLOCK_CKSUM on resident steps (device API, CUDA events), with the
flag off and on, the two handles alternating step by step so that both see the same machine:

  verify      a 16 GiB uncompressed stream (128 KiB records): every block is checked logically
              against its key on the input's K1 sums
  recompress  the `zfs send -c` form of a 1 GiB stream whose keys say "written with
              compression=lz4" (tests/block_ref.py): frames checked on the input

Prints one JSON line (and writes it to --out): per workload the mean step time of each leg, the
difference, the block counters, and the GPU name and power limit the numbers were taken on.
usage: tools/block_cksum_cost.py [--verify-gib 16] [--recompress-gib 1] [--steps 10] [--warmup 2] [--out F]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

RECSIZE = 131072


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


def time_legs(mode, s, steps, warm, out_cap):
    """mean ms per resident step (dev_submit + dev_finish), flag off vs on, alternating"""
    import numpy as np
    import torch
    from manatee_b200 import GpuSnapshotStage, index_host
    recs, used = index_host(s)
    assert used == s.size
    d_in = torch.empty(s.size + 512, dtype=torch.uint8, device="cuda")
    d_in[:s.size].copy_(torch.from_numpy(s))
    d_recs = torch.from_numpy(recs.view(np.uint8).copy()).cuda()
    d_out = torch.empty(out_cap, dtype=torch.uint8, device="cuda") if out_cap else None
    st = torch.cuda.Stream()
    legs = {"off": GpuSnapshotStage(mode, block_checksums=False), "on": GpuSnapshotStage(mode, block_checksums=True)}
    ms = {"off": [], "on": []}
    outs = {}
    try:
        for i in range(warm + steps):
            for name in (("off", "on") if i % 2 == 0 else ("on", "off")):
                g = legs[name]
                e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record(st)
                g.dev_submit(d_in.data_ptr(), s.size, d_recs.data_ptr(), len(recs),
                             d_out.data_ptr() if d_out is not None else 0, out_cap, cuda_stream=st.cuda_stream)
                ob, _, _ = g.dev_finish(carry_in=(0, 0, 0, 0), carry_out_in=(0, 0, 0, 0))
                e1.record(st)
                torch.cuda.synchronize()
                if i >= warm:
                    ms[name].append(e0.elapsed_time(e1))
                if i == warm + steps - 1 and d_out is not None:
                    outs[name] = (ob, d_out[:ob].view(torch.int64).sum().item())    # records are 8-byte aligned
        res = {}
        for name in ("off", "on"):
            v = sorted(ms[name])
            res[name + "_ms_mean"] = sum(v) / len(v)
            res[name + "_ms_median"] = v[len(v) // 2]
            res[name + "_ms_min"] = v[0]
        res["diff_ms_mean"] = res["on_ms_mean"] - res["off_ms_mean"]
        res["diff_pct_mean"] = 100.0 * res["diff_ms_mean"] / res["off_ms_mean"]
        res["block_stats"] = legs["on"].block_stats()
        res["records"] = int(len(recs))
        res["stream_bytes"] = int(s.size)
        if outs:
            res["outputs_equal"] = outs["off"] == outs["on"]
        return res
    finally:
        for g in legs.values():
            g.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--verify-gib", type=float, default=16.0)
    ap.add_argument("--recompress-gib", type=float, default=1.0)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("block_cksum_cost.py measures device time: it needs a GPU")
    import oracle as O
    import block_ref as R
    O.build()
    nth = os.cpu_count() or 1
    result = {"tool": "block_cksum_cost", **gpu_info(), "steps": args.steps, "warmup": args.warmup}
    n = max(1, int(args.verify_gib * (1 << 30)) // (RECSIZE + 312))
    s = O.synth_stream(n, RECSIZE, O.PAYLOAD_PCG, nthreads=nth)
    result["verify"] = time_legs("verify", s, args.steps, args.warmup, 0)
    del s
    n = max(1, int(args.recompress_gib * (1 << 30)) // (RECSIZE + 312))
    raw = O.synth_stream(n, RECSIZE, O.PAYLOAD_PGPAGE, nthreads=nth)
    disk, _ = R.as_on_disk(O, raw)
    c = R.as_send_c(O, disk)
    result["recompress"] = time_legs("recompress", c, args.steps, args.warmup, raw.size + (1 << 20))
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
