#!/usr/bin/env python
"""Cost of MTZ_FLAG_BLOCK_SHA256 (SHA-256 block keys hashed on the device by k_block_sha256), each leg
against MTZ_FLAG_BLOCK_CKSUM alone on the same stream, the two handles alternating step by step so
that both see the same machine:

  verify      a resident 16 GiB uncompressed stream of 128 KiB records with SHA-256 keys (device
              API, CUDA events): step time, k_block_sha256's device time (torch.profiler, in a pass
              of its own) and the bytes it hashes per second
  host        mtz_process_host VERIFY at the default batch size, 128 KiB and 1 MiB records (host
              clock around the synchronous call): SHA-256 is serial per record, so a batch of
              1 MiB records gives the kernel few threads and shows the latency of one hash
  recompress  the `zfs send -c` form of a resident 1 GiB stream whose SHA-256 keys say "written with
              compression=lz4": the kernel runs on the post stream ahead of the stamp chain

tools/block_sha512_cost.py runs the same legs for MTZ_FLAG_BLOCK_SHA512 (main("sha512")).

Prints one JSON line (and writes it to --out) with the GPU name and power limit the numbers were
taken on.
usage: tools/block_sha256_cost.py [--verify-gib 16] [--host-gib 2] [--recompress-gib 1] [--steps 10]
                                  [--warmup 2] [--out F]"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from block_cksum_cost import gpu_info  # noqa: E402

# the hash a run measures: its leg is the flag on top of MTZ_FLAG_BLOCK_CKSUM; `block` = the bytes of
# one compression block (a message of a 128 KiB record hashes 128 KiB + one padding block)
HASHES = {"sha256": {"kernel": "k_block_sha256", "block": 64},
          "sha512": {"kernel": "k_block_sha512", "block": 128}}
LEGS = ("cksum", "sha256")


def _stage(mode, leg):
    from manatee_b200 import GpuSnapshotStage
    return GpuSnapshotStage(mode, block_checksums=True, **({"block_" + leg: True} if leg in HASHES else {}))


def _summary(ms):
    res = {}
    for name in LEGS:
        v = sorted(ms[name])
        res[name + "_ms_mean"] = sum(v) / len(v)
        res[name + "_ms_median"] = v[len(v) // 2]
        res[name + "_ms_min"] = v[0]
        res[name + "_ms_max"] = v[-1]
    res["diff_ms_mean"] = res[LEGS[1] + "_ms_mean"] - res["cksum_ms_mean"]
    res["diff_pct_mean"] = 100.0 * res["diff_ms_mean"] / res["cksum_ms_mean"]
    return res


def resident_legs(mode, s, steps, warm, out_cap, profile_steps=0):
    """mean ms per resident step (dev_submit + dev_finish), BLOCK_CKSUM vs BLOCK_CKSUM|the hash's flag"""
    import numpy as np
    import torch
    from manatee_b200 import index_host
    recs, used = index_host(s)
    assert used == s.size
    d_in = torch.empty(s.size + 512, dtype=torch.uint8, device="cuda")
    d_in[:s.size].copy_(torch.from_numpy(s))
    d_recs = torch.from_numpy(recs.view(np.uint8).copy()).cuda()
    d_out = torch.empty(out_cap, dtype=torch.uint8, device="cuda") if out_cap else None
    st = torch.cuda.Stream()
    legs = {name: _stage(mode, name) for name in LEGS}
    ms = {name: [] for name in LEGS}
    outs = {}

    def step(g):
        g.dev_submit(d_in.data_ptr(), s.size, d_recs.data_ptr(), len(recs),
                     d_out.data_ptr() if d_out is not None else 0, out_cap, cuda_stream=st.cuda_stream)
        return g.dev_finish(carry_in=(0, 0, 0, 0), carry_out_in=(0, 0, 0, 0))[0]

    try:
        for i in range(warm + steps):
            for name in (LEGS if i % 2 == 0 else LEGS[::-1]):
                e0 = torch.cuda.Event(enable_timing=True)
                e1 = torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record(st)
                ob = step(legs[name])
                e1.record(st)
                torch.cuda.synchronize()
                if i >= warm:
                    ms[name].append(e0.elapsed_time(e1))
                if i == warm + steps - 1 and d_out is not None:
                    outs[name] = (ob, d_out[:ob].view(torch.int64).sum().item())    # records are 8-byte aligned
        res = _summary(ms)
        res["block_stats"] = legs[LEGS[1]].block_stats()
        res["records"] = int(len(recs))
        res["stream_bytes"] = int(s.size)
        if outs:
            res["outputs_equal"] = outs["cksum"] == outs[LEGS[1]]
        if profile_steps:
            res.update(kernel_time(lambda: step(legs[LEGS[1]]), profile_steps))
        return res
    finally:
        for g in legs.values():
            g.close()


def kernel_time(fn, n):
    """device time per step of the hash kernel (torch.profiler, CUDA activities), over n steps"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    kern = HASHES[LEGS[1]]["kernel"]
    us, calls = 0.0, 0
    for e in prof.key_averages():
        if kern in e.key:
            us += getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            calls += e.count
    return {kern + "_ms_per_step": us / 1000.0 / n, kern + "_launches_per_step": calls / n}


def host_legs(s, steps, warm):
    """mtz_process_host VERIFY, default batch size: mean wall ms per pass of the whole stream"""
    legs = {name: _stage("verify", name) for name in LEGS}
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
        res = _summary(ms)
        for name in LEGS:
            res[name + "_gbps"] = s.size / (res[name + "_ms_mean"] * 1e6)
        res["block_stats"] = legs[LEGS[1]].block_stats()
        res["stream_bytes"] = int(s.size)
        return res
    finally:
        for g in legs.values():
            g.close()


def main(hash_name="sha256"):
    global LEGS
    LEGS = ("cksum", hash_name)
    kern, blk = HASHES[hash_name]["kernel"], HASHES[hash_name]["block"]
    ap = argparse.ArgumentParser()
    ap.add_argument("--verify-gib", type=float, default=16.0)
    ap.add_argument("--host-gib", type=float, default=2.0)
    ap.add_argument("--recompress-gib", type=float, default=1.0)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--host-steps", type=int, default=4)
    ap.add_argument("--profile-steps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("block_%s_cost.py measures device time: it needs a GPU" % hash_name)
    import oracle as O
    import block_sha512_ref as R
    O.build()
    nth = os.cpu_count() or 1
    rekey = R.as_sha256 if hash_name == "sha256" else R.as_sha512
    result = {"tool": "block_%s_cost" % hash_name, **gpu_info(), "steps": args.steps, "warmup": args.warmup}

    rs = 131072
    n = max(1, int(args.verify_gib * (1 << 30)) // (rs + 312))
    s = rekey(O, O.synth_stream(n, rs, O.PAYLOAD_PCG, nthreads=nth), threads=nth)
    v = resident_legs("verify", s, args.steps, args.warmup, 0, args.profile_steps)
    hashed = v["block_stats"][hash_name] // (args.steps + args.warmup) * (rs + blk)
    v["hashed_bytes_per_step"] = hashed
    if v.get(kern + "_ms_per_step"):
        v[kern + "_gbps"] = hashed / (v[kern + "_ms_per_step"] * 1e6)
    result["verify"] = v
    del s

    result["host"] = {}
    for rs in (131072, 1 << 20):
        n = max(1, int(args.host_gib * (1 << 30)) // (rs + 312))
        s = rekey(O, O.synth_stream(n, rs, O.PAYLOAD_PCG, nthreads=nth), threads=nth)
        result["host"]["recsize_%d" % rs] = host_legs(s, args.host_steps, 1)
        del s

    rs = 131072
    n = max(1, int(args.recompress_gib * (1 << 30)) // (rs + 312))
    raw = O.synth_stream(n, rs, O.PAYLOAD_PGPAGE, nthreads=nth)
    disk, _ = R.as_lz4_on_disk(O, raw)
    c = R.as_send_c(O, rekey(O, disk, threads=nth))
    result["recompress"] = resident_legs("recompress", c, args.steps, args.warmup, raw.size + (1 << 20),
                                         args.profile_steps)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
