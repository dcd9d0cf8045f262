#!/usr/bin/env python
"""Cost of MTZ_FLAG_BLOCK_LZJB (VERIFY encodes an lzjb or zle frame for every raw block whose key covers
one on disk: k_frame_plan, k_lzjb_encode / k_zle_encode, k_frame_sums), each leg against
MTZ_FLAG_BLOCK_CKSUM alone on the same stream, the two handles alternating step by step.  The legs and
their measurement are tools/block_frames_cost.py's; the streams are the generator's pg-page records
re-keyed as ZFS with compression=lzjb (or zle) at ashift 9 writes them, sent without -c.

  verify  a resident 16 GiB stream of 128 KiB lzjb-keyed records (device API, CUDA events), with the
          device time of the frame kernels per step (torch.profiler, in a pass of its own)
  host    mtz_process_host VERIFY with 128 KiB and 1 MiB records, at 32 MiB and at 256 MiB batches
  ring    the ring API, acquire + commit, at the default batch size of each leg
  zle     the verify leg on a 4 GiB stream of 128 KiB zle-keyed records

Prints one JSON line (and writes it to --out) with the GPU name, power limit and max SM clock.
usage: tools/block_lzjb_cost.py [--verify-gib 16] [--host-gib 2] [--ring-gib 8] [--zle-gib 4] [--steps 10]
                                [--warmup 2] [--out F]"""
import argparse
import json
import os
import sys
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import block_frames_cost as F  # noqa: E402
from block_cksum_cost import gpu_info  # noqa: E402

F.KERNELS = ("k_lzjb_encode", "k_zle_encode", "k_frame_sums", "k_frame_plan")


def _stage(mode, leg, **kw):
    """leg "frames" of block_frames_cost's legs is the one with MTZ_FLAG_BLOCK_LZJB here"""
    from manatee_b200 import GpuSnapshotStage
    return GpuSnapshotStage(mode, block_checksums=True, block_lzjb=(leg == "frames"), **kw)


F._stage = _stage


def keyed(O, s, threads, codec):
    """block_ref.as_on_disk(O, s, 9, codec) with the frames and their Fletcher-4 taken on `threads`
    threads (the C restatement releases the GIL)"""
    import numpy as np
    import block_ref as R
    s = np.array(s, dtype=np.uint8, copy=True)
    todo = [(off, po, pl) for off, po, pl, t in R.records(s) if t == 3 and s[off + 50] == 0]

    def key(job):
        _, po, pl = job
        logical = s[po:po + pl]
        fr = R.disk_frame(O, logical, 9, codec)
        if fr is None:
            return O.fletcher4(logical), R.prop(pl, pl, R.DC_OFF)
        return O.fletcher4(np.ascontiguousarray(fr)), R.prop(pl, fr.size, codec)

    with ThreadPoolExecutor(threads) as ex:
        keys = list(ex.map(key, todo, chunksize=256))
    for (off, _, _), (k, p) in zip(todo, keys):
        R.set_key(s, off, R.FLETCHER4, k, p)
    assert O.stream_restamp(s)[0] == 0
    return s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--verify-gib", type=float, default=16.0)
    ap.add_argument("--host-gib", type=float, default=2.0)
    ap.add_argument("--ring-gib", type=float, default=8.0)
    ap.add_argument("--zle-gib", type=float, default=4.0)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--host-steps", type=int, default=4)
    ap.add_argument("--ring-steps", type=int, default=3)
    ap.add_argument("--profile-steps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("block_lzjb_cost.py measures device time: it needs a GPU")
    import oracle as O
    import block_ref as R
    O.build()
    nth = os.cpu_count() or 1
    result = {"tool": "block_lzjb_cost", **gpu_info(), "steps": args.steps, "warmup": args.warmup}

    def stream(gib, rs, codec):
        n = max(1, int(gib * (1 << 30)) // (rs + 312))
        return keyed(O, O.synth_stream(n, rs, O.PAYLOAD_PGPAGE, nthreads=nth), nth, codec)

    s = stream(args.verify_gib, 131072, R.DC_LZJB)
    result["verify"] = F.resident_legs(s, args.steps, args.warmup, args.profile_steps)
    del s
    result["host"] = {}
    for rs in (131072, 1 << 20):
        s = stream(args.host_gib, rs, R.DC_LZJB)
        for bb in (32 << 20, 256 << 20):
            result["host"]["recsize_%d_batch_%dMiB" % (rs, bb >> 20)] = F.host_legs(s, args.host_steps, 1, bb)
        del s
    s = stream(args.ring_gib, 131072, R.DC_LZJB)
    result["ring"] = F.ring_legs(s, args.ring_steps)
    del s
    s = stream(args.zle_gib, 131072, R.DC_ZLE)
    result["zle"] = F.resident_legs(s, args.steps, args.warmup, args.profile_steps)
    del s
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
