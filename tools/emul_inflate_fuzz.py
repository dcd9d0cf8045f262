#!/usr/bin/env python
"""Long mutation fuzz of k_inflate (manatee_b200/csrc/kernels_inflate.cuh) on the SIMT emulator, off the
suite: the seeded bit flips, truncations and inserted bytes of tests/test_emul_gzip_in.py over more
seeds and mutants, each frame compared with zlib byte for byte and verdict for verdict inside
guard-page buffers.  Test infrastructure only.
usage: tools/emul_inflate_fuzz.py [--seeds N] [--mutants M]"""
import argparse
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_emul_gzip_in as E  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--seeds", type=int, default=20)
    ap.add_argument("--mutants", type=int, default=200)
    a = ap.parse_args()
    inf = E.build_inflate(tempfile.mkdtemp(prefix="emul_inflate"))
    acc = rej = 0
    for seed in range(a.seeds):
        x, y = E.fuzz(inf, seed, a.mutants)
        acc, rej = acc + x, rej + y
        print("seed %d: %d accepted, %d refused, all as zlib says" % (seed, x, y), flush=True)
    print("TOTAL %d frames agree with zlib (%d accepted, %d refused)" % (acc + rej, acc, rej))
    return 0


if __name__ == "__main__":
    sys.exit(main())
