#!/usr/bin/env python
"""Cost of MTZ_FLAG_BLOCK_SHA512 (SHA-512/256 block keys hashed on the device by k_block_sha512): the
three legs of tools/block_sha256_cost.py -- resident 16 GiB VERIFY of 128 KiB records (step time,
k_block_sha512's device time from torch.profiler, bytes hashed per second), mtz_process_host VERIFY
at 128 KiB and 1 MiB records, resident RECOMPRESS of a 1 GiB `send -c` stream -- on streams with
SHA-512 keys, each against MTZ_FLAG_BLOCK_CKSUM alone, the two handles alternating step by step.

Prints one JSON line (and writes it to --out) with the GPU name and power limit the numbers were
taken on.
usage: tools/block_sha512_cost.py [--verify-gib 16] [--host-gib 2] [--recompress-gib 1] [--steps 10]
                                  [--warmup 2] [--out F]"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from block_sha256_cost import main  # noqa: E402

if __name__ == "__main__":
    main("sha512")
