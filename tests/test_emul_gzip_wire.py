"""MTZ_FLAG_GZIP_WIRE on the CPU: the library built for the SIMT emulator (tests/emul/make_emul_lib.py), whose
every device buffer ends at a guard page -- cb.dec_gz, k_inflate's job table, included: an access past its
rec_cap entries faults.  COMPRESS -> DECOMPRESS round trips of gzip-1 / 6 / 9 and mixed gzip / lz4 / lzjb /
raw pools at 512 B to 1 MiB records, a corrupted gzip frame re-stamped past the stream checksum failing at
its record on the receiver, and the device API across the emulated build's 700-record sub-batch edge,
where the second sub-batch's k_plan_jobs refills the other scratch set's dec_gz, also under the
adversarial stream scheduler (MTZ_EMUL_ASYNC)."""
import os
import subprocess
import sys

import pytest

import test_gpu_gzip_wire as S
from test_emul_block_cksum import HostMem, emul_library  # noqa: F401  (fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ME = os.path.abspath(__file__)

CASES = [("round_trip-%s-%d" % (c, rs), S.test_round_trip_equals_the_model, (c, rs))
         for c in ("gzip-1", "gzip-6", "gzip-9", "mixed") for rs in (512, 8192, 131072)]
CASES += [
    ("round_trip-gzip-6-1MiB", S.test_round_trip_equals_the_model, ("gzip-6", 1 << 20)),
    ("round_trip-mixed-1MiB", S.test_round_trip_equals_the_model, ("mixed", 1 << 20)),
    ("ecodec", S.test_a_corrupted_frame_is_ecodec_at_the_receiver, ()),
    ("eformat", S.test_a_receiver_without_the_flag_refuses_the_gzip_wire, ()),
    ("lz4_wire", S.test_the_flag_changes_nothing_on_an_lz4_wire, ()),
    ("ring_api-4093", S.ring_api, (4093,)),
]


@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_gzip_wire_case_on_the_emulated_library(emul_library, oracle, name):  # noqa: F811
    fn, args = {c[0]: (c[1], c[2]) for c in CASES}[name]
    fn(oracle, *args)


def test_device_api_across_the_emulated_subbatch_edge(emul_library, oracle):  # noqa: F811
    """800 records: the first sub-batch fills all 700 entries of dec_gz, up to its guard page"""
    S.device_api(oracle, HostMem(), n=800, recsize=1024, codec="gzip-6")


def test_device_api_of_a_mixed_pool_on_the_emulated_library(emul_library, oracle):  # noqa: F811
    S.device_api(oracle, HostMem(), n=900, recsize=1024, codec="mixed")


@pytest.mark.parametrize("seed", [1, 5])
def test_under_adversarial_scheduling(emul_library, seed):  # noqa: F811
    """any order the stream / event graph allows: K2 and k_inflate of a sub-batch read the job tables its
    plan wrote, k_layout reads their verdicts, and the next sub-batch of the same scratch set must not
    plan before they are done"""
    env = dict(os.environ, MTZ_EMUL_SO=emul_library._name, MTZ_EMUL_ASYNC=str(seed))
    code = ("import sys, pytest; import manatee_b200._native as N; N.SO_PATH=%r; N._lib=None; "
            "sys.exit(pytest.main(['-q', '-x', '-p', 'no:cacheprovider', %r, '-k', %r]))"
            % (emul_library._name, ME, "device_api_ or ring_api-4093"))
    r = subprocess.run([sys.executable, "-c", code], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True,
                       env=env, cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert " passed" in r.stdout
