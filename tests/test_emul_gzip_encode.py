"""MTZ_FLAG_GZIP_ENCODE on the CPU: the library built for the SIMT emulator (tests/emul/make_emul_lib.py), whose
every device buffer ends at a guard page -- cb.gz and cb.d_gz included, so a frame written past its slot
faults.  mtz_k_gzip_encode and COMPRESS equal the reference model (tests/gzip_encode_ref.py) frame for frame on
every payload family and at 512 B to 1 MiB records, DECOMPRESS with MTZ_FLAG_GZIP_WIRE gives the input back,
and the device API crosses the emulated build's 700-record sub-batch edge, also under the adversarial
stream scheduler (MTZ_EMUL_ASYNC)."""
import os
import subprocess
import sys

import pytest

import test_gpu_gzip_encode as S
from test_emul_block_cksum import HostMem, emul_library  # noqa: F401  (fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ME = os.path.abspath(__file__)


def _kernel_on_host_memory(oracle):
    """mtz_k_gzip_encode through the emulated runtime: host buffers stand in for device ones"""
    import ctypes as C
    import numpy as np
    from manatee_b200 import _native as N
    pays = S.kernel_payloads(oracle)

    def enc(src, dst_bytes, jobs):
        dst = np.zeros(dst_bytes + 64, dtype=np.uint8)
        j = np.array(jobs, copy=True)
        with S._stage("verify") as g:
            rc = N.lib().mtz_k_gzip_encode(g._h, src.ctypes.data, dst.ctypes.data, j.ctypes.data, len(j), None)
            assert rc == 0, N.lib().mtz_last_error(g._h)
        return dst, j
    for p, (n, f) in zip(pays, S.encode_jobs(enc, pays)):
        z = S.E.frame(oracle, p)
        assert (n == p.size) if z is None else (n == len(z) and f.tobytes() == z)
    del C


CASES = [
    ("kernel", _kernel_on_host_memory, ()),
    ("compress-pgpage", S.test_compress_equals_the_model, ("pgpage", 131072)),
    ("compress-mixed-8192", S.test_compress_equals_the_model, ("mixed", 8192)),
    ("compress-mixed-1MiB", S.test_compress_equals_the_model, ("mixed", 1 << 20)),
    ("compressed_input", S.test_with_compressed_input_and_the_gzip_wire, ()),
    ("eformat", S.test_a_receiver_without_the_flag_refuses_the_wire, ()),
    ("ring_api-4093", S.ring_api, (4093, 4)),
]


@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_gzip_encode_case_on_the_emulated_library(emul_library, oracle, name):  # noqa: F811
    fn, args = {c[0]: (c[1], c[2]) for c in CASES}[name]
    fn(oracle, *args)


def test_device_api_across_the_emulated_subbatch_edge(emul_library, oracle):  # noqa: F811
    """800 records: the first sub-batch fills all 700 entries of gz, up to its guard page"""
    S.device_api(oracle, HostMem(), n=800, recsize=2048)


@pytest.mark.parametrize("seed", [1, 5])
def test_under_adversarial_scheduling(emul_library, seed):  # noqa: F811
    """k_deflate_from_lz4 reads K3's frames and k_layout / k_assemble read its verdicts in any order the
    stream / event graph allows"""
    env = dict(os.environ, MTZ_EMUL_SO=emul_library._name, MTZ_EMUL_ASYNC=str(seed))
    code = ("import sys, pytest; import manatee_b200._native as N; N.SO_PATH=%r; N._lib=None; "
            "sys.exit(pytest.main(['-q', '-x', '-p', 'no:cacheprovider', %r, '-k', %r]))"
            % (emul_library._name, ME, "device_api_ or ring_api-4093"))
    r = subprocess.run([sys.executable, "-c", code], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True,
                       env=env, cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert " passed" in r.stdout
