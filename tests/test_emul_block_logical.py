"""MTZ_FLAG_BLOCK_LOGICAL on the CPU: the cases of tests/test_gpu_block_logical.py run against the whole
library built for the SIMT emulator (tests/emul/make_emul_lib.py: k_logical_plan, the encoders, the
frame sums, the checks and the library's launch sites, unchanged): mtz_process_host, the ring engine,
the device API across the emulated build's sub-batch edge (700 records; COMPRESS with 1 KiB records
to keep the emulated K3 affordable) and deferred shards, for every subset of the SHA and lzjb flags;
COMPRESS handed records that are already LZ4, which it cannot decode; the same
under the adversarial stream scheduler (MTZ_EMUL_ASYNC) and in a build with -fsanitize=alignment,
where a misaligned load the GPU would fault on aborts the child.  Test infrastructure only."""
import os
import shutil
import subprocess
import sys

import pytest

import test_gpu_block_logical as S
from test_emul_block_cksum import HostMem, emul_library  # noqa: F401  (fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL = os.path.join(ROOT, "tests", "emul")
ME = os.path.abspath(__file__)

INVARIANT = S.test_the_compressed_wire_counts_what_verify_counts
CASES = [("invariant-" + ("+".join(k for k in f if f[k]) or "fletcher4"), INVARIANT, (f,)) for f in S.SUBSETS] + [
    ("flag_off", S.test_without_the_flag_the_modes_count_what_they_did, ()),
    ("verify_unchanged", S.test_verify_accepts_the_flag_and_does_not_change, ()),
    ("einval", S.test_the_flag_without_block_checksums_is_einval, ()),
    ("corrupted-fletcher4", S.test_a_corrupted_raw_keyed_lz4_record_fails_the_recompress_relay, ("fletcher4",)),
    ("corrupted-sha256", S.test_a_corrupted_raw_keyed_lz4_record_fails_the_recompress_relay, ("sha256",)),
    ("corrupted-sha512", S.test_a_corrupted_raw_keyed_lz4_record_fails_the_recompress_relay, ("sha512",)),
    ("ring_api-4093", S.test_ring_api, (4093,)),
    ("ring_api-1MiB", S.test_ring_api, (1 << 20,)),
]


@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_block_logical_case_on_the_emulated_library(emul_library, oracle, name):  # noqa: F811
    fn, args = {c[0]: (c[1], c[2]) for c in CASES}[name]
    fn(oracle, *args)


def test_device_api_across_the_emulated_subbatch_edge(emul_library, oracle):  # noqa: F811
    S.device_api_subbatched(oracle, HostMem(), 800, modes=("decompress", "recompress"))


def test_device_api_compress_across_the_emulated_subbatch_edge(emul_library, oracle):  # noqa: F811
    """1 KiB records keep the emulated K3 affordable and still leave room for a 512-byte lzjb / zle frame"""
    S.device_api_subbatched(oracle, HostMem(), 800, modes=("compress",), recsize=1024)


def test_compress_of_lz4_records_on_the_emulated_library(emul_library, oracle):  # noqa: F811
    S.compress_of_lz4_records(oracle, HostMem())


def test_deferred_shards_on_the_emulated_library(emul_library, oracle):  # noqa: F811
    S.deferred_shards(oracle, HostMem())


def _child(so, select, env_extra, timeout=280):
    """this file's cases named by `select` in a child process on the library `so`"""
    env = dict(os.environ, MTZ_EMUL_SO=so, **env_extra)
    code = ("import sys, pytest; import manatee_b200._native as N; N.SO_PATH=%r; N._lib=None; "
            "sys.exit(pytest.main(['-q', '-x', '-p', 'no:cacheprovider', %r, '-k', %r]))" % (so, ME, select))
    r = subprocess.run([sys.executable, "-c", code], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True,
                       env=env, cwd=ROOT, timeout=timeout)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert " passed" in r.stdout


PATHS = "ring_api-4093 or device_api_across_the_emulated or deferred_shards or corrupted-sha256"


@pytest.mark.parametrize("seed", [1, 5])
def test_under_adversarial_scheduling(emul_library, seed):  # noqa: F811
    """any order the stream / event graph allows: the check's jobs read the input batch, K2's output and
    the job tables on the post stream, and the next sub-batch of the same scratch set must not start
    its K2 before they are done"""
    _child(emul_library._name, PATHS, {"MTZ_EMUL_ASYNC": str(seed)})


def test_no_misaligned_access_in_an_alignment_sanitized_build(tmp_path):
    """x86 forgives a misaligned load, the GPU faults: the library built with -fsanitize=alignment
    -fno-sanitize-recover aborts on the first one (input payloads at header + 312, K2's 16-aligned
    slots, the check's own slots)"""
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    probe = subprocess.run(["g++", "-fsanitize=alignment", "-x", "c++", "-", "-o", os.path.join(str(tmp_path), "p")],
                           input="int main(){return 0;}", text=True, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    if probe.returncode != 0:
        pytest.skip("g++ has no -fsanitize=alignment runtime")
    sys.path.insert(0, EMUL)
    import make_emul_lib as M
    gen, n = M.rewrite_launches(open(os.path.join(M.CSRC, "mtz_lib.cu")).read())
    gen = "#define EMU_SUBBATCH_RECORDS 700\n" + gen.replace("65536, scratch)", "EMU_SUBBATCH_RECORDS, scratch)")
    gen_path = os.path.join(str(tmp_path), "mtz_lib_ubsan.cc")
    with open(gen_path, "w") as f:
        f.write(gen + M.TAIL)
    so = os.path.join(str(tmp_path), "libmanatee_gpu_ubsan.so")
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-w", "-fno-extern-tls-init", "-pthread", "-shared", "-fPIC",
                        "-fsanitize=alignment", "-fno-sanitize-recover=alignment", "-I" + M.HERE, "-I" + M.CSRC,
                        "-o", so, gen_path, os.path.join(M.HERE, "warp_emul.cc")],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    ub = subprocess.run(["g++", "-print-file-name=libubsan.so"], stdout=subprocess.PIPE, text=True).stdout.strip()
    _child(so, "invariant-sha256+sha512+lzjb or deferred_shards_on", {"LD_PRELOAD": ub})
