"""js/src/binding.cc EXECUTED without Node: the addon source is compiled together with a
miniature in-process N-API (tests/stubs/napi_mock.cc) and driven by tests/stubs/napi_harness.cc
in the order js/lib/gpuSnapshotStage.js calls it (open, watch, write..., flush, peek/consume on
every wake-up, stats, endChecksum, unwatch, close).

  CPU:  linked against tests/stubs/mtz_mock.cc (in-memory stand-in, bytes unchanged): argument
        marshalling, the eventfd -> poll thread -> threadsafe-function wake-up path, external
        ArrayBuffers, 64-bit BigInts, thrown errors carrying MTZ_E* codes and mtz_last_error;
        and against the REAL libmanatee_gpu.so, where open() must throw MTZ_ENOGPU here.
  GPU:  linked against the real library: a stream goes through the binding and the H100 and
        comes back verified / compressed exactly as the oracle says.
(The file sorts last on purpose: it is the newest test of the suite.)"""
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STUBS = os.path.join(ROOT, "tests", "stubs")
BINDING = os.path.join(ROOT, "js", "src", "binding.cc")


def _build(tmp, real):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = os.path.join(str(tmp), "napi_harness_real" if real else "napi_harness_mock")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I" + STUBS, "-pthread", "-o", exe,
           BINDING, os.path.join(STUBS, "napi_mock.cc"), os.path.join(STUBS, "napi_harness.cc")]
    if real:
        libdir = os.path.join(ROOT, "manatee_b200")
        cmd += ["-L" + libdir, "-lmanatee_gpu", "-Wl,-rpath," + libdir]
    else:
        cmd += [os.path.join(STUBS, "mtz_mock.cc")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def _run(exe, mode, data, tmp, chunk=1 << 20, env=None, name="io"):
    pi, po = os.path.join(str(tmp), name + ".in"), os.path.join(str(tmp), name + ".out")
    np.asarray(data, dtype=np.uint8).tofile(pi)
    e = dict(os.environ)
    e.update(env or {})
    r = subprocess.run([exe, str(mode), pi, po, str(chunk)], stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                       text=True, env=e, timeout=240)
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert line, (r.returncode, r.stdout, r.stderr)
    out = np.fromfile(po, dtype=np.uint8) if os.path.exists(po) else np.zeros(0, np.uint8)
    return r.returncode, json.loads(line[-1]), out


@pytest.fixture(scope="module")
def mock_exe(tmp_path_factory):
    return _build(tmp_path_factory.mktemp("napi_mock"), real=False)


@pytest.fixture(scope="module")
def real_exe(tmp_path_factory):
    return _build(tmp_path_factory.mktemp("napi_real"), real=True)


def test_binding_runs_against_the_mock_library(mock_exe, tmp_path):
    rng = np.random.default_rng(3)
    data = rng.integers(0, 256, 3_000_001, dtype=np.uint8)
    for chunk in (70_000, 1 << 20, 1):                    # partial acceptance, ring-sized, degenerate
        d = data if chunk != 1 else data[:3000]
        rc, js, out = _run(mock_exe, 0, d, tmp_path, chunk=chunk, name="c%d" % chunk)
        assert rc == 0 and js["ok"] and js["fed"] == d.size == js["out"] == js["bytesIn"] == js["bytesOut"]
        assert np.array_equal(out, d) and js["wakes"] >= 1
        # 64-bit words survive the trip as BigInts (a double would lose the low bits)
        assert js["endChecksum"] == ["1111111111111111", "ffffffffffffffff", "0000000000000003",
                                     "0000000000000004"]
    rc, js, out = _run(mock_exe, 0, np.zeros(0, np.uint8), tmp_path, name="empty")
    assert rc == 0 and js["ok"] and js["out"] == 0


def test_binding_throws_with_code_and_last_error(mock_exe, tmp_path):
    data = np.zeros(3_000_000, dtype=np.uint8)
    rc, js, _ = _run(mock_exe, 0, data, tmp_path, chunk=70_000, env={"MTZ_MOCK_FAIL_AFTER": "1000000"})
    assert rc == 3 and js["code"] == "-5" and "checksum mismatch at record 7" in js["message"]
    rc, js, _ = _run(mock_exe, 0, data, tmp_path, env={"MTZ_MOCK_NOGPU": "1"})
    assert rc == 3 and js["threw"] == "open" and js["code"] == "-10"
    rc, js, _ = _run(mock_exe, 9, data, tmp_path)         # bad mode -> MTZ_EINVAL from open
    assert rc == 3 and js["threw"] == "open" and js["code"] == "-1"


def test_binding_links_the_real_library_and_fails_loudly_without_a_gpu(real_exe, tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present: covered by the gpu-marked test")
    rc, js, _ = _run(real_exe, 0, np.zeros(4096, np.uint8), tmp_path)
    assert rc == 3 and js["threw"] == "open" and js["code"] == "-10", js     # MTZ_ENOGPU: no CPU fallback


def _check_binding_end_to_end(exe, tmp_path, oracle, nrec):
    s = oracle.synth_stream(nrec, recsize=131072, kind=oracle.PAYLOAD_PGPAGE)
    rc_o, st = oracle.stream_verify(s)
    want_ck = ["%016x" % x for x in st.end_cksum.tuple()]
    rc, js, out = _run(exe, 0, s, tmp_path, chunk=300_000, name="verify")
    assert rc == 0 and js["ok"], js
    assert np.array_equal(out, s) and js["records"] == st.records and js["endChecksum"] == want_ck
    rc_c, want, cst = oracle.stream_compress(s)
    rc, js, out = _run(exe, 1, s, tmp_path, chunk=1 << 20, name="compress")
    assert rc == 0 and js["ok"], js
    assert np.array_equal(out, want) and js["lz4Encoded"] == cst.lz4_out
    assert js["endChecksum"] == ["%016x" % x for x in cst.end_cksum.tuple()]
    bad = s.copy()
    bad[(nrec // 2) * 131384 + 5000] ^= 1
    rc, js, _ = _run(exe, 0, bad, tmp_path, name="bad")
    assert rc == 3 and js["code"] == "-5", js              # MTZ_ECKSUM surfaces as a thrown error


@pytest.mark.gpu
def test_binding_moves_a_stream_through_the_gpu(real_exe, tmp_path, oracle):
    _check_binding_end_to_end(real_exe, tmp_path, oracle, 40)


def test_binding_moves_a_stream_through_the_emulated_library(tmp_path_factory, tmp_path, oracle, emul_so):
    """the same end-to-end check with the binding linked against the WHOLE library built for the
    SIMT emulator (tests/emul/make_emul_lib.py): binding.cc -> C ABI -> engine thread -> kernels,
    all on the CPU"""
    import sys
    d = os.path.dirname(emul_so)                     # the session's one emulated build (conftest.py)
    exe = os.path.join(str(tmp_path_factory.mktemp("napi_emul")), "napi_harness_emul")
    cmd = ["g++", "-std=c++17", "-O1", "-I" + STUBS, "-pthread", "-o", exe, BINDING,
           os.path.join(STUBS, "napi_mock.cc"), os.path.join(STUBS, "napi_harness.cc"),
           "-L" + str(d), "-lmanatee_gpu_emul", "-Wl,-rpath," + str(d)]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert r.returncode == 0, r.stderr
    _check_binding_end_to_end(exe, tmp_path, oracle, 8)
