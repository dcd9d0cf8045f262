"""gpu.blockLogical through js/src/binding.cc without Node (tests/test_zz_napi_harness.py's method): the
addon, a miniature N-API and tests/stubs/napi_harness_blocks.cc, which opens the handle with the flags
js/lib/gpuSnapshotStage.js computes and reads blockStats() as the stage publishes it, linked against
the whole library built for the SIMT emulator.  The JS sources cannot run here, so the flag values
they carry are held to include/manatee_gpu.h as text."""
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import block_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STUBS = os.path.join(ROOT, "tests", "stubs")
CKSUM, LZJB, LOGICAL = 4, 64, 128


def test_the_js_stages_carry_the_header_flag_value():
    hdr = open(os.path.join(ROOT, "include", "manatee_gpu.h")).read()
    assert int(re.search(r"#define MTZ_FLAG_BLOCK_LOGICAL (\d+)u", hdr).group(1)) == LOGICAL
    snap = open(os.path.join(ROOT, "js", "lib", "gpuSnapshotStage.js")).read()
    assert re.search(r"var BLOCK_LOGICAL = %d;" % LOGICAL, snap)
    assert re.search(r"\(options\.blockLogical \? BLOCK_LOGICAL : 0\)", snap)
    fan = open(os.path.join(ROOT, "js", "lib", "gpuFanoutStage.js")).read()
    assert re.search(r"\(options\.blockLogical \? %d : 0\)" % LOGICAL, fan)
    from manatee_b200 import _native as N
    assert N.FLAG_BLOCK_LOGICAL == LOGICAL


def test_block_logical_through_the_binding_on_the_emulated_library(tmp_path, oracle, emul_so):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    d = os.path.dirname(emul_so)
    exe = os.path.join(str(tmp_path), "napi_harness_blocks")
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-I" + STUBS, "-pthread", "-o", exe,
                        os.path.join(ROOT, "js", "src", "binding.cc"), os.path.join(STUBS, "napi_mock.cc"),
                        os.path.join(STUBS, "napi_harness_blocks.cc"), "-L" + d, "-lmanatee_gpu_emul",
                        "-Wl,-rpath," + d], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert r.returncode == 0, r.stderr
    x, dcs = R.as_on_disk(oracle, oracle.synth_stream(12, recsize=8192, kind=oracle.PAYLOAD_PGPAGE), 9, R.DC_LZJB)
    ncomp = sum(1 for v in dcs.values() if v == R.DC_LZJB)
    assert ncomp > 0
    pi = os.path.join(str(tmp_path), "in")
    x.tofile(pi)
    got = {}
    for flags in (CKSUM | LZJB, CKSUM | LZJB | LOGICAL, LOGICAL):
        po = os.path.join(str(tmp_path), "out%d" % flags)
        r = subprocess.run([exe, "1", str(flags), pi, po], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True,
                           timeout=240)
        line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
        assert line, (r.returncode, r.stdout, r.stderr)
        got[flags] = (r.returncode, json.loads(line[-1]), np.fromfile(po, dtype=np.uint8))
    rc, off, out_off = got[CKSUM | LZJB]
    assert rc == 0 and off["skipped"] == ncomp and off["logicalChecked"] == off["lzjbEncoded"] == 0
    rc, on, out_on = got[CKSUM | LZJB | LOGICAL]
    assert rc == 0 and on["skipped"] == 0 and on["frameOk"] == on["lzjbEncoded"] == on["logicalChecked"] == ncomp
    assert on["logicalOk"] == off["logicalOk"] == len(dcs) - ncomp and on["firstFrameMiss"] == -1
    assert np.array_equal(out_on, out_off) and np.array_equal(out_on, oracle.stream_compress(x)[1])
    rc, js, _ = got[LOGICAL]                              # without blockChecksums: MTZ_EINVAL from open
    assert rc == 3 and js["threw"] == "open" and js["code"] == "-1"
