"""CPU: libmanatee_gpu.so loads and exports every symbol include/manatee_gpu.h
declares (no compute calls: there is no GPU here)."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_symbols():
    src = open(os.path.join(ROOT, "include", "manatee_gpu.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(mtz_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol(native):
    from manatee_b200 import _native
    hdr = _header_symbols()
    assert len(hdr) >= 20
    assert sorted(_native.SYMBOLS) == hdr, "binding table and header disagree"
    out = subprocess.check_output(["nm", "-D", "--defined-only", _native.SO_PATH]).decode()
    exported = set(re.findall(r" T (mtz_[a-z0-9_]+)", out))
    missing = [s for s in hdr if s not in exported]
    assert not missing, missing
    assert native.mtz_abi_version() == 2


def test_error_strings_and_null_handles(native):
    assert native.mtz_strerror(0) == b"ok"
    assert b"checksum" in native.mtz_strerror(-5)
    assert b"no CPU fallback" in native.mtz_strerror(-10)
    assert native.mtz_close(None) == -1
    assert native.mtz_get_stats(None, None) == -1


def test_open_without_gpu_fails_loudly(native):
    """No silent CPU fallback: on a box without an H100 mtz_open returns MTZ_ENOGPU."""
    import ctypes as C
    import torch
    from manatee_b200 import _native as N
    if torch.cuda.is_available():
        return
    cfg = N.Config()
    cfg.struct_size = C.sizeof(N.Config)
    h = C.c_void_p()
    rc = native.mtz_open(C.byref(cfg), C.byref(h))
    assert rc == N.ENOGPU
    assert b"no CPU fallback" in native.mtz_last_error(None)


def test_host_index_matches_oracle(native, oracle):
    """mtz_index_host is host-side product logic (DRR parse): same record table as the oracle."""
    import numpy as np
    from manatee_b200 import index_host
    s = oracle.synth_stream(17, recsize=4096, kind=oracle.PAYLOAD_PCG)
    recs, used = index_host(s)
    cnt, offs = oracle.stream_index(s)
    assert used == s.size and len(recs) == cnt
    assert np.array_equal(recs["off"], offs)
    assert list(recs["type"][:3]) == [0, 1, 3] and recs["type"][-1] == 5
    assert set(recs["payload"][2:-1]) == {4096}
    # a compressed stream exposes lsize/comp
    sp = oracle.synth_stream(6, recsize=131072, kind=oracle.PAYLOAD_PGPAGE)
    rc, c, st = oracle.stream_compress_plain(sp)
    recs, used = index_host(c)
    assert used == c.size
    w = recs[recs["type"] == 3]
    assert set(w["comp"]) == {15} and set(w["lsize"]) == {131072}
    assert all(w["payload"] % 512 == 0) and all(w["payload"] < 131072)
    # truncated tail: only whole records are reported
    recs2, used2 = index_host(s[:-100])
    assert len(recs2) == cnt - 1 and used2 == int(offs[-1])


def test_napi_binding_type_checks_against_the_header():
    """js/src/binding.cc is what a manatee maintainer compiles; Node is absent here, so the
    least we can do is type-check it against include/manatee_gpu.h with a stub of the N-API
    declarations, and check that the JS wrapper only calls exports the binding defines."""
    import re
    import shutil
    import subprocess
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    src = os.path.join(ROOT, "js", "src", "binding.cc")
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-Wextra", "-Werror",
                        "-I" + os.path.join(ROOT, "tests", "stubs"), src],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert r.returncode == 0, r.stderr
    text = open(src).read()
    exported = set(re.findall(r'\{"(\w+)", 0, \w+, 0, 0, 0, napi_default, 0\}', text))
    assert {"open", "write", "flush", "peek", "consume", "eventFd", "stats", "close", "acquire", "commit",
            "endChecksum"} <= exported
    js = open(os.path.join(ROOT, "js", "lib", "gpuSnapshotStage.js")).read()
    used = set(re.findall(r"this\._addon\.(\w+)\(", js))
    assert used and used <= exported, used - exported
    # every C entry point the binding calls is declared in the public header
    called = set(re.findall(r"\b(mtz_[a-z_0-9]+)\(", text))
    header = open(os.path.join(ROOT, "include", "manatee_gpu.h")).read()
    for fn in called:
        assert re.search(r"\b%s\(" % fn, header), fn


def test_record_alignment_is_part_of_the_format(native, oracle):
    """Records of a send stream are 8-byte aligned; the kernels use 64-bit header loads.  A
    length that would break that (WRITE/SPILL/BEGIN payload not a multiple of 8) is a format
    error in the host parser and in the oracle alike -- never a misaligned device access."""
    import numpy as np
    from manatee_b200 import index_host
    from manatee_b200 import _native as N

    def hdr(t, fields):
        h = np.zeros(312, dtype=np.uint8)
        h[0:4] = np.array([t], dtype=np.uint32).view(np.uint8)
        for off, (val, width) in fields.items():
            h[off:off + width] = np.array([val], dtype={4: np.uint32, 8: np.uint64}[width]).view(np.uint8)
        return h

    begin = hdr(0, {8: (0x2F5bacbac, 8), 16: (1, 8)})
    end = hdr(5, {})
    ok = np.concatenate([begin, hdr(7, {8: (8, 8), 16: (520, 8)}), np.zeros(520, np.uint8), end])
    assert len(index_host(ok)[0]) == 3 and oracle.stream_index(ok)[0] == 3
    for bad in (
        np.concatenate([begin, hdr(7, {8: (8, 8), 16: (516, 8)}), np.zeros(516, np.uint8), end]),   # SPILL 4 mod 8
        np.concatenate([begin, hdr(3, {8: (8, 8), 32: (1028, 8)}), np.zeros(1028, np.uint8), end]),  # WRITE 4 mod 8
        np.concatenate([hdr(0, {8: (0x2F5bacbac, 8), 16: (1, 8), 4: (12, 4)}), np.zeros(12, np.uint8), end]),
    ):
        with pytest.raises(N.MtzError) as ei:
            index_host(bad)
        assert ei.value.code == N.EFORMAT
        assert oracle.stream_index(bad)[0] == oracle.EFORMAT


def test_host_parser_agrees_with_the_oracle_on_mutated_headers(native, oracle):
    """mtz_index_host is product code that runs on the CPU (the streaming path parses DRR
    headers as bytes arrive): fuzz it against the oracle's walker.  Random header-field
    mutations of a stream that uses every record type must be judged the same way: same
    record table when the stream still parses, and a format error or a short parse (a length
    that now runs past the end is 'incomplete' for a streaming parser) when it does not."""
    import numpy as np
    from manatee_b200 import index_host
    from manatee_b200 import _native as N
    from test_gpu_codec import _all_types_stream
    s = _all_types_stream(oracle, seed=21)
    cnt, offs = oracle.stream_index(s)
    rng = np.random.default_rng(77)
    fields = [(0, 4), (4, 4), (8, 8), (16, 8), (28, 4), (32, 8), (50, 1), (52, 4), (96, 8)]
    agree_ok = agree_bad = 0
    for _ in range(400):
        m = s.copy()
        r = int(rng.integers(0, cnt))
        off, width = fields[int(rng.integers(0, len(fields)))]
        kind = int(rng.integers(0, 3))
        if kind == 0:
            m[int(offs[r]) + off + int(rng.integers(0, width))] ^= 1 << int(rng.integers(0, 8))
        elif kind == 1:
            m[int(offs[r]) + off:int(offs[r]) + off + width] = rng.integers(0, 256, width, dtype=np.uint8)
        else:
            m[int(offs[r]) + off:int(offs[r]) + off + width] = 0
        ocnt, ooffs = oracle.stream_index(m)
        try:
            recs, used = index_host(m)
            host_ok = used == m.size
        except N.MtzError as e:
            assert e.code == N.EFORMAT
            host_ok, recs = False, None
        if ocnt >= 0:
            assert host_ok and len(recs) == ocnt and np.array_equal(recs["off"], ooffs), (r, off, kind)
            agree_ok += 1
        else:
            assert ocnt == oracle.EFORMAT and not host_ok, (r, off, kind)
            agree_bad += 1
    assert agree_ok > 50 and agree_bad > 50, (agree_ok, agree_bad)      # both outcomes were exercised


def test_unaligned_logical_size_is_a_format_error_everywhere(native, oracle):
    """ADVICE r1 (medium): drr_logical_size becomes a PAYLOAD length in DECOMPRESS / RECOMPRESS
    output, so an LZ4 record with lsize = 1001 would misalign every record behind it (a
    misaligned-address fault on the GPU).  The host parser, the GPU parser and the oracle all
    refuse it up front, like a payload length that is not a multiple of 8."""
    import numpy as np
    from manatee_b200 import index_host
    from manatee_b200 import _native as N
    s = oracle.synth_stream(6, recsize=4096, kind=oracle.PAYLOAD_PGPAGE)
    rc, c, _ = oracle.stream_compress_plain(s)
    cnt, offs = oracle.stream_index(c)
    bad = c.copy()
    o = int(offs[3])
    assert int.from_bytes(bad[o:o + 4].tobytes(), "little") == 3 and bad[o + 50] == 15
    bad[o + 32:o + 40] = np.frombuffer((1001).to_bytes(8, "little"), dtype=np.uint8)
    assert oracle.stream_verify(bad)[0] == oracle.EFORMAT
    assert oracle.stream_recompress(bad)[0] == oracle.EFORMAT
    with pytest.raises(N.MtzError) as ei:
        index_host(bad)
    assert ei.value.code == N.EFORMAT
