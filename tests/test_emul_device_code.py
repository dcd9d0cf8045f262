"""The DEVICE code itself, on the CPU: manatee_b200/csrc/kernels_lz4.cuh (and fletcher.cuh) are
compiled by g++ against tests/emul/cuda_runtime.h -- a stub that maps the warp intrinsics onto
32 fibers switched at every *_sync -- and the very functions the GPU kernels call
(warp_lz4_encode3 in all three table flavours, warp_zfs_lz4_compress, warp_lz4_decode,
warp_fletcher / group_fletcher) are fuzzed against the oracle, inside guard-page buffers so an
out-of-bounds access is a crash.  Far more inputs than the GPU suite can afford, no GPU needed;
it is also how a kernel change can be checked for bit-exactness before it ever sees an H100.
Test infrastructure only: the product has no CPU path."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import lz4_payloads as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL = os.path.join(ROOT, "tests", "emul")
ECODEC = -6


FLAGS = ["-std=c++17", "-Wall", "-Wextra", "-Wno-unused-variable", "-Wno-unused-function", "-Wno-unknown-pragmas",
         "-fno-extern-tls-init",      # `extern __shared__` maps to `extern thread_local`
         "-I" + EMUL, "-shared", "-fPIC"]


def build(so, extra):
    r = subprocess.run(["g++"] + extra + FLAGS + ["-o", so, os.path.join(EMUL, "warp_emul.cc"),
                                                  os.path.join(EMUL, "emul_kernels.cc")],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert r.returncode == 0, r.stderr


def bind(so):
    L = C.CDLL(so)
    vp, u32, i32, sz = C.c_void_p, C.c_uint32, C.c_int, C.c_size_t
    L.emu_zfs_lz4_compress.argtypes = [vp, u32, vp, i32]
    L.emu_zfs_lz4_compress.restype = u32
    L.emu_lz4_encode_block.argtypes = [vp, u32, vp, u32, i32]
    L.emu_lz4_encode_block.restype = u32
    L.emu_zfs_lz4_decode.argtypes = [vp, u32, vp, u32]
    L.emu_zfs_lz4_decode.restype = C.c_int32
    L.emu_lz4_certify.argtypes = [vp, u32, vp, u32, i32]
    L.emu_lz4_certify.restype = C.c_int32
    L.emu_k1.argtypes = [vp, vp, u32, vp, u32, i32, u32]
    L.emu_k1.restype = C.c_int32
    L.emu_recsums_size.restype = u32
    L.emu_scan_verify.argtypes = [vp, u32, vp, vp]
    L.emu_scan_verify.restype = C.c_int32
    L.emu_codec.argtypes = [u32, vp, vp, u32, vp, vp, i32, vp]
    L.emu_codec.restype = C.c_int32
    L.emu_index.argtypes = [vp, C.c_uint64, vp, C.c_uint64, vp]
    L.emu_index.restype = C.c_int32
    L.emu_fold_carry.argtypes = [vp, u32, vp]
    L.emu_fold_carry.restype = C.c_int32
    L.emu_guard_alloc.argtypes = [sz, sz, sz]
    L.emu_guard_alloc.restype = vp
    L.emu_guard_free.argtypes = [vp, sz, sz, sz]
    return L


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    so = os.path.join(str(tmp_path_factory.mktemp("emul")), "libemul.so")
    build(so, ["-O2"])
    return bind(so)


class Guarded(object):
    """numpy view of `size` bytes whose end sits `slack` bytes before an inaccessible page"""

    def __init__(self, L, size, slack=0, front=16, data=None):
        self.L, self.size, self.slack, self.front = L, size, slack, front
        self.ptr = L.emu_guard_alloc(size, slack, front)
        assert self.ptr
        self.a = np.ctypeslib.as_array((C.c_uint8 * max(size, 1)).from_address(self.ptr))[:size]
        if data is not None:
            self.a[:] = data

    def free(self):
        self.L.emu_guard_free(self.ptr, self.size, self.slack, self.front)


def _inputs(oracle, rng, n):
    """one payload of a family of tests/lz4_payloads.py (random, zeros, periodic, tiny alphabet, far
    repeats, mixtures, ...), picked and seeded by rng"""
    return P.payload(P.FAMILIES[int(rng.integers(len(P.FAMILIES)))], int(rng.integers(0, 1 << 20)), n)


def test_k3_encoder_source_is_bit_exact_on_the_cpu(emu, oracle):
    """warp_lz4_encode3<TabU16|TabU32|Tab17> vs the oracle's serial greedy encoder: every block
    flavour, sizes on both sides of every switch, output limits that do and do not fit."""
    rng = np.random.default_rng(2024)
    sizes = [13, 14, 20, 64, 100, 1000, 1024, 4096, 8192, 20000, 65535, 65546, 65547, 65548, 100000, 131072]
    checked = 0
    for rnd in range(3):
        for n in sizes:
            p = _inputs(oracle, rng, n)
            src = Guarded(emu, n, slack=8, data=p)
            for osize in sorted({n + n // 100 + 32, n - (n >> 3) - 4 if n >= 64 else n + 32}):
                if osize <= 0:
                    continue
                want = oracle.lz4_compress_block(p, osize=osize)
                flavours = [0] if n < 65547 else [1, 2]
                for fl in flavours:
                    dst = Guarded(emu, osize, slack=0)
                    got = emu.emu_lz4_encode_block(src.ptr, n, dst.ptr, osize, fl)
                    assert got != 0xffffffff, "result not warp-uniform"
                    assert got == want.size, (n, osize, fl, got, want.size)
                    assert np.array_equal(dst.a[:got], want), (n, osize, fl)
                    dst.free()
                    checked += 1
            src.free()
    assert checked >= 100


def test_k3_zfs_frame_rules_on_the_cpu(emu, oracle):
    rng = np.random.default_rng(7)
    for n in [512, 1023, 1024, 1536, 4096, 65536, 131072]:
        for _ in range(3):
            p = _inputs(oracle, rng, n)
            ps, frame = oracle.zfs_lz4_compress(p)
            src = Guarded(emu, n, slack=8, data=p)
            for compact in ((0, 1) if n >= 65547 else (0,)):
                dst = Guarded(emu, n, slack=0)
                got = emu.emu_zfs_lz4_compress(src.ptr, n, dst.ptr, compact)
                assert got == ps, (n, compact, got, ps)
                if ps < n:
                    assert np.array_equal(dst.a[:ps], frame[:ps])
                dst.free()
            src.free()


def test_k2_decoder_source_on_the_cpu_valid_and_malformed(emu, oracle):
    """warp_lz4_decode on valid frames (== input) and on thousands of corrupted ones: it must
    agree with the oracle's safe decoder on accept / reject, produce the same bytes when it
    accepts, and never touch a byte outside [src, src+psize) or [dst, dst+lsize)."""
    rng = np.random.default_rng(99)
    n_ok = n_bad = 0
    for n in [1024, 4096, 8192, 65536, 131072]:
        for _ in range(4):
            p = _inputs(oracle, rng, n)
            ps, frame = oracle.zfs_lz4_compress(p)
            if ps >= n:
                continue
            frame = frame[:ps].copy()
            src = Guarded(emu, ps, slack=0, data=frame)
            dst = Guarded(emu, n, slack=0)
            assert emu.emu_zfs_lz4_decode(src.ptr, ps, dst.ptr, n) == 0 and np.array_equal(dst.a, p)
            clen = int.from_bytes(frame[:4].tobytes(), "big")
            for _ in range(60 if n <= 8192 else 12):
                bad = frame.copy()
                k = int(rng.integers(0, 4))
                if k == 0:
                    bad[int(rng.integers(0, clen + 4))] ^= 1 << int(rng.integers(0, 8))
                elif k == 1:
                    i = int(rng.integers(4, clen + 4))
                    bad[i:i + 4] = 255
                elif k == 2:
                    bad[:4] = np.frombuffer(int(rng.integers(0, 2 * ps)).to_bytes(4, "big"), dtype=np.uint8)
                else:
                    i = int(rng.integers(4, clen + 4))
                    bad[i:i + 2] = 0
                src.a[:] = bad
                dst.a[:] = 0xEE
                rc = emu.emu_zfs_lz4_decode(src.ptr, ps, dst.ptr, n)
                orc, oout = oracle.zfs_lz4_decompress(bad, n)
                assert rc in (0, ECODEC), rc
                assert (rc == 0) == (orc == 0), (n, k, rc, orc)
                if rc == 0:
                    assert np.array_equal(dst.a, oout)
                    n_ok += 1
                else:
                    n_bad += 1
            src.free()
            dst.free()
    assert n_ok > 5 and n_bad > 100, (n_ok, n_bad)


def _verify_on_emulator(emu, stream, lanes, grid=2, carry_in=(0, 0, 0, 0)):
    from manatee_b200 import index_host
    recs, used = index_host(stream)
    assert used == stream.size
    buf = Guarded(emu, stream.size, slack=(-stream.size) % 16, data=stream)     # 16-byte aligned, padded
    assert buf.ptr % 16 == 0
    sums = np.zeros(len(recs) * emu.emu_recsums_size(), dtype=np.uint8)
    assert emu.emu_k1(buf.ptr, recs.ctypes.data, len(recs), sums.ctypes.data, 280, lanes, grid) == 0
    cin = np.array(carry_in, dtype=np.uint64)
    out = np.zeros(15, dtype=np.uint64)
    assert emu.emu_scan_verify(sums.ctypes.data, len(recs), cin.ctypes.data, out.ctypes.data) == 0
    buf.free()
    return {"bad": int(out[0]), "end_seen": int(out[1]), "end_ck": tuple(int(x) for x in out[2:6]),
            "carry": tuple(int(x) for x in out[6:10]), "agg": tuple(int(x) for x in out[10:15]), "nrec": len(recs)}


def test_k1_and_scan_kernels_on_the_cpu(emu, oracle):
    """k1_record_sums / k1_record_sums_g<16|8|4> + k_scan_tiles / k_scan_spine / k_scan_verify,
    launched as mtz_lib.cu launches them: END checksum, carry, aggregate and the index of the
    first corrupted record must be the oracle's, for every lane-group width, record sizes from
    512 B to 1 MiB (chunked rows), every record type, sub-streams, all-ones payloads."""
    from test_gpu_codec import _all_types_stream
    NONE = 0xffffffff
    cases = [oracle.synth_stream(9, recsize=512, kind=oracle.PAYLOAD_PCG),
             oracle.synth_stream(300, recsize=4096, kind=oracle.PAYLOAD_PGPAGE),       # > 1 scan tile
             oracle.synth_stream(20, recsize=131072, kind=oracle.PAYLOAD_PCG),
             oracle.synth_stream(2, recsize=1 << 20, kind=oracle.PAYLOAD_PGPAGE),
             oracle.synth_stream(0),
             _all_types_stream(oracle, seed=12)]
    ones = oracle.synth_stream(6, recsize=65536, kind=oracle.PAYLOAD_ZERO).copy()
    cnt, offs = oracle.stream_index(ones)
    for k in range(2, cnt - 1):
        ones[int(offs[k]) + 312:int(offs[k + 1])] = 255                                  # carries everywhere
    assert oracle.stream_restamp(ones)[0] == 0
    cases.append(ones)
    cases.append(np.concatenate([cases[0], cases[5], cases[0]]))                         # checksum restarts
    rng = np.random.default_rng(5)
    for s in cases:
        rc, st = oracle.stream_verify(s)
        assert rc == 0
        whole = oracle.fletcher4_partial(s)
        for lanes in (32, 16, 8, 4):
            r = _verify_on_emulator(emu, s, lanes)
            assert r["bad"] == NONE and r["end_seen"] == 1 and r["end_ck"] == st.end_cksum.tuple(), lanes
            assert r["nrec"] == st.records
            if s is not cases[-1]:                     # one BEGIN at the start: the aggregate is the plain sum
                assert r["agg"][1:] == whole[1:] and (r["agg"][0] & ((1 << 63) - 1)) == whole[0], lanes
        # one flipped bit anywhere: same verdict and same record index as the oracle
        for _ in range(3):
            bad = s.copy()
            bad[int(rng.integers(0, s.size))] ^= 1 << int(rng.integers(0, 8))
            orc, ost = oracle.stream_verify(bad)
            if orc == oracle.EFORMAT:
                continue
            lanes = int(rng.choice([32, 16, 8, 4]))
            r = _verify_on_emulator(emu, bad, lanes)
            if orc == 0:                               # a flip inside an unverified legacy field
                assert r["bad"] == NONE
            else:
                assert r["bad"] == ost.bad_record, (lanes, r["bad"], ost.bad_record)
    # shard semantics: the second half of a stream verified with the first half's carry
    s = cases[2]
    cnt, offs = oracle.stream_index(s)
    cut = int(offs[cnt // 2])
    first = oracle.fletcher4(s[:cut])
    from manatee_b200 import index_host
    recs, _ = index_host(s[cut:])
    tail = np.ascontiguousarray(s[cut:])
    r = _verify_on_emulator(emu, tail, 32, carry_in=first)
    assert r["bad"] == NONE and r["end_ck"] == oracle.stream_verify(s)[1].end_cksum.tuple()


def _codec_on_emulator(emu, mode, stream, lanes=32, carry=(0, 0, 0, 0)):
    from manatee_b200 import index_host
    recs, used = index_host(stream)
    assert used == stream.size
    buf = Guarded(emu, stream.size, slack=(-stream.size) % 16, data=stream)
    worst = int(sum(312 + max(int(r["payload"]), int(r["lsize"]) if r["type"] == 3 else 0) for r in recs))
    out = Guarded(emu, worst, slack=(-worst) % 16)
    out.a[:] = 0x77
    res = np.zeros(13, dtype=np.uint64)
    cin = np.array(carry, dtype=np.uint64)
    rc = emu.emu_codec(mode, buf.ptr, recs.ctypes.data, len(recs), out.ptr, cin.ctypes.data, lanes, res.ctypes.data)
    assert rc == 0
    got = out.a[:int(res[0])].copy()
    buf.free()
    out.free()
    return got, {"bad": int(res[1]), "n_dec": int(res[2]), "n_enc": int(res[3]),
                 "end_ck": tuple(int(x) for x in res[4:8]), "carry": tuple(int(x) for x in res[8:12]),
                 "end_seen": int(res[12])}


def test_codec_kernels_on_the_cpu(emu, oracle):
    """plan / K2 / K3 / layout / assemble / K1(out) / stamp chain, in the order mtz_lib.cu launches
    them, on the emulator: COMPRESS, DECOMPRESS and RECOMPRESS outputs must be the oracle's byte
    for byte (headers, frames, every re-stamped checksum) -- every record type, mixed payload
    kinds, both table flavours, a few hundred tiny records in one batch."""
    from test_gpu_codec import _all_types_stream, _mixed_stream
    NONE = 0xffffffff
    cases = [(_all_types_stream(oracle, seed=3), 32),
             (_mixed_stream(oracle, n=12, recsize=131072), 32),            # compact (17-bit) tables
             (_mixed_stream(oracle, n=30, recsize=16384), 16),
             (_mixed_stream(oracle, n=300, recsize=4096), 4),              # > 1 plan CTA, lane groups of 4
             (oracle.synth_stream(40, recsize=1024, kind=oracle.PAYLOAD_PGPAGE), 4),
             (oracle.synth_stream(0), 32),
             # two sub-streams in one batch: the stamp chain restarts at the second BEGIN
             (np.concatenate([oracle.synth_stream(5, recsize=8192, kind=oracle.PAYLOAD_PGPAGE),
                              _all_types_stream(oracle, seed=4)]), 8)]
    for s, lanes in cases:
        rc, want_c, cst = oracle.stream_compress_plain(s)
        assert rc == 0
        got_c, r = _codec_on_emulator(emu, 1, s, lanes)
        assert np.array_equal(got_c, want_c), ("compress", s.size)
        assert r["bad"] == NONE and r["n_enc"] == cst.lz4_out and r["end_seen"] == 1
        assert r["end_ck"] == cst.end_cksum.tuple()
        got_d, r = _codec_on_emulator(emu, 2, want_c, lanes)
        assert np.array_equal(got_d, s), ("decompress", s.size)
        assert r["bad"] == NONE and r["n_dec"] == cst.lz4_out
        rc, want_r, rst = oracle.stream_recompress(want_c)
        got_r, r = _codec_on_emulator(emu, 3, want_c, lanes)
        assert np.array_equal(got_r, want_r), ("recompress", s.size)
        assert r["end_ck"] == rst.end_cksum.tuple()
    # a frame that does not decode is reported with its record index, nothing is written past it
    s = _mixed_stream(oracle, n=12, recsize=131072)
    rc, c, _ = oracle.stream_compress_plain(s)
    cnt, offs = oracle.stream_index(c)
    k = 5
    bad = c.copy()
    bad[int(offs[k]) + 312:int(offs[k]) + 316] = 255                         # absurd BE32 length
    _, r = _codec_on_emulator(emu, 2, bad, 32)
    assert r["bad"] == k


def _index_on_emulator(emu, stream, cap=None):
    from manatee_b200.stage import REC_DTYPE
    # 4-byte aligned like mtz_dev_index demands; at most 3 spare bytes: the parse must not read past n
    buf = Guarded(emu, stream.size, slack=(-stream.size) % 4, data=stream)
    assert buf.ptr % 4 == 0
    cap = cap if cap is not None else stream.size // 312 + 8
    recs = np.zeros(cap, dtype=REC_DTYPE)
    res = np.zeros(3, dtype=np.int64)
    assert emu.emu_index(buf.ptr, stream.size, recs.ctypes.data, cap, res.ctypes.data) == 0
    buf.free()
    return recs[:int(res[0])], int(res[1]), int(res[2])


def test_gpu_side_parser_and_carry_fold_on_the_cpu(emu, oracle):
    """k_index (speculative strided header walk; the cooperative grid emulated with one CTA)
    must build the record table the host parser builds -- on valid streams, truncated ones and
    a few hundred header mutations -- and k_fold_carry must equal the oracle's fold."""
    from manatee_b200 import index_host
    from manatee_b200 import _native as N
    from test_gpu_codec import _all_types_stream
    EFORMAT, ENOSPC = -4, -7
    base = _all_types_stream(oracle, seed=17)
    streams = [base, oracle.synth_stream(0), oracle.synth_stream(700, recsize=512, kind=oracle.PAYLOAD_PCG),
               oracle.synth_stream(9, recsize=131072, kind=oracle.PAYLOAD_PGPAGE),
               np.concatenate([base, oracle.synth_stream(5, recsize=4096), base])]
    rc, comp, _ = oracle.stream_compress_plain(streams[3])
    streams.append(comp)                                              # ragged record lengths
    for s in streams:
        for cut in (0, 100, 312 + 77):
            t = s[:s.size - cut] if cut else s
            hrecs, hused = index_host(t)
            drecs, dused, dst = _index_on_emulator(emu, t)
            assert dst == 0 and dused == hused and len(drecs) == len(hrecs), (s.size, cut)
            for f in ("off", "payload", "type", "lsize", "comp"):
                assert np.array_equal(drecs[f], hrecs[f]), (f, s.size, cut)
    # too small a table is reported, not overrun
    _, _, st = _index_on_emulator(emu, streams[2], cap=10)
    assert st == ENOSPC
    # header mutations: same verdict as the host parser
    cnt, offs = oracle.stream_index(base)
    rng = np.random.default_rng(123)
    fields = [(0, 4), (4, 4), (8, 8), (28, 4), (32, 8), (50, 1), (52, 4), (96, 8), (16, 8)]
    n_bad = 0
    for _ in range(150):
        m = base.copy()
        r = int(rng.integers(0, cnt))
        off, width = fields[int(rng.integers(0, len(fields)))]
        if rng.integers(0, 2):
            m[int(offs[r]) + off + int(rng.integers(0, width))] ^= 1 << int(rng.integers(0, 8))
        else:
            m[int(offs[r]) + off:int(offs[r]) + off + width] = rng.integers(0, 256, width, dtype=np.uint8)
        try:
            hrecs, hused = index_host(m)
            hst = 0
        except N.MtzError as e:
            hst = e.code
        drecs, dused, dst = _index_on_emulator(emu, m)
        assert dst == hst, (r, off, dst, hst)
        if hst == 0:
            assert dused == hused and len(drecs) == len(hrecs) and np.array_equal(drecs["off"], hrecs["off"])
        else:
            assert dst == EFORMAT
            n_bad += 1
    assert n_bad > 10
    # carry fold == applying the earlier shards' aggregates in order
    parts = [oracle.fletcher4_partial(rng.integers(0, 256, 4 * int(rng.integers(1, 5000)), dtype=np.uint8))
             for _ in range(6)]
    aggs = np.array([list(p) for p in parts], dtype=np.uint64)
    for rank in range(7):
        want = (0, 0, 0, 0)
        for p in parts[:rank]:
            want = oracle.fletcher4_apply(want, p)
        got = np.zeros(4, dtype=np.uint64)
        emu.emu_fold_carry(aggs.ctypes.data, rank, got.ctypes.data)
        assert tuple(int(x) for x in got) == want


def test_no_misaligned_access_in_device_code(tmp_path):
    """x86 tolerates misaligned loads and stores, a GPU faults on them.  The kernel-level tests
    again, in a child process, against a harness built with -fsanitize=alignment
    -fno-sanitize-recover: one misaligned access anywhere in the device code aborts the child."""
    import sys
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    so = os.path.join(str(tmp_path), "libemul_ubsan.so")
    probe = subprocess.run(["g++", "-fsanitize=alignment", "-x", "c++", "-", "-o", os.path.join(str(tmp_path), "p")],
                           input="int main(){return 0;}", stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    if probe.returncode != 0:
        pytest.skip("no UBSan runtime")
    # alignment is the one a GPU punishes; signed overflow / shifts / array bounds come for free
    build(so, ["-O1", "-g", "-fsanitize=alignment,signed-integer-overflow,shift,bounds", "-fno-sanitize-recover=all"])
    r = subprocess.run([sys.executable, os.path.join(EMUL, "ubsan_driver.py"), so], stdout=subprocess.PIPE,
                       stderr=subprocess.PIPE, text=True, timeout=280)
    assert r.returncode == 0 and "UBSAN-CLEAN" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]
