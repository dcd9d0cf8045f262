"""MTZ_FLAG_GZIP_IN on the CPU.  k_inflate (manatee_b200/csrc/kernels_inflate.cuh, launched as the
pipeline launches it) runs on the SIMT emulator inside guard-page buffers -- the payload ending at a page
boundary, and the output slot too -- and is compared with zlib byte for byte and verdict for verdict
(tests/gzip_in_ref.py's acceptance rule): levels 1..9, every strategy, stored blocks, flushes, the longest
and farthest matches, overlapping copies, 512 B .. 1 MiB records, the payload families of
tests/lz4_payloads.py, one hand-built frame per rejection rule and a seeded mutation fuzz.  Then the cases
of tests/test_gpu_gzip_in.py run against the whole library built for the emulator.  Test infrastructure
only."""
import ctypes as C
import os
import shutil
import subprocess
import zlib

import numpy as np
import pytest

import gzip_in_ref as G
import lz4_payloads as P
import test_emul_device_code as D
import test_gpu_gzip_in as S
from test_emul_block_cksum import HostMem, emul_library  # noqa: F401  (fixture)
from test_gzip_in_oracle import malformed_frames

EMUL = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul")
GZ6 = G.DC_GZIP[6]


def build_inflate(d):
    """(k_inflate's library of tests/emul/emul_inflate.cc, emul_kernels.cc's build for guard pages) in d"""
    so = os.path.join(d, "libinflate.so")
    r = subprocess.run(["g++", "-O2"] + D.FLAGS + ["-o", so, os.path.join(EMUL, "warp_emul.cc"),
                                                   os.path.join(EMUL, "emul_inflate.cc")],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert r.returncode == 0, r.stderr
    L = C.CDLL(so)
    u32 = C.c_uint32
    L.emu_inflate.argtypes = [u32, C.c_void_p, u32, C.c_void_p, u32, u32, u32, u32]
    L.emu_inflate.restype = C.c_int32
    g = os.path.join(d, "libemul.so")
    D.build(g, ["-O2"])
    return L, D.bind(g)


@pytest.fixture(scope="module")
def inf(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    return build_inflate(str(tmp_path_factory.mktemp("emul_gzip")))


def inflate(inf, frame, lsize, comp=GZ6, slot=0, njobs=1, grid=1):
    """the stage's inflate of `frame` inside guard pages: (status, output)"""
    L, Gd = inf
    frame = bytes(frame)
    src = D.Guarded(Gd, len(frame), data=np.frombuffer(frame, dtype=np.uint8))
    dst = D.Guarded(Gd, lsize)
    try:
        rc = L.emu_inflate(comp, src.ptr, len(frame), dst.ptr, lsize, slot, njobs, grid)
        return rc, dst.a.tobytes()
    finally:
        src.free()
        dst.free()


def same_as_zlib(inf, frame, lsize, **kw):
    """k_inflate agrees with the model on `frame`; returns whether it was accepted"""
    want = G.inflate(frame, lsize)
    rc, got = inflate(inf, frame, lsize, **kw)
    if want is None:
        assert rc == D.ECODEC, (rc, len(frame), lsize)
        return False
    assert rc == 0 and got == want, (rc, len(frame), lsize)
    return True


def deflate(data, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, flushes=()):
    """a zlib stream of data, with `flushes` = [(offset, zlib flush mode)] inside it"""
    c = zlib.compressobj(level, zlib.DEFLATED, 15, 9, strategy)
    out, at = [], 0
    for off, mode in flushes:
        out += [c.compress(data[at:off]), c.flush(mode)]
        at = off
    return b"".join(out + [c.compress(data[at:]), c.flush()])


def pg(size, seed=3):
    return P.payload("pgpage", seed, size).tobytes()


@pytest.mark.parametrize("level", range(1, 10))
def test_levels(inf, level):
    for size in (512, 8192, 131072):
        d = pg(size, level)
        f = zlib.compress(d, level)
        assert same_as_zlib(inf, f + bytes(-len(f) % 512), size)
        assert same_as_zlib(inf, f, size)                               # no padding at all


@pytest.mark.parametrize("strategy", [zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FIXED])
def test_strategies(inf, strategy):
    for fam in ("pgpage", "text", "zeros", "periodic"):
        d = P.payload(fam, 7, 32768).tobytes()
        assert same_as_zlib(inf, deflate(d, 6, strategy), len(d))


def test_stored_blocks_and_flushes(inf):
    rng = np.random.default_rng(5)
    noise = rng.integers(0, 256, 70000, dtype=np.uint8).tobytes()
    d = pg(40000) + noise + pg(20000, 9)                  # incompressible spans: stored blocks
    assert same_as_zlib(inf, zlib.compress(d, 6), len(d))
    assert same_as_zlib(inf, zlib.compress(noise[:1000], 0), 1000)     # level 0: stored only
    d = pg(65536)
    for mode in (zlib.Z_SYNC_FLUSH, zlib.Z_FULL_FLUSH):
        f = deflate(d, 6, flushes=[(1, mode), (4097, mode), (30000, mode), (30000, mode)])
        assert same_as_zlib(inf, f, len(d))


def test_longest_and_farthest_matches(inf):
    rng = np.random.default_rng(8)
    a = rng.integers(0, 256, 32768, dtype=np.uint8).tobytes()
    d = a + a + a[:4000]                                   # distance 32768, length 258 runs
    assert same_as_zlib(inf, zlib.compress(d, 9), len(d))
    for period in (1, 2, 3, 7, 31, 32, 33, 100, 257, 258, 259):
        d = (rng.integers(0, 256, period, dtype=np.uint8).tobytes() * (20000 // period + 1))[:20000]
        assert same_as_zlib(inf, zlib.compress(d, 6), len(d))          # overlapping copies


@pytest.mark.parametrize("size", [512, 4096, 65536, 1 << 20])
def test_record_sizes(inf, size):
    d = pg(size, 11)
    assert same_as_zlib(inf, zlib.compress(d, 6), size)


@pytest.mark.parametrize("family", P.FAMILIES)
def test_payload_families(inf, family):
    for size in (1024, 131072):
        d = P.payload(family, 13, size).tobytes()
        for level in (1, 9):
            assert same_as_zlib(inf, zlib.compress(d, level), size)
        fr = G.gzip_frame(d, G.DC_GZIP[6])
        if fr is not None:
            assert same_as_zlib(inf, fr, size)


def test_jobs_and_grids(inf):
    d = pg(8192, 2)
    f = zlib.compress(d, 6)
    for slot, njobs, grid in ((0, 1, 1), (3, 5, 1), (9, 10, 2), (40, 64, 3)):
        rc, got = inflate(inf, f, len(d), slot=slot, njobs=njobs, grid=grid)
        assert rc == 0 and got == d
    for comp in (G.DC_GZIP[1], G.DC_GZIP[9]):
        assert inflate(inf, f, len(d), comp=comp)[0] == 0
    for comp in (0, 3, 4, 14, 15, 16):                   # not gzip: the job is left alone
        assert inflate(inf, f, len(d), comp=comp)[0] == 77


def test_one_frame_per_rejection_rule(inf):
    names = set()
    for name, frame, lsize in malformed_frames():
        assert G.inflate(frame, lsize) is None, name
        rc, _ = inflate(inf, frame, lsize)
        assert rc == D.ECODEC, name
        names.add(name)
    assert len(names) >= 20


def mutants(rng, frame, n):
    """n seeded mutations of frame: bit flips, truncations, inserted bytes"""
    for _ in range(n):
        b = bytearray(frame)
        k = int(rng.integers(3))
        if k == 0:
            for _ in range(int(rng.integers(1, 4))):
                b[int(rng.integers(len(b)))] ^= 1 << int(rng.integers(8))
        elif k == 1:
            b = b[:int(rng.integers(len(b)))]
        else:
            at = int(rng.integers(len(b) + 1))
            b[at:at] = rng.integers(0, 256, int(rng.integers(1, 4)), dtype=np.uint8).tobytes()
        yield bytes(b)


def fuzz(inf, seed, n):
    """the mutation fuzz over frames of a few families and levels; (accepted, refused)"""
    rng = np.random.default_rng(seed)
    acc = rej = 0
    for fam in ("pgpage", "text", "sparse", "periodic"):
        d = P.payload(fam, seed, 4096).tobytes()
        for level in (1, 6, 9):
            for f in mutants(rng, zlib.compress(d, level), n):
                if same_as_zlib(inf, f, len(d)):
                    acc += 1
                else:
                    rej += 1
    return acc, rej


def test_mutation_fuzz(inf):
    acc, rej = fuzz(inf, 2024, 25)
    assert rej > 200


CASES = [
    ("output-gzip-1", S.test_inflated_output_equals_the_model, ("gzip-1", 8192)),
    ("output-gzip-9", S.test_inflated_output_equals_the_model, ("gzip-9", 8192)),
    ("output-mixed", S.test_inflated_output_equals_the_model, ("mixed", 8192)),
    ("ecodec", S.test_corrupted_frames_and_zstd_are_ecodec, ()),
    ("einval", S.test_gzip_input_needs_compressed_input, ()),
    ("block", S.test_gzip_block_counters, (True, True)),
    ("ring_api-4093", S.ring_api, (4093,)),
]


@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_gzip_in_case_on_the_emulated_library(emul_library, oracle, name):  # noqa: F811
    fn, args = {c[0]: (c[1], c[2]) for c in CASES}[name]
    fn(oracle, *args)


def test_device_api_on_the_emulated_library(emul_library, oracle):  # noqa: F811
    S.device_api(oracle, HostMem())
