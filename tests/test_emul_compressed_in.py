"""MTZ_FLAG_COMPRESSED_IN on the CPU.  The decoders themselves (k_lzjb_decode, k_zle_decode of
manatee_b200/csrc/kernels_lzjb.cuh, launched as the pipeline launches them) run on the SIMT emulator
inside guard-page buffers: bit-exact against ZFS's frames of every payload family of
tests/lz4_payloads.py at buffer phases 0 and 5, MTZ_ECODEC exactly where the model
(tests/compressed_in_ref.py) calls a frame malformed, and no access outside [src, src+src_len) and
[dst, dst+lsize).  Then the cases of tests/test_gpu_compressed_in.py run against the whole library
built for the emulator (tests/emul/make_emul_lib.py).  Test infrastructure only."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import compressed_in_ref as M
import lz4_payloads as P
import lzjb_ref as Z
import test_emul_device_code as D
import test_gpu_compressed_in as S
from test_emul_block_cksum import HostMem, emul_library  # noqa: F401  (fixture)

EMUL = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul")


@pytest.fixture(scope="module")
def dec(tmp_path_factory):
    """(decoder library of tests/emul/emul_decoders.cc, emul_kernels.cc's build for guard pages)"""
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    d = str(tmp_path_factory.mktemp("emul_cin"))
    so = os.path.join(d, "libdec.so")
    r = subprocess.run(["g++", "-O2"] + D.FLAGS + ["-o", so, os.path.join(EMUL, "warp_emul.cc"),
                                                   os.path.join(EMUL, "emul_decoders.cc")],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert r.returncode == 0, r.stderr
    L = C.CDLL(so)
    u32 = C.c_uint32
    L.emu_cin_decode.argtypes = [u32, C.c_void_p, u32, C.c_void_p, u32, u32, u32, u32]
    L.emu_cin_decode.restype = C.c_int32
    g = os.path.join(d, "libemul.so")
    D.build(g, ["-O2"])
    return L, D.bind(g)


def _decode(dec, comp, frame, lsize, slot=0, njobs=1, grid=1):
    """the stage's decode of `frame` inside guard pages: (status, output)"""
    L, G = dec
    frame = bytes(frame)
    src = D.Guarded(G, len(frame), data=np.frombuffer(frame, dtype=np.uint8))
    dst = D.Guarded(G, lsize)
    try:
        rc = L.emu_cin_decode(comp, src.ptr, len(frame), dst.ptr, lsize, slot, njobs, grid)
        return rc, dst.a.tobytes()
    finally:
        src.free()
        dst.free()


def _frames(comp, p, phase):
    if comp == M.DC_LZJB:
        (_, fr), c_len = Z.zfs_lzjb_compress(p, phase)
    else:
        (_, fr), c_len = Z.zfs_zle_compress(p)
    return fr, c_len


@pytest.mark.parametrize("family", P.FAMILIES)
def test_decoders_on_zfs_frames(dec, oracle, family):
    """every frame ZFS makes decodes to its block, sector-padded or cut at the encoder's end"""
    n = 0
    for size in (1024, 4096, 131072):
        p = P.payload(family, 11, size)
        for comp, phases in ((M.DC_LZJB, (0, 5)), (M.DC_ZLE, (0,))):
            for phase in phases:
                fr, c_len = _frames(comp, p, phase)
                if fr is None:
                    continue
                for f in (fr, fr[:c_len]):
                    assert M.decode(oracle, comp, f, size) == p.tobytes()
                    rc, got = _decode(dec, comp, f, size, slot=n % 3, njobs=3, grid=1 + n % 2)
                    assert rc == 0 and got == p.tobytes(), (family, size, comp, phase)
                n += 1
    if family not in ("random", "mixture"):
        assert n > 0


def _corruptions(rng, comp, fr, lsize):
    """frames derived from `fr` by the corruptions a stage must survive"""
    fr = bytes(fr)
    out = [fr[:k] for k in sorted({0, 1, len(fr) // 2, len(fr) - 1})]            # truncated sources
    if comp == M.DC_LZJB:
        items = M.lzjb_items(fr, lsize)
        matches = [it for it in items if it[1]]
        for pos, _, op in matches[:3] + matches[-2:]:
            for off in (0, op + 1, 1023):                                           # bad offsets
                b = bytearray(fr)
                b[pos] = (b[pos] & 0xfc) | (off >> 8)
                b[pos + 1] = off & 0xff
                out.append(bytes(b))
        end = max(p for p, _, _ in items) + 1
        out.append(fr[:end - 1])
    else:
        toks = M.zle_tokens(fr, lsize)
        for tp, _, zero in toks[-3:]:
            b = bytearray(fr)
            b[tp] = 255 if zero else 63                                             # runs past lsize
            out.append(bytes(b))
    for _ in range(12):                                                             # random byte flips
        b = bytearray(fr)
        for k in rng.integers(0, len(b), 3):
            b[int(k)] = int(rng.integers(0, 256))
        out.append(bytes(b))
    return out


@pytest.mark.parametrize("comp", [M.DC_LZJB, M.DC_ZLE])
def test_corrupted_frames_fail_exactly_where_the_model_says(dec, oracle, comp):
    rng = np.random.default_rng(comp)
    bad = good = 0
    for family in ("pgpage", "sparse", "text", "zeros", "ints", "far"):
        p = P.payload(family, 5, 8192)
        fr, c_len = _frames(comp, p, 0)
        if fr is None:
            continue
        for f in _corruptions(rng, comp, fr, p.size):
            want = M.decode(oracle, comp, f, p.size)
            rc, got = _decode(dec, comp, f, p.size)
            if want is None:
                assert rc == D.ECODEC, (family, len(f))
                bad += 1
            else:
                assert rc == 0 and got == want, family
                good += 1
    assert bad > 10


CASES = [
    ("output-lzjb", S.test_output_equals_the_model, ("lzjb", 8192)),
    ("output-zle", S.test_output_equals_the_model, ("zle", 8192)),
    ("output-lz4-12", S.test_output_equals_the_model, ("lz4-12", 8192)),
    ("output-mixed", S.test_output_equals_the_model, ("mixed", 8192)),
    ("forwarded", S.test_lz4_payloads_are_forwarded_as_they_arrive, ()),
    ("preamble-embed", S.test_the_preamble_says_what_plain_send_would_have_said, (M.FEAT_EMBED_DATA, True)),
    ("preamble-plain", S.test_the_preamble_says_what_plain_send_would_have_said, (0, True)),
    ("ecodec", S.test_corrupted_frames_and_unknown_compressions_are_ecodec, ()),
    ("other_modes", S.test_the_other_modes_do_not_change, ()),
    ("block-lzjb", S.test_block_counters_are_those_of_verify, (False,)),
    ("block-logical", S.test_block_counters_are_those_of_verify, (True,)),
    ("ring_api-4093", S.ring_api, (4093,)),
]


@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_compressed_in_case_on_the_emulated_library(emul_library, oracle, name):  # noqa: F811
    fn, args = {c[0]: (c[1], c[2]) for c in CASES}[name]
    fn(oracle, *args)


def test_device_api_on_the_emulated_library(emul_library, oracle):  # noqa: F811
    S.device_api(oracle, HostMem())
