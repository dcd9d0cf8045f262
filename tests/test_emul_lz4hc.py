"""MTZ_FLAG_LZ4_HC on the CPU: K3h (kernels_lz4hc.cuh) through mtz_k_lz4hc_encode of the whole library
built for the SIMT emulator (tests/emul/make_emul_lib.py), every source block ending at an inaccessible
page (rounded up to its 4-byte boundary) and every frame slot exactly lsize bytes before one: the frames
equal the CPU restatement (tests/lz4hc_ref.py) byte for byte, and the kernel reads and writes nothing
outside its block and its slot.  Then COMPRESS with the flag through process_host and the ring API of
the emulated library.  Test infrastructure only."""
import numpy as np
import pytest

import lz4hc_ref as R
import test_gpu_lz4hc as G
from test_emul_block_cksum import emul_library  # noqa: F401  (fixture)
from test_emul_device_code import Guarded, emu  # noqa: F401  (fixture)


def _payloads(oracle):
    out = []
    for kind in (oracle.PAYLOAD_PGPAGE, oracle.PAYLOAD_PCG, oracle.PAYLOAD_ZERO):
        for r, n in enumerate((1024, 4096, 16384 + 8, 65536 + 512, 131072)):
            out.append(oracle.gen_payload(kind, 10 * kind + r, n))
    rng = np.random.default_rng(9)
    out += [np.tile(rng.integers(0, 256, per, dtype=np.uint8), 9000)[:8192].copy() for per in (1, 2, 3, 7)]
    out.append(rng.integers(0, 3, 20000, dtype=np.uint8))                        # hash clashes
    return out


@pytest.mark.parametrize("mis", [0, 1, 3])
def test_k3h_equals_the_oracle_inside_guard_pages(emul_library, emu, oracle, mis):  # noqa: F811
    from manatee_b200 import GpuSnapshotStage
    pays = _payloads(oracle)
    bufs, jobs = [], np.zeros(len(pays), dtype=G.JOB)
    for i, p in enumerate(pays):
        src = Guarded(emu, p.size + mis, slack=(-(p.size + mis)) % 4, front=16)
        src.a[mis:] = p
        dst = Guarded(emu, p.size, slack=0)
        jobs[i]["src_off"], jobs[i]["dst_off"], jobs[i]["lsize"] = src.ptr + mis, dst.ptr, p.size
        bufs.append((src, dst))
    with GpuSnapshotStage("verify") as g:
        assert emul_library.mtz_k_lz4hc_encode(g._h, None, None, jobs.ctypes.data, len(jobs), None) == 0
    for i, (p, (src, dst)) in enumerate(zip(pays, bufs)):
        want_n, want = R.zfs_lz4hc_compress(p)
        assert jobs[i]["status"] == 0 and jobs[i]["out_len"] == want_n, (i, p.size)
        if want is not None:
            assert np.array_equal(dst.a[:want_n], want), (i, p.size)
        src.free()
        dst.free()


def test_compress_on_the_emulated_library(emul_library, oracle):  # noqa: F811
    s = np.ascontiguousarray(np.concatenate([
        oracle.synth_stream(6, recsize=131072, kind=oracle.PAYLOAD_PGPAGE),
        oracle.synth_stream(20, recsize=4096, kind=oracle.PAYLOAD_PGPAGE, first_rec=50),
        oracle.synth_stream(2, recsize=65536, kind=oracle.PAYLOAD_PCG)]))
    rc, want, wst = R.stream_compress(s, hc=True)
    out, st = G._run("compress", s, True, batch_bytes=1 << 18)
    assert np.array_equal(out, want) and st["lz4_encoded"] == wst.lz4_out
    back, _ = G._run("decompress", out, False)
    assert np.array_equal(back, s)
    for mode, inp in (("verify", s), ("decompress", out)):
        a, b = G._run(mode, inp, False), G._run(mode, inp, True)
        assert np.array_equal(a[0], b[0]) and a[1] == b[1], mode
