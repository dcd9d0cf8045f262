"""GPU: MTZ_FLAG_LZ4_HC -- COMPRESS with the high-ratio LZ4 encoder (K3h, kernels_lz4hc.cuh).  Every
output equals the CPU restatement (tests/lz4hc_ref.py): the kernel on thousands of jobs through
mtz_k_lz4hc_encode, and COMPRESS through process_host, the ring API, the device API and a device group.
DECOMPRESS (no flag) restores the input, the other modes ignore the flag, and the block check counts
what the reference model (tests/block_ref.py) counts for the HC frames."""
import hashlib

import numpy as np
import pytest

import block_ref as BR
import lz4hc_ref as R
import test_gpu_block_cksum as B
from test_host_pipeline import _run_restore, fakezfs  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

JOB = np.dtype([("src_off", "<u8"), ("dst_off", "<u8"), ("src_len", "<u4"), ("lsize", "<u4"),
                ("out_len", "<u4"), ("status", "<i4")])


def encode_jobs(enc, payloads, src_mis=0):
    """the frames of `payloads` from `enc(src_base_ptr, dst_base_ptr, jobs)` -> [(out_len, frame)];
    the blocks sit at 8-byte offsets + src_mis in one source buffer, the frame slots in one output buffer"""
    jobs = np.zeros(len(payloads), dtype=JOB)
    so = do = 0
    srcs = []
    for i, p in enumerate(payloads):
        jobs[i]["src_off"] = so + src_mis
        jobs[i]["dst_off"] = do
        jobs[i]["lsize"] = p.size
        srcs.append((so + src_mis, p))
        so += (p.size + src_mis + 7) & ~7
        do += (p.size + 7) & ~7
    src = np.zeros(so + 8, dtype=np.uint8)
    for o, p in srcs:
        src[o:o + p.size] = p
    dst, out = enc(src, do, jobs)
    res = []
    for i, p in enumerate(payloads):
        assert out[i]["status"] == 0
        n = int(out[i]["out_len"])
        o = int(jobs[i]["dst_off"])
        res.append((n, dst[o:o + n].copy() if n < p.size else None))
    return res


def _torch_enc(src, dst_bytes, jobs):
    import torch
    from manatee_b200 import GpuSnapshotStage, _native as N
    d_src = torch.from_numpy(src).cuda()
    d_dst = torch.zeros(dst_bytes + 64, dtype=torch.uint8, device="cuda")
    d_jobs = torch.from_numpy(jobs.view(np.uint8).copy()).cuda()
    with GpuSnapshotStage("verify") as g:
        rc = N.lib().mtz_k_lz4hc_encode(g._h, d_src.data_ptr(), d_dst.data_ptr(), d_jobs.data_ptr(),
                                        len(jobs), None)
        assert rc == 0, N.lib().mtz_last_error(g._h)
        torch.cuda.synchronize()
    return d_dst.cpu().numpy(), d_jobs.cpu().numpy().view(JOB)


def _assert_oracle(payloads, got):
    for i, (p, (n, fr)) in enumerate(zip(payloads, got)):
        want_n, want = R.zfs_lz4hc_compress(p)
        assert n == want_n, (i, p.size, n, want_n)
        if want is not None:
            assert np.array_equal(fr, want), (i, p.size)


def test_kernel_equals_the_oracle_on_thousands_of_jobs(oracle):
    rng = np.random.default_rng(3)
    sizes = [4096, 8192, 16384, 65536, 131072, 1 << 20]
    kinds = [oracle.PAYLOAD_PGPAGE] * 6 + [oracle.PAYLOAD_PCG, oracle.PAYLOAD_ZERO]
    payloads = []
    for i in range(3000):
        n = sizes[int(rng.integers(0, 5))] if i % 100 else sizes[5]
        payloads.append(oracle.gen_payload(kinds[i % len(kinds)], i, n))
    payloads.append(oracle.gen_payload(oracle.PAYLOAD_PGPAGE, 77, 16 << 20))
    _assert_oracle(payloads, encode_jobs(_torch_enc, payloads))


def test_kernel_on_unaligned_blocks_and_odd_sizes(oracle):
    rng = np.random.default_rng(4)
    payloads = [oracle.gen_payload(oracle.PAYLOAD_PGPAGE, i, int(n))
                for i, n in enumerate(rng.integers(1, 70000, 200) * 8)]
    payloads += [np.tile(rng.integers(0, 256, per, dtype=np.uint8), 20000)[:65536].copy() for per in (1, 2, 3, 7)]
    for mis in (0, 1, 3):
        _assert_oracle(payloads, encode_jobs(_torch_enc, payloads, mis))


def _stream(oracle):
    """pg pages at several record sizes, a few incompressible and zero records, several BEGIN..END"""
    parts = [oracle.synth_stream(40, recsize=131072, kind=oracle.PAYLOAD_PGPAGE),
             oracle.synth_stream(6, recsize=65536, kind=oracle.PAYLOAD_PCG),
             oracle.synth_stream(50, recsize=8192, kind=oracle.PAYLOAD_PGPAGE, first_rec=100),
             oracle.synth_stream(4, recsize=131072, kind=oracle.PAYLOAD_ZERO),
             oracle.synth_stream(3, recsize=1 << 20, kind=oracle.PAYLOAD_PGPAGE, first_rec=300)]
    return np.ascontiguousarray(np.concatenate(parts))


def _run(mode, s, hc, **kw):
    """process_host -> (output, stats without the timing fields); the output of VERIFY is the input"""
    from manatee_b200 import GpuSnapshotStage
    out = None if mode == "verify" else np.zeros(s.size * 3 + (1 << 20), dtype=np.uint8)
    with GpuSnapshotStage(mode, lz4_hc=hc, **kw) as g:
        n = g.process_host(s, out)
        st = g.stats()
    for k in B.TIMING:
        st.pop(k)
    return (s if out is None else out[:n].copy()), st


def test_process_host_compress_equals_the_oracle_and_decompresses(oracle):
    s = _stream(oracle)
    rc, want, wst = R.stream_compress(s, hc=True)
    assert rc == 0
    for batch in (0, 1 << 20):
        out, st = _run("compress", s, True, batch_bytes=batch)
        assert np.array_equal(out, want), batch
        assert st["lz4_encoded"] == wst.lz4_out
    plain, _ = _run("compress", s, False)
    assert out.size < plain.size
    back, _ = _run("decompress", out, False)
    assert np.array_equal(back, s)


def test_the_other_modes_ignore_the_flag(oracle):
    s = _stream(oracle)
    rc, wire, _ = oracle.stream_compress(s)
    for mode, inp in (("verify", s), ("decompress", wire), ("recompress", oracle.wire_strip(wire))):
        a, b = _run(mode, inp, False), _run(mode, inp, True)
        assert np.array_equal(a[0], b[0]) and a[1] == b[1], mode


@pytest.mark.parametrize("chunk", [4093, 65536, 1 << 20])
def test_ring_api(oracle, chunk):
    from manatee_b200 import GpuSnapshotStage
    s = _stream(oracle)
    rc, want, wst = R.stream_compress(s, hc=True)
    with GpuSnapshotStage("compress", lz4_hc=True, batch_bytes=1 << 20) as g:
        out, err = B._pump(g, s.tobytes(), chunk)
        assert not err, err
        assert out == want.tobytes() and g.stats()["lz4_encoded"] == wst.lz4_out


def test_device_api(oracle):
    from manatee_b200 import GpuSnapshotStage, index_host
    mem = B.TorchMem()
    s = _stream(oracle)
    rc, want, wst = R.stream_compress(s, hc=True)
    want = oracle.wire_strip(want)                      # the device API emits no wire preamble
    recs, _ = index_host(s)
    d_in, p_in = mem.put(s)
    d_recs, p_recs = mem.put(recs.view(np.uint8))
    cap = s.size + (1 << 20)
    d_out, p_out = mem.zeros(cap)
    with GpuSnapshotStage("compress", lz4_hc=True) as g:
        g.dev_submit(p_in, s.size, p_recs, len(recs), p_out, cap)
        ob, _, _ = g.dev_finish()
        assert np.array_equal(mem.get(d_out, ob), want)
        assert g.stats()["lz4_encoded"] == wst.lz4_out


def test_device_group(oracle):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    s = _stream(oracle)
    rc, want, _ = R.stream_compress(s, hc=True)
    out, _ = _run("compress", s, True, devices=[0, 1], batch_bytes=1 << 20)
    assert np.array_equal(out, want)


def test_fanout_of_two_peers(oracle):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from manatee_b200 import GpuSnapshotStage
    s = _stream(oracle)
    rc, want, _ = R.stream_compress(s, hc=True)
    with GpuSnapshotStage("compress", lz4_hc=True, devices=[0, 1], batch_bytes=1 << 20) as g:
        for p in (0, 1):
            g.fanout_attach(p)
        g.write(s)
        g.flush()
        for p in (0, 1):
            got = []
            while True:
                b = g.read_peer(p, 1 << 20)
                if b is None:
                    break
                got.append(b)
            assert b"".join(got) == want.tobytes(), p


@pytest.mark.parametrize("logical", [False, True])
def test_block_check_counts_the_hc_frames(oracle, logical):
    """COMPRESS + HC compares LZ4-on-disk keys with its own frames (nearly always frame_miss); the
    receiver's DECOMPRESS counts what the sender counted"""
    s, _ = BR.as_on_disk(oracle, oracle.synth_stream(30, recsize=8192, kind=oracle.PAYLOAD_PGPAGE), 9)
    flags = dict(logical=True) if logical else {}
    out, st, bs = B._run(oracle, "compress", s, lz4_hc=True, **flags)
    rc, want_out, _ = R.stream_compress(s, hc=True)
    assert np.array_equal(out, want_out)
    _, want = B._want(oracle, "compress", s, out, **flags)
    B._same(bs, want)
    if logical:
        _, _, rbs = B._run(oracle, "decompress", out, **flags)
        assert {k: rbs[k] for k in BR.TRANSFER} == {k: bs[k] for k in BR.TRANSFER}


def test_host_pipeline_compress_hc_to_a_plain_decompress(fakezfs, tmp_path, oracle):  # noqa: F811
    s = fakezfs["stream"]
    wire = {}
    for hc in (False, True):
        res, cli, _ = _run_restore(fakezfs, sender_gpu={"mode": "compress", "lz4Hc": hc},
                                   recv_gpu={"mode": "decompress"})
        assert res["err"] is None, res
        digest, n = open(fakezfs["recv_out"]).read().split()
        assert int(n) == s.size and digest == hashlib.sha256(s.tobytes()).hexdigest()
        job = cli._restoreObject
        assert job.get("wire") == "lz4-stage-v1"
        wire[hc] = job["gpu"]["bytes_out"]
    assert wire[True] < wire[False], wire
