"""GPU: MTZ_FLAG_GZIP_ENCODE -- COMPRESS re-codes K3's LZ4 frames as zlib frames (k_deflate_from_lz4) and
sends each record in the smaller form.  Every output byte and counter is the reference model's
(tests/gzip_encode_ref.py): mtz_k_gzip_encode, mtz_process_host, the ring API and the device API; DECOMPRESS
with MTZ_FLAG_GZIP_WIRE gives the input back, a receiver without it refuses the wire, and the flag combines
with MTZ_FLAG_COMPRESSED_IN and MTZ_FLAG_GZIP_WIRE."""
import numpy as np
import pytest

import block_ref as B
import compressed_in_ref as M
import gzip_encode_ref as E
import gzip_in_ref as G
import gzip_wire_ref as W
import lz4_payloads as P
import test_gpu_block_cksum as K
import test_gpu_gzip_in as GI
from test_gpu_lz4hc import JOB, encode_jobs

pytestmark = pytest.mark.gpu

SEND = dict(gzip_encode=True)
RECV = dict(gzip_wire=True)
TIMING = ("gpu_ms", "k1_ms", "codec_ms", "k3_ms", "kernel_launches", "k1_launches", "k3_launches", "batches")


def _stage(mode, **kw):
    from manatee_b200 import GpuSnapshotStage
    return GpuSnapshotStage(mode, **kw)


def _run(mode, x, cap=None, **kw):
    """process_host -> (output, stats without the timing fields, compressed-in stats); `cap` output bytes
    (default: twice the input's)"""
    out = np.zeros(x.size * 2 + (1 << 20) if cap is None else cap, dtype=np.uint8)
    with _stage(mode, **kw) as g:
        n = g.process_host(x, None if mode in ("verify", "passthrough") else out)
        st = {k: v for k, v in g.stats().items() if k not in TIMING}
        return (x if mode in ("verify", "passthrough") else out[:n].copy()), st, g.compressed_in_stats()


def raw_stream(oracle, kind="mixed", n=24, recsize=131072):
    if kind == "pgpage":
        return oracle.synth_stream(n, recsize=recsize, kind=oracle.PAYLOAD_PGPAGE).copy()
    from test_gpu_codec import _mixed_stream
    return _mixed_stream(oracle, n=n, recsize=recsize)


def gzip_on_wire(oracle, wire, x):
    """DRR_WRITEs that left as the stage's gzip-1 frame: gzip_encoded"""
    xb, wb = np.asarray(x, dtype=np.uint8), oracle.wire_strip(wire)
    return sum(1 for (xo, _, _, t), (wo, _, _, _) in zip(B.records(xb), B.records(wb))
               if t == 3 and wb[wo + 50] == E.DC_GZIP1 and not G.is_gzip(int(xb[xo + 50])))


def check(oracle, x, out, st, cst, want, back_to=None):
    assert out.size == want.size and np.array_equal(out, want)
    assert all(f & W.WIRE_F_GZIP for f in W.pre_flags(oracle, out))
    assert st["bad_record"] == B.NONE
    assert st["lz4_encoded"] == M.encoded(oracle, out, x)
    assert cst["gzip_encoded"] == gzip_on_wire(oracle, out, x)
    want_back = x if back_to is None else back_to
    back, _, _ = _run("decompress", out, cap=want_back.size + (1 << 20), **RECV)
    assert np.array_equal(back, want_back)


def encode_kernel(payloads):
    def enc(src, dst_bytes, jobs):
        import torch
        from manatee_b200 import _native as N
        d_src = torch.from_numpy(src).cuda()
        d_dst = torch.zeros(dst_bytes + 64, dtype=torch.uint8, device="cuda")
        d_jobs = torch.from_numpy(jobs.view(np.uint8).copy()).cuda()
        with _stage("verify") as g:
            rc = N.lib().mtz_k_gzip_encode(g._h, d_src.data_ptr(), d_dst.data_ptr(), d_jobs.data_ptr(), len(jobs), None)
            assert rc == 0, N.lib().mtz_last_error(g._h)
            torch.cuda.synchronize()
        return d_dst.cpu().numpy(), d_jobs.cpu().numpy().view(JOB)
    return encode_jobs(enc, payloads)


def kernel_payloads(oracle):
    out = [oracle.gen_payload(oracle.PAYLOAD_PGPAGE, r, n) for r, n in enumerate((512, 4096, 65536, 131072, 1 << 20))]
    for fam in P.FAMILIES:
        out += [P.payload(fam, 3, n) for n in (8192, 131072)]
    return out


def test_kernel_equals_the_model(oracle):
    pays = kernel_payloads(oracle)
    for p, (n, f) in zip(pays, encode_kernel(pays)):
        z = E.frame(oracle, p)
        if z is None:
            assert n == p.size
        else:
            assert n == len(z) and f.tobytes() == z


@pytest.mark.parametrize("kind,recsize", [("pgpage", 131072), ("mixed", 8192), ("mixed", 131072), ("mixed", 1 << 20)])
def test_compress_equals_the_model(oracle, kind, recsize):
    x = raw_stream(oracle, kind, n={8192: 60, 131072: 24, 1 << 20: 4}[recsize], recsize=recsize)
    out, st, cst = _run("compress", x, **SEND)
    check(oracle, x, out, st, cst, E.expected(oracle, x))
    base, bst, _ = _run("compress", x)
    assert out.size < base.size or recsize == 8192
    assert st["lz4_encoded"] + cst["gzip_encoded"] == bst["lz4_encoded"]
    assert cst == {"lz4_passed": 0, "lzjb_decoded": 0, "zle_decoded": 0, "gzip_encoded": cst["gzip_encoded"]}
    if kind == "pgpage":
        assert cst["gzip_encoded"] > 0


def test_with_compressed_input_and_the_gzip_wire(oracle):
    """lzjb / zle records are decoded and deflated; LZ4 and gzip records are forwarded as they arrive"""
    x = GI.send_c_stream(oracle, "mixed", n=30)
    out, st, cst = _run("compress", x, compressed_input=True, gzip_wire=True, **SEND)
    check(oracle, x, out, st, cst, E.splice(oracle, W.expected(oracle, x), x), back_to=G.plain(oracle, x))
    assert cst["gzip_passed"] == W.verdict(oracle, x)[1]["gzip_passed"] > 0
    lx = M.send_c(oracle, raw_stream(oracle, "mixed", n=30, recsize=8192), 9, B.mixed_codecs)
    out, st, cst = _run("compress", lx, compressed_input=True, **SEND)
    check(oracle, lx, out, st, cst, E.expected(oracle, lx, compressed_in=True), back_to=M.plain(oracle, lx))


def test_a_receiver_without_the_flag_refuses_the_wire(oracle):
    from manatee_b200._native import MtzError, EFORMAT
    x = raw_stream(oracle, "pgpage", n=8)
    w, _, _ = _run("compress", x, **SEND)
    with _stage("decompress") as g:
        with pytest.raises(MtzError) as ei:
            g.process_host(w, np.zeros(w.size * 4, dtype=np.uint8))
        assert ei.value.code == EFORMAT


def test_einval_and_the_other_modes(oracle):
    from manatee_b200._native import MtzError, EINVAL
    for kw in (dict(lz4_hc=True), dict(compressed_input=True, gzip_input=True)):
        with pytest.raises(MtzError) as ei:
            _stage("compress", **dict(SEND, **kw))
        assert ei.value.code == EINVAL, kw
    x = raw_stream(oracle, "mixed", n=20, recsize=8192)
    cap = x.size + (1 << 20)
    rc, lz, _ = oracle.stream_compress_plain(x)
    for mode, src in (("verify", x), ("recompress", lz), ("passthrough", x)):
        a, b = _run(mode, src, cap=cap), _run(mode, src, cap=cap, **SEND)
        assert np.array_equal(a[0], b[0]) and a[1] == b[1], mode
    w, _, _ = _run("compress", x)
    a, b = _run("decompress", w, cap=cap), _run("decompress", w, cap=cap, **SEND)
    assert np.array_equal(a[0], b[0]) and a[1] == b[1]


def test_block_counters(oracle):
    """a raw record with an LZ4 key that leaves as gzip is a frame_miss at the sender, never an error; the
    receiver skips the stage's gzip-1 records"""
    s, _ = B.as_on_disk(oracle, raw_stream(oracle, "pgpage", n=12), 9)
    x = np.ascontiguousarray(B.as_send_c(oracle, s))
    p = M.plain(oracle, x)
    out, st, bs = K._run(oracle, "compress", p, **SEND)
    assert np.array_equal(out, E.expected(oracle, p))
    ng = E.counts(oracle, out)[1]
    assert ng > 0 and bs["frame_miss"] >= ng and bs["logical_ok"] + bs["frame_ok"] + bs["frame_miss"] > 0
    back, _, rbs = K._run(oracle, "decompress", out, **RECV)
    assert np.array_equal(back, p)
    assert rbs["skipped"] >= ng


def ring_api(oracle, chunk, n=12):
    x = raw_stream(oracle, "mixed", n=n, recsize=131072)
    want = E.expected(oracle, x)
    with _stage("compress", batch_bytes=1 << 20, **SEND) as g:
        out, err = K._pump(g, x.tobytes(), chunk)
        assert not err, err
        assert np.array_equal(np.frombuffer(out, dtype=np.uint8), want)
        assert g.compressed_in_stats()["gzip_encoded"] == gzip_on_wire(oracle, want, x)


@pytest.mark.parametrize("chunk", [4093, 1 << 20])
def test_ring_api(oracle, chunk):
    ring_api(oracle, chunk)


def device_api(oracle, mem, n=20, recsize=8192, model=True):
    """COMPRESS on the device API gives the wire without preambles; more records than one codec sub-batch
    holds take the other scratch set's gz table across the sub-batch edge.  `model` False: the wire of
    mtz_process_host stands in for the model's (too many records for the Python model)"""
    from manatee_b200 import index_host
    x = raw_stream(oracle, "mixed", n=n, recsize=recsize)
    full = E.expected(oracle, x) if model else _run("compress", x, **SEND)[0]
    want = oracle.wire_strip(full)
    recs, _ = index_host(x)
    d_in, p_in = mem.put(x)
    d_recs, p_recs = mem.put(recs.view(np.uint8))
    d_out, p_out = mem.zeros(x.size + (1 << 20))
    with _stage("compress", **SEND) as g:
        g.dev_submit(p_in, x.size, p_recs, len(recs), p_out, x.size + (1 << 20))
        ob, _, _ = g.dev_finish()
        assert np.array_equal(mem.get(d_out, ob), want)
        assert g.compressed_in_stats()["gzip_encoded"] == gzip_on_wire(oracle, full, x)


def test_device_api(oracle):
    device_api(oracle, K.TorchMem(), n=40, recsize=131072)


def test_device_api_across_the_subbatch_edge(oracle):
    device_api(oracle, K.TorchMem(), n=70000, recsize=2048, model=False)


def test_device_group(oracle):
    import test_gpu_compressed_in as CI
    CI._two_gpus()
    x = raw_stream(oracle, "mixed", n=24, recsize=131072)
    out, st, cst = _run("compress", x, devices=[0, 1], batch_bytes=1 << 20, **SEND)
    check(oracle, x, out, st, cst, E.expected(oracle, x))
