"""K2, K3, K3h and RECOMPRESS's certificate (K3c) on the H100 over every payload family of
tests/lz4_payloads.py, against the oracle.

Direct kernel calls: K3 encodes thousands of jobs of every family at sizes on both sides of each table
switch (and once more under MTZ_K3_FORCE_COMPACT for the 128 KiB class); K2 decodes foreign,
synthesized and malformed frames; K3h encodes the families.  Every job's output window is followed by
canary bytes that must come back untouched.

RECOMPRESS streams through process_host: the output must be the oracle's bit for bit with the oracle's
END checksum, and `lz4_certified` must be the number of blocks lz4_payloads.expected_certified
accepts -- which catches a missed certificate as well as a false one.  Records of 65547..131072 bytes
are certified under Tab17 only when every DRR_WRITE of the batch is of that class
(mtz_lib.cu all_compact_blocks), so the same records run once beside a 16 KiB record (TabU32) and
once alone (Tab17).  The malformed frames were run on the emulator inside guard pages first
(tests/test_emul_lz4_families.py)."""
import os

import numpy as np
import pytest

import lz4_frames as F
import lz4_payloads as P
import lz4hc_ref

pytestmark = pytest.mark.gpu

JOB = np.dtype([("src_off", "<u8"), ("dst_off", "<u8"), ("src_len", "<u4"), ("lsize", "<u4"),
                ("out_len", "<u4"), ("status", "<i4")])
CANARY = 64
CODEC_BATCH = 256 << 20             # mtz_open: default batch_bytes of the re-encoding modes


# ---- direct kernel calls ------------------------------------------------------------------------------
def _kernel(kind, srcs, windows, env=None):
    """mtz_k_<kind> over one job per (src bytes, output window size); returns [(status, out_len,
    window bytes)] and asserts the canaries after every window are intact"""
    import torch
    from manatee_b200 import GpuSnapshotStage, _native as N
    jobs = np.zeros(len(srcs), dtype=JOB)
    so = do = 0
    for i, (s, (w, lsize)) in enumerate(zip(srcs, windows)):
        jobs[i]["src_off"], jobs[i]["dst_off"] = so, do
        jobs[i]["src_len"], jobs[i]["lsize"] = s.size, lsize
        so += (s.size + 15) & ~15
        do += ((w + 15) & ~15) + CANARY
    src = np.zeros(so + 16, np.uint8)
    dst = np.full(do, 0xCD, np.uint8)
    for i, s in enumerate(srcs):
        o = int(jobs[i]["src_off"])
        src[o:o + s.size] = s
    d_src = torch.from_numpy(src).cuda()
    d_dst = torch.from_numpy(dst).cuda()
    d_jobs = torch.from_numpy(jobs.view(np.uint8).copy()).cuda()
    saved = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    try:
        with GpuSnapshotStage("verify") as g:
            rc = getattr(N.lib(), "mtz_k_" + kind)(g._h, d_src.data_ptr(), d_dst.data_ptr(), d_jobs.data_ptr(),
                                                  len(jobs), None)
            assert rc == 0, N.lib().mtz_last_error(g._h)
            torch.cuda.synchronize()
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    out, rj = d_dst.cpu().numpy(), d_jobs.cpu().numpy().view(JOB)
    res = []
    for i, (w, _) in enumerate(windows):
        o = int(jobs[i]["dst_off"])
        end = o + ((w + 15) & ~15) + CANARY
        assert (out[o + w:end] == 0xCD).all(), ("canary", kind, i, w)
        res.append((int(rj[i]["status"]), int(rj[i]["out_len"]), out[o:o + w]))
    return res


def _encode_payloads():
    pays = []
    for fam in P.FAMILIES:
        for n, seeds in ((1024, 60), (4096, 40), (16384, 16), (65536, 3), (P.SIZES_64K_EDGE[0], 2),
                         (P.SIZES_64K_EDGE[1], 2), (P.SIZES_64K_EDGE[2], 2), (66048, 3), (131072, 3),
                         (262144, 1), (1 << 20, 1)):
            pays += [P.payload(fam, s, n) for s in range(seeds)]
    pays.append(P.payload("pgpage", 1, P.SIZE_HUGE))
    return pays


def _assert_encoded(oracle, pays, res):
    for i, (p, (st, n, win)) in enumerate(zip(pays, res)):
        ps, want = oracle.zfs_lz4_compress(p)
        assert st == 0 and n == ps, (i, p.size, n, ps)
        if want is not None:
            assert np.array_equal(win[:ps], want), (i, p.size)


def test_k3_encodes_every_family_like_the_oracle(oracle):
    P.check_thresholds()
    pays = _encode_payloads()
    assert len(pays) > 1200
    _assert_encoded(oracle, pays, _kernel("lz4_encode", pays, [(p.size, p.size) for p in pays]))
    # the compact (Tab17) launch, which the entry point picks per call from MTZ_K3_FORCE_COMPACT
    cls = [p for p in pays if P.LZ4_64KLIMIT <= p.size <= P.COMPACT_MAX]
    assert {p.size for p in cls} == {P.SIZES_64K_EDGE[1], P.SIZES_64K_EDGE[2], 66048, 131072}
    _assert_encoded(oracle, cls, _kernel("lz4_encode", cls, [(p.size, p.size) for p in cls],
                                         env={"MTZ_K3_FORCE_COMPACT": "1"}))


def test_k3h_encodes_every_family_like_the_reference(oracle):
    pays = [P.payload(fam, s, n) for fam in P.FAMILIES for s, n in
            ((0, 4096), (1, 16384), (2, 65536), (3, P.SIZES_64K_EDGE[1]), (4, 131072), (5, 1 << 20))]
    res = _kernel("lz4hc_encode", pays, [(p.size, p.size) for p in pays])
    for i, (p, (st, n, win)) in enumerate(zip(pays, res)):
        want_n, want = lz4hc_ref.zfs_lz4hc_compress(p)
        assert st == 0 and n == want_n, (i, p.size, n, want_n)
        if want is not None:
            assert np.array_equal(win[:n], want), (i, p.size)


def test_k2_on_foreign_synthesized_and_malformed_frames(oracle):
    cases = []                      # (name, frame, lsize)
    rng = np.random.default_rng(8)
    for fam in P.FAMILIES:
        for seed, n in ((1, 4096), (2, 65536), (3, P.SIZES_64K_EDGE[1]), (4, 131072), (5, 1 << 20)):
            d = P.payload(fam, seed, n)
            ps, fr = oracle.zfs_lz4_compress(d)
            blocks = P.foreign_blocks(d)
            if fr is not None:
                blocks += [("oracle", P.block_of(fr))] + P.mutated_blocks(P.block_of(fr), rng)[:2]
            for name, b in blocks:
                cases.append(((fam, n, name), P.frame_of(b), n))
            cases += [((fam, n, m), f, ls) for m, f, ls in P.malformed(blocks[0][1], d)]
    for name, blk, data in P.synthesized_blocks(4):
        cases.append((name, P.frame_of(blk), len(data)))
        cases += [((name, m), f, ls) for m, f, ls in P.malformed(blk, data)]
    res = _kernel("lz4_decode", [f for _, f, _ in cases], [(ls, ls) for _, _, ls in cases])
    ok = bad = 0
    for (name, f, ls), (st, n, win) in zip(cases, res):
        orc, want = oracle.zfs_lz4_decompress(f, ls)
        assert st in (0, oracle.ECODEC) and (st == 0) == (orc == 0), (name, st, orc)
        if st == 0:
            assert n == ls and np.array_equal(win, want), name
            ok += 1
        else:
            bad += 1
    assert ok > 500 and bad > 300, (ok, bad)


# ---- streams ------------------------------------------------------------------------------------------
def _family_stream(oracle, recs):
    """raw send stream whose DRR_WRITE payloads are [(family, seed, lsize)], in that order (lsize a
    multiple of 8, as every DRR_WRITE's)"""
    s = oracle.synth_stream(1, 4096, oracle.PAYLOAD_PGPAGE)
    cnt, offs = oracle.stream_index(s)
    heads = [s[int(offs[k]):int(offs[k + 1]) if k + 1 < cnt else s.size] for k in range(cnt)]
    assert [int(h[0]) for h in heads] == [0, 1, 3, 5]                  # BEGIN OBJECT WRITE END
    parts = heads[:2]
    for i, (fam, seed, n) in enumerate(recs):
        assert n % 8 == 0
        h = heads[2][:312].copy()
        h[32:40] = np.array([n], np.uint64).view(np.uint8)              # drr_logical_size
        h[24:32] = np.array([i << 24], np.uint64).view(np.uint8)        # drr_offset
        parts += [h, P.payload(fam, seed, n)]
    raw = np.ascontiguousarray(np.concatenate(parts + [heads[3]]))
    assert oracle.stream_restamp(raw)[0] == 0
    return raw


def _write_sizes(oracle, stream):
    cnt, offs = oracle.stream_index(stream)
    return [int(stream[int(o) + 32:int(o) + 40].view(np.uint64)[0]) for o in offs if int(stream[int(o)]) == 3]


def all_compact_blocks(sizes):
    """mtz_lib.cu all_compact_blocks over the DRR_WRITE sizes of one batch"""
    return all(P.LZ4_64KLIMIT <= n <= P.COMPACT_MAX for n in sizes)


def _want_certified(oracle, stream):
    sizes = _write_sizes(oracle, stream)
    n = 0
    for w, blk in F.blocks_of(oracle, stream):
        fr = P.frame_of(blk)
        rc, data = oracle.zfs_lz4_decompress(fr, sizes[w])
        assert rc == 0
        n += P.expected_certified(fr, data)
    return n


def _recompress(oracle, src, **kw):
    from manatee_b200 import GpuSnapshotStage
    rc, want, st = oracle.stream_recompress(src)
    assert rc == 0
    with GpuSnapshotStage("recompress", **kw) as g:
        out = np.empty(want.size + (1 << 20), np.uint8)
        n = g.process_host(src, out)
        gs, end = g.stats(), g.end_checksum()
    assert np.array_equal(out[:n], want)
    assert end == st.end_cksum.tuple()
    assert gs["lz4_certified"] == _want_certified(oracle, src), gs
    return gs


def _streams(oracle):
    uni = {n: _family_stream(oracle, [(f, s, n) for f in P.FAMILIES for s in range(2 if n <= 131072 else 1)])
           for n in (16384, 65536, 66048, 131072, 262144, 1 << 20)}
    cls = [(f, s, n) for f in P.FAMILIES for s, n in ((7, 66048), (8, 131072), (9, P.STREAM_64K_EDGE))]
    mixed = []
    for i, r in enumerate(cls):
        mixed.append(r)
        if i % 3 == 2:
            mixed.append(("pgpage", 100 + i, 16384))
    return uni, _family_stream(oracle, mixed), _family_stream(oracle, cls)


def test_recompress_family_streams(oracle):
    uni, mixed, compact = _streams(oracle)
    for n, raw in list(uni.items()) + [("mixed", mixed), ("compact", compact)]:
        assert raw.size < CODEC_BATCH                                  # one batch each
        rc, lz, _ = oracle.stream_compress_plain(raw)
        assert rc == 0
        gs = _recompress(oracle, np.ascontiguousarray(lz))
        assert gs["lz4_certified"] > 0, n
    # by construction: the mixed stream's batch is not compact (K3c certifies its 128 KiB class with
    # TabU32), the same records alone are (Tab17)
    assert not all_compact_blocks(_write_sizes(oracle, mixed))
    assert all_compact_blocks(_write_sizes(oracle, compact))


def test_recompress_spliced_mutated_and_foreign_frames(oracle):
    uni, mixed, compact = _streams(oracle)
    rng = np.random.default_rng(12)
    for name, raw in (("u16k", uni[16384]), ("u64k", uni[65536]), ("u1m", uni[1 << 20]),
                      ("mixed", mixed), ("compact", compact)):
        rc, lz, _ = oracle.stream_compress_plain(raw)
        lz = np.ascontiguousarray(lz)
        sizes = _write_sizes(oracle, lz)
        changes = {}
        for i, (w, blk) in enumerate(F.blocks_of(oracle, lz)):
            if i % 3 == 0:
                m = P.mutated_blocks(blk, rng)
                if m:
                    changes[w] = m[int(rng.integers(len(m)))][1]
            elif i % 3 == 1:
                rc, data = oracle.zfs_lz4_decompress(P.frame_of(blk), sizes[w])
                fb = P.foreign_blocks(data)
                changes[w] = fb[int(rng.integers(len(fb)))][1]
        assert len(changes) > 5, name
        spliced = F.splice(oracle, lz, changes)
        gs = _recompress(oracle, spliced)
        assert gs["lz4_certified"] < len(F.blocks_of(oracle, lz)), name
        # DECOMPRESS of the foreign frames (behind the wire preamble COMPRESS puts before the BEGIN):
        # the oracle's logical stream
        from manatee_b200 import GpuSnapshotStage
        rc, wire, _ = oracle.stream_compress(raw)
        assert rc == 0 and wire[:8].tobytes() == oracle.WIRE_MAGIC
        src = np.ascontiguousarray(np.concatenate([wire[:oracle.WIRE_PRE_BYTES], spliced]))
        rc, want, _ = oracle.stream_decompress(src)
        assert rc == 0
        with GpuSnapshotStage("decompress") as g:
            out = np.empty(want.size + (1 << 20), np.uint8)
            n = g.process_host(src, out)
        assert np.array_equal(out[:n], want), name


def test_compress_family_streams(oracle):
    from manatee_b200 import GpuSnapshotStage
    uni, mixed, compact = _streams(oracle)
    for raw in list(uni.values()) + [mixed, compact, _family_stream(oracle, [("pgpage", 3, P.SIZE_HUGE)])]:
        rc, want, st = oracle.stream_compress(raw)
        assert rc == 0
        with GpuSnapshotStage("compress") as g:
            out = np.empty(want.size + (1 << 20), np.uint8)
            n = g.process_host(raw, out)
            end = g.end_checksum()
        assert np.array_equal(out[:n], want) and end == st.end_cksum.tuple()


def test_huge_record_takes_the_encoder(oracle):
    """16 MiB: the encoder compresses it, the certificate refuses lsize >= 2^24 (24-bit parse positions)"""
    raw = _family_stream(oracle, [("pgpage", 3, P.SIZE_HUGE), ("text", 3, 131072)])
    rc, lz, _ = oracle.stream_compress_plain(raw)
    lz = np.ascontiguousarray(lz)
    assert len(F.blocks_of(oracle, lz)) == 2
    gs = _recompress(oracle, lz)
    assert gs["lz4_certified"] == 1 and gs["lz4_encoded"] == 2
