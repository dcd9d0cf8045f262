"""Send streams of the shape a dataset with many files produces (test infrastructure): long runs of
312..632-byte metadata records -- one DRR_OBJECT per dnode, DRR_FREE / DRR_FREEOBJECTS for holes and
unused object ranges -- with WRITE_EMBEDDED, SPILL and rare small DRR_WRITEs mixed in, large WRITEs
where the caller puts them, and optionally several BEGIN ... END sub-streams back to back.  Header
layouts as tests/test_gpu_codec.py::_all_types_stream.  Stamped by the oracle.

The metadata mix averages under 400 bytes a record, so a stream smaller than a batch's byte budget
can hold more records than the batch's record table: the batch is then cut on record count."""
import numpy as np

BEGIN, OBJECT, FREEOBJECTS, WRITE, FREE, END, SPILL, WRITE_EMBEDDED = 0, 1, 2, 3, 4, 5, 7, 8
HDR = 312
MIX = ((OBJECT, 0.41), (FREE, 0.29), (FREEOBJECTS, 0.22), (WRITE_EMBEDDED, 0.04), (SPILL, 0.0375),
       (WRITE, 0.0025))
SMALL_WRITES = (512, 1024, 2048, 4096, 8192, 16384)
SWEEP_BONUS = 16      # a 328-byte OBJECT: 41 * 8, so 64 in a row start at every 8-byte residue mod 512


def meta_stream(oracle, seed, subs, big=None, sweep=0):
    """A stamped stream of len(subs) sub-streams; sub-stream k is BEGIN, `sweep` OBJECTs with a
    SWEEP_BONUS-byte bonus, subs[k] - sweep records of the metadata mix, END.  `big` maps a record
    index of the whole stream (never a BEGIN or END) to the size of a pg-page DRR_WRITE put there."""
    rng = np.random.default_rng(seed)
    subs = [subs] if np.isscalar(subs) else list(subs)
    big = dict(big or {})
    n = sum(subs) + 2 * len(subs)
    kinds = np.array([k for k, _ in MIX], dtype=np.uint32)
    t = kinds[rng.choice(len(MIX), size=n, p=[p for _, p in MIX])]
    first = np.cumsum([0] + [m + 2 for m in subs[:-1]])
    last = first + np.array(subs) + 1
    t[first] = BEGIN
    t[last] = END
    assert sweep <= min(subs)
    for f in first:
        t[f + 1:f + 1 + sweep] = OBJECT
    for i in big:
        assert t[i] not in (BEGIN, END), i
        t[i] = WRITE

    h = np.zeros((n, HDR), dtype=np.uint8)
    h32, h64 = h.view(np.uint32), h.view(np.uint64)        # (n, 78) and (n, 39): field offset / 4 or / 8
    idx = np.arange(n, dtype=np.uint64)
    h32[:, 0] = t
    obj = 64 + idx // 4
    pl = np.zeros(n, dtype=np.int64)

    m = t == BEGIN
    h64[m, 1] = 0x2F5bacbac
    h64[m, 2] = 1 | (0x4 << 2)
    m = t == OBJECT
    bonus = rng.integers(0, 321, size=n)
    for f in first:
        bonus[f + 1:f + 1 + sweep] = SWEEP_BONUS
    h64[m, 1] = obj[m]
    h32[m, 4] = 19                                          # DMU_OT_PLAIN_FILE_CONTENTS
    h32[m, 5] = 44                                          # DMU_OT_SA
    h32[m, 6] = 131072
    h32[m, 7] = bonus[m]
    pl[m] = (bonus[m] + 7) & ~7
    m = t == FREEOBJECTS
    h64[m, 1] = obj[m]
    h64[m, 2] = rng.integers(1, 1 << 12, size=int(m.sum()))
    m = t == FREE
    h64[m, 1] = obj[m]
    h64[m, 2] = rng.integers(0, 1 << 20, size=int(m.sum())).astype(np.uint64) << np.uint64(17)
    h64[m, 3] = np.uint64((1 << 64) - 1)                   # to the end of the object
    m = t == WRITE_EMBEDDED
    psize = rng.integers(1, 113, size=n)
    h64[m, 1] = obj[m]
    h64[m, 3] = 4096
    h[m, 40] = 15                                           # ZIO_COMPRESS_LZ4 (the payload is opaque)
    h32[m, 12] = 4096
    h32[m, 13] = psize[m]
    pl[m] = (psize[m] + 7) & ~7
    m = t == SPILL
    h64[m, 1] = obj[m]
    spill = rng.integers(1, 33, size=n) * 8
    h64[m, 2] = spill[m]
    pl[m] = spill[m]
    m = t == WRITE
    wsize = np.array(SMALL_WRITES)[rng.integers(0, len(SMALL_WRITES), size=n)]
    for i, size in big.items():
        wsize[i] = size
    h64[m, 1] = obj[m]
    h32[m, 4] = 19
    h64[m, 3] = idx[m] << np.uint64(17)
    h64[m, 4] = wsize[m]
    h[m, 48] = 7                                            # ZIO_CHECKSUM_FLETCHER_4
    pl[m] = wsize[m]

    offs = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(HDR + pl, out=offs[1:])
    s = np.frombuffer(rng.bytes(int(offs[-1])), dtype=np.uint8).copy()     # every other payload: random
    w64 = s.view(np.uint64)
    cols = np.arange(HDR // 8, dtype=np.int64)
    for a in range(0, n, 1 << 16):
        b = min(n, a + (1 << 16))
        w64[(offs[a:b, None] >> 3) + cols] = h64[a:b]
    kinds = (oracle.PAYLOAD_PGPAGE, oracle.PAYLOAD_PCG, oracle.PAYLOAD_ZERO)
    for i in np.flatnonzero(t == WRITE):
        kind = oracle.PAYLOAD_PGPAGE if int(i) in big else kinds[int(i) % 3]
        s[offs[i] + HDR:offs[i + 1]] = oracle.gen_payload(kind, int(i), int(pl[i]))
    assert oracle.stream_restamp(s)[0] == 0 and oracle.stream_verify(s)[0] == 0
    return s


def body_residues(offs, mod, body_from=280):
    """the residues mod `mod` of every record's K1 body start (VERIFY sums from header byte 280)"""
    return set(((np.asarray(offs, dtype=np.int64) + body_from) % mod).tolist())
