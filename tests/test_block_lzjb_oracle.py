"""CPU: the lzjb / zle restatements (tests/lzjb_ref.py) and the model of MTZ_FLAG_BLOCK_LZJB
(tests/block_ref.py).  The pure-Python encoders equal ZFS's C code (tests/lzjb_zfs.c) on fuzzed and
edge inputs, every frame decodes to its input in both languages, a few answers are derived by hand,
lzjb's dependence on the buffer's address phase is shown, and turning the flag off skips exactly the
lzjb / zle keys (none on streams without them) and changes no other verdict."""
import numpy as np
import pytest

import block_ref as R
import lzjb_ref as Z
import test_block_cksum_oracle as T
import test_gpu_block_lzjb as G

SIZES = [512, 1024, 4096, 8192, 65536, 131072, 1 << 20]


def _payloads(oracle, size, seed):
    """every synth payload kind at `size`, plus sparse and low-entropy bytes"""
    rng = np.random.default_rng(seed)
    out = [oracle.gen_payload(k, seed, size).tobytes()
           for k in (oracle.PAYLOAD_PCG, oracle.PAYLOAD_PGPAGE, oracle.PAYLOAD_ZERO)]
    out.append((rng.integers(0, 256, size, dtype=np.uint8) * (rng.random(size) < 0.3)).astype(np.uint8).tobytes())
    out.append(rng.integers(0, 4, size, dtype=np.uint8).tobytes())
    return out


def _both(x):
    """(python, C) results of both encoders for x: the c_len and frame of each"""
    pl, cl = Z.py_lzjb_compress(x), Z.zfs_lzjb_compress(x)
    pz, cz = Z.py_zle_compress(x), Z.zfs_zle_compress(x)
    return (pl, cl), (pz, cz)


def _check(x):
    n = len(x)
    for (py, (zio, c_len)), dec_py, dec_c in (
            (_both(x)[0], Z.py_lzjb_decompress, Z.zfs_lzjb_decompress),
            (_both(x)[1], Z.py_zle_decompress, Z.zfs_zle_decompress)):
        assert py[0] == c_len
        assert Z.zio_rule(py[0], py[1], n) == zio
        if py[1] is not None:
            assert zio[1] is None or zio[1][:len(py[1])] == py[1]
            assert dec_py(py[1], n) == x and dec_c(py[1], n) == x


@pytest.mark.parametrize("size", SIZES)
def test_python_encoders_equal_the_c_code_on_every_payload_kind(oracle, size):
    for seed in range(3 if size <= 131072 else 1):
        for x in _payloads(oracle, size, seed):
            _check(x)


def test_fuzzed_lengths_and_contents(oracle):
    rng = np.random.default_rng(7)
    for k in range(150):
        n = int(rng.integers(512, 12000))
        p = rng.random()
        x = (rng.integers(0, 256, n, dtype=np.uint8) * (rng.random(n) < p)).astype(np.uint8)
        if k % 3 == 0:                                   # repeats at every distance up to 1023
            d = int(rng.integers(1, 1024))
            x[d:] = x[:n - d] if k % 2 else x[d:]
        _check(x.tobytes())


def test_lzjb_gives_up_exactly_at_the_copymap_test():
    """random bytes: the encoder gives up at the first copymap byte at or past d_len - 17; with a
    compressible prefix of varying length the give-up moves across copymap boundaries"""
    rng = np.random.default_rng(3)
    seen = set()
    for n in (512, 520, 1024, 4096):
        for pre in range(0, 200, 7):
            x = bytes(pre) + rng.integers(0, 256, n - pre, dtype=np.uint8).tobytes()
            py = Z.py_lzjb_compress(x)
            assert py[0] == Z.zfs_lzjb_compress(x)[1]
            seen.add(py[0] == n)
    assert seen == {True, False}


def test_lzjb_positions_at_s_len_minus_66():
    """the last position that is hashed (s_len - 66) matches up to the end; later ones are literals"""
    for n in (512, 1024, 4096):
        for tail in range(60, 72):
            x = bytearray(np.random.default_rng(n + tail).integers(0, 256, n, dtype=np.uint8).tobytes())
            start = n - tail
            x[start:start + 66] = x[start - 100:start - 34]      # a 66-byte repeat starting near s_len - 66
            x = bytes(x)
            _check(x)


@pytest.mark.parametrize("run", [191, 192, 193])
def test_zle_zero_runs_at_the_length_byte_edge(run):
    for lead in (1, 63, 64):
        x = b"\x07" * lead + bytes(run) + b"\x05" * 700
        _check(x)
        x = bytes(run) + b"\x01\x02" * 400
        _check(x)


@pytest.mark.parametrize("lit", [63, 64, 65])
def test_zle_literal_runs_at_the_length_byte_edge(lit):
    for gap in (0, 1, 2):
        x = (b"\x09" * lit + bytes(gap)) * 40 + bytes(2000)
        _check(x)
        x = bytes(300) + bytes(range(1, lit + 1)) + b"\x00\x03" * 30 + bytes(1500)
        _check(x)


def test_known_answers():
    """Derived by hand.
    lzjb, 1024 bytes of 0x01: position 0 finds slot h(1,1,1) never written, offset (0 - 0) & 1023 = 0,
    a literal; position 1 finds it written by 0, offset 1, a match of the maximum 66 bytes; positions
    67, 133, ... find it written by the previous match start, offset 66, 66 bytes each.  The last
    hashed position is 1024 - 66 = 958: matches start at 1 + 66k for k = 0..14 (925), ending at 991;
    33 literals follow (items 16..48).  49 items -> 7 copymaps; 7 + 1 + 15 * 2 + 33 = 71 bytes, the last
    two the copymap of item 48 (0: a literal) and that literal.  The first copymap
    has item 0 a literal and items 1..7 matches: 0xfe; a match at offset 1 is ((66 - 3) << 2, 1) =
    (252, 1), at offset 66 (252, 66).
    zle, 1024 zero bytes: five runs of 192 (length byte 192 - 1 + 64 = 255) and one of 64 (127):
    6 bytes, padded to 512 < 1024, so ZFS stores the frame."""
    c_len, fr = Z.py_lzjb_compress(b"\x01" * 1024)
    assert c_len == 71 and fr[:8] == bytes([0xfe, 1, 252, 1, 252, 66, 252, 66])
    assert fr[-2:] == b"\x00\x01" and fr[-11:-2] == b"\x00" + b"\x01" * 8      # items 40..47
    assert Z.zfs_lzjb_compress(b"\x01" * 1024)[1] == 71
    assert Z.py_zle_compress(bytes(1024)) == (6, bytes([255] * 5 + [127]))
    assert Z.zfs_zle_compress(bytes(1024))[0] == (512, bytes([255] * 5 + [127]) + bytes(506))
    # 512 zero bytes: 3 bytes, but the pad reaches LSIZE: stored raw
    assert Z.zfs_zle_compress(bytes(512))[0] == (512, None)
    # random bytes: every encoder gives up, the block is stored raw
    x = np.random.default_rng(0).integers(0, 256, 8192, dtype=np.uint8).tobytes()
    assert Z.py_lzjb_compress(x)[0] == Z.py_zle_compress(x)[0] == 8192


def _phase_block(seed):
    """960 random bytes, a 65-byte copy of them ending on byte 1024, two new bytes, ~400 more random
    bytes, then the trigram at byte 1024 once more (and zeros up to 4 KiB): its slot may be first
    touched there, where the never-written entry's offset is the address phase"""
    rng = np.random.default_rng(seed)
    a = bytearray(rng.integers(0, 256, 960, dtype=np.uint8).tobytes())
    a += a[100:165]                                      # bytes 960..1024
    a += rng.integers(0, 256, 2, dtype=np.uint8).tobytes()
    a += rng.integers(0, 256, 400 + seed % 64, dtype=np.uint8).tobytes()
    a += a[1024:1027] + a[1027:1100]
    a += bytes(4096 - len(a))                            # zeros: the block compresses by > 1/8
    return bytes(a)


def test_lzjb_depends_on_the_buffer_phase():
    """phase 0 (the declared model, the GPU's) and phase 512 give different frames for some input;
    both decode to it, and phase 0 is the Python restatement's"""
    differ = 0
    for seed in range(64):
        x = _phase_block(seed)
        (_, f0), c0 = Z.zfs_lzjb_compress(x, 0)
        (_, f5), c5 = Z.zfs_lzjb_compress(x, 512)
        py = Z.py_lzjb_compress(x)
        assert py[0] == c0 and (f0 is None or f0[:c0] == py[1])
        if f0 is not None and f5 is not None and f0 != f5:
            differ += 1
            assert Z.zfs_lzjb_decompress(f0, len(x)) == x == Z.zfs_lzjb_decompress(f5, len(x))
    assert differ > 0


def test_most_data_does_not_depend_on_the_phase(oracle):
    same = 0
    for seed in range(20):
        x = oracle.gen_payload(oracle.PAYLOAD_PGPAGE, seed, 131072).tobytes()
        same += Z.zfs_lzjb_compress(x, 0) == Z.zfs_lzjb_compress(x, 512)
    assert same >= 18


def test_the_model_with_the_flag_off_is_the_existing_one(oracle):
    s, dcs = G._mixed(oracle)
    c = R.as_send_c(oracle, s)
    ncomp = sum(1 for x in dcs.values() if x in (R.DC_LZJB, R.DC_ZLE))
    for frames in (False, True):
        assert T.flag_off(oracle, s, R.VERIFY, None, "lzjb", frames=frames) == ncomp
        assert T.flag_off(oracle, c, R.VERIFY, None, "lzjb", frames=frames) == ncomp
    assert T.flag_off(oracle, c, R.RECOMPRESS, oracle.stream_recompress(c)[1], "lzjb") == ncomp


def test_the_model_without_lzjb_or_zle_keys_is_the_existing_one(oracle):
    from test_gpu_codec import _mixed_stream
    s, _ = R.as_on_disk(oracle, _mixed_stream(oracle, n=20, recsize=8192))
    for frames in (False, True):
        assert T.flag_off(oracle, s, R.VERIFY, None, "lzjb", frames=frames) == 0


def test_the_model_checks_every_lzjb_and_zle_key(oracle):
    s, dcs = G._mixed(oracle)
    v, st = R.block_check(oracle, s, R.VERIFY, lzjb=True)
    nl = sum(1 for x in dcs.values() if x == R.DC_LZJB)
    nz = sum(1 for x in dcs.values() if x == R.DC_ZLE)
    assert nl > 0 and nz > 0 and st["lzjb_encoded"] == nl and st["zle_encoded"] == nz
    assert st["frame_ok"] == nl + nz and st["frame_miss"] == 0
    # the send -c form: the same frames arrive as they are, nothing is encoded
    c = R.as_send_c(oracle, s)
    _, sc = R.block_check(oracle, c, R.VERIFY, lzjb=True)
    assert sc["frame_ok"] == st["frame_ok"] + sum(1 for x in dcs.values() if x == R.DC_LZ4)
    assert sc["lzjb_encoded"] == sc["zle_encoded"] == 0
