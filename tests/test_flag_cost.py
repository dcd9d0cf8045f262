"""CPU: the parts of tools/flag_cost.py that do not need a GPU -- its threaded re-keying of a stream
as ZFS writes it, each subcommand's options and defaults, and the refusal to run without a device."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.append(os.path.join(ROOT, "tools"))

import block_ref as R  # noqa: E402
import flag_cost  # noqa: E402

SHA = dict(verify_gib=16.0, host_gib=2.0, recompress_gib=1.0, steps=10, warmup=2, host_steps=4, profile_steps=3)
FRAMES = dict(verify_gib=16.0, host_gib=2.0, ring_gib=8.0, steps=10, warmup=2, host_steps=4, ring_steps=3,
              profile_steps=3)
DEFAULTS = {
    "block_cksum": dict(verify_gib=16.0, recompress_gib=1.0, steps=10, warmup=2),
    "block_sha256": SHA,
    "block_sha512": SHA,
    "block_frames": FRAMES,
    "block_lzjb": dict(FRAMES, zle_gib=4.0),
    "block_logical": dict(gib=1.0, large_gib=4.0, host_gib=2.0, steps=10, warmup=2, host_steps=4, profile_steps=3),
    "lz4hc": dict(gib=1.0, host_gib=1.0, steps=5, warmup=1, host_steps=3, profile_steps=2),
}


@pytest.mark.parametrize("codec", [R.DC_LZ4, R.DC_LZJB, R.DC_ZLE])
@pytest.mark.parametrize("threads", [1, 8])
def test_keyed_is_as_on_disk(oracle, codec, threads):
    s = oracle.synth_stream(24, recsize=16384, kind=oracle.PAYLOAD_PGPAGE)
    want, dcs = R.as_on_disk(oracle, s, 9, codec)
    assert codec in dcs.values()            # some blocks are stored compressed, not all raw
    got = flag_cost.keyed(oracle, s, threads, codec)
    assert got.tobytes() == want.tobytes()


@pytest.mark.parametrize("workload", sorted(DEFAULTS))
def test_defaults(workload):
    a = vars(flag_cost.parse_args([workload]))
    assert a.pop("workload") == workload and a.pop("out") is None
    assert a == DEFAULTS[workload]
    assert all(type(v) is type(DEFAULTS[workload][k]) for k, v in a.items())
    assert flag_cost.parse_args([workload, "--steps", "3", "--out", "f.json"]).steps == 3


@pytest.mark.parametrize("workload", sorted(DEFAULTS))
def test_needs_a_gpu(workload, monkeypatch):
    import torch
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(SystemExit) as e:
        flag_cost.main([workload])
    assert e.value.code == "flag_cost.py %s measures device time: it needs a GPU" % workload
