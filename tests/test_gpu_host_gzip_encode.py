"""GPU, host mirror: deflate on the compressed wire.  A `compress` sender with gpu.gzipEncode whose requester posted
`acceptGzip: true` sets job.wireGzip and opens COMPRESS with MTZ_FLAG_GZIP_ENCODE; the receiver's DECOMPRESS,
opened with MTZ_FLAG_GZIP_WIRE, inflates the gzip-1 records and hands `zfs recv` the stream `zfs send` produced.
A requester without acceptGzip gets today's wire."""
import hashlib

import pytest

from test_host_pipeline import _run_restore, fakezfs  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

SENDER = {"mode": "compress", "gzipEncode": True}


def _digest(path):
    digest, n = open(path).read().split()
    return digest, int(n)


@pytest.mark.parametrize("accept", [True, False])
def test_the_deflated_wire_only_for_a_receiver_that_accepts_gzip(fakezfs, accept):  # noqa: F811
    s = fakezfs["stream"]
    recv = {"mode": "decompress", "acceptGzip": True} if accept else {"mode": "decompress"}
    res, cli, _ = _run_restore(fakezfs, sender_gpu=SENDER, recv_gpu=recv)
    assert res["err"] is None, res
    assert _digest(fakezfs["recv_out"]) == (hashlib.sha256(s.tobytes()).hexdigest(), s.size)
    job = cli._restoreObject
    assert job["wire"] == "lz4-stage-v1" and job["wireGzip"] is accept
    cin = job["gpu"]["compressed_in"]
    if accept:
        assert cin["gzip_encoded"] > 0
        assert cin["gzip_encoded"] + job["gpu"]["lz4_encoded"] == 24
    else:
        assert "gzip_encoded" not in cin and job["gpu"]["lz4_encoded"] == 24
