"""manatee_b200 -- H100-native snapshot-stream stage for TritonDataCenter/manatee's
peer-bootstrap pipeline (lib/backupSender.js -> lib/backupServer.js ->
lib/zfsClient.js).  See DESIGN.md; the product is ``libmanatee_gpu.so`` (C ABI in
``include/manatee_gpu.h``), this package is its host-side mirror."""
from . import _native  # noqa: F401
from .stage import GpuSnapshotStage, PinnedBuffer, comm_unique_id, index_host  # noqa: F401

__all__ = ["GpuSnapshotStage", "PinnedBuffer", "comm_unique_id", "index_host"]
