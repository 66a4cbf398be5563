"""SM partitions: a fixed set of a GPU's SMs (a CUDA green context) with streams bound to it.

The communication kernels of this library run on an SM *budget* (expert parallelism: 24 of an H100's 132 SMs).  A grid
size only bounds how many CTAs a kernel brings; a partition also fixes where they run, so a GEMM that was launched first
cannot keep the dispatch kernel waiting behind its waves, and the complementary partition keeps compute off the
communication SMs.  Native side: ``csrc/common/sm_partition.{h,cc}``; the reference probes the same driver feature in
``experimental/misc/cuda_greenctx.cu``.

    comm_sms, compute_sms = SmPartition.split(24)           # 24 SMs (rounded up to the granularity) and the rest
    buffer.set_num_sms(min(24, comm_sms.sm_count))           # every CTA of a launch must be resident at once
    with compute_sms:                                        # torch work goes to the big partition ...
        y = experts(x)
    with comm_sms:                                           # ... the all-to-all to its own SMs
        recv, *_ = buffer.dispatch(...)

Lifetime: a partition owns its streams.  Release tensors that were allocated while one of them was the current stream
(and synchronise) before dropping the partition, as with any stream that outlives its users.

Kernels of this library synchronise their CTAs with each other and with the same CTA on peer GPUs: never launch them
on a partition with fewer SMs than their budget.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from .. import _native


class SmPartition:
    """One side of a split.  Use :meth:`split`; instances are context managers that make the partition's stream the
    current torch stream (the previous current stream is waited for on entry and waits for the partition on exit)."""

    def __init__(self, native, total_sms: int):
        self._p = native
        self.total_sms = int(total_sms)
        self._streams = {}
        self._ctx = []

    # ------------------------------------------------------------------ construction
    @staticmethod
    def supported(device: Optional[int] = None) -> Tuple[bool, str]:
        """(True, "") where the driver can partition `device`; otherwise (False, reason)."""
        if not torch.cuda.is_available():
            return False, "no CUDA device"
        dev = torch.cuda.current_device() if device is None else int(device)
        ok, why = _native.C().util.SmPartition.supported(dev)
        return bool(ok), str(why)

    @classmethod
    def split(cls, sm_count: int, device: Optional[int] = None, fine_grained: bool = False
              ) -> Tuple["SmPartition", Optional["SmPartition"]]:
        """Carve at least `sm_count` SMs out of `device` (default: the current one).  Returns ``(partition, rest)``;
        `rest` is None when the partition took the whole device.  `fine_grained` lowers the granularity of
        the split (2 SMs instead of 8) and gives up large thread-block clusters inside the partitions."""
        ok, why = cls.supported(device)
        if not ok:
            raise RuntimeError(f"uccl_b200: SM partitions are unavailable: {why}")
        dev = torch.cuda.current_device() if device is None else int(device)
        U = _native.C().util.SmPartition
        total = int(U.device_sm_count(dev))
        part, rest = U.split(dev, int(sm_count), bool(fine_grained))
        return cls(part, total), (cls(rest, total) if rest is not None else None)

    # ------------------------------------------------------------------ properties
    @property
    def device(self) -> int:
        return int(self._p.device)

    @property
    def sm_count(self) -> int:
        return int(self._p.sm_count)

    def stream(self, priority: int = 0) -> "torch.cuda.Stream":
        """The partition's stream of that priority as a torch stream (owned by the partition)."""
        s = self._streams.get(priority)
        if s is None:
            s = torch.cuda.ExternalStream(int(self._p.stream(int(priority))), device=torch.device("cuda", self.device))
            self._streams[priority] = s
        return s

    # ------------------------------------------------------------------ context manager
    def __enter__(self) -> "SmPartition":
        s = self.stream()
        prev = torch.cuda.current_stream(s.device)
        s.wait_stream(prev)
        cm = torch.cuda.stream(s)
        cm.__enter__()
        self._ctx.append((cm, prev, s))
        return self

    def __exit__(self, *exc) -> None:
        cm, prev, s = self._ctx.pop()
        cm.__exit__(*exc)
        prev.wait_stream(s)

    def sm_ids(self, blocks: Optional[int] = None, hold_us: int = 50) -> "torch.Tensor":
        """Sorted ids of the SMs a probe kernel of `blocks` CTAs (default: 4 per SM of the device) lands on when it
        is launched on this partition's stream -- the check that the partition is physical."""
        return sm_ids(self.stream(), blocks or 4 * self.total_sms, hold_us)

    def __repr__(self) -> str:
        return f"SmPartition(device={self.device}, sm_count={self.sm_count} of {self.total_sms})"


def sm_ids(stream: Optional["torch.cuda.Stream"] = None, blocks: int = 1024, hold_us: int = 50) -> "torch.Tensor":
    """Sorted unique SM ids hit by a `blocks`-CTA probe kernel on `stream` (default: the current stream)."""
    st = stream if stream is not None else torch.cuda.current_stream()
    with torch.cuda.stream(st):
        out = torch.full((int(blocks),), -1, dtype=torch.int32, device=st.device)
        _native.C().util.smid_probe(out.data_ptr(), int(blocks), int(hold_us) * 1000, st.cuda_stream)
    st.synchronize()
    return torch.unique(out.cpu())
