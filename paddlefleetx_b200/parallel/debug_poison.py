"""Debug mode for the peer-memory protocols (``PFX_DEBUG_POISON=1``).

The kernels in ``comm_nvls.cu`` / ``comm_p2p.cu`` / the fused GEMM+collective modes synchronise with flags and barriers instead of
stream-ordered NCCL calls.  The failure mode of such a protocol is *silent*: a consumer that runs ahead of its producer reads the previous
step's bytes, which look like perfectly good numbers.  This mode makes those bugs loud:

* **poisoned buffers** — symmetric allocations and the receive side of every collective are filled with NaN before the producer is
  allowed to write, so data consumed before it arrived turns the loss into NaN on the first step instead of degrading convergence;
  ``check_finite`` names the buffer, the rank and the first bad element;
* **epoch-skew check** — every rank must have issued the same number of barriers on every channel; ``barrier_skew_check`` compares the
  host-side counters across the group (a mismatch means some rank will satisfy another rank's *next* barrier with a stale arrival);
* race detection itself is ``compute-sanitizer --tool racecheck`` around ``tools/gpu_selftest.py <check>``.

Everything here costs host synchronisation and memory traffic; nothing runs unless the environment variable is set.
"""
from __future__ import annotations

import os
from typing import Dict, Optional

import torch


def enabled() -> bool:
    return os.environ.get("PFX_DEBUG_POISON", "0") == "1"


def poison(t: Optional[torch.Tensor]) -> None:
    """NaN for floating dtypes, 0x7F.. for integers (flags / counters must never be poisoned: callers pass data buffers only)."""
    if t is None or not enabled() or t.numel() == 0:
        return
    if t.is_floating_point():
        t.fill_(float("nan"))
    else:
        t.fill_(torch.iinfo(t.dtype).max)


def check_finite(t: torch.Tensor, what: str, rank: Optional[int] = None) -> None:
    if not enabled() or t.numel() == 0 or not t.is_floating_point():
        return
    bad = ~torch.isfinite(t.reshape(-1))
    if bool(bad.any()):
        first = int(bad.nonzero()[0])
        raise RuntimeError(f"PFX_DEBUG_POISON: {what}: non-finite value at element {first} of {t.numel()}"
                           f"{'' if rank is None else f' on rank {rank}'} — a consumer read this buffer before its producer wrote it "
                           f"(or the producer wrote NaN); {int(bad.sum())} elements affected")


def barrier_skew_check(counts: Dict[int, int], group=None) -> None:
    """``counts``: barriers issued so far per channel on this rank (``VmmSymmetricAllocator._bar_counts``).  Collective, host side."""
    if not enabled():
        return
    import torch.distributed as dist

    if not (dist.is_available() and dist.is_initialized()):
        return
    pg = getattr(group, "process_group", group)
    world = dist.get_world_size(pg)
    mine = [int(counts.get(c, 0)) for c in range(8)]
    gathered = [None] * world
    dist.all_gather_object(gathered, mine, group=pg)
    for ch in range(8):
        vals = [g[ch] for g in gathered]
        if len(set(vals)) > 1:
            raise RuntimeError(f"PFX_DEBUG_POISON: barrier epoch skew on channel {ch}: per-rank counts {vals} — the ranks did not issue the same "
                               f"sequence of symmetric-memory barriers; the next barrier on this channel can be satisfied by a stale arrival")
