"""The evaluation programs (vcr_validate, sort_story) on `WORLD_SIZE` processes, one per GPU as torchrun starts them.

Every rank reads the same record stream and evaluates the global batches k with k % world == rank (sort_story.eval_batches);
rank 0 puts the ranks' per-batch results back in global batch order and writes the one output file.  The collectives carry
host objects only (prefixes, status, per-batch results), so they are small:

  * `broadcast`  -- rank 0's object to every rank (the checkpoint to evaluate next, the prefix to restore)
  * `agree`      -- before each gather: an all-reduce of a failed flag; when a rank failed, every rank raises RankFailure with
                    the failing ranks' messages, so no rank is left waiting in the gather
  * `all_gather` -- every rank's object, in rank order

With WORLD_SIZE unset or 1 there is no process group and every collective is the identity.
"""
from __future__ import annotations

import contextlib
import os
from typing import Any, Callable, Iterator, List, Optional, Sequence


class RankFailure(RuntimeError):
    """An evaluation step failed on at least one rank; raised on every rank with the failing ranks' messages."""


def local_device_index() -> int:
    """LOCAL_RANK's GPU.  With more local ranks than GPUs (as when measuring several ranks on one card) ranks share GPUs
    round-robin."""
    import torch
    return int(os.environ.get("LOCAL_RANK", "0")) % max(1, torch.cuda.device_count())


def backend() -> str:
    """NCCL when every local rank has a GPU of its own, gloo otherwise (NCCL takes one rank per GPU) or without CUDA."""
    import torch
    local_world = int(os.environ.get("LOCAL_WORLD_SIZE", os.environ.get("WORLD_SIZE", "1")))
    return "nccl" if torch.cuda.is_available() and local_world <= torch.cuda.device_count() else "gloo"


class EvalGroup:
    """This process's rank among `world` evaluation processes, and the collectives of the evaluation programs."""

    def __init__(self, rank: int = 0, world: int = 1, dist=None):
        self.rank, self.world, self.dist = rank, world, dist

    def _flag_device(self):
        import torch
        return torch.device("cuda", torch.cuda.current_device()) if self.dist.get_backend() == "nccl" else torch.device("cpu")

    def broadcast(self, obj: Any) -> Any:
        """Rank 0's `obj` on every rank (the argument of the other ranks is ignored)."""
        if self.world == 1:
            return obj
        box = [obj]
        self.dist.broadcast_object_list(box, src=0)
        return box[0]

    def all_gather(self, obj: Any) -> List[Any]:
        if self.world == 1:
            return [obj]
        out = [None] * self.world
        self.dist.all_gather_object(out, obj)
        return out

    def agree(self, error: Optional[str]) -> None:
        """Every rank passes its error message (None when it succeeded).  Raises RankFailure on every rank if any rank failed."""
        if self.world == 1:
            if error is not None:
                raise RankFailure(error)
            return
        import torch
        failed = torch.tensor([0 if error is None else 1], dtype=torch.int32, device=self._flag_device())
        self.dist.all_reduce(failed)
        if int(failed.item()):
            messages = self.all_gather(error)
            raise RankFailure("; ".join(f"rank {r}: {m}" for r, m in enumerate(messages) if m is not None))

    def run_and_gather(self, fn: Callable[[], Any]) -> List[Any]:
        """fn() on every rank, then every rank's result in rank order.  With one rank fn's exceptions propagate unchanged;
        with several, an exception on any rank becomes RankFailure on every rank."""
        if self.world == 1:
            return [fn()]
        try:
            out, error = fn(), None
        except Exception as e:  # handed to every rank by agree()
            out, error = None, f"{type(e).__name__}: {e}"
        self.agree(error)
        return self.all_gather(out)

    def on_rank0(self, fn: Callable[[], Any]) -> Any:
        """fn() on rank 0 only (writing the output files); its result there, None on the other ranks.  With several ranks a
        failure on rank 0 raises RankFailure on every rank."""
        if self.world == 1:
            return fn()
        out, error = None, None
        if self.rank == 0:
            try:
                out = fn()
            except Exception as e:  # handed to every rank by agree()
                error = f"{type(e).__name__}: {e}"
        self.agree(error)
        return out

    def shared_prefixes(self, follow: Callable[[Callable[[float], None]], Iterator[str]],
                        sleep: Callable[[float], None]) -> Iterator[str]:
        """The checkpoint prefixes rank 0's `follow(sleep)` yields, on every rank, in its order; every rank ends when it ends.
        Rank 0 broadcasts each prefix, then "stop" (or its error).  After each of rank 0's polls it also broadcasts "wait",
        so the other ranks wait in a collective at most one poll interval at a time, far below the collectives' timeout."""
        if self.world == 1:
            yield from follow(sleep)
            return
        if self.rank == 0:
            def sleep_then_wait(seconds):
                sleep(seconds)
                self.broadcast(("wait", None))
            try:
                for prefix in follow(sleep_then_wait):
                    self.broadcast(("prefix", prefix))
                    yield prefix
            except Exception as e:
                self.broadcast(("error", f"{type(e).__name__}: {e}"))
                raise
            self.broadcast(("stop", None))
            return
        while True:
            kind, value = self.broadcast(None)
            if kind == "stop":
                return
            if kind == "error":
                raise RankFailure(f"rank 0: {value}")
            if kind == "prefix":
                yield value


def in_batch_order(per_rank: Sequence[Sequence[Any]]) -> List[Any]:
    """Per-rank lists of per-batch results (rank r holds global batches r, r + world, ...) -> one list in global batch order."""
    world = len(per_rank)
    n = sum(len(x) for x in per_rank)
    for r, x in enumerate(per_rank):
        if len(x) != len(range(r, n, world)):
            raise RuntimeError(f"rank {r} evaluated {len(x)} of {n} batches, expected {len(range(r, n, world))}")
    return [per_rank[k % world][k // world] for k in range(n)]


@contextlib.contextmanager
def eval_group() -> Iterator[EvalGroup]:
    """Set this process's GPU (LOCAL_RANK) and, with WORLD_SIZE > 1, join the process group (env:// rendezvous as torchrun
    sets it up; an existing default group is used as is).  A group this function created is destroyed on exit."""
    import torch
    if torch.cuda.is_available():
        torch.cuda.set_device(local_device_index())
    if int(os.environ.get("WORLD_SIZE", "1")) <= 1:
        yield EvalGroup()
        return
    import torch.distributed as dist
    created = not dist.is_initialized()
    if created:
        dist.init_process_group(backend=backend())
    try:
        yield EvalGroup(dist.get_rank(), dist.get_world_size(), dist)
    finally:
        if created:
            dist.destroy_process_group()
