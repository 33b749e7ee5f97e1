"""Every rank of a tensor-parallel world in one process, for tests: a stand-in for tensor_p._all_gather_flat.

Loopback.run(fns) calls fns[r]() on a thread of its own for each rank r, and the threads take turns: only the thread whose turn it
is runs, so no two of them are ever inside the library at once.  A rank that reaches a gather registers (out_flat, in_flat) and
hands the turn to the next rank; the last rank copies every rank's slice into every rank's output, out_r[s*n:(s+1)*n] <- in_s,
and hands the turn back to rank 0.  All threads issue their work on the stream that was current where run() was called, so the
copies are stream-ordered after every rank's segment with no host synchronisation.  torch.distributed is never touched.

A failure on any thread releases the others and is re-raised by run(); every wait has a timeout, so a bug fails the test rather
than hanging it.  A thread still running after the timeouts may be inside a library call: run() then sets `stuck`, and the
caller must not free anything that thread may still use (the decoders' handles).
"""
from __future__ import annotations

import contextlib
import threading

import torch

WAIT_S = 120.0


class _Released(Exception):
    """Raised on a waiting thread when another rank has failed."""


class Loopback:
    def __init__(self, world: int, wait_s: float = WAIT_S):
        self.world, self.wait_s = world, wait_s
        self.cv = threading.Condition()
        self.turn = 0
        self.failed: BaseException | None = None
        self.slots: list = [None] * world
        self.rounds = 0                 # gathers completed
        self.stuck = False              # a rank's thread outlived run(): its library handles must stay alive
        self.local = threading.local()

    def _wait(self, rank: int):
        with self.cv:
            if not self.cv.wait_for(lambda: self.failed is not None or self.turn == rank, timeout=self.wait_s):
                self.failed = TimeoutError(f"rank {rank} waited {self.wait_s:.0f} s for its turn")
                self.cv.notify_all()
            if self.failed is not None:
                raise _Released()

    def _pass(self, rank: int):
        with self.cv:
            self.turn = (rank + 1) % self.world
            self.cv.notify_all()

    def gather(self, out_flat: torch.Tensor, in_flat: torch.Tensor):
        """tensor_p._all_gather_flat: out_flat[s * n:(s + 1) * n] <- rank s's in_flat, on every rank."""
        rank, done = self.local.rank, self.rounds
        self.slots[rank] = (out_flat, in_flat)
        if rank == self.world - 1:
            n = in_flat.numel()
            if not all(s is not None and s[1].numel() == n and s[0].numel() == n * self.world for s in self.slots):
                raise RuntimeError("the ranks reached different gathers")
            for out, _ in self.slots:
                for s, (_, src) in enumerate(self.slots):
                    out[s * n:(s + 1) * n].copy_(src)
            self.slots = [None] * self.world
            self.rounds += 1
        self._pass(rank)
        self._wait(rank)
        if self.rounds == done:         # the turn came back without the last rank's copies: a rank left without this gather
            raise RuntimeError(f"rank {rank} gathered, and a rank finished its call without that gather")

    def run(self, fns) -> list:
        """fns[r]() on rank r's thread, in turns; returns their results in rank order."""
        assert len(fns) == self.world
        stream = torch.cuda.current_stream() if torch.cuda.is_available() else None       # (CPU tensors: the host-logic test)
        results = [None] * self.world
        self.turn, self.failed, self.slots = 0, None, [None] * self.world

        def body(rank):
            self.local.rank = rank
            try:
                with contextlib.nullcontext() if stream is None else torch.cuda.stream(stream):
                    self._wait(rank)
                    results[rank] = fns[rank]()
                self._pass(rank)
            except _Released:
                pass
            except BaseException as e:       # noqa: BLE001 -- handed to the caller below
                with self.cv:
                    if self.failed is None:
                        self.failed = e
                    self.cv.notify_all()

        threads = [threading.Thread(target=body, args=(r,), name=f"tp-rank-{r}", daemon=True) for r in range(self.world)]
        for t in threads:
            t.start()
        for t in threads:
            t.join(self.wait_s * 2)
        if any(t.is_alive() for t in threads):
            with self.cv:
                if self.failed is None:
                    self.failed = TimeoutError("a rank did not finish")
                self.cv.notify_all()
            for t in threads:
                t.join(self.wait_s)
            self.stuck = any(t.is_alive() for t in threads)
            raise TimeoutError(f"ranks still running: {[t.name for t in threads if t.is_alive()]}") from self.failed
        if self.failed is not None:
            raise self.failed
        return results
