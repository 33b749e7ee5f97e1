"""The one-process loopback the single-GPU tensor-parallel tests run every rank through (tests/tp_loopback.py), on CPU tensors:
TPContext.all_gather_cols over it gives every rank the whole row, in place at one row and through the scratch above; a rank's
failure, or ranks that disagree on their gathers, fail the call instead of hanging it."""
import time

import pytest
import torch

from tp_loopback import Loopback


def _gathers(world, rows, n):
    from exllamav2_b200.model import PRESETS
    from exllamav2_b200.tensor_p import TPContext
    cfg = PRESETS["test-small"]()
    nl = n // world

    def rank_fn(r):
        def f():
            tp = TPContext(cfg, r, world)
            full = torch.full((rows, n), -1.0)
            if rows == 1:                       # the rank's own columns of the replicated buffer, gathered in place
                full[:, r * nl:(r + 1) * nl] = torch.arange(r * nl, (r + 1) * nl, dtype=torch.float32)
                tp.all_gather_cols(full, full[:, r * nl:(r + 1) * nl])
            else:
                local = torch.arange(rows * n, dtype=torch.float32).view(rows, n)[:, r * nl:(r + 1) * nl].clone()
                tp.all_gather_cols(full, local)
            return full
        return f
    return [rank_fn(r) for r in range(world)]


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("rows", [1, 3])
def test_all_gather_cols_over_loopback(world, rows, monkeypatch):
    from exllamav2_b200 import tensor_p
    loop = Loopback(world, wait_s=20)
    monkeypatch.setattr(tensor_p, "_all_gather_flat", loop.gather)
    n = 64
    want = torch.arange(rows * n, dtype=torch.float32).view(rows, n) if rows > 1 else torch.arange(n, dtype=torch.float32)[None]
    for _ in range(2):                          # the same Loopback serves consecutive calls
        outs = loop.run(_gathers(world, rows, n))
        for r, out in enumerate(outs):
            assert torch.equal(out, want), f"rank {r}"
    assert loop.rounds == 2


def test_failure_on_one_rank_releases_the_others():
    loop = Loopback(4, wait_s=20)
    got = []

    def fn(r):
        def f():
            x = torch.zeros(8)
            loop.gather(x, x[2 * r:2 * r + 2])
            if r == 2:
                raise ValueError("rank 2 failed")
            loop.gather(x, x[2 * r:2 * r + 2])
            got.append(r)
        return f

    t0 = time.monotonic()
    with pytest.raises(ValueError, match="rank 2 failed"):
        loop.run([fn(r) for r in range(4)])
    assert time.monotonic() - t0 < 10 and got == []


def test_ranks_that_disagree_on_gathers_fail():
    loop = Loopback(3, wait_s=20)

    def fn(r):
        def f():
            x = torch.zeros(6)
            for _ in range(2 if r == 0 else 1):         # rank 0 gathers once more than the others
                loop.gather(x, x[2 * r:2 * r + 2])
        return f

    with pytest.raises(RuntimeError, match="without that gather"):
        loop.run([fn(r) for r in range(3)])


def test_a_rank_that_never_hands_on_times_out():
    loop = Loopback(2, wait_s=1)

    def fn(r):
        def f():
            if r == 0:
                time.sleep(3)                          # holds the turn past rank 1's wait
        return f

    with pytest.raises(TimeoutError):
        loop.run([fn(r) for r in range(2)])


def test_a_rank_still_running_after_the_timeouts_is_reported_stuck():
    loop = Loopback(2, wait_s=0.5)
    done = []

    def fn(r):
        def f():
            if r == 0:
                time.sleep(3)                          # outlives both joins of run()
                done.append(r)
        return f

    with pytest.raises(TimeoutError, match="still running"):
        loop.run([fn(r) for r in range(2)])
    assert loop.stuck and not done
    time.sleep(3)
    assert done == [0]
