"""The split-KV scratch of the fused decode attention (csrc/attn_q4.cu, attn_scratch) is allocated once per (device, stream)
at a fixed bound and never moves, so CUDA graphs captured on a stream keep valid pointers.  Here the bound is checked against
every launch attn_launch_plan can make (restated by tests/attn_regimes.py nsplit_of): partial results of B * H * nsplit
(head, sequence, chunk) slots of hd + 2 floats each, and one arrival counter per (sequence, head)."""
import pytest

import attn_regimes as ar

SMS = [1, 66, 78, 114, 132]
# every cache capacity up to the one where the split stops growing (by_ctx reaches its cap of 16 at 8192), then long ones
MAX_CTX = list(range(ar.PAGE, 8192 + 2 * ar.PAGE, ar.PAGE)) + [12288, 16384, 32768, 65536]


def bound(sms: int) -> tuple[int, int]:
    """attn_q4.cu attn_scratch: 2 * SMs * (128 + 2) floats and SMs counters"""
    return 2 * sms * (128 + 2), sms


@pytest.mark.parametrize("sms", SMS)
def test_every_split_launch_fits_the_scratch(sms):
    ws_floats, n_cnt = bound(sms)
    worst = 0
    for H in range(1, 129):
        for B in range(1, 65):
            for max_ctx in MAX_CTX:
                ns = ar.nsplit_of(1, max_ctx, H, B, sms)
                if ns == 1:
                    continue                      # no split: the launch uses no scratch
                assert H * B <= sms, (H, B, max_ctx, ns)
                assert B * H <= n_cnt
                for hd in (64, 128):
                    need = B * H * ns * (hd + 2)
                    assert need <= ws_floats, (H, B, hd, max_ctx, ns, need, ws_floats)
                    worst = max(worst, need)
    # the bound is reached (B * H * nsplit = 2 * SMs at hd 128), so it cannot be lowered
    assert worst == ws_floats
