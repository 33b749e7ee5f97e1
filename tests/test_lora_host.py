"""Host side of the LoRA adapters (no GPU): how one launch stacks adapters (include/exl2_b200.h exl2b_lora_stack), the stage
bound, the shim's checks of the tensors q_attn_set_loras / q_mlp_set_loras receive, and that both names never reach a stock
extension."""
import pytest
import torch


def _ext():
    from exllamav2_b200 import build
    build.build()
    from exllamav2_b200 import ext
    return ext


def test_stacking_offsets():
    ext = _ext()
    # two adapters over q|k|v: ranks are stacked adapter by adapter, projection by projection, each in whole groups of 8 columns
    segs, total = ext.lora_stack([[16, 0, 16], [8, 8, 8]])
    assert segs == [(0, 0, 0), (0, 2, 16), (1, 0, 32), (1, 1, 40), (1, 2, 48)]
    assert total == 56
    segs, total = ext.lora_stack([[12, 4, 0]])           # ranks that are not multiples of 8 take the next multiple
    assert segs == [(0, 0, 0), (0, 1, 16)] and total == 24
    segs, total = ext.lora_stack([[0, 0], [0, 0]])
    assert segs == [] and total == 0


def test_stage_bound():
    ext = _ext()
    assert ext.LORA_MAX_RANK == 512
    segs, total = ext.lora_stack([[128, 128, 128], [128, 0, 0]])   # exactly at the bound
    assert total == 512
    with pytest.raises(RuntimeError, match="512"):
        ext.lora_stack([[128, 128, 128], [128, 8, 0]])
    assert ext.lora_stack([[250, 250, 0]])[1] == 512
    with pytest.raises(RuntimeError, match="512"):
        ext.lora_stack([[250, 250, 1]])                    # 250 takes 256 columns, 1 takes 8 more


def _h(*shape, dtype=torch.half):
    return torch.zeros(shape, dtype=dtype)


@pytest.mark.parametrize("case", ["b_missing", "a_missing", "rank_mismatch", "one_dim", "dtype", "non_contiguous", "rank_bound",
                                  "cpu", "too_many"])
def test_set_loras_rejects(case):
    ext = _ext()
    a, b = _h(512, 16), _h(16, 512)
    qa, qb = {1: a}, {1: b}
    match = {"b_missing": "has A but no B", "a_missing": "has B but no A", "rank_mismatch": "incompatible shapes",
             "one_dim": "2-D", "dtype": "incorrect datatype", "non_contiguous": "contiguous", "rank_bound": "outside 1..512",
             "cpu": "CUDA tensor", "too_many": "at most 8"}[case]
    if case == "b_missing":
        qb = {}
    elif case == "a_missing":
        qa = {}
    elif case == "rank_mismatch":
        qb = {1: _h(8, 512)}
    elif case == "one_dim":
        qa = {1: _h(512)}
    elif case == "dtype":
        qa, qb = {1: _h(512, 16, dtype=torch.float32)}, {1: _h(16, 512, dtype=torch.float32)}
    elif case == "non_contiguous":
        qa = {1: _h(16, 512).t()}
    elif case == "rank_bound":
        qa, qb = {1: _h(512, 600)}, {1: _h(600, 512)}
    elif case == "too_many":
        qa, qb = {i: a for i in range(9)}, {i: b for i in range(9)}
    with pytest.raises(RuntimeError, match=match):
        ext.q_attn_set_loras(0, qa, qb, {}, {}, {}, {}, {}, {})
    with pytest.raises(RuntimeError, match=match):
        ext.q_mlp_set_loras(0, {}, {}, {}, {}, qa, qb)


def test_set_loras_never_reach_a_stock_extension():
    """The stock binding would reinterpret one of this library's handles as its own QAttn / QMLP (ext_qattn.cpp:206)."""
    ext = _ext()

    class Stock:
        def __getattr__(self, name):
            raise AssertionError(f"{name} was forwarded to the stock extension")

    assert {"q_attn_set_loras", "q_mlp_set_loras"} <= set(ext.HOT_PATH_EXPORTS)
    saved = ext._stock_ext
    ext.set_stock_extension(Stock())
    try:
        assert ext.q_attn_set_loras.__module__ == ext.__name__ and ext.q_mlp_set_loras.__module__ == ext.__name__
        with pytest.raises(RuntimeError, match="null argument"):      # reaches this library (no handle here), not the stub
            ext.q_attn_set_loras(0, {}, {}, {}, {}, {}, {}, {}, {})
        with pytest.raises(RuntimeError, match="null argument"):
            ext.q_mlp_set_loras(0, {}, {}, {}, {}, {}, {})
    finally:
        ext._stock_ext = saved
