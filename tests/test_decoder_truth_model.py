"""Self-checks of the fp64 decoder truth (tests/decoder_truth.py) that need no GPU: it must be right before it judges anything.

  * incremental == full: with a lossless cache, feeding a sequence token by token (each call teacher-forced on the K/V the
    earlier calls produced) gives exactly the one-shot causal forward over the whole sequence -- MHA and GQA, and for chunks
    of several tokens.  This pins the causal mask, the past/new split of the keys and the position of every token.
  * RoPE is relative: shifting every position by a constant leaves q.k unchanged, and a whole forward started at another
    offset gives the same hidden states and logits.
  * the fp16-storage mode (the floor the GPU tests scale their bounds by) is a rounding-level perturbation of the exact forward."""
import numpy as np
import pytest

import decoder_truth as dt


def _tables(hd, n, base=10000.0):
    inv = 1.0 / base ** (np.arange(0, hd, 2, dtype=np.float64) / hd)
    emb = np.outer(np.arange(n, dtype=np.float64), inv)
    emb = np.concatenate([emb, emb], axis=-1)
    return np.sin(emb), np.cos(emb)


def _model(H, KVH, hd=16, hidden=64, inter=96, vocab=50, layers=2, seed=0):
    rng = np.random.default_rng(seed)

    def w(k, n):
        return rng.normal(0, 1 / np.sqrt(k), size=(k, n))

    ls = [dt.TruthLayer(input_norm=1 + 0.1 * rng.normal(size=hidden), post_norm=1 + 0.1 * rng.normal(size=hidden),
                        wq=w(hidden, H * hd), wk=w(hidden, KVH * hd), wv=w(hidden, KVH * hd), wo=w(H * hd, hidden),
                        wg=w(hidden, inter), wu=w(hidden, inter), wd=w(inter, hidden)) for _ in range(layers)]
    sin, cos = _tables(hd, 4096)
    return dt.TruthModel(ls, 1 + 0.1 * rng.normal(size=hidden), w(hidden, vocab), 0.5 * rng.normal(size=(vocab, hidden)),
                         sin, cos, H, KVH, hd, 1e-5)


def _empty(m):
    return [np.zeros((0, m.KVH, m.hd)) for _ in m.layers]


@pytest.mark.parametrize("H,KVH", [(4, 4), (4, 2), (8, 1)], ids=["mha", "gqa2", "mqa"])
@pytest.mark.parametrize("chunk", [1, 3])
def test_incremental_equals_full_forward(H, KVH, chunk):
    m = _model(H, KVH, seed=H * 10 + KVH)
    ids = np.random.default_rng(1).integers(0, 50, size=13)
    full = m.forward(ids, 0, _empty(m), _empty(m))
    pk, pv = _empty(m), _empty(m)
    for t0 in range(0, len(ids), chunk):
        r = m.forward(ids[t0:t0 + chunk], t0, pk, pv)
        n = r.hidden.shape[0]
        for a, b in ((r.hidden, full.hidden[t0:t0 + n]), (r.logits, full.logits[t0:t0 + n])):
            assert np.abs(a - b).max() <= 1e-12 * max(1.0, np.abs(b).max())
        for li in range(len(m.layers)):
            assert np.abs(r.k[li] - full.k[li][t0:t0 + n]).max() <= 1e-12
            assert np.abs(r.v[li] - full.v[li][t0:t0 + n]).max() <= 1e-12
        pk = [np.concatenate([a, b]) for a, b in zip(pk, r.k)]
        pv = [np.concatenate([a, b]) for a, b in zip(pv, r.v)]


def test_causal_mask_hides_the_future():
    """A query attends to its own position and earlier ones: changing a later token leaves earlier outputs unchanged."""
    m = _model(4, 2, seed=3)
    ids = np.random.default_rng(2).integers(0, 50, size=9)
    a = m.forward(ids, 0, _empty(m), _empty(m))
    ids2 = ids.copy()
    ids2[6] = (ids2[6] + 1) % 50
    b = m.forward(ids2, 0, _empty(m), _empty(m))
    assert np.abs(a.logits[:6] - b.logits[:6]).max() <= 1e-12
    assert np.abs(a.logits[6] - b.logits[6]).max() > 1e-3


@pytest.mark.parametrize("shift", [1, 37, 300])
def test_rope_scores_depend_only_on_relative_position(shift):
    hd = 64
    sin, cos = _tables(hd, 2048)
    rng = np.random.default_rng(shift)
    q = rng.normal(size=(5, 1, hd))
    k = rng.normal(size=(5, 1, hd))
    pq = np.array([3, 10, 11, 100, 500])
    pk = np.array([0, 10, 4, 99, 2])
    s0 = (dt.rope_neox(q, sin, cos, pq) * dt.rope_neox(k, sin, cos, pk)).sum(-1)
    s1 = (dt.rope_neox(q, sin, cos, pq + shift) * dt.rope_neox(k, sin, cos, pk + shift)).sum(-1)
    assert np.abs(s0 - s1).max() <= 1e-12 * np.abs(s0).max()
    # and the rotation is not the identity: the absolute position does reach the keys
    assert np.abs(dt.rope_neox(k, sin, cos, pk + shift) - dt.rope_neox(k, sin, cos, pk)).max() > 1e-3


@pytest.mark.parametrize("H,KVH", [(4, 4), (4, 2)], ids=["mha", "gqa"])
def test_forward_is_invariant_under_a_position_shift(H, KVH):
    m = _model(H, KVH, seed=7)
    ids = np.random.default_rng(4).integers(0, 50, size=10)
    a = m.forward(ids, 0, _empty(m), _empty(m))
    # the same tokens at positions [123, 133): tables that start 123 rows later rotate every query and key 123 steps further
    sin, cos = m.sin, m.cos
    m.sin, m.cos = sin[123:], cos[123:]
    b = m.forward(ids, 0, _empty(m), _empty(m))
    m.sin, m.cos = sin, cos
    assert np.abs(a.logits - b.logits).max() <= 1e-12 * np.abs(a.logits).max()
    assert np.abs(a.hidden - b.hidden).max() <= 1e-12 * np.abs(a.hidden).max()


@pytest.mark.parametrize("H,KVH,hidden", [(4, 2, 64), (7, 1, 48), (14, 2, 160)], ids=["gqa2", "gqa7-narrow", "gqa7-wide"])
@pytest.mark.parametrize("fp16", [False, True], ids=["exact", "fp16"])
def test_torch_forward_equals_numpy_forward(H, KVH, hidden, fp16):
    """The torch fp64 restatement the full-size GPU tests use (decoder_truth.TorchTruthModel, chunked products) is the numpy
    forward, on CPU: GQA ratios of 2 and 7, attention wider (112 vs 48) and narrower (224 vs 160) than the hidden size, a past
    of 6 positions, and column chunks small enough that every product takes several.  In fp16-storage mode a last-bit difference
    of the two fp64 sums may round an intermediate to the neighbouring fp16 value, and one such flip moves these toy models by up
    to ~4e-4, so there the two are held to 1e-3 rel-L2 instead of 1e-12."""
    import torch
    m = _model(H, KVH, hidden=hidden, seed=H * 100 + hidden)
    tl = [dt.TruthLayer(**{f: torch.from_numpy(getattr(L, f)) for f in L.__dataclass_fields__}) for L in m.layers]
    tm = dt.TorchTruthModel(tl, m.final_norm, torch.from_numpy(m.head), m.embed, m.sin, m.cos, m.H, m.KVH, m.hd, m.eps, "cpu",
                            chunk_bytes=8 * 64 * 16)
    ids = np.random.default_rng(6).integers(0, 50, size=10)
    past = m.forward(ids[:6], 0, _empty(m), _empty(m))
    a = m.forward(ids[6:], 6, past.k, past.v, fp16=fp16)
    b = tm.forward(ids[6:], 6, past.k, past.v, fp16=fp16)
    for x, y in ((a.logits, b.logits), (a.hidden, b.hidden), *zip(a.k, b.k), *zip(a.v, b.v)):
        assert x.shape == y.shape
        if fp16:
            assert np.linalg.norm(x - y) <= 1e-3 * np.linalg.norm(x)
        else:
            assert np.abs(x - y).max() <= 1e-12 * max(1.0, np.abs(x).max())


@pytest.mark.parametrize("H,KVH", [(4, 4), (4, 2)], ids=["mha", "gqa"])
def test_fp16_storage_mode_is_a_rounding_level_perturbation(H, KVH):
    m = _model(H, KVH, seed=11)
    ids = np.random.default_rng(5).integers(0, 50, size=8)
    a = m.forward(ids, 0, _empty(m), _empty(m))
    b = m.forward(ids, 0, _empty(m), _empty(m), fp16=True)
    for x, y in ((a.logits, b.logits), (a.hidden, b.hidden), (a.k[1], b.k[1])):
        d = np.linalg.norm(x - y) / np.linalg.norm(x)
        assert 1e-6 < d < 5e-3, d
    # every stored intermediate is representable in fp16
    assert np.array_equal(b.k[0], b.k[0].astype(np.float16).astype(np.float64))
    assert np.array_equal(b.hidden, b.hidden.astype(np.float16).astype(np.float64))
