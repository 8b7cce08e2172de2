"""Chunk planning of the fused vocabulary cross-entropy backward (ops.xent_chunks): no GPU needed."""
import pytest

from cogview_b200 import ops

V4B = 58240


def _check(chunks, M, V, budget):
    assert chunks[0][0] == 0 and chunks[-1][1] == V
    for (a0, a1), (b0, b1) in zip(chunks, chunks[1:]):
        assert a1 == b0                                   # in order, no gap, no overlap
    for v0, v1 in chunks:
        assert v1 > v0
    if len(chunks) > 1:
        widths = [v1 - v0 for v0, v1 in chunks]
        assert all(w % 256 == 0 for w in widths[:-1]) and len(set(widths[:-1])) <= 1
        assert widths[-1] <= widths[0]
        if widths[0] > 256:
            assert M * widths[0] * 2 <= budget            # the bf16 dlogits chunk fits the budget
        assert M * (widths[0] + 256) * 2 > budget or widths[0] + 256 > V   # and is the widest that does


@pytest.mark.parametrize("M", [1, 127, 2176, 4352, 8192, 8704])
@pytest.mark.parametrize("V", [V4B, 1000, 256, 300])
@pytest.mark.parametrize("budget", [1 << 20, 16 << 20, 100 << 20, ops.XENT_CHUNK_BYTES, 4 << 30])
def test_chunks_cover_the_vocabulary_within_the_budget(M, V, budget):
    _check(ops.xent_chunks(M, V, budget), M, V, budget)


def test_one_chunk_when_the_whole_dlogits_fits():
    assert ops.xent_chunks(2176, V4B) == [(0, V4B)]                 # the training benchmark's 2 x 1088 tokens
    assert ops.xent_chunks(2304, V4B, ops.XENT_CHUNK_BYTES) == [(0, V4B)]
    # exactly the padded size fits: one chunk even though V is not a multiple of 256
    assert ops.xent_chunks(100, V4B, 100 * V4B * 2) == [(0, V4B)]
    assert len(ops.xent_chunks(100, V4B, 100 * V4B * 2 - 1)) == 2


def test_a_budget_below_one_256_column_chunk_still_gives_256():
    chunks = ops.xent_chunks(8192, 1000, 1024)
    assert chunks == [(0, 256), (256, 512), (512, 768), (768, 1000)]


def test_many_chunks_with_a_partial_last_one():
    M = 8192
    chunks = ops.xent_chunks(M, V4B, ops.XENT_CHUNK_BYTES)
    assert [v1 - v0 for v0, v1 in chunks] == [16384, 16384, 16384, V4B - 3 * 16384]


def test_default_budget_is_the_module_constant(monkeypatch):
    monkeypatch.setattr(ops, "XENT_CHUNK_BYTES", 8192 * 512 * 2)
    assert ops.xent_chunks(8192, 2048) == [(0, 512), (512, 1024), (1024, 1536), (1536, 2048)]
