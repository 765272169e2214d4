"""Host planning of refilled generation (no GPU): the slots and queue chunks of `ProGen.generate` with prefill='decode',
and which calls keep one launch per chunk (`plan_launches`)."""
import numpy as np
import pytest

from progen_b200.progen import QUEUE_ROWS_PER_SLOT, plan_launches, plan_queue


@pytest.mark.parametrize('n_rows,batch_size', [(2, 64), (5, 5), (90, 64), (90, 12), (7, 8), (64, 64), (192, 3)])
def test_one_queue_of_every_row_in_row_order(n_rows, batch_size):
    slots, chunks = plan_queue(n_rows, batch_size)
    assert slots == min(batch_size, n_rows)
    assert len(chunks) == 1 and chunks[0].dtype == np.int64
    np.testing.assert_array_equal(chunks[0], np.arange(n_rows))


@pytest.mark.parametrize('n_rows,batch_size', [(64 * 64 + 1, 64), (3 * 64 * 8, 8), (10 ** 5, 40), (129, 2)])
def test_chunk_cap(n_rows, batch_size):
    """at most QUEUE_ROWS_PER_SLOT rows per slot and launch, the fewest such chunks, each with a row for every slot"""
    slots, chunks = plan_queue(n_rows, batch_size)
    cap = QUEUE_ROWS_PER_SLOT * slots
    assert len(chunks) == -(-n_rows // cap)
    assert all(slots <= len(c) <= cap for c in chunks)
    np.testing.assert_array_equal(np.concatenate(chunks), np.arange(n_rows))


@pytest.mark.parametrize('n_rows,batch_size', [(1, 64), (1, 1), (30, 1)])
def test_one_row_per_launch_keeps_plan_launches(n_rows, batch_size):
    """a launch of one row runs the single-stream kernel, which has no queue"""
    assert plan_queue(n_rows, batch_size) is None
    launches = plan_launches([3] * n_rows, batch_size)
    assert [real for _, real in launches] == [1] * n_rows


def test_forward_prefill_keeps_plan_launches(monkeypatch):
    """prefill='forward' plans per-length launches (plan_launches), never a queue"""
    import progen_b200.progen as P
    calls = []

    def no_queue(*a):
        raise AssertionError('forward prefill planned a queue')

    monkeypatch.setattr(P, 'plan_queue', no_queue)

    class Stop(Exception):
        pass

    def fake_launches(lengths, batch_size, by_length=False):
        calls.append(('launches', by_length))
        raise Stop

    monkeypatch.setattr(P, 'plan_launches', fake_launches)
    monkeypatch.setattr(P.ProGen, '_generate_decoder', lambda self, params, batch: None)
    monkeypatch.setattr(P.ProGen, '_ensure_loaded', lambda self, params: None)
    model = P.ProGen(num_tokens=256, dim=64, seq_len=32, depth=1, window_size=8, heads=2, dim_head=32)
    with pytest.raises(Stop):
        model.generate({}, ['MK', 'A'], num_samples=4, prefill='forward')
    assert calls == [('launches', True)]
