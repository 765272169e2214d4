"""The host side of the cut training step (DESIGN.md §3.10): data.group_by_length, and the cut length of the seeded
uniform rows bench.py and train.py --synthetic train on."""
import numpy as np
import pytest

from progen_b200.data import collate, group_by_length, synthetic_iterator
from progen_b200.engine import counted_length, cut_length


def _group(sizes, seed, n=256):
    rng = np.random.default_rng(seed)
    seqs = [''.join(chr(65 + c) for c in rng.integers(0, 20, int(rng.integers(5, n)))) for _ in range(sum(sizes))]
    out, r0 = [], 0
    for b in sizes:
        out.append(collate(seqs[r0:r0 + b], n))
        r0 += b
    return out


def _key(rows):
    return [r.tobytes() for r in rows]


@pytest.mark.parametrize('sizes', [(4, 4, 4, 4), (4, 4, 3), (1,), (2, 5, 1)])
def test_group_by_length_is_a_sorted_permutation_of_the_group(sizes):
    batches = _group(sizes, seed=sum(sizes))
    out = group_by_length(batches)
    assert [len(b) for b in out] == list(sizes)                         # micro-batch sizes kept, a ragged last one too
    rows_in, rows_out = np.concatenate(batches), np.concatenate(out)
    assert sorted(_key(rows_in)) == sorted(_key(rows_out))               # the same sequences
    lens = counted_length(rows_out[:, 1:])
    assert (np.diff(lens) >= 0).all()                                    # non-decreasing across the micro-batches
    again = group_by_length(batches)
    assert all(np.array_equal(a, b) for a, b in zip(out, again))         # deterministic
    assert all(a.dtype == b.dtype for a, b in zip(out, batches))


def test_group_by_length_is_stable():
    """rows of equal counted length keep their order: all-full-length rows come back as they were"""
    rng = np.random.default_rng(3)
    batches = [rng.integers(1, 256, (3, 129)).astype(np.uint16) for _ in range(3)]
    out = group_by_length(batches)
    assert all(np.array_equal(a, b) for a, b in zip(out, batches))
    assert group_by_length([]) == []


@pytest.mark.parametrize('seed,B,n', [(42, 2, 1024), (43, 4, 1024), (10042, 64, 1024), (42, 4, 1024), (52, 4, 1024)])
def test_uniform_rows_run_at_full_length(seed, B, n):
    """bench.py's rows (default_rng(42 | 43 | 10042).integers(0, 256, (B, n + 1))) and train.py --synthetic's
    (synthetic_iterator, seed 42 + rank and 42 + 10 000) end on a non-pad label: their cut length is n, so those
    workloads make the full-length step's launches"""
    rows = np.random.default_rng(seed).integers(0, 256, (B, n + 1))
    assert cut_length(rows[:, 1:]) == n
    it = synthetic_iterator(n, B, seed=seed)
    for _ in range(4):
        assert cut_length(next(it)[:, 1:]) == n


def test_check_length_rule():
    from progen_b200 import lib as L
    from progen_b200.engine import check_length
    rows = collate(['A' * 200, 'C' * 20], 512)
    assert check_length(rows[:, 1:], None, 'x') == 256
    assert check_length(rows[:, 1:], 256, 'x') == 256 and check_length(rows[:, 1:], 512, 'x') == 512
    for bad in (100, 128, 640, 0, -128, 256.0, True):
        with pytest.raises(L.ProgenError, match='cut_length of these rows: 256|length must be'):
            check_length(rows[:, 1:], bad, 'x')
