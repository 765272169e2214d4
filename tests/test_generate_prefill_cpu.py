"""Forward prefill without a device: the `prefill` argument is checked before any device work, and the launch planner of
ProGen.generate (a pure function) keeps today's chunks for 'decode' and splits at prompt-length boundaries for 'forward'."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KW = dict(num_tokens=256, dim=64, seq_len=64, depth=2, window_size=16, global_mlp_depth=1, heads=2, dim_head=32)


@pytest.mark.parametrize('value', ['Forward', 'prefill', '', None, 1, True, b'forward', ['forward']])
def test_prefill_rejects_invalid_values_without_a_device(value):
    from progen_b200 import ProGen
    from progen_b200.lib import ProgenError
    model = ProGen(**KW)
    with pytest.raises(ProgenError):
        model.generate({}, 'MK', prefill=value)
    assert model._engine is None and model._gen_decoder is None


@pytest.mark.parametrize('prompts,kwargs', [
    ('#' * 63, {}),
    ('abcd', dict(max_length=5)),
    ([np.array([0, 5])], {}),
    ('a', dict(temperature=-0.1)),
    ('a', dict(min_new_tokens=63)),
])
def test_forward_prefill_checks_the_other_arguments_first(prompts, kwargs):
    from progen_b200 import ProGen
    from progen_b200.lib import ProgenError
    model = ProGen(**KW)
    with pytest.raises(ProgenError):
        model.generate({}, prompts, prefill='forward', **kwargs)
    assert model._engine is None and model._gen_decoder is None


def _old_chunks(N, batch_size):
    """the chunking of ProGen.generate before forward prefill existed (row ranges, ragged chunk padded to its class)"""
    per = min(batch_size, N)
    lo = 9 if per > 8 else (2 if per > 1 else 1)
    out = []
    for r0 in range(0, N, per):
        r1 = min(N, r0 + per)
        pad = max(0, lo - (r1 - r0))
        out.append((np.concatenate([np.arange(r0, r1), np.full(pad, r1 - 1)]).astype(np.int64), r1 - r0))
    return out


@pytest.mark.parametrize('N,batch_size', [(1, 64), (5, 64), (90, 64), (90, 12), (90, 30), (3, 8), (9, 8), (10, 3), (7, 1)])
def test_decode_plan_is_the_previous_chunking(N, batch_size):
    from progen_b200.progen import plan_launches
    rng = np.random.default_rng(N * 100 + batch_size)
    got = plan_launches(rng.integers(0, 5, N), batch_size)
    want = _old_chunks(N, batch_size)
    assert len(got) == len(want)
    for (a, ra), (b, rb) in zip(got, want):
        assert a.dtype == np.int64 and ra == rb
        np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize('batch_size', [64, 12, 8, 5, 1])
def test_forward_plan_splits_at_prompt_lengths(batch_size):
    """every launch holds rows of one prompt length, in row order; each row runs exactly once; a ragged launch is padded
    with its last row up to the class of min(batch_size, N).  The rows are also the launch's sample ids (row r of a
    prompt-major call is sample r % num_samples of prompt r // num_samples and draws from stream r)."""
    from progen_b200.progen import plan_launches
    lengths = [0, 5, 3, 5, 17]                             # prompt lengths; 5 appears twice (different prompts)
    num_samples = 7
    N = len(lengths) * num_samples
    row_len = [lengths[r // num_samples] for r in range(N)]
    plan = plan_launches(row_len, batch_size, by_length=True)
    per = min(batch_size, N)
    lo = 9 if per > 8 else (2 if per > 1 else 1)
    seen = []
    for rows, real in plan:
        assert rows.dtype == np.int64 and 1 <= real <= per
        assert len(rows) == max(real, lo)
        assert (rows[real:] == rows[real - 1]).all()
        assert (np.diff(rows[:real]) > 0).all()
        assert len({row_len[r] for r in rows}) == 1
        seen += rows[:real].tolist()
    assert sorted(seen) == list(range(N))
    # the launches of one length take that length's rows in order, per_launch at a time
    for L in set(lengths):
        mine = [rows[:real] for rows, real in plan if row_len[rows[0]] == L]
        flat = np.concatenate(mine)
        np.testing.assert_array_equal(flat, [r for r in range(N) if row_len[r] == L])
        assert all(len(m) == per for m in mine[:-1])


def test_forward_plan_of_one_length_is_the_decode_plan():
    from progen_b200.progen import plan_launches
    for N, bs in ((64, 64), (100, 64), (20, 8), (3, 2)):
        a, b = plan_launches([4] * N, bs, by_length=True), plan_launches([4] * N, bs)
        assert [r for _, r in a] == [r for _, r in b]
        for (x, _), (y, _) in zip(a, b):
            np.testing.assert_array_equal(x, y)


def test_cli_rejects_an_unknown_prefill_mode(tmp_path):
    from progen_b200.checkpoint import file_save_checkpoint
    from progen_b200 import ProGen
    (tmp_path / 'ckpts').mkdir()
    file_save_checkpoint(tmp_path / 'ckpts', dict(next_seq_index=0, params=ProGen(**KW).init(1), optim_state=None,
                                                  model_config=KW, run_id=None))
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'generate.py'), '--checkpoint_path', str(tmp_path / 'ckpts'),
                        '--prefill', 'prompt', '--output', str(tmp_path / 'x.fasta')],
                       cwd=str(tmp_path), env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=600)
    assert r.returncode != 0
    assert '--prefill' in r.stderr, r.stderr[-2000:]
    assert not (tmp_path / 'x.fasta').exists()
