"""Host side of position-specific generation constraints (no GPU): the tables `ProGen.generate` builds from `fixed` and
`position_bias`, their checks, the split of queue chunks under the table byte budget, and generate.py's --fix."""
import os
import subprocess
import sys

import numpy as np
import pytest

from progen_b200.lib import ProgenError
from progen_b200.progen import plan_queue, position_tables, launch_tables
import progen_b200.progen as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KW = dict(num_tokens=256, dim=64, seq_len=64, depth=2, window_size=16, global_mlp_depth=1, heads=2, dim_head=32)
V, N = 256, 64


def test_fixed_residues_become_one_hot_rows_with_eos_banned_before_the_last():
    tables, pt = position_tables([3], V, N, N, fixed={2: 'H', 5: 20})
    assert pt.tolist() == [0] and len(tables) == 1
    t = tables[0]
    assert t.shape == (5, V) and t.dtype == np.float32
    h = ord('H') + 1                                      # encoded like training text
    for j, c in ((1, h), (4, 20)):
        assert t[j, c] == 0.0 and np.isneginf(np.delete(t[j], c)).all()
    for j in (0, 2, 3):                                   # earlier free offsets: only EOS banned
        assert t[j, 0] == -np.inf and (t[j, 1:] == 0.0).all()


def test_fixed_adds_to_the_prompts_position_bias():
    rng = np.random.default_rng(0)
    b = rng.standard_normal((7, V)).astype(np.float32)
    tables, pt = position_tables([1], V, N, N, position_bias=b, fixed={3: 'A'})
    t = tables[pt[0]]
    assert t.shape == (7, V)
    a = ord('A') + 1
    assert t[2, a] == b[2, a] and np.isneginf(np.delete(t[2], a)).all()
    assert t[0, 0] == t[1, 0] == -np.inf
    np.testing.assert_array_equal(t[0, 1:], b[0, 1:])
    np.testing.assert_array_equal(t[3:], b[3:])           # past the last fixed offset: the bias alone (EOS allowed)
    # a fixed offset past the bias's end lengthens the table
    t2 = position_tables([1], V, N, N, position_bias=b[:2], fixed={5: 'A'})[0][0]
    assert t2.shape == (5, V) and t2[4, a] == 0.0
    np.testing.assert_array_equal(t2[1, 1:], b[1, 1:])


def test_identical_tables_are_stored_once():
    b = np.zeros((4, V), np.float32)
    b[1, 5] = -np.inf
    tables, pt = position_tables([1, 3, 5, 2], V, N, N, position_bias=[b, b.copy(), None, b], fixed=[None, None, {1: 9}, None])
    assert len(tables) == 2 and pt.tolist() == [0, 0, 1, 0]
    tables, pt = position_tables([1] * 9, V, N, N, position_bias=b)      # one array for every prompt
    assert len(tables) == 1 and pt.tolist() == [0] * 9
    tables, pt = position_tables([1, 2], V, N, N)
    assert tables == [] and pt.tolist() == [-1, -1]


def test_launch_tables_stack_the_used_tables_zero_padded():
    t0, t1, t2 = (np.full((k, V), float(k), np.float32) for k in (2, 5, 3))
    row_table = np.array([1, -1, 2, 1, 0, -1])
    stack, m = launch_tables([t0, t1, t2], row_table, np.array([0, 1, 2, 3]))
    assert stack.shape == (2, 5, V) and m.dtype == np.int32 and m.tolist() == [0, -1, 1, 0]
    np.testing.assert_array_equal(stack[0], t1)
    np.testing.assert_array_equal(stack[1, :3], t2)
    assert (stack[1, 3:] == 0).all()
    assert launch_tables([t0, t1, t2], row_table, np.array([1, 5])) is None


@pytest.mark.parametrize('kwargs,words', [
    (dict(fixed={0: 'A'}), ('prompt 0', 'offset 0')),
    (dict(fixed={-2: 'A'}), ('prompt 0',)),
    (dict(fixed={62: 'A'}), ('prompt 0', '62')),          # start 3: offsets 1 .. 61 fit before max_length 64
    (dict(fixed={1: 'Ā'}), ('prompt 0', 'vocabulary')),   # encodes to id 257
    (dict(fixed={1: 0}), ('vocabulary',)),                # EOS is not a residue
    (dict(fixed={1: 256}), ('vocabulary',)),
    (dict(fixed={1: 'AB'}), ('one character',)),
    (dict(fixed={1.0: 'A'}), ('prompt 0',)),
    (dict(fixed=[{1: 'A'}]), ('list of 2',)),             # per-prompt list of the wrong length
    (dict(position_bias=[np.zeros((2, V))] * 3), ('list of 2',)),
    (dict(position_bias=np.zeros((2, V - 1))), ('shape',)),
    (dict(position_bias=np.zeros((N + 1, V))), ('shape',)),
    (dict(position_bias=np.zeros((0, V))), ('shape',)),
    (dict(position_bias=np.full((2, V), np.nan)), ('NaN',)),
    (dict(position_bias=np.full((2, V), np.inf)), ('NaN',)),
    (dict(position_bias=np.full((2, V), 1e300)), ('NaN',)),   # +inf in float32
])
def test_bad_tables_are_refused_naming_prompt_and_offset(kwargs, words):
    with pytest.raises(ProgenError) as e:
        position_tables([3, 1], V, N, N, **kwargs)
    for w in words:
        assert w in str(e.value), str(e.value)


def test_no_candidate_is_refused():
    a = ord('A') + 1
    lb = np.zeros(V, np.float32)
    lb[a] = -np.inf
    with pytest.raises(ProgenError, match='prompt 1 .* offset 4'):       # a fixed residue banned by logit_bias
        position_tables([1, 2], V, N, N, fixed=[None, {4: 'A'}], logit_bias=lb)
    only_eos = np.full((3, V), -np.inf, np.float32)
    only_eos[:, 0] = 0.0
    tables, _ = position_tables([1], V, N, N, position_bias=only_eos)   # EOS alone is legal: it ends the row
    assert len(tables) == 1
    with pytest.raises(ProgenError, match='offset 1'):                  # ... unless min_new_tokens bans it
        position_tables([1], V, N, N, position_bias=only_eos, min_new_tokens=1)
    b = np.zeros((3, V), np.float32)
    b[2, a] = -np.inf
    with pytest.raises(ProgenError, match='offset 3'):                  # the prompt's own bias bans the fixed residue
        position_tables([1], V, N, N, position_bias=b, fixed={3: 'A'})
    # a row past max_length is never drawn, so it is not checked
    dead = np.zeros((10, V), np.float32)
    dead[9] = -np.inf
    position_tables([1], V, N, 10, position_bias=dead)
    with pytest.raises(ProgenError, match='offset 10'):
        position_tables([1], V, N, 11, position_bias=dead)


@pytest.mark.parametrize('kwargs', [
    dict(fixed={0: 'A'}), dict(fixed={70: 'A'}), dict(fixed=[{1: 'A'}, None]), dict(fixed={1: 'Ā'}),
    dict(position_bias=np.zeros((3, 7))), dict(fixed={1: 'A'}, logit_bias=np.where(np.arange(256) == 66, -np.inf, 0.0)),
])
def test_generate_refuses_bad_tables_without_a_device(kwargs):
    from progen_b200 import ProGen
    model = ProGen(**KW)
    with pytest.raises(ProgenError):
        model.generate({}, 'MK', **kwargs)
    assert model._engine is None and model._gen_decoder is None


def test_queue_chunks_split_under_the_table_budget(monkeypatch):
    row_table = np.repeat(np.arange(40), 3)              # 120 rows, 40 distinct tables, 3 rows each
    slots, base = plan_queue(120, 8)
    assert len(base) == 1
    assert plan_queue(120, 8, row_table, 1 << 20)[1][0].size == 120       # 40 MiB: under the default budget
    monkeypatch.setattr(P, 'QUEUE_TABLE_BYTES', 10 << 20)                 # 10 tables of 1 MiB per launch
    slots, chunks = plan_queue(120, 8, row_table, 1 << 20)
    assert slots == 8
    np.testing.assert_array_equal(np.concatenate(chunks), np.arange(120))
    assert [c.size for c in chunks] == [30, 30, 30, 30]
    assert all(len(np.unique(row_table[c])) <= 10 for c in chunks)
    # never below `slots` rows: a short tail joins the chunk before it
    slots, chunks = plan_queue(32, 8, np.arange(32), 1 << 20)
    assert [c.size for c in chunks] == [10, 10, 12]
    monkeypatch.setattr(P, 'QUEUE_TABLE_BYTES', 1)
    slots, chunks = plan_queue(20, 8, np.arange(20), 1 << 20)
    assert [c.size for c in chunks] == [8, 12]
    # rows without a table cost nothing
    slots, chunks = plan_queue(20, 8, np.full(20, -1), 1 << 20)
    assert [c.size for c in chunks] == [20]


def test_parse_fix():
    from generate import parse_fix
    assert parse_fix('12=H,57=D,102=S') == {12: 'H', 57: 'D', 102: 'S'}
    assert parse_fix(' 3 = C ') == {3: 'C'}
    for bad in ('', '12', '12=', '12=HH', 'x=H', '-1=H', '1=H,1=C', '1=H,,2=C'):
        with pytest.raises(ProgenError, match='--fix'):
            parse_fix(bad)


@pytest.fixture(scope='module')
def ckpt(tmp_path_factory):
    from progen_b200.checkpoint import file_save_checkpoint
    from progen_b200 import ProGen
    d = tmp_path_factory.mktemp('ck')
    (d / 'ckpts').mkdir()
    file_save_checkpoint(d / 'ckpts', dict(next_seq_index=0, params=ProGen(**KW).init(1), optim_state=None,
                                           model_config=KW, run_id=None))
    return d


def _cli(ckpt, *args):
    out = ckpt / 'x.fasta'
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'generate.py'), '--checkpoint_path', str(ckpt / 'ckpts'),
                        '--output', str(out), *args], cwd=str(ckpt), env=dict(os.environ, PYTHONPATH=ROOT),
                       capture_output=True, text=True, timeout=600)
    assert r.returncode != 0
    assert 'Traceback' not in r.stderr, r.stderr[-2000:]
    assert not out.exists()
    return r.stderr


def test_cli_fixed_residue_outside_the_alphabet(ckpt):
    err = _cli(ckpt, '--alphabet', 'ACDE', '--fix', '3=W')
    assert 'ProgenError' in err and 'offset 3' in err, err


def test_cli_bad_fix_and_position_bias(ckpt):
    assert '--fix' in _cli(ckpt, '--fix', '3W')
    assert 'offset 99' in _cli(ckpt, '--fix', '99=A')
    np.save(ckpt / 'b64.npy', np.zeros((4, 256), np.float64))
    assert 'float32' in _cli(ckpt, '--position_bias', str(ckpt / 'b64.npy'))
    np.save(ckpt / 'bv.npy', np.zeros((4, 100), np.float32))
    assert 'shape' in _cli(ckpt, '--position_bias', str(ckpt / 'bv.npy'))
    assert 'cannot read' in _cli(ckpt, '--position_bias', str(ckpt / 'missing.npy'))
