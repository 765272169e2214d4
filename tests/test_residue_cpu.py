"""Per-residue fine-tuning without a GPU: the float64 reference the GPU tests compare against (its gradient against finite
differences, for both tasks), the residue -> position alignment, every refusal of the target contract (all before any
device work), the per-residue file of fitness.py, the package's `level` default and the CLI's flag checks."""
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import progen_ref as O
from oracle import progen_torch as T
from property_oracle import HEAD
from residue_oracle import residue_head_loss, residue_loss_and_grads

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _tiny():
    kw = dict(num_tokens=32, dim=16, seq_len=16, depth=2, window_size=8, global_mlp_depth=1, heads=2, dim_head=8)
    cfg = O.make_config(**kw)
    return cfg, O.randomize_params(O.init_params(cfg, 1), 2)


@pytest.mark.parametrize('task', ['regression', 'classification'])
def test_oracle_gradient_matches_finite_differences(task):
    cfg, params = _tiny()
    rng = np.random.default_rng(3)
    rows = rng.integers(1, 32, (3, 17)).astype(np.int64)
    rows[:, 0] = 0
    rows[1, 9:] = 0
    C = 3
    head = {HEAD: {'w': rng.standard_normal((16, C)) * 0.5, 'b': rng.standard_normal(C) * 0.1}}
    if task == 'regression':
        y = rng.standard_normal((3, 16, C))
        y[:, 0] = np.nan
        y[1, 9:] = np.nan
        y[2, 3] = np.nan
    else:
        y = rng.integers(0, C, (3, 16))
        y[:, 0] = -1
        y[1, 9:] = -1
        y[0, 5] = -1
    loss, grads, hgrads, p, row = residue_loss_and_grads(params, head, rows, y, cfg, task)
    lab = (~np.isnan(y).all(-1)) if task == 'regression' else y >= 0
    assert p.shape == (3, 16, C) and np.isclose(loss, row[lab].sum() / lab.sum()) and (row[~lab] == 0).all()

    def f(prm_np, head_np):
        prm = T.to_torch(prm_np)
        _, h = T.forward(prm, torch.as_tensor(rows[:, :-1]), cfg, return_hidden=True)
        w = torch.tensor(head_np[HEAD]['w'], dtype=torch.float64)
        b = torch.tensor(head_np[HEAD]['b'], dtype=torch.float64)
        return float(residue_head_loss(h, w, b, y, task)[0])

    eps = 1e-6
    probes = [(HEAD, 'w', (4, 1)), (HEAD, 'b', (2,)), (O.P + 'layer_norm', 'scale', (5,)),
              (O.P + 'attn1/~/linear', 'w', (3, 7)), (O.P + 'ff0/~/linear', 'w', (2, 9))]
    for m, k, idx in probes:
        src = head if m == HEAD else params
        plus = {mm: {kk: np.array(vv, np.float64) for kk, vv in d.items()} for mm, d in src.items()}
        minus = {mm: {kk: np.array(vv, np.float64) for kk, vv in d.items()} for mm, d in src.items()}
        plus[m][k][idx] += eps
        minus[m][k][idx] -= eps
        if m == HEAD:
            fd = (f(params, plus) - f(params, minus)) / (2 * eps)
            got = hgrads[HEAD][k][idx]
        else:
            fd = (f(plus, head) - f(minus, head)) / (2 * eps)
            got = grads[m][k][idx]
        assert abs(fd - got) <= 1e-5 * max(1.0, abs(fd)), (m, k, fd, got)


# ------------------------------------------------------------------------------------------------ the contract
def _rows():
    from progen_b200.data import collate
    return collate(['MKTAY', 'AC', 'WWWWWWWW'], 8).astype(np.int32)      # seq_len 8: up to 7 residues per row


def test_residue_positions_follow_collate():
    """position t >= 1 holds residue t - 1: the input id there is that residue's byte + 1"""
    from progen_b200.property import residue_label_array, residue_positions
    rows = _rows()
    m = residue_positions(rows)
    assert m.tolist()[0] == [False, True, True, True, True, True, False, False]
    assert m[1].sum() == 2 and m[2].sum() == 7                 # the eighth W has no input position: dropped
    for b, s in enumerate(['MKTAY', 'AC', 'WWWWWWW']):
        for i, ch in enumerate(s):
            assert rows[b, i + 1] == ord(ch) + 1 and m[b, i + 1]
    y = residue_label_array(['ab.ba', 'bb', 'aaaaaaab'], 'classification', ['a', 'b'], 8)
    assert y[0].tolist() == [-1, 0, 1, -1, 1, 0, -1, -1]
    assert y[2].tolist() == [-1, 0, 0, 0, 0, 0, 0, 0]          # the eighth label went with its residue
    v = residue_label_array([np.array([1.0, np.nan, 3.0])], 'regression', None, 8)
    assert np.isnan(v[0, [0, 2, 4, 5, 6, 7]]).all() and v[0, 1] == 1.0 and v[0, 3] == 3.0


def test_check_residue_targets_layout_and_refusals():
    from progen_b200.lib import ProgenError
    from progen_b200.property import check_residue_targets
    rows = _rows()
    cls = np.full((3, 8), -1, np.int64)
    cls[0, 1], cls[2, 7] = 2, 0
    out, lab = check_residue_targets(rows, cls, 'classification', 3, 'w')
    assert out.dtype == np.int32 and lab.sum() == 2 and out[0, 1] == 2
    y = np.full((3, 8), np.nan)
    y[1, 2] = 0.5
    out, lab = check_residue_targets(rows, y, 'regression', 1, 'w')
    assert out.shape == (3, 8, 1) and out.dtype == np.float32 and lab.sum() == 1

    def refused(targets, task, C, match):
        with pytest.raises(ProgenError, match=match):
            check_residue_targets(rows, targets, task, C, 'w')

    bad = cls.copy(); bad[0, 0] = 1
    refused(bad, 'classification', 3, r'\(0, 0\).*BOS')
    bad = cls.copy(); bad[1, 3] = 0
    refused(bad, 'classification', 3, r'\(1, 3\).*pad')
    bad = cls.copy(); bad[2, 4] = 3
    refused(bad, 'classification', 3, r'\(2, 4\) has class 3')
    bad = cls.copy(); bad[0, 2] = -2
    refused(bad, 'classification', 3, r'\(0, 2\) has class -2')
    refused(np.full((3, 8), -1), 'classification', 3, 'no labelled position')
    refused(cls.astype(np.float32), 'classification', 3, 'integer class indices')
    refused(cls[:, :7], 'classification', 3, r'shape \(3, 8\)')
    y3 = np.full((3, 8, 2), np.nan)
    y3[0, 1] = [1.0, np.nan]
    refused(y3, 'regression', 2, r'\(0, 1\) has only some')
    y3[0, 1] = [1.0, np.inf]
    refused(y3, 'regression', 2, r'\(0, 1\) has a value that is not finite')
    y3[0, 1] = [1.0, 1e39]
    refused(y3, 'regression', 2, 'not finite in float32')
    refused(np.full((3, 8, 2), np.nan), 'regression', 2, 'no labelled position')
    refused(np.zeros((3, 8)), 'regression', 2, r'shape \(3, 8, 2\)')
    y1 = np.full((3, 8), np.nan); y1[1, 5] = 1.0
    refused(y1, 'regression', 1, r'\(1, 5\).*pad')


def test_residue_length_covers_labelled_positions():
    from progen_b200.lib import ProgenError
    from progen_b200.property import residue_length
    rows = np.zeros((2, 513), np.int32)
    rows[0, 1:100] = 5
    lab = np.zeros((2, 512), bool)
    lab[0, 99] = True
    assert residue_length(rows, lab, None, 'w') == 128
    assert residue_length(rows, lab, 512, 'w') == 512
    # a residue after a pad inside the row: its own input position 256 is past the counted length (256), so the cut
    # grows to cover its label
    rows[1, 256] = 7
    lab[1, 256] = True
    assert residue_length(rows, lab, None, 'w') == 384
    with pytest.raises(ProgenError, match='cuts off labelled position 256'):
        residue_length(rows, lab, 256, 'w')


# ------------------------------------------------------------------------------------------------ fitness.py
def test_read_residue_labelled():
    from progen_b200.lib import ProgenError
    from progen_b200.property import read_residue_labelled
    seqs, labels = read_residue_labelled(['MKT\tHH.\n', '\n', 'AC\tEC\n'], 'classification')
    assert seqs == ['MKT', 'AC'] and labels == ['HH.', 'EC']
    seqs, labels = read_residue_labelled(['MKT\t1.5,nan,-2\n'], 'regression')
    assert seqs == ['MKT'] and np.isnan(labels[0][1]) and labels[0][2] == -2.0
    for lines, task, match in ((['MKT\tHH\n'], 'classification', 'line 1: 2 labels for a sequence of 3'),
                               (['MKT\t1,2\n'], 'regression', '2 labels'),
                               (['MKT\t1,x,2\n'], 'regression', 'comma-separated'),
                               (['MKT\t1,inf,2\n'], 'regression', 'finite or nan'),
                               (['MKT\n'], 'classification', '0 tabs'),
                               (['AC\tEC\n', '\tEC\n'], 'classification', 'line 2: empty sequence')):
        with pytest.raises(ProgenError, match=match):
            read_residue_labelled(lines, task)


def test_residue_head_cfg_targets_and_metric():
    import fitness
    cfg = fitness.residue_head_cfg(['HH.E', 'CE'], 'classification')
    assert cfg['classes'] == ['C', 'E', 'H'] and cfg['num_outputs'] == 3 and cfg['level'] == 'residue'
    t = fitness.residue_targets(['HH.E', 'CE'], cfg, 8)
    assert t[0].tolist() == [-1, 2, 2, -1, 1, -1, -1, -1]
    pred = np.zeros((2, 8, 3), np.float32)
    pred[0, [1, 2], 2] = 1.0                     # H, H right; elsewhere class 0 (C): right for row 1's C only
    assert fitness.residue_metric(cfg, pred, t) == 'accuracy 0.6000'
    reg = fitness.residue_head_cfg([np.array([1.0, np.nan, 3.0])], 'regression')
    assert reg['num_outputs'] == 1 and np.allclose(reg['target_mean'], [2.0]) and np.allclose(reg['target_std'], [1.0])
    z = fitness.residue_targets([np.array([1.0, np.nan, 3.0])], reg, 8)
    assert z[0, 1] == -1.0 and np.isnan(z[0, 2]) and z[0, 3] == 1.0
    with pytest.raises(Exception, match='at least 2 classes'):
        fitness.residue_head_cfg(['HH.'], 'classification')


def test_package_level_defaults_to_sequence():
    import fitness
    assert fitness.head_level({'task': 'regression'}) == 'sequence'
    assert fitness.head_level({'task': 'regression', 'level': 'residue'}) == 'residue'


def _run(*args):
    env = dict(os.environ, PYTHONPATH=ROOT)
    return subprocess.run([sys.executable, os.path.join(ROOT, 'fitness.py'), *args], cwd=ROOT, env=env,
                          capture_output=True, text=True)


def test_cli_level_flag_checks(tmp_path):
    """--level is checked before any model work: an unknown level, and a resumed run whose package has another level
    (a package without `level` is a sequence-level run)"""
    (tmp_path / 't.tsv').write_text('MKT\tHH.\n')
    out = _run('train', '--train', str(tmp_path / 't.tsv'), '--level', 'atom', '--checkpoint_path', str(tmp_path / 'x'))
    assert out.returncode != 0 and "'atom' is not one of" in out.stderr
    ck = tmp_path / 'fit'
    ck.mkdir()
    pkg = {'head': {'task': 'classification', 'num_outputs': 2}, 'lora': {'rank': 8, 'alpha': 8.0},
           'base_checkpoint': 'nowhere', 'next_index': 0}
    with open(ck / 'ckpt_0', 'wb') as f:
        pickle.dump(pkg, f)
    out = _run('train', '--train', str(tmp_path / 't.tsv'), '--level', 'residue', '--checkpoint_path', str(ck))
    assert out.returncode != 0 and '--level residue' in out.stderr and 'holds a run with sequence' in out.stderr, out.stderr
