"""Host side of property fine-tuning (DESIGN.md §3.9): a head on the pooled sequence embedding, trained with low-rank
adapters on the frozen base.  Input checks for `ProGen.property_loss_and_grad`, `Trainer.property_step` and
`ProGen.predict` (all before any device work), the labelled-sequence file of fitness.py, target standardization and the
Spearman rank correlation of its validation metric."""
import math

import numpy as np

from . import lib as L
from .lora import HEAD

TASKS = {'regression': L.TASK_REGRESSION, 'classification': L.TASK_CLASSIFICATION}


def check_task(task):
    """'regression' | 'classification' -> its task code"""
    if not isinstance(task, str) or task not in TASKS:
        raise L.ProgenError(f"task must be 'regression' or 'classification', got {task!r}")
    return TASKS[task]


def _host(a):
    import torch
    return a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)


def check_head(cfg, head, task=None, what='head'):
    """Validate a head tree {'property_head': {'w': [dim, C], 'b': [C]}} -> C.  ProgenError names the offending part: the
    tree's keys, a shape that disagrees with the model's dim or with the other leaf, C outside [1,
    PROPERTY_MAX_OUTPUTS] (classification: [2, ...]), a non-finite value."""
    if not isinstance(head, dict) or set(head) != {HEAD} or not isinstance(head[HEAD], dict) or \
            set(head[HEAD]) != {'w', 'b'}:
        raise L.ProgenError(f"{what} must be {{'{HEAD}': {{'w': [dim, C], 'b': [C]}}}} (ProGen.init_head)")
    w, b = _host(head[HEAD]['w']), _host(head[HEAD]['b'])
    d = cfg['dim']
    if w.ndim != 2 or w.shape[0] != d:
        raise L.ProgenError(f'{what}: {HEAD}/w must have shape [dim = {d}, C], got {w.shape}')
    C = w.shape[1]
    if b.shape != (C,):
        raise L.ProgenError(f'{what}: {HEAD}/b must have shape ({C},) like the columns of w, got {b.shape}')
    if not 1 <= C <= L.PROPERTY_MAX_OUTPUTS:
        raise L.ProgenError(f'{what}: {C} outputs; a property head has 1 to {L.PROPERTY_MAX_OUTPUTS}')
    if task is not None and check_task(task) == L.TASK_CLASSIFICATION and C < 2:
        raise L.ProgenError(f'{what}: classification needs at least 2 classes, the head has {C} output')
    for name, a in (('w', w), ('b', b)):
        if not np.issubdtype(a.dtype, np.number) or not np.isfinite(a.astype(np.float64)).all():
            raise L.ProgenError(f'{what}: {HEAD}/{name} has a non-finite value')
    return C


def init_head(dim, seed, num_outputs):
    """w ~ TruncatedNormal(1 / sqrt(dim)), b = 0 (the hk.Linear default)"""
    from .progen import _trunc_normal
    if isinstance(num_outputs, (bool, np.bool_)) or not isinstance(num_outputs, (int, np.integer)) or \
            not 1 <= num_outputs <= L.PROPERTY_MAX_OUTPUTS:
        raise L.ProgenError(f'num_outputs must be an integer in [1, {L.PROPERTY_MAX_OUTPUTS}], got {num_outputs!r}')
    g = np.random.default_rng(seed)
    return {HEAD: {'w': _trunc_normal(g, (dim, int(num_outputs)), dim ** -0.5), 'b': np.zeros(int(num_outputs), np.float32)}}


def check_rows(rows, seq_len, what):
    a = np.asarray(rows)
    if a.ndim != 2 or a.shape[1] != seq_len + 1:
        raise L.ProgenError(f'{what}: rows must be (B, seq_len + 1 = {seq_len + 1}) integer rows, got shape {a.shape}')
    if a.dtype.kind not in 'iu':
        raise L.ProgenError(f'{what}: rows must hold integer token ids, got dtype {a.dtype}')
    return a.astype(np.int32)


def check_targets(targets, task, C, B, what):
    """-> regression: float32 [B, C] (a [B] vector when C == 1), finite in float32; classification: int32 [B] in [0, C)"""
    code = check_task(task)
    if code == L.TASK_REGRESSION:
        try:
            y = np.asarray(targets, np.float64)
        except (TypeError, ValueError):
            raise L.ProgenError(f'{what}: targets must be numbers, shape ({B}, {C})') from None
        if C == 1 and y.shape == (B,):
            y = y[:, None]
        if y.shape != (B, C):
            raise L.ProgenError(f'{what}: targets must have shape ({B}, {C}) (rows, head outputs), got {y.shape}')
        with np.errstate(over='ignore'):
            y32 = y.astype(np.float32)
        if not np.isfinite(y32).all():
            raise L.ProgenError(f'{what}: targets must be finite (in float32); missing values are not supported')
        return y32
    t = np.asarray(targets)
    if t.shape != (B,):
        raise L.ProgenError(f'{what}: targets must have shape ({B},) (one class index per row), got {t.shape}')
    if t.dtype.kind not in 'iu':
        raise L.ProgenError(f'{what}: classification targets must be integer class indices, got dtype {t.dtype}')
    if B and (t.min() < 0 or t.max() >= C):
        raise L.ProgenError(f'{what}: class indices must be in [0, {C}) (the head has {C} classes), got '
                            f'{int(t.min())}..{int(t.max())}')
    return t.astype(np.int32)


# ------------------------------------------------------------------------------------------------ fitness.py data
def read_labelled(lines, task):
    """Labelled sequences of a text file: `sequence<TAB>value[<TAB>value...]` (regression, the same number of values on
    every line) or `sequence<TAB>class_name` (classification).  Blank lines are skipped.  Returns (sequences, labels):
    labels a float64 [N, C] array or a list of class names.  A bad line raises ProgenError naming it (1-based)."""
    code = check_task(task)
    seqs, labels, width = [], [], None
    for i, line in enumerate(lines, start=1):
        line = line.rstrip('\r\n')
        if not line.strip():
            continue
        parts = line.split('\t')
        seq = parts[0].strip()
        if not seq or len(parts) < 2:
            raise L.ProgenError(f'line {i}: expected `sequence<TAB>value`, got {len(parts) - 1} tabs'
                                if seq else f'line {i}: empty sequence')
        if code == L.TASK_CLASSIFICATION:
            if len(parts) != 2 or not parts[1].strip():
                raise L.ProgenError(f'line {i}: expected `sequence<TAB>class_name` (one non-empty class name)')
            labels.append(parts[1].strip())
        else:
            try:
                v = [float(p) for p in parts[1:]]
            except ValueError:
                raise L.ProgenError(f'line {i}: values must be numbers, got {parts[1:]!r}') from None
            if not all(math.isfinite(x) for x in v):
                raise L.ProgenError(f'line {i}: values must be finite (missing values are not supported)')
            if width is not None and len(v) != width:
                raise L.ProgenError(f'line {i}: {len(v)} values, earlier lines have {width}')
            width = len(v)
            labels.append(v)
        seqs.append(seq)
    if code == L.TASK_REGRESSION:
        labels = np.asarray(labels, np.float64).reshape(len(seqs), width or 0)
    return seqs, labels


def standardize(y, mean=None, std=None):
    """(y - mean) / std per output, mean and std of y itself by default (a constant output keeps std 1) ->
    (z float32, mean float64 [C], std float64 [C])"""
    y = np.asarray(y, np.float64)
    if mean is None:
        mean = y.mean(0)
        std = y.std(0)
        std = np.where(std > 0, std, 1.0)
    return ((y - mean) / std).astype(np.float32), np.asarray(mean, np.float64), np.asarray(std, np.float64)


def destandardize(z, mean, std):
    """the inverse of standardize, in float64"""
    return np.asarray(z, np.float64) * np.asarray(std, np.float64) + np.asarray(mean, np.float64)


def rankdata(x):
    """ranks 1..N of x with ties given their average rank"""
    x = np.asarray(x, np.float64)
    order = np.argsort(x, kind='mergesort')
    xs = x[order]
    starts = np.flatnonzero(np.r_[True, xs[1:] != xs[:-1]])
    ends = np.r_[starts[1:], len(xs)]
    avg = (starts + ends + 1) / 2.0                       # mean of the 1-based ranks starts+1 .. ends
    ranks = np.empty(len(x), np.float64)
    ranks[order] = np.repeat(avg, ends - starts)
    return ranks


def spearman(x, y):
    """Spearman's rank correlation: the Pearson correlation of the average ranks (nan when either side is constant)"""
    rx, ry = rankdata(x), rankdata(y)
    rx, ry = rx - rx.mean(), ry - ry.mean()
    den = math.sqrt(float((rx * rx).sum()) * float((ry * ry).sum()))
    return float((rx * ry).sum()) / den if den > 0 else float('nan')


def softmax(logits):
    """row softmax in float64"""
    z = np.asarray(logits, np.float64)
    z = np.exp(z - z.max(-1, keepdims=True))
    return z / z.sum(-1, keepdims=True)
