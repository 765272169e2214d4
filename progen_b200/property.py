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


# ------------------------------------------------------------------------------------------------ per-residue labels
def residue_positions(rows):
    """rows (B, n+1) of the `collate` contract -> bool [B, n]: the positions that hold a residue.  The input id at
    position t >= 1 is residue t - 1; position 0 (BOS) and pad inputs hold none."""
    m = np.asarray(rows)[:, :-1] != 0
    m[:, 0] = False
    return m


def check_residue_targets(rows, targets, task, C, what):
    """Per-residue targets of checked rows (B, n+1) -> (targets, labelled [B, n] bool) in the layout the engine reads:
    regression float32 [B, n, C] with NaN at unlabelled positions, classification int32 [B, n] with -1 there.
    Regression targets are float [B, n, C] (or [B, n] when C == 1): a position is unlabelled when all of its values are
    NaN; one with only some of them NaN, or with a value that is not finite in float32, is refused.  Classification
    targets are integers [B, n] in [0, C), -1 meaning unlabelled.  A label at position 0 (BOS) or on a pad input is
    refused, and so is a batch without a labelled position.  ProgenError names the first offending (row, position)."""
    code = check_task(task)
    B, n = rows.shape[0], rows.shape[1] - 1
    first = lambda bad: tuple(int(i) for i in np.argwhere(bad)[0])
    if code == L.TASK_REGRESSION:
        try:
            y = np.asarray(targets, np.float64)
        except (TypeError, ValueError):
            raise L.ProgenError(f'{what}: targets must be numbers, shape ({B}, {n}, {C})') from None
        if C == 1 and y.shape == (B, n):
            y = y[..., None]
        if y.shape != (B, n, C):
            raise L.ProgenError(f'{what}: targets must have shape ({B}, {n}, {C}) (rows, positions, head outputs), '
                                f'got {y.shape}')
        nan = np.isnan(y)
        labelled = ~nan.all(-1)
        part = nan.any(-1) & labelled
        if part.any():
            raise L.ProgenError(f'{what}: (row, position) {first(part)} has only some of its {C} values NaN; mark an '
                                f'unlabelled position with NaN in every output')
        with np.errstate(over='ignore', invalid='ignore'):
            y32 = y.astype(np.float32)
        bad = labelled & ~np.isfinite(y32).all(-1)
        if bad.any():
            raise L.ProgenError(f'{what}: (row, position) {first(bad)} has a value that is not finite in float32')
        out = np.where(labelled[..., None], y32, np.float32(np.nan)).astype(np.float32)
    else:
        t = np.asarray(targets)
        if t.shape != (B, n):
            raise L.ProgenError(f'{what}: targets must have shape ({B}, {n}) (one class index per position), got {t.shape}')
        if t.dtype.kind not in 'iu':
            raise L.ProgenError(f'{what}: classification targets must be integer class indices, got dtype {t.dtype}')
        bad = (t < -1) | (t >= C)
        if bad.any():
            raise L.ProgenError(f'{what}: (row, position) {first(bad)} has class {int(t[first(bad)])}; classes are in '
                                f'[0, {C}) (the head has {C} classes), -1 marks an unlabelled position')
        labelled = t >= 0
        out = np.where(labelled, t, -1).astype(np.int32)
    stray = labelled & ~residue_positions(rows)
    if stray.any():
        b, p = first(stray)
        raise L.ProgenError(f'{what}: (row, position) {(b, p)} is labelled but holds no residue '
                            f'({"position 0 is BOS" if p == 0 else "its input is pad"}); position t labels residue t - 1')
    if not labelled.any():
        raise L.ProgenError(f'{what}: no labelled position in the batch')
    return out, labelled


def residue_length(rows, labelled, length, what):
    """the row length of a residue step or forward over rows (B, n+1) whose labelled (or predicted) positions are
    `labelled` [B, n]: engine.check_length of the rows (None: their cut_length), which must also cover every labelled
    position; None grows the cut to cover them (only rows with a pad inside a sequence need that)"""
    from .engine import CUT_ALIGN, check_length
    n = rows.shape[1] - 1
    cut = check_length(rows[:, 1:], length, what)
    cols = np.flatnonzero(np.asarray(labelled).any(0))
    need = int(cols[-1]) + 1 if cols.size else 1
    if need <= cut:
        return cut
    if length is not None:
        raise L.ProgenError(f'{what}: length {length} cuts off labelled position {need - 1}')
    return min(n, -(-need // CUT_ALIGN) * CUT_ALIGN)


def read_residue_labelled(lines, task):
    """Per-residue labels of a text file, one `sequence<TAB>labels` line per sequence (blank lines skipped):
    classification labels are one class character per residue, `.` for an unlabelled residue; regression labels are
    comma-separated numbers, one per residue, `nan` for an unlabelled one.  The label count must equal the sequence's
    length.  Returns (sequences, labels): labels a list of strings (classification) or of float64 arrays (regression).
    A bad line raises ProgenError naming it (1-based)."""
    code = check_task(task)
    seqs, labels = [], []
    for i, line in enumerate(lines, start=1):
        line = line.rstrip('\r\n')
        if not line.strip():
            continue
        parts = line.split('\t')
        seq = parts[0].strip()
        if not seq:
            raise L.ProgenError(f'line {i}: empty sequence')
        if len(parts) != 2:
            raise L.ProgenError(f'line {i}: expected `sequence<TAB>labels`, got {len(parts) - 1} tabs')
        lab = parts[1].strip()
        if code == L.TASK_CLASSIFICATION:
            got = lab
        else:
            try:
                got = np.array([float(v) for v in lab.split(',')], np.float64)
            except ValueError:
                raise L.ProgenError(f'line {i}: per-residue values must be comma-separated numbers (nan: unlabelled)') \
                    from None
            if np.isinf(got).any():
                raise L.ProgenError(f'line {i}: values must be finite or nan (unlabelled)')
        if len(got) != len(seq):
            raise L.ProgenError(f'line {i}: {len(got)} labels for a sequence of {len(seq)} residues')
        seqs.append(seq)
        labels.append(got)
    return seqs, labels


def residue_label_array(labels, task, classes, seq_len):
    """file labels (read_residue_labelled) -> per-position targets of their `collate` rows: classification int32
    [N, seq_len] (class index, -1 unlabelled), regression float64 [N, seq_len] (NaN unlabelled).  Residue i sits at
    position i + 1; residues past position seq_len - 1 have no representation and are dropped, as collate truncates.
    ProgenError names a class character that is not one of `classes`."""
    code = check_task(task)
    N = len(labels)
    if code == L.TASK_CLASSIFICATION:
        index = {c: k for k, c in enumerate(classes)}
        out = np.full((N, seq_len), -1, np.int32)
        for r, lab in enumerate(labels):
            for i, ch in enumerate(lab[:seq_len - 1]):
                if ch == '.':
                    continue
                if ch not in index:
                    raise L.ProgenError(f'sequence {r}: class {ch!r} is not one of the training classes {classes}')
                out[r, i + 1] = index[ch]
        return out
    out = np.full((N, seq_len), np.nan, np.float64)
    for r, lab in enumerate(labels):
        v = np.asarray(lab, np.float64)[:seq_len - 1]
        out[r, 1:1 + len(v)] = v
    return out


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
