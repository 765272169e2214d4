"""Input checks and the pairs file of preference (DPO) fine-tuning: `ProGen.preference_loss_and_grad`,
`Trainer.preference_step` and dpo.py.  Everything here runs on the host, before any device work."""
import math

import numpy as np

from . import lib as L


def _rows(a, what, seq_len):
    a = np.asarray(a)
    if a.ndim != 2 or a.shape[1] != seq_len + 1:
        raise L.ProgenError(f'{what} must be (P, seq_len + 1 = {seq_len + 1}) integer rows, got shape {a.shape}')
    if a.dtype.kind not in 'iu':
        raise L.ProgenError(f'{what} must hold integer token ids, got dtype {a.dtype}')
    return a


def _ref(a, what, P):
    try:
        r = np.asarray(a, np.float64)
    except (TypeError, ValueError):
        raise L.ProgenError(f'{what} must be {P} floats (log-likelihoods from `score`)') from None
    if r.shape != (P,):
        raise L.ProgenError(f'{what} must have shape ({P},) (one log-likelihood per pair), got {r.shape}')
    with np.errstate(over='ignore'):
        r32 = r.astype(np.float32)
    if not np.isfinite(r32).all():
        raise L.ProgenError(f'{what} must be finite (in float32)')
    return r32


def check_pairs(chosen, rejected, ref_chosen, ref_rejected, beta, global_pairs, seq_len, what='preference_loss_and_grad',
                allow_empty=False):
    """Check one preference batch and return (rows, ref, beta, global_pairs): rows (2P, seq_len + 1) int32, the chosen
    rows then the rejected rows; ref [2P] float32 in the same order; beta a float; global_pairs an int (default P).
    Raises ProgenError naming the bad input.  allow_empty: P = 0 is accepted (a data-parallel rank without pairs), with
    global_pairs >= 1 given."""
    c = _rows(chosen, f'{what}: chosen', seq_len)
    r = _rows(rejected, f'{what}: rejected', seq_len)
    if c.shape != r.shape:
        raise L.ProgenError(f'{what}: chosen and rejected must have the same shape, got {c.shape} and {r.shape}')
    P = c.shape[0]
    if P < 1 and not allow_empty:
        raise L.ProgenError(f'{what}: needs at least one pair (P >= 1)')
    rc = _ref(ref_chosen, f'{what}: ref_chosen', P)
    rr = _ref(ref_rejected, f'{what}: ref_rejected', P)
    ok = not isinstance(beta, (bool, np.bool_)) and isinstance(beta, (int, float, np.integer, np.floating))
    if ok:
        with np.errstate(over='ignore'):
            b32 = float(np.float32(beta))
        ok = math.isfinite(float(beta)) and math.isfinite(b32) and b32 > 0
    if not ok:
        raise L.ProgenError(f'{what}: beta must be a finite number > 0 (in float32), got {beta!r}')
    if global_pairs is None:
        if P < 1:
            raise L.ProgenError(f'{what}: a rank without pairs needs global_pairs')
        global_pairs = P
    if isinstance(global_pairs, (bool, np.bool_)) or not isinstance(global_pairs, (int, np.integer)) or \
            global_pairs < max(P, 1):
        raise L.ProgenError(f'{what}: global_pairs must be an integer >= the pairs given ({max(P, 1)}), got {global_pairs!r}')
    rows = np.concatenate([c, r]).astype(np.int32)
    return rows, np.concatenate([rc, rr]), float(beta), int(global_pairs)


def read_pairs(lines):
    """Pairs of a text file: one pair per line, `chosen<TAB>rejected`, each side a text sequence as in train.py
    --text_file.  Blank lines are skipped.  Returns (chosen, rejected) lists of strings; a line without exactly one tab
    or with an empty side raises ProgenError naming the line (1-based)."""
    chosen, rejected = [], []
    for i, line in enumerate(lines, start=1):
        line = line.rstrip('\r\n')
        if not line.strip():
            continue
        parts = line.split('\t')
        if len(parts) != 2:
            raise L.ProgenError(f'pairs line {i}: expected `chosen<TAB>rejected` (exactly one tab), found {len(parts) - 1} tabs')
        c, r = parts[0].strip(), parts[1].strip()
        if not c or not r:
            raise L.ProgenError(f'pairs line {i}: the chosen and the rejected sequence must both be non-empty')
        chosen.append(c)
        rejected.append(r)
    return chosen, rejected
