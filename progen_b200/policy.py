"""Host side of policy-gradient fine-tuning (DESIGN.md §3.14): `ProGen.policy_loss_and_grad`, `Trainer.policy_step` and
design.py.  `samples_to_rows` turns `generate`'s samples into training rows and the spans of their generated tokens,
`group_advantages` turns rewards into group-relative advantages, and `check_policy_batch` checks one batch before any
device work."""
import math

import numpy as np

from . import lib as L


def samples_to_rows(samples):
    """`ProGen.generate`'s (or `Trainer.generate`'s) dict -> (rows (N, seq_len + 1) int32, span (N, 2) int32).  rows are
    the tokens plus a zero column; span [start - 1, start - 1 + length) holds the label positions of the generated
    tokens, EOS included, so an unfinished row (no EOS before max_length) counts no trailing pad."""
    tok = np.asarray(samples['tokens'])
    start, length = np.asarray(samples['start']), np.asarray(samples['length'])
    N = tok.shape[0]
    rows = np.zeros((N, tok.shape[1] + 1), np.int32)
    rows[:, :-1] = tok
    span = np.stack([start - 1, start - 1 + length], -1).astype(np.int32)
    return rows, span


def group_advantages(rewards, group_size, scale='std'):
    """rewards [N] (N a multiple of group_size; rows of one group consecutive, as `generate` orders a prompt's samples)
    -> float64 advantages [N]: A = r - mean(group), divided by (population std(group) + 1e-6) when scale='std' (as-is
    with scale='none').  A group of equal rewards gives 0."""
    r = np.asarray(rewards, np.float64)
    if isinstance(group_size, (bool, np.bool_)) or not isinstance(group_size, (int, np.integer)) or group_size < 1:
        raise L.ProgenError(f'group_advantages: group_size must be an integer >= 1, got {group_size!r}')
    if r.ndim != 1 or r.size == 0 or r.size % group_size:
        raise L.ProgenError(f'group_advantages: rewards must be a non-empty 1-D array whose length is a multiple of '
                            f'group_size ({group_size}), got shape {r.shape}')
    if not np.isfinite(r).all():
        raise L.ProgenError(f'group_advantages: reward {int(np.argmin(np.isfinite(r)))} is not finite')
    if scale not in ('std', 'none'):
        raise L.ProgenError(f"group_advantages: scale must be 'std' or 'none', got {scale!r}")
    g = r.reshape(-1, group_size)
    a = g - g.mean(-1, keepdims=True)
    if scale == 'std':
        a = a / (g.std(-1, keepdims=True) + 1e-6)
    a[g.max(-1) == g.min(-1)] = 0.0
    return a.reshape(-1)


def check_beta(beta, what):
    """beta: a finite number >= 0 (in float32) -> float; ProgenError otherwise"""
    ok = not isinstance(beta, (bool, np.bool_)) and isinstance(beta, (int, float, np.integer, np.floating))
    if ok:
        with np.errstate(over='ignore'):
            ok = math.isfinite(float(beta)) and math.isfinite(float(np.float32(beta))) and beta >= 0
    if not ok:
        raise L.ProgenError(f'{what}: beta must be a finite number >= 0 (in float32), got {beta!r}')
    return float(beta)


def check_policy_batch(rows, span, advantages, beta, global_rows, seq_len, what='policy_loss_and_grad', allow_empty=False):
    """Check one policy-gradient batch and return (rows (B, seq_len + 1) int32, span (B, 2) int32, advantages [B]
    float32, beta float, global_rows int).  Every span is non-empty, inside the row and inside its counted positions (the
    loss mask of `loss_and_grad`, Q8); advantages are finite in float32; beta is finite and >= 0; global_rows (default B)
    >= B.  Raises ProgenError naming the bad input and the row.  allow_empty: B = 0 (a data-parallel rank without rows)
    with global_rows >= 1 given."""
    from .engine import counted_length
    r = np.asarray(rows)
    if r.ndim != 2 or r.shape[1] != seq_len + 1 or r.dtype.kind not in 'iu':
        raise L.ProgenError(f'{what}: rows must be (B, seq_len + 1 = {seq_len + 1}) integer token ids, got shape '
                            f'{r.shape} of {r.dtype}')
    B = r.shape[0]
    if B < 1 and not allow_empty:
        raise L.ProgenError(f'{what}: needs at least one row')
    s = np.asarray(span)
    if s.shape != (B, 2) or (B and s.dtype.kind not in 'iu'):
        raise L.ProgenError(f'{what}: span must be ({B}, 2) integers (lo, hi), got shape {s.shape}')
    s = s.astype(np.int64)
    labels = r[:, 1:]
    if B:
        pad = labels == 0
        counted = ~pad | ((np.cumsum(pad, axis=-1) == 1) & pad)
        reach = counted_length(labels)
        for i in range(B):
            lo, hi = int(s[i, 0]), int(s[i, 1])
            if not 0 <= lo < hi <= seq_len:
                raise L.ProgenError(f'{what}: row {i}: span ({lo}, {hi}) must satisfy 0 <= lo < hi <= seq_len ({seq_len})')
            if hi > reach[i] or not counted[i, lo:hi].all():
                raise L.ProgenError(f'{what}: row {i}: span ({lo}, {hi}) covers positions the loss mask does not count '
                                    f'(pad labels after the first one)')
    try:
        a = np.asarray(advantages, np.float64)
    except (TypeError, ValueError):
        raise L.ProgenError(f'{what}: advantages must be {B} floats') from None
    if a.shape != (B,):
        raise L.ProgenError(f'{what}: advantages must have shape ({B},), got {a.shape}')
    with np.errstate(over='ignore'):
        a32 = a.astype(np.float32)
    bad = ~np.isfinite(a32)
    if bad.any():
        raise L.ProgenError(f'{what}: row {int(np.argmax(bad))}: advantage {a[np.argmax(bad)]!r} is not finite in float32')
    beta = check_beta(beta, what)
    if global_rows is None:
        if B < 1:
            raise L.ProgenError(f'{what}: a rank without rows needs global_rows')
        global_rows = B
    if isinstance(global_rows, (bool, np.bool_)) or not isinstance(global_rows, (int, np.integer)) or \
            global_rows < max(B, 1):
        raise L.ProgenError(f'{what}: global_rows must be an integer >= the rows given ({max(B, 1)}), got {global_rows!r}')
    return r.astype(np.int32), s.astype(np.int32), a32, beta, int(global_rows)
