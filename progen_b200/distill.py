"""Input checks and the teacher length rule of distillation (DESIGN.md §3.13): `ProGen.distill_loss_and_grad`,
`Trainer.distill_step` and train.py --teacher_checkpoint.  Everything here runs on the host, before any device work."""
import math

from . import lib as L
from .engine import CUT_ALIGN


def check_objective(temperature, alpha, what='distill'):
    """temperature tau (finite, > 0, with a finite float32 reciprocal) and mix alpha (in [0, 1]) -> (tau, alpha) as
    floats; ProgenError otherwise"""
    try:
        tau, a = float(temperature), float(alpha)
    except (TypeError, ValueError):
        raise L.ProgenError(f'{what}: temperature and alpha must be numbers, got {temperature!r} and {alpha!r}') from None
    if isinstance(temperature, bool) or not math.isfinite(tau) or not tau >= 1e-30:
        raise L.ProgenError(f'{what}: temperature must be finite and > 0 (at least 1e-30), got {temperature!r}')
    if isinstance(alpha, bool) or not 0.0 <= a <= 1.0:
        raise L.ProgenError(f'{what}: alpha must lie in [0, 1], got {alpha!r}')
    return tau, a


def check_teacher(student, teacher, what='distill'):
    """`teacher` (a ProGen, or its config dict) can teach `student` (the same): not the student object itself, the same
    vocabulary, and a seq_len at least the student's.  ProgenError otherwise."""
    if teacher is None:
        raise L.ProgenError(f'{what}: needs a teacher model')
    if teacher is student:
        raise L.ProgenError(f'{what}: the teacher is the student model itself; pass a second model (it may have the '
                            f'same config and parameters)')
    s = student if isinstance(student, dict) else student.config
    t = teacher if isinstance(teacher, dict) else teacher.config
    if t['num_tokens'] != s['num_tokens']:
        raise L.ProgenError(f"{what}: the teacher's vocabulary ({t['num_tokens']} tokens) differs from the student's "
                            f"({s['num_tokens']})")
    if t['seq_len'] < s['seq_len']:
        raise L.ProgenError(f"{what}: the teacher's seq_len ({t['seq_len']}) is below the student's ({s['seq_len']})")


def teacher_length(length, teacher_seq_len):
    """the row length L_t the teacher's forward runs at for a student step of row length `length`: `length` itself when
    it is a valid row length of the teacher (its seq_len, or a multiple of CUT_ALIGN below it), otherwise the smallest
    valid one above it"""
    if length == teacher_seq_len or (0 < length < teacher_seq_len and length % CUT_ALIGN == 0):
        return int(length)
    return min(int(teacher_seq_len), -(-int(length) // CUT_ALIGN) * CUT_ALIGN)
