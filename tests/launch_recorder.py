"""A stand-in kernel library for recording an engine's launches on the CPU — test infrastructure.

`record_steps()` builds engines on the CPU with a library object that records every C-ABI call instead of running it,
and returns, per workload (objective x full / LoRA x fp32 / bf16 x full / cut length x resident / recompute), the calls
one `Engine.train_step` makes: the function name and its arguments, with every pointer replaced by the order in which
the step first passed it (so the record does not depend on where the host allocator put the buffers) and every
`progen_gemm` descriptor spelled out field by field.  tests/golden/train_launches.json holds the sha256 of each
workload's record as the engine made them before distillation existed (tests/golden/make_launches.py)."""
import ctypes
import hashlib
import json
from types import SimpleNamespace

import numpy as np
import torch

TINY = dict(num_tokens=256, dim=128, seq_len=256, depth=2, window_size=64, heads=2, dim_head=64, global_mlp_depth=1,
            ff_mult=4, ff_glu=True, shift_tokens=True, attn_dim=None, clamp_gate=True)


class StandInLib:
    """records calls; `progen_optim_workspace_floats` and the version queries answer, everything else returns 0"""

    def __init__(self, prototypes):
        self.protos = prototypes
        self.calls = None

    def __getattr__(self, name):
        if not name.startswith('progen_'):
            raise AttributeError(name)
        proto = self.protos[name]

        def call(*args):
            if name == 'progen_optim_workspace_floats':
                return 64
            if self.calls is not None:
                self.calls.append((name, proto, args))
            return 0
        return call


def _canonical(calls, gemm_desc):
    """[(name, argtypes, args)] -> a JSON-able list with pointers renumbered by first use"""
    ids = {}

    def ptr(v):
        v = int(v or 0)
        if v == 0:
            return 'null'
        return 'p%d' % ids.setdefault(v, len(ids))

    out = []
    for name, proto, args in calls:
        row = [name]
        for t, a in zip(proto, args):
            if t is ctypes.c_void_p:
                row.append(ptr(a))
            elif t is ctypes.c_float:
                row.append(float(np.float32(a)))
            elif name == 'progen_gemm' and hasattr(a, '_obj'):
                d = a._obj
                row.append({f: (ptr(getattr(d, f)) if ft is ctypes.c_void_p else int(getattr(d, f)))
                            for f, ft in gemm_desc._fields_})
            else:
                row.append(int(a))
        out.append(row)
    return out


def workloads():
    """(name, objective, lora, mixed_precision, cut, recompute) of every recorded step"""
    out = []
    for obj in ('lm', 'preference', 'property', 'residue'):
        for lora in ((False, True) if obj in ('lm', 'preference') else (True,)):
            for mp in (False, True):
                for cut in (False, True):
                    for rc in (False, True):
                        out.append((f'{obj}-{"lora" if lora else "full"}-{"bf16" if mp else "fp32"}-'
                                    f'{"cut" if cut else "full"}-{"recompute" if rc else "resident"}', obj, lora, mp,
                                    cut, rc))
    return out


def record_steps(monkeypatch):
    """{workload name: canonical launch list of one train_step} (see the module docstring)"""
    from progen_b200 import lib as L
    from progen_b200 import engine as E
    from progen_b200.lora import Adapters, init_adapters
    from progen_b200.property import init_head
    stand_in = StandInLib(L.PROTOTYPES)
    monkeypatch.setattr(L, 'load', lambda: stand_in)
    monkeypatch.setattr(L, 'require_device', lambda: None)
    monkeypatch.setattr(L, 'stream', lambda: 0)
    monkeypatch.setattr(torch.cuda, 'get_device_properties', lambda dev: SimpleNamespace(multi_processor_count=132))
    cfg = dict(TINY)
    n, B = cfg['seq_len'], 4
    rng = np.random.default_rng(0)
    rows = rng.integers(1, 256, (B, n + 1)).astype(np.int32)
    rows[:, 100:] = 0                                     # counted length 100: the cut step runs at 128
    out = {}
    for name, obj, lora, mp, cut, rc in workloads():
        eng = E.Engine(cfg, mp, device='cpu', recompute=rc)
        length = 128 if cut else n
        if lora:
            eng.lora = Adapters(eng, 8, 8.0, head_outputs=3 if obj in ('property', 'residue') else 0)
            eng.lora.load(init_adapters(cfg, 1, 8), init_head(cfg['dim'], 2, 3) if eng.lora.head_outputs else None)
            eng.grads = None
        if obj == 'lm':
            eng.load_batch(rows, length)
            objective, gr = (), B
        elif obj == 'preference':
            eng.load_preference(rows, np.zeros(B, np.float32), length)
            objective, gr = ('preference', 0.1), B // 2
        elif obj == 'property':
            eng.load_property(rows, L.TASK_REGRESSION, np.zeros((B, 3), np.float32), length)
            objective, gr = ('property', L.TASK_REGRESSION), B
        else:
            y = np.full((B, n, 3), np.nan, np.float32)
            y[:, 1:50] = 0.5
            eng.load_residue(rows, L.TASK_REGRESSION, y, length)
            objective, gr = ('residue', L.TASK_REGRESSION), B
        stand_in.calls = []
        eng.train_step(objective, gr, length=length)
        out[name] = _canonical(stand_in.calls, L.GemmDesc)
        stand_in.calls = None
    return out


def digest(record):
    return hashlib.sha256(json.dumps(record, sort_keys=True).encode()).hexdigest()
