"""Writes tests/golden/train_launches.json: the sha256 of every workload's launch record (tests/launch_recorder.py).
It was run at the commit before distillation was added, so the file pins the launches the LM, preference, property and
residue steps made then.  Usage: python tests/golden/make_launches.py"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

if __name__ == '__main__':
    import pytest
    from launch_recorder import digest, record_steps
    with pytest.MonkeyPatch.context() as mp:
        rec = record_steps(mp)
    with open(os.path.join(HERE, 'train_launches.json'), 'w') as f:
        json.dump({k: digest(v) for k, v in rec.items()}, f, indent=1, sort_keys=True)
        f.write('\n')
