"""File-system checkpoints with the reference's package layout and naming (progen_transformer/checkpoint.py:12-37,
train.py:196-202): cloudpickle of {next_seq_index, params, optim_state, model_config, run_id} to ckpt_<unix>.pkl, newest =
lexicographically last, keep-last-N.  `params` is the haiku-shaped nested dict of NumPy arrays, so the PARAMETERS of a
checkpoint interchange with the reference once its jax arrays are converted to NumPy.  `optim_state` does not: here it is
{count, mu, nu, acc, every} (Trainer.optim_state), not optax's (ClipState, (ScaleByAdamState, ...), ApplyEvery) tuple —
resuming a reference checkpoint re-initialises the optimizer state (train.py warns), and the reference cannot resume ours.
The GCS twin is out of scope (no network)."""
import os
import time
from functools import partial
from pathlib import Path
from shutil import rmtree

from cloudpickle import pickle


def file_reset_checkpoint(path):
    rmtree(str(path), ignore_errors=True)
    path.mkdir(exist_ok=True, parents=True)


def file_get_last_checkpoint(path):
    checkpoints = sorted(path.glob('**/ckpt_*'))
    if len(checkpoints) == 0:
        return None
    with open(str(checkpoints[-1]), 'rb') as f:
        return pickle.load(f)


def file_save_checkpoint(path, package, keep_last_n=None):
    unix_time = int(time.time())
    checkpoints = sorted(path.glob('**/ckpt_*'))
    target = path / f'ckpt_{unix_time}.pkl'
    while target.exists():                      # two saves within one second must not overwrite each other
        unix_time += 1
        target = path / f'ckpt_{unix_time}.pkl'
    with open(str(target), 'wb') as f:
        pickle.dump(package, f)
    if keep_last_n is None:
        return
    for old in checkpoints[:max(0, len(checkpoints) - keep_last_n)]:
        try:
            os.remove(old)
        except OSError:
            pass


def get_checkpoint_fns(path):
    if str(path).startswith('gs://'):
        raise NotImplementedError('GCS checkpoints are out of scope of this engine (local files only)')
    obj = Path(path)
    obj.mkdir(exist_ok=True, parents=True)
    return tuple(partial(fn, obj) for fn in (file_reset_checkpoint, file_get_last_checkpoint, file_save_checkpoint))
