"""File-system checkpoints with the reference's package layout and naming (progen_transformer/checkpoint.py:12-37,
train.py:196-202): cloudpickle of {next_seq_index, params, optim_state, model_config, run_id} to ckpt_<unix>.pkl, newest =
lexicographically last, keep-last-N.  `params` is the haiku-shaped nested dict of NumPy arrays, so the PARAMETERS of a
checkpoint interchange with the reference once its jax arrays are converted to NumPy.  `optim_state` does not: here it is
{count, mu, nu, acc, every} (Trainer.optim_state), not optax's (ClipState, (ScaleByAdamState, ...), ApplyEvery) tuple —
resuming a reference checkpoint re-initialises the optimizer state (train.py warns), and the reference cannot resume ours.
The GCS twin is out of scope (no network).

A low-rank adapter package (train.py --lora_rank) stores {adapters, lora: {rank, alpha}, optim_state (the adapters'),
model_config, next_seq_index, base_checkpoint (absolute path of the base checkpoint file), num_params (the base's)}
and no base parameters; `package_params` resolves either kind of package to the parameters to run."""
import os
import time
from functools import partial
from pathlib import Path
from shutil import rmtree

import numpy as np
from cloudpickle import pickle


def file_reset_checkpoint(path):
    rmtree(str(path), ignore_errors=True)
    path.mkdir(exist_ok=True, parents=True)


def last_checkpoint_file(path):
    """the newest checkpoint file under directory `path` (absolute), or None"""
    checkpoints = sorted(Path(path).glob('**/ckpt_*'))
    return str(checkpoints[-1].resolve()) if checkpoints else None


def load_checkpoint_file(file):
    with open(str(file), 'rb') as f:
        return pickle.load(f)


def file_get_last_checkpoint(path):
    last = last_checkpoint_file(path)
    return None if last is None else load_checkpoint_file(last)


def count_params(params):
    return int(sum(np.size(a) for leaves in params.values() for a in leaves.values()))


def package_params(package):
    """The parameters a checkpoint package runs with: its `params`, or for a low-rank adapter package the base
    checkpoint's params with the adapters merged in (W + (alpha / rank) A B, in float64, cast to float32).  Raises
    ProgenError when the base checkpoint file is missing or its parameter count is not the one the package recorded."""
    if 'adapters' not in package:
        return package['params']
    from .lib import ProgenError
    from .lora import check_adapters, check_rank_alpha, merge_adapters
    base_file = package['base_checkpoint']
    if not os.path.isfile(base_file):
        raise ProgenError(f'adapter checkpoint: its base checkpoint {base_file} is missing (the adapters are trained on '
                          f'that exact file)')
    base = load_checkpoint_file(base_file)['params']
    if count_params(base) != package['num_params']:
        raise ProgenError(f'adapter checkpoint: base checkpoint {base_file} has {count_params(base)} parameters, the '
                          f'adapters were trained on {package["num_params"]}')
    from .progen import ProGen
    cfg = ProGen(**package['model_config']).config
    rank, alpha = check_rank_alpha(check_adapters(cfg, package['adapters']), package['lora']['alpha'])
    if rank != package['lora']['rank']:
        raise ProgenError(f'adapter checkpoint: adapters of rank {rank}, the package records rank {package["lora"]["rank"]}')
    return merge_adapters(base, package['adapters'], alpha / rank)


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
