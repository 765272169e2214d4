"""design.py without a device: --help carries the on-policy note, argument errors stop before any device work, and the
iteration helpers (prompt rotation, seeds, micro-steps)."""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)


def _run(*args, cwd=ROOT):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES='', PYTHONPATH=ROOT)
    return subprocess.run([sys.executable, os.path.join(ROOT, 'design.py'), *args], cwd=cwd, env=env,
                          capture_output=True, text=True, timeout=300)


def test_help_needs_no_device_and_states_the_on_policy_condition():
    r = _run('--help')
    assert r.returncode == 0, r.stderr
    text = ' '.join(r.stdout.split())
    assert 'on-policy only' in text and 'temperature 1' in text
    for flag in ('--reward_checkpoint', '--reward_output', '--reward_class', '--group_size', '--prompts_per_step',
                 '--lora_rank', '--grad_accum_every', '--batch_size', '--checkpoint_path', '--min_new_tokens'):
        assert flag in r.stdout, flag


@pytest.mark.parametrize('args,message', [
    ([], 'reward_checkpoint'),
    (['--reward_checkpoint', 'R'], 'exactly one of --reward_output'),
    (['--reward_checkpoint', 'R', '--reward_output', '0', '--reward_class', 'a'], 'exactly one of --reward_output'),
    (['--reward_checkpoint', 'R', '--reward_output', '0', '--beta', '-1'], 'beta'),
    (['--reward_checkpoint', 'R', '--reward_output', '0', '--group_size', '0'], '--group_size must be >= 1'),
    (['--reward_checkpoint', 'R', '--reward_output', '0', '--grad_accum_every', '0'], '--grad_accum_every'),
    (['--reward_checkpoint', 'R', '--reward_output', '0', '--lora_alpha', '4'], '--lora_alpha needs --lora_rank'),
])
def test_argument_errors_need_no_device(tmp_path, args, message):
    r = _run(*args, '--checkpoint_path', str(tmp_path / 'out'), cwd=str(tmp_path))
    assert r.returncode != 0
    assert message in ' '.join(r.stderr.split()), r.stderr


def test_a_new_run_needs_init_checkpoint(tmp_path):
    r = _run('--reward_checkpoint', str(tmp_path / 'r'), '--reward_output', '0', '--checkpoint_path', str(tmp_path / 'o'))
    assert r.returncode != 0 and 'needs --init_checkpoint' in r.stderr, r.stderr


def test_iteration_helpers():
    import design
    assert design.iteration_prompts(['a', 'b', 'c'], 0, 2) == ['a', 'b']
    assert design.iteration_prompts(['a', 'b', 'c'], 1, 2) == ['c', 'a']
    assert design.iteration_seed(0, 3) == design.iteration_seed(0, 3) != design.iteration_seed(0, 4)
    assert design.micro_batches(64, 64) == [(0, 64)]
    assert design.micro_batches(10, 4) == [(0, 4), (4, 8), (8, 10)]
