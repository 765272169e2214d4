"""train.py — drop-in for the reference CLI (lucidrains/progen train.py:36-57: same flags and defaults), running the
H100 engine.  Additions: --synthetic (uniform-random tokens, the BASELINE workload), --num_steps, --text_file (one
sequence per line, instead of TFRecords whose reader needs tensorflow), --group_by_length (sort the rows of each
effective batch by counted length before splitting it into micro-batches), --recompute (keep one residual checkpoint
per layer and re-run each layer's forward in the backward pass, DESIGN.md §3.12; a resumed run may switch it).
Launch with torchrun for --data_parallel.

Every micro-step runs at its rows' cut length (`engine.cut_length`: the longest counted length rounded up to 128);
under data parallelism every rank runs the cut length of the global micro-batch.

Fine-tuning: --init_checkpoint DIR starts from the newest checkpoint there (its params and model_config).  With
--lora_rank R (and --lora_alpha, default R) only low-rank adapters train on the frozen base; the checkpoints written
are adapter packages that name the base checkpoint file instead of storing its parameters (checkpoint.py).  A resumed
run keeps its mode and adapter settings: --lora_rank / --lora_alpha / --init_checkpoint that disagree with the
checkpoint in --checkpoint_path are refused.

Distillation: --teacher_checkpoint DIR trains the student (a config from --config_path / --model_name, or
--init_checkpoint, optionally with --lora_rank) on (1 - alpha) tau^2 KL(teacher || student) + alpha CE at temperature tau
(--distill_temperature, default 2.0) and mix alpha (--distill_alpha, default 0.5), DESIGN.md §3.13.  The teacher is the
newest package in DIR (an adapter package is merged), runs with its own config in --mixed_precision mode, and keeps no
training state.  Validation reports the student's CE and the KL.  Packages record distill = {teacher_checkpoint (the
teacher's file), temperature, alpha}; a resumed run refuses flags that disagree with them.  The student's packages stay
plain packages that sample.py, generate.py, score.py and variants.py load.

The loop is the reference's (train.py:184-222): for each effective batch, grad_accum_every micro-steps of
loss+grads -> optim.update -> apply_updates; checkpoint / validate / sample on the same cadence."""
import os
import time
from pathlib import Path

import click
import numpy as np
import toml
import torch

from progen_b200 import ProGen
from progen_b200 import parallel as PAR
from progen_b200.checkpoint import count_params, get_checkpoint_fns, last_checkpoint_file, load_checkpoint_file
from progen_b200.checkpoint import package_params
from progen_b200.distill import check_objective, check_teacher
from progen_b200.lib import ProgenError
from progen_b200.data import decode_tokens, iterator_from_sequences, iterator_from_tfrecords_folder, synthetic_iterator
from progen_b200.data import group_by_length as length_grouped
from progen_b200.engine import counted_length, cut_length
from progen_b200.utils import sample, confirm, exists


@click.command()
@click.option('--seed', default=42)
@click.option('--batch_size', default=4)
@click.option('--grad_accum_every', default=4)
@click.option('--learning_rate', default=2e-4)
@click.option('--weight_decay', default=1e-3)
@click.option('--data_parallel', default=False, is_flag=True)
@click.option('--max_grad_norm', default=0.5)
@click.option('--validate_every', default=100)
@click.option('--sample_every', default=500)
@click.option('--checkpoint_every', default=1000)
@click.option('--checkpoint_path', default='./ckpts')
@click.option('--checkpoint_keep_n', default=500)
@click.option('--config_path', default='./configs/model')
@click.option('--model_name', default='default')
@click.option('--prime_length', default=25)
@click.option('--seq_len', default=1024)
@click.option('--mixed_precision', default=False, is_flag=True)
@click.option('--data_path', default='./train_data')
@click.option('--wandb_off', default=False, is_flag=True)
@click.option('--wandb_project_name', default='progen-training')
@click.option('--new', default=False, is_flag=True)
@click.option('--synthetic', default=False, is_flag=True, help='uniform-random tokens instead of --data_path')
@click.option('--text_file', default=None, help='one sequence per line (train); last 5%% of lines validate')
@click.option('--num_steps', default=None, type=int, help='stop after this many effective batches')
@click.option('--cuda_graph', default=False, is_flag=True, help='single GPU: capture the training step into a CUDA graph and replay it')
@click.option('--init_checkpoint', default=None, help='fine-tune: start from the newest checkpoint in this directory')
@click.option('--lora_rank', default=None, type=int, help='train low-rank adapters of this rank on the frozen --init_checkpoint')
@click.option('--lora_alpha', default=None, type=float, help='adapter scale alpha (s = alpha / rank; default: the rank)')
@click.option('--group_by_length', default=False, is_flag=True,
              help='sort the rows of each effective batch by length into its micro-batches (each runs at its cut length)')
@click.option('--recompute', default=False, is_flag=True,
              help='recompute activations in the backward pass: one residual checkpoint per layer (less memory, more time)')
@click.option('--teacher_checkpoint', default=None,
              help='distil: train on the logits of the newest package in this directory (the teacher)')
@click.option('--distill_temperature', default=None, type=float, help='distillation temperature tau (default 2.0)')
@click.option('--distill_alpha', default=None, type=float,
              help='weight of the label cross entropy in the distillation loss, in [0, 1] (default 0.5)')
def main(seed, batch_size, grad_accum_every, learning_rate, weight_decay, data_parallel, max_grad_norm, validate_every,
         sample_every, checkpoint_every, checkpoint_path, checkpoint_keep_n, config_path, model_name, prime_length, seq_len,
         mixed_precision, data_path, wandb_off, wandb_project_name, new, synthetic, text_file, num_steps, cuda_graph,
         init_checkpoint, lora_rank, lora_alpha, group_by_length, recompute, teacher_checkpoint, distill_temperature,
         distill_alpha):
    if data_parallel and 'RANK' in os.environ:
        import torch.distributed as dist
        torch.cuda.set_device(int(os.environ.get('LOCAL_RANK', '0')))
        dist.init_process_group('nccl')
    rank, world = PAR.world()
    reset_checkpoint, get_last_checkpoint, save_checkpoint = get_checkpoint_fns(checkpoint_path)
    if new and rank == 0:
        if not confirm('are you sure you want to clear all your checkpoints and restart training?'):
            if world > 1:
                import torch.distributed as dist
                dist.destroy_process_group()
            exit()
        reset_checkpoint()
    if world > 1:
        # every rank must start from the SAME state: rank 0 (which may just have cleared the folder) reads the checkpoint
        # and broadcasts the package; without this the other ranks could load the old files before rank 0 removes them
        import torch.distributed as dist
        box = [get_last_checkpoint() if rank == 0 else None]
        dist.broadcast_object_list(box, src=0)
        last_checkpoint = box[0]
    else:
        last_checkpoint = get_last_checkpoint()
    lora = exists(last_checkpoint) and 'adapters' in last_checkpoint
    base_file = None
    # a resumed run keeps its own mode and adapter settings: flags that would change them are refused, not ignored
    if lora:
        base_file = last_checkpoint['base_checkpoint']          # resume an adapter run: its base, its adapters
        got = last_checkpoint['lora']
        if lora_rank is not None and lora_rank != got['rank']:
            raise click.UsageError(f"--lora_rank {lora_rank}: {checkpoint_path} holds adapters of rank {got['rank']}")
        if lora_alpha is not None and float(lora_alpha) != float(got['alpha']):
            raise click.UsageError(f"--lora_alpha {lora_alpha}: {checkpoint_path} holds adapters with alpha {got['alpha']}")
        if init_checkpoint is not None and last_checkpoint_file(init_checkpoint) != base_file:
            raise click.UsageError(f'--init_checkpoint {init_checkpoint}: its newest checkpoint is not {base_file}, the base '
                                   f'of the adapters in {checkpoint_path}')
    elif exists(last_checkpoint):
        if lora_rank is not None or lora_alpha is not None:
            raise click.UsageError(f'--lora_rank / --lora_alpha: {checkpoint_path} holds a full-parameter checkpoint; '
                                   f'train adapters into another --checkpoint_path')
    elif lora_alpha is not None and lora_rank is None:
        raise click.UsageError('--lora_alpha needs --lora_rank')
    elif not exists(last_checkpoint) and lora_rank is not None and init_checkpoint is None:
        raise click.UsageError('--lora_rank needs --init_checkpoint (the base the adapters are trained on)')
    elif not exists(last_checkpoint) and init_checkpoint is not None:
        base_file = last_checkpoint_file(init_checkpoint)
        assert base_file is not None, f'no checkpoint found in --init_checkpoint {init_checkpoint}'
        lora = lora_rank is not None
    distill = resolve_distill(last_checkpoint, checkpoint_path, teacher_checkpoint, distill_temperature, distill_alpha)
    base = load_checkpoint_file(base_file) if base_file is not None else None
    if exists(last_checkpoint):
        model_kwargs = last_checkpoint['model_config']          # resume: config comes from the checkpoint (train.py:99-100)
    elif base is not None:
        model_kwargs = base['model_config']
    else:
        cfg_file = Path(config_path) / f'{model_name}.toml'
        assert cfg_file.exists(), f'path to your model config {str(cfg_file)} does not exist'
        model_kwargs = toml.loads(cfg_file.read_text())

    model = ProGen(**{**model_kwargs, 'mixed_precision': mixed_precision}, recompute=recompute)
    teacher = teacher_params = None
    if distill is not None:
        teacher_pkg = load_checkpoint_file(distill['teacher_checkpoint'])
        teacher = ProGen(**{**teacher_pkg['model_config'], 'mixed_precision': mixed_precision})
        check_teacher(model, teacher, '--teacher_checkpoint')
        teacher_params = package_params(teacher_pkg)
    adapters, lora_cfg = None, None
    if lora and exists(last_checkpoint):
        params = base['params']
        assert count_params(params) == last_checkpoint['num_params'], f'base checkpoint {base_file} has changed'
        adapters, lora_cfg = last_checkpoint['adapters'], last_checkpoint['lora']
        optim_state, start_seq_index = last_checkpoint['optim_state'], last_checkpoint['next_seq_index']
    elif exists(last_checkpoint):
        params, optim_state, start_seq_index = last_checkpoint['params'], last_checkpoint['optim_state'], last_checkpoint['next_seq_index']
    elif base is not None:
        params, optim_state, start_seq_index = base['params'], None, 0
        if lora:
            adapters = model.init_adapters(seed, lora_rank, alpha=lora_alpha)
            lora_cfg = dict(rank=lora_rank, alpha=float(lora_rank if lora_alpha is None else lora_alpha))
    else:
        params, optim_state, start_seq_index = model.init(seed), None, 0
    trainer = model.trainer(params, learning_rate=learning_rate, weight_decay=weight_decay, max_grad_norm=max_grad_norm,
                            grad_accum_every=grad_accum_every, optim_state=optim_state, data_parallel=data_parallel,
                            cuda_graph=cuda_graph, adapters=adapters, lora_alpha=None if lora_cfg is None else lora_cfg['alpha'],
                            teacher=teacher, teacher_params=teacher_params)
    seq_len = model_kwargs['seq_len']                           # the --seq_len flag is dead in the reference too (train.py:137)
    num_params = model.engine.num_params
    if rank == 0 and lora:
        print(f"adapters: rank {lora_cfg['rank']}, alpha {lora_cfg['alpha']}, {trainer.lora.num_params} parameters on base {base_file}")
    if rank == 0 and distill is not None:
        print(f"distilling {distill['teacher_checkpoint']} at temperature {distill['temperature']}, alpha {distill['alpha']}")

    if synthetic:
        total_train_seqs = 10 ** 9
        train_dataset = synthetic_iterator(seq_len, batch_size, seed=seed + rank)
        valid_dataset = synthetic_iterator(seq_len, batch_size, seed=seed + 10_000)
    elif text_file:
        lines = [l.strip() for l in open(text_file) if l.strip()]
        cut = max(1, int(len(lines) * 0.95))
        total_train_seqs = cut
        train_dataset = iterator_from_sequences(lines[:cut], seq_len, batch_size, skip=start_seq_index, loop=False)
        valid_dataset = iterator_from_sequences(lines[cut:] or lines[:1], seq_len, batch_size, loop=True)
    else:
        # the reference's data layout (train.py:154-170): gzip TFRecords under --data_path, read without tensorflow
        total_train_seqs, get_train_dataset = iterator_from_tfrecords_folder(data_path, data_type='train')
        total_valid_seqs, get_valid_dataset = iterator_from_tfrecords_folder(data_path, data_type='valid')
        assert total_train_seqs > 0, 'no protein sequences found for training'
        assert total_valid_seqs > 0, 'no protein sequences found for validation'
        train_dataset = get_train_dataset(seq_len=seq_len, batch_size=batch_size, skip=start_seq_index)
        valid_dataset = get_valid_dataset(seq_len=seq_len, batch_size=batch_size, loop=True)
    if rank == 0:
        print(f'params: {num_params}')
        print(f'sequence length: {seq_len}')
        print(f'num sequences: {total_train_seqs}')
        print(f'starting from sequence {start_seq_index}')

    effective_batch_size = batch_size * grad_accum_every
    run_id = None
    t0, tokens, counted = time.time(), 0, 0
    for i, seq_index in enumerate(range(start_seq_index, total_train_seqs, effective_batch_size)):
        if num_steps is not None and i >= num_steps:
            break
        group = []
        for _ in range(grad_accum_every):
            try:
                group.append(next(train_dataset))
            except StopIteration:
                break
        # (Adam and the clipping see the micro-steps of a grouped effective batch in another order: hence opt-in)
        for data in length_grouped(group) if group_by_length else group:
            local = PAR.shard_batch(data) if world > 1 else data
            # every rank holds the global micro-batch: the ranks agree on its cut length without communicating
            length = cut_length(data[:, 1:]) if world > 1 else None
            if distill is None:
                loss = trainer.step(local, sync_loss=True, global_batch=data.shape[0], length=length)
            else:
                loss = trainer.distill_step(local, distill['temperature'], distill['alpha'], sync_loss=True,
                                            global_batch=data.shape[0], length=length)
            tokens += data.shape[0] * seq_len
            counted += int(counted_length(data[:, 1:]).sum())
        if len(group) < grad_accum_every:
            return
        if rank == 0:
            print(f'loss: {loss.item()}')
        if i % checkpoint_every == 0 and rank == 0:
            package = {'next_seq_index': seq_index + effective_batch_size, 'optim_state': trainer.optim_state(),
                       'model_config': model_kwargs, 'run_id': run_id}
            if lora:
                package.update(adapters=trainer.adapters(), lora=lora_cfg, base_checkpoint=base_file, num_params=num_params)
            else:
                package['params'] = trainer.params()
            if distill is not None:
                package['distill'] = dict(distill)
            save_checkpoint(package, checkpoint_keep_n)
            print(f"checkpoint to start at sequence index of {package['next_seq_index']}")
        if i % validate_every == 0:
            valid_data = next(valid_dataset)
            if distill is None:
                vloss = trainer.evaluate(valid_data)
                if rank == 0:
                    print(f'valid_loss: {vloss.item()}')
            else:
                trainer.evaluate_distill(valid_data, distill['temperature'], distill['alpha'])
                st = trainer.distill_stats()
                if rank == 0:
                    print(f"valid_loss: {float(st['ce'].mean())}")      # the student's CE, comparable with an LM run
                    print(f"valid_kl: {float(st['kl'].mean())}")
        if i % sample_every == 0 and rank == 0:
            valid_data = next(valid_dataset)[0]
            prime = valid_data[:prime_length]
            prime_str = decode_tokens(prime)
            cur = model.merge_adapters(params, trainer.adapters(), lora_alpha=lora_cfg['alpha']) if lora else trainer.params()
            sampled = sample(seed, model.apply, cur, prime, seq_len, top_k=25)
            if lora:
                trainer.eng.load_params(params)            # the engine's base again (apply loaded the merged weights)
            print(prime_str, '\n', '*' * 40, '\n', decode_tokens(sampled[prime_length:]))
    if rank == 0:
        elapsed = max(1e-9, time.time() - t0)
        print(f'tokens/sec (host clock, incl. logging syncs): {tokens / elapsed:.0f}')
        print(f'counted tokens/sec (the positions the loss counts, same clock): {counted / elapsed:.0f}')
    if world > 1:
        import torch.distributed as dist
        trainer._graph = None                      # a captured step references the communicator: drop it before NCCL goes away
        torch.cuda.synchronize()
        dist.barrier()
        dist.destroy_process_group()


def resolve_distill(last_checkpoint, checkpoint_path, teacher_checkpoint, temperature, alpha):
    """the run's distillation settings {teacher_checkpoint (file), temperature, alpha}, or None for an LM run: from the
    flags on a new run, from the package on a resumed one (flags that disagree with it are refused)"""
    got = last_checkpoint.get('distill') if exists(last_checkpoint) else None
    if exists(last_checkpoint) and got is None:
        if teacher_checkpoint is not None or temperature is not None or alpha is not None:
            raise click.UsageError(f'--teacher_checkpoint / --distill_temperature / --distill_alpha: {checkpoint_path} '
                                   f'holds a checkpoint of a run without a teacher; distil into another --checkpoint_path')
        return None
    if got is not None:
        if teacher_checkpoint is not None and last_checkpoint_file(teacher_checkpoint) != got['teacher_checkpoint']:
            raise click.UsageError(f"--teacher_checkpoint {teacher_checkpoint}: its newest package is not "
                                   f"{got['teacher_checkpoint']}, the teacher of the run in {checkpoint_path}")
        if temperature is not None and float(temperature) != float(got['temperature']):
            raise click.UsageError(f"--distill_temperature {temperature}: the run in {checkpoint_path} distils at "
                                   f"temperature {got['temperature']}")
        if alpha is not None and float(alpha) != float(got['alpha']):
            raise click.UsageError(f"--distill_alpha {alpha}: the run in {checkpoint_path} distils with alpha {got['alpha']}")
        return dict(got)
    if teacher_checkpoint is None:
        if temperature is not None or alpha is not None:
            raise click.UsageError('--distill_temperature / --distill_alpha need --teacher_checkpoint')
        return None
    teacher_file = last_checkpoint_file(teacher_checkpoint)
    if teacher_file is None:
        raise click.UsageError(f'--teacher_checkpoint {teacher_checkpoint}: no checkpoint found there')
    try:
        tau, a = check_objective(2.0 if temperature is None else temperature, 0.5 if alpha is None else alpha,
                                 '--distill_temperature / --distill_alpha')
    except ProgenError as e:
        raise click.UsageError(str(e)) from None
    return dict(teacher_checkpoint=teacher_file, temperature=tau, alpha=a)


if __name__ == '__main__':
    main()
