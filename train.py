"""train.py — drop-in for the reference CLI (lucidrains/progen train.py:36-57: same flags and defaults), running the
H100 engine.  Additions: --synthetic (uniform-random tokens, the BASELINE workload), --num_steps, --text_file (one
sequence per line, instead of TFRecords whose reader needs tensorflow).  Launch with torchrun for --data_parallel.

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
from progen_b200.checkpoint import get_checkpoint_fns
from progen_b200.data import decode_tokens, iterator_from_sequences, iterator_from_tfrecords_folder, synthetic_iterator
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
def main(seed, batch_size, grad_accum_every, learning_rate, weight_decay, data_parallel, max_grad_norm, validate_every,
         sample_every, checkpoint_every, checkpoint_path, checkpoint_keep_n, config_path, model_name, prime_length, seq_len,
         mixed_precision, data_path, wandb_off, wandb_project_name, new, synthetic, text_file, num_steps, cuda_graph):
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
    if not exists(last_checkpoint):
        cfg_file = Path(config_path) / f'{model_name}.toml'
        assert cfg_file.exists(), f'path to your model config {str(cfg_file)} does not exist'
        model_kwargs = toml.loads(cfg_file.read_text())
    else:
        model_kwargs = last_checkpoint['model_config']          # resume: config comes from the checkpoint (train.py:99-100)

    model = ProGen(**{**model_kwargs, 'mixed_precision': mixed_precision})
    if exists(last_checkpoint):
        params, optim_state, start_seq_index = last_checkpoint['params'], last_checkpoint['optim_state'], last_checkpoint['next_seq_index']
    else:
        params, optim_state, start_seq_index = model.init(seed), None, 0
    trainer = model.trainer(params, learning_rate=learning_rate, weight_decay=weight_decay, max_grad_norm=max_grad_norm,
                            grad_accum_every=grad_accum_every, optim_state=optim_state, data_parallel=data_parallel,
                            cuda_graph=cuda_graph)
    seq_len = model_kwargs['seq_len']                           # the --seq_len flag is dead in the reference too (train.py:137)
    num_params = model.engine.num_params

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
    t0, tokens = time.time(), 0
    for i, seq_index in enumerate(range(start_seq_index, total_train_seqs, effective_batch_size)):
        if num_steps is not None and i >= num_steps:
            break
        for _ in range(grad_accum_every):
            try:
                data = next(train_dataset)
            except StopIteration:
                return
            local = PAR.shard_batch(data) if world > 1 else data
            loss = trainer.step(local, sync_loss=True, global_batch=data.shape[0])
            tokens += data.shape[0] * seq_len
        if rank == 0:
            print(f'loss: {loss.item()}')
        if i % checkpoint_every == 0 and rank == 0:
            package = {'next_seq_index': seq_index + effective_batch_size, 'params': trainer.params(),
                       'optim_state': trainer.optim_state(), 'model_config': model_kwargs, 'run_id': run_id}
            save_checkpoint(package, checkpoint_keep_n)
            print(f"checkpoint to start at sequence index of {package['next_seq_index']}")
        if i % validate_every == 0:
            valid_data = next(valid_dataset)
            vloss = trainer.evaluate(valid_data)
            if rank == 0:
                print(f'valid_loss: {vloss.item()}')
        if i % sample_every == 0 and rank == 0:
            valid_data = next(valid_dataset)[0]
            prime = valid_data[:prime_length]
            prime_str = decode_tokens(prime)
            cur = trainer.params()
            sampled = sample(seed, model.apply, cur, prime, seq_len, top_k=25)
            print(prime_str, '\n', '*' * 40, '\n', decode_tokens(sampled[prime_length:]))
    if rank == 0:
        print(f'tokens/sec (host clock, incl. logging syncs): {tokens / max(1e-9, time.time() - t0):.0f}')
    if world > 1:
        import torch.distributed as dist
        trainer._graph = None                      # a captured step references the communicator: drop it before NCCL goes away
        torch.cuda.synchronize()
        dist.barrier()
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
