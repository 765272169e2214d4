"""dpo.py — preference (DPO) fine-tuning of a checkpoint on chosen / rejected sequence pairs, on one GPU.

    python dpo.py --init_checkpoint ./ckpts --pairs pairs.tsv --checkpoint_path ./ckpts_dpo --beta 0.1 \\
        --learning_rate 1e-6 --batch_pairs 8 --grad_accum_every 1 --epochs 1 --seed 0 [--mixed_precision] [--cuda_graph] \\
        [--recompute]

--pairs has one pair per line, `chosen<TAB>rejected`; each side is a text sequence, tokenized like train.py --text_file
(data.collate).  Blank lines are skipped.  The reference model is the newest checkpoint under --init_checkpoint: the
log-likelihood of every row under it is computed once with ProGen.score, in the same precision as training.  The policy
starts from it too, or, when --checkpoint_path already holds a checkpoint, resumes from that checkpoint's parameters,
optimizer state and next_pair_index (the reference stays the init checkpoint).  Every epoch visits the pairs in an order
shuffled with --seed; each step (one Trainer.preference_step of --batch_pairs pairs) logs the loss, the mean margin z and
the accuracy (the fraction of pairs with z > 0).  A checkpoint is written at the end of every epoch and of the run."""
import click
import numpy as np

from progen_b200 import ProGen
from progen_b200.checkpoint import get_checkpoint_fns
from progen_b200.data import collate
from progen_b200.lib import ProgenError
from progen_b200.preference import read_pairs


def epoch_order(num_pairs, epoch, seed):
    """the pair indices of one epoch, in the order it visits them"""
    return np.random.default_rng([seed, epoch]).permutation(num_pairs)


@click.command()
@click.option('--init_checkpoint', required=True, help='folder whose newest checkpoint is the reference and the start')
@click.option('--pairs', 'pairs_path', required=True, help='text file, one `chosen<TAB>rejected` pair per line')
@click.option('--checkpoint_path', default='./ckpts_dpo')
@click.option('--beta', default=0.1)
@click.option('--learning_rate', default=1e-6)
@click.option('--batch_pairs', default=8)
@click.option('--grad_accum_every', default=1)
@click.option('--epochs', default=1)
@click.option('--seed', default=0)
@click.option('--checkpoint_keep_n', default=500)
@click.option('--mixed_precision', default=False, is_flag=True, help='bf16 tensor-core engine')
@click.option('--cuda_graph', default=False, is_flag=True, help='capture the step into a CUDA graph and replay it')
@click.option('--recompute', default=False, is_flag=True,
              help='recompute activations in the backward pass: one residual checkpoint per layer (less memory, more time)')
def main(init_checkpoint, pairs_path, checkpoint_path, beta, learning_rate, batch_pairs, grad_accum_every, epochs, seed,
         checkpoint_keep_n, mixed_precision, cuda_graph, recompute):
    if batch_pairs < 1 or grad_accum_every < 1 or epochs < 1:
        raise click.UsageError('--batch_pairs, --grad_accum_every and --epochs must be >= 1')
    try:
        with open(pairs_path) as f:
            chosen, rejected = read_pairs(f)
    except ProgenError as e:
        raise click.ClickException(f'{pairs_path}: {e}')
    if not chosen:
        raise click.ClickException(f'{pairs_path}: no pairs')
    init = get_checkpoint_fns(init_checkpoint)[1]()
    if init is None:
        raise click.ClickException(f'no checkpoints found at {init_checkpoint}')
    model_kwargs = init['model_config']
    seq_len = model_kwargs['seq_len']
    model = ProGen(**{**model_kwargs, 'mixed_precision': mixed_precision}, recompute=recompute)
    c_rows, r_rows = collate(chosen, seq_len), collate(rejected, seq_len)
    # the reference's log-likelihoods, once, before the trainer loads the policy into the same engine
    ref_c = model.score(init['params'], c_rows)['log_likelihood']
    ref_r = model.score(init['params'], r_rows)['log_likelihood']

    _, get_last_checkpoint, save_checkpoint = get_checkpoint_fns(checkpoint_path)
    last = get_last_checkpoint()
    if last is not None:
        params, optim_state, start = last['params'], last['optim_state'], int(last['next_pair_index'])
    else:
        params, optim_state, start = init['params'], None, 0
    trainer = model.trainer(params, learning_rate=learning_rate, grad_accum_every=grad_accum_every, optim_state=optim_state,
                            data_parallel=False, cuda_graph=cuda_graph)
    N = len(chosen)
    print(f'{N} pairs, sequence length {seq_len}, beta {beta}, starting from pair {start}')

    def save(next_pair_index):
        # train.py's package keys; a train.py run resumed from it starts its own data at sequence 0
        save_checkpoint({'next_seq_index': 0, 'next_pair_index': next_pair_index, 'params': trainer.params(),
                         'optim_state': trainer.optim_state(), 'model_config': model_kwargs, 'run_id': None},
                        checkpoint_keep_n)
        print(f'checkpoint to start at pair index {next_pair_index}')

    k, step = start, 0
    while k < epochs * N:
        epoch, pos = divmod(k, N)
        idx = epoch_order(N, epoch, seed)[pos:pos + batch_pairs]
        loss = float(trainer.preference_step(c_rows[idx], r_rows[idx], ref_c[idx], ref_r[idx], beta=beta).item())
        st = trainer.preference_stats()
        k += len(idx)
        print(f'step {step} epoch {epoch} pairs {k - len(idx)}-{k - 1}: loss {loss:.6f} margin {float(st["margin"].mean()):.6f} '
              f'accuracy {float((st["margin"] > 0).mean()):.3f}')
        step += 1
        if k % N == 0:
            save(k)
    if step == 0:
        print('nothing to do: every epoch is done')


if __name__ == '__main__':
    main()
