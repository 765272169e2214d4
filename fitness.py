"""fitness.py — fit a property head on labelled sequences with low-rank adapters on a frozen base, and predict with it,
on one GPU.

    python fitness.py train --init_checkpoint ./ckpts --train train.tsv [--valid valid.tsv] --task regression \\
        --lora_rank 16 [--lora_alpha 16] --checkpoint_path ./ckpts_fit --learning_rate 1e-4 --batch_size 8 --epochs 3 \\
        --seed 0 [--mixed_precision] [--cuda_graph]
    python fitness.py predict --checkpoint_path ./ckpts_fit --input seqs.txt --output preds.tsv

Training lines are `sequence<TAB>value[<TAB>value...]` (regression: one column per output, e.g. DMS fitness or a
stability ddG) or `sequence<TAB>class_name` (classification); sequences are tokenized like train.py --text_file
(data.collate).  Regression targets are standardized with the training set's mean and std per output, and predictions
are written in the original units; class names are indexed in sorted order.  Both are stored in the package.  Every
epoch visits the training rows in an order shuffled with --seed and ends with a checkpoint, the mean training loss and,
with --valid, the validation metric: Spearman's rho per output (regression) or the accuracy (classification).  A run
resumes from the newest package under --checkpoint_path, at its next_index.

The package is the adapter package of train.py --lora_rank (adapters, lora, optim_state, model_config, base_checkpoint,
num_params; no base parameters) plus head: {params, task, num_outputs, target_mean, target_std, classes} and
next_index, so `checkpoint.package_params` (score.py, generate.py, ...) runs it as the adapted language model."""
import click
import numpy as np

from progen_b200 import ProGen
from progen_b200.checkpoint import (count_params, get_checkpoint_fns, last_checkpoint_file, load_checkpoint_file,
                                    package_params)
from progen_b200.data import collate
from progen_b200.lib import ProgenError
from progen_b200.property import destandardize, read_labelled, softmax, spearman, standardize


def epoch_order(num_rows, epoch, seed):
    """the row indices of one epoch, in the order it visits them"""
    return np.random.default_rng([seed, epoch]).permutation(num_rows)


def _read(path, task):
    try:
        with open(path) as f:
            seqs, labels = read_labelled(f, task)
    except ProgenError as e:
        raise click.ClickException(f'{path}: {e}')
    if not seqs:
        raise click.ClickException(f'{path}: no labelled sequences')
    return seqs, labels


def _targets(labels, head_cfg, path):
    """file labels -> the head's targets: standardized float32 [N, C] or class indices [N]"""
    if head_cfg['task'] == 'regression':
        if labels.shape[1] != head_cfg['num_outputs']:
            raise click.ClickException(f"{path}: {labels.shape[1]} values per line, the head has {head_cfg['num_outputs']} outputs")
        return standardize(labels, head_cfg['target_mean'], head_cfg['target_std'])[0]
    index = {c: i for i, c in enumerate(head_cfg['classes'])}
    unknown = sorted(set(labels) - set(index))
    if unknown:
        raise click.ClickException(f'{path}: class {unknown[0]!r} is not one of the training classes {head_cfg["classes"]}')
    return np.array([index[c] for c in labels], np.int32)


def _metric(head_cfg, pred, labels):
    """validation metric of predictions (head outputs) against the file labels"""
    if head_cfg['task'] == 'regression':
        rho = [spearman(pred[:, c], labels[:, c]) for c in range(pred.shape[1])]
        return 'spearman ' + ' '.join(f'{r:.4f}' for r in rho)
    index = {c: i for i, c in enumerate(head_cfg['classes'])}
    truth = np.array([index[c] for c in labels])
    return f'accuracy {float((pred.argmax(-1) == truth).mean()):.4f}'


@click.group()
def cli():
    pass


@cli.command()
@click.option('--init_checkpoint', default=None, help='folder whose newest checkpoint is the frozen base')
@click.option('--train', 'train_path', required=True, help='labelled sequences, `sequence<TAB>value...` per line')
@click.option('--valid', 'valid_path', default=None, help='labelled sequences for the per-epoch validation metric')
@click.option('--task', type=click.Choice(['regression', 'classification']), default=None)
@click.option('--lora_rank', default=None, type=int, help='adapter rank (multiple of 8 in [8, 64])')
@click.option('--lora_alpha', default=None, type=float, help='adapter scale alpha (s = alpha / rank; default: the rank)')
@click.option('--checkpoint_path', default='./ckpts_fit')
@click.option('--learning_rate', default=1e-4)
@click.option('--weight_decay', default=1e-3)
@click.option('--max_grad_norm', default=0.5)
@click.option('--batch_size', default=8)
@click.option('--grad_accum_every', default=1)
@click.option('--epochs', default=1)
@click.option('--seed', default=0)
@click.option('--checkpoint_keep_n', default=500)
@click.option('--mixed_precision', default=False, is_flag=True, help='bf16 tensor-core engine')
@click.option('--cuda_graph', default=False, is_flag=True, help='capture the step into a CUDA graph and replay it')
def train(init_checkpoint, train_path, valid_path, task, lora_rank, lora_alpha, checkpoint_path, learning_rate, weight_decay,
          max_grad_norm, batch_size, grad_accum_every, epochs, seed, checkpoint_keep_n, mixed_precision, cuda_graph):
    if batch_size < 1 or grad_accum_every < 1 or epochs < 1:
        raise click.UsageError('--batch_size, --grad_accum_every and --epochs must be >= 1')
    _, get_last_checkpoint, save_checkpoint = get_checkpoint_fns(checkpoint_path)
    last = get_last_checkpoint()
    if last is not None:
        # a resumed run keeps its base, task and adapter settings: flags that would change them are refused
        if 'head' not in last:
            raise click.UsageError(f'{checkpoint_path} holds no property-head package; train into another --checkpoint_path')
        head_cfg, lora_cfg, base_file = last['head'], last['lora'], last['base_checkpoint']
        for flag, got, want in (('--task', task, head_cfg['task']), ('--lora_rank', lora_rank, lora_cfg['rank']),
                                ('--lora_alpha', None if lora_alpha is None else float(lora_alpha), lora_cfg['alpha'])):
            if got is not None and got != want:
                raise click.UsageError(f'{flag} {got}: {checkpoint_path} holds a run with {want}')
        if init_checkpoint is not None and last_checkpoint_file(init_checkpoint) != base_file:
            raise click.UsageError(f'--init_checkpoint {init_checkpoint}: its newest checkpoint is not {base_file}, the base '
                                   f'of the run in {checkpoint_path}')
        task = head_cfg['task']
    else:
        if init_checkpoint is None or task is None or lora_rank is None:
            raise click.UsageError('a new run needs --init_checkpoint, --task and --lora_rank')
        base_file = last_checkpoint_file(init_checkpoint)
        if base_file is None:
            raise click.ClickException(f'no checkpoints found at {init_checkpoint}')
    seqs, labels = _read(train_path, task)
    base = load_checkpoint_file(base_file)
    params, model_kwargs = base['params'], base['model_config']
    seq_len = model_kwargs['seq_len']
    model = ProGen(**{**model_kwargs, 'mixed_precision': mixed_precision})
    if last is not None:
        if count_params(params) != last['num_params']:
            raise click.ClickException(f'base checkpoint {base_file} has changed')
        adapters, head, optim_state, start = last['adapters'], last['head']['params'], last['optim_state'], int(last['next_index'])
    else:
        if task == 'regression':
            _, mean, std = standardize(labels)
            head_cfg = dict(task=task, num_outputs=labels.shape[1], target_mean=mean, target_std=std, classes=None)
        else:
            classes = sorted(set(labels))
            if len(classes) < 2:
                raise click.ClickException(f'{train_path}: classification needs at least 2 classes, found {classes}')
            head_cfg = dict(task=task, num_outputs=len(classes), target_mean=None, target_std=None, classes=classes)
        try:
            adapters = model.init_adapters(seed, lora_rank, alpha=lora_alpha)
            head = model.init_head(seed, head_cfg['num_outputs'])
        except ProgenError as e:
            raise click.UsageError(str(e))
        lora_cfg = dict(rank=lora_rank, alpha=float(lora_rank if lora_alpha is None else lora_alpha))
        optim_state, start = None, 0
    rows, targets = collate(seqs, seq_len), _targets(labels, head_cfg, train_path)
    valid = None
    if valid_path is not None:
        v_seqs, v_labels = _read(valid_path, task)
        _targets(v_labels, head_cfg, valid_path)            # the same checks as the training file
        valid = (collate(v_seqs, seq_len), v_labels)
    trainer = model.trainer(params, adapters=adapters, head=head, task=task, lora_alpha=lora_cfg['alpha'],
                            learning_rate=learning_rate, weight_decay=weight_decay, max_grad_norm=max_grad_norm,
                            grad_accum_every=grad_accum_every, optim_state=optim_state, data_parallel=False,
                            cuda_graph=cuda_graph)
    N = len(seqs)
    print(f"{N} sequences, task {task}, {head_cfg['num_outputs']} outputs, adapters: rank {lora_cfg['rank']}, alpha "
          f"{lora_cfg['alpha']}, {trainer.lora.num_params} trained parameters on base {base_file}, starting from row {start}")

    def save(next_index):
        package = {'adapters': trainer.adapters(), 'lora': lora_cfg, 'optim_state': trainer.optim_state(),
                   'model_config': model_kwargs, 'next_seq_index': 0, 'base_checkpoint': base_file,
                   'num_params': count_params(params), 'head': {**head_cfg, 'params': trainer.head()},
                   'next_index': next_index}
        save_checkpoint(package, checkpoint_keep_n)
        print(f'checkpoint to start at row index {next_index}')

    k, losses = start, []
    while k < epochs * N:
        epoch, pos = divmod(k, N)
        idx = epoch_order(N, epoch, seed)[pos:pos + batch_size]
        losses.append(float(trainer.property_step(rows[idx], targets[idx]).item()))
        k += len(idx)
        if k % N == 0:
            msg = f'epoch {epoch}: train loss {np.mean(losses):.6f}'
            if valid is not None:
                merged = model.merge_adapters(params, trainer.adapters(), lora_alpha=lora_cfg['alpha'])
                pred = model.predict(merged, trainer.head(), valid[0], batch_size=max(batch_size, 64))['prediction']
                trainer.eng.load_params(params)              # the engine's base again (predict loaded the merged weights)
                model._loaded = None
                if task == 'regression':
                    pred = destandardize(pred, head_cfg['target_mean'], head_cfg['target_std'])
                msg += f', valid {_metric(head_cfg, pred, valid[1])}'
            print(msg)
            losses = []
            save(k)
    if k == start:
        print('nothing to do: every epoch is done')


@cli.command()
@click.option('--checkpoint_path', required=True, help='folder of a fitness.py train run')
@click.option('--input', 'input_path', required=True, help='text file, one sequence per line')
@click.option('--output', default='preds.tsv', help='TSV: index, residues, then the values or the class and its probabilities')
@click.option('--batch_size', default=64, help='sequences per forward pass')
@click.option('--mixed_precision', default=False, is_flag=True, help='bf16 tensor-core engine')
def predict(checkpoint_path, input_path, output, batch_size, mixed_precision):
    pkg = get_checkpoint_fns(checkpoint_path)[1]()
    if pkg is None or 'head' not in pkg:
        raise click.ClickException(f'no property-head package found at {checkpoint_path}')
    try:
        params = package_params(pkg)                     # base + merged adapters
    except ProgenError as e:
        raise click.ClickException(str(e))
    head_cfg = pkg['head']
    model = ProGen(**{**pkg['model_config'], 'mixed_precision': mixed_precision})
    seq_len = pkg['model_config']['seq_len']
    with open(input_path) as f:
        seqs = [l.strip() for l in f if l.strip()]
    pred = model.predict(params, head_cfg['params'], collate(seqs, seq_len), batch_size=batch_size)['prediction']
    with open(output, 'w') as f:
        if head_cfg['task'] == 'regression':
            vals = destandardize(pred, head_cfg['target_mean'], head_cfg['target_std'])
            f.write('index\tresidues\t' + '\t'.join(f'value_{c}' for c in range(vals.shape[1])) + '\n')
            for i, s in enumerate(seqs):
                f.write(f'{i}\t{min(len(s.encode()), seq_len)}\t' + '\t'.join(f'{v:.9g}' for v in vals[i]) + '\n')
        else:
            prob, classes = softmax(pred), head_cfg['classes']
            f.write('index\tresidues\tclass\t' + '\t'.join(f'p_{c}' for c in classes) + '\n')
            for i, s in enumerate(seqs):
                f.write(f'{i}\t{min(len(s.encode()), seq_len)}\t{classes[int(prob[i].argmax())]}\t' +
                        '\t'.join(f'{p:.6g}' for p in prob[i]) + '\n')
    print(f'wrote {output}: {len(seqs)} sequences')


if __name__ == '__main__':
    cli()
