"""fitness.py — fit a property head on labelled sequences (or on labelled residues) with low-rank adapters on a frozen
base, and predict with it, on one GPU.

    python fitness.py train --init_checkpoint ./ckpts --train train.tsv [--valid valid.tsv] --task regression \\
        --lora_rank 16 [--lora_alpha 16] --checkpoint_path ./ckpts_fit --learning_rate 1e-4 --batch_size 8 --epochs 3 \\
        --seed 0 [--mixed_precision] [--cuda_graph] [--recompute]
    python fitness.py train ... --level residue --train residues.tsv --task classification ...
    python fitness.py predict --checkpoint_path ./ckpts_fit --input seqs.txt --output preds.tsv

Training lines are `sequence<TAB>value[<TAB>value...]` (regression: one column per output, e.g. DMS fitness or a
stability ddG) or `sequence<TAB>class_name` (classification); sequences are tokenized like train.py --text_file
(data.collate).  Regression targets are standardized with the training set's mean and std per output, and predictions
are written in the original units; class names are indexed in sorted order.  Both are stored in the package.  Every
epoch visits the training rows in an order shuffled with --seed and ends with a checkpoint, the mean training loss and,
with --valid, the validation metric: Spearman's rho per output (regression) or the accuracy (classification).  A run
resumes from the newest package under --checkpoint_path, at its next_index.

With --level residue the head is trained on per-residue labels (DESIGN.md §3.11): the head is applied at every position,
and position t >= 1 holds residue t - 1.  Lines are `sequence<TAB>labels`: one class character per residue (`.`
unlabelled; the classes are the sorted set of characters seen) or comma-separated values, one per residue (`nan`
unlabelled; one output, standardized over the labelled residues).  Residues past the row's capacity (seq_len - 1) are
dropped, as collate truncates, and sequences left without a labelled residue are skipped.  The validation metric is the
accuracy or Spearman's rho over labelled residues.  ProGen is causal: a residue's representation has seen it and the
residues before it only, so labels that depend on downstream context are harder for it than for a bidirectional model.

The package is the adapter package of train.py --lora_rank (adapters, lora, optim_state, model_config, base_checkpoint,
num_params; no base parameters) plus head: {params, task, num_outputs, target_mean, target_std, classes} and
next_index, so `checkpoint.package_params` (score.py, generate.py, ...) runs it as the adapted language model.  The
head's `level` is 'sequence' or 'residue'; a package without it is 'sequence'."""
import click
import numpy as np

from progen_b200 import ProGen
from progen_b200.checkpoint import (count_params, get_checkpoint_fns, last_checkpoint_file, load_checkpoint_file,
                                    package_params)
from progen_b200.data import collate
from progen_b200.lib import ProgenError
from progen_b200.property import (destandardize, read_labelled, read_residue_labelled, residue_label_array, softmax,
                                  spearman, standardize)

LEVELS = ('sequence', 'residue')


def head_level(head_cfg):
    """the level of a package's head: 'sequence' (per-sequence labels, the default of packages without one) or 'residue'"""
    return head_cfg.get('level', 'sequence')


def epoch_order(num_rows, epoch, seed):
    """the row indices of one epoch, in the order it visits them"""
    return np.random.default_rng([seed, epoch]).permutation(num_rows)


def _read(path, task, level='sequence'):
    try:
        with open(path) as f:
            seqs, labels = (read_residue_labelled if level == 'residue' else read_labelled)(f, task)
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


def residue_head_cfg(labels, task):
    """the head settings of a new residue-level run from its training labels (read_residue_labelled)"""
    if task == 'regression':
        v = np.concatenate([np.asarray(l, np.float64) for l in labels])
        v = v[~np.isnan(v)]
        if v.size == 0:
            raise ProgenError('no labelled residue (every value is nan)')
        _, mean, std = standardize(v[:, None])
        return dict(task=task, num_outputs=1, target_mean=mean, target_std=std, classes=None, level='residue')
    classes = sorted(set(''.join(labels)) - {'.'})
    if len(classes) < 2:
        raise ProgenError(f'classification needs at least 2 classes, found {classes}')
    return dict(task=task, num_outputs=len(classes), target_mean=None, target_std=None, classes=classes, level='residue')


def residue_targets(labels, head_cfg, seq_len):
    """file labels -> the per-position targets of their collate rows: standardized float32 [N, seq_len] with NaN where
    unlabelled (regression), or class indices int32 [N, seq_len] with -1 (classification)"""
    y = residue_label_array(labels, head_cfg['task'], head_cfg['classes'], seq_len)
    if head_cfg['task'] == 'regression':
        return ((y - head_cfg['target_mean'][0]) / head_cfg['target_std'][0]).astype(np.float32)
    return y


def residue_metric(head_cfg, pred, targets):
    """validation metric over the labelled residues: pred [N, n, C] head outputs, targets of residue_targets"""
    if head_cfg['task'] == 'regression':
        lab = ~np.isnan(targets)
        return f'spearman {spearman(pred[..., 0][lab], targets[lab]):.4f}'
    lab = targets >= 0
    return f'accuracy {float((pred.argmax(-1)[lab] == targets[lab]).mean()):.4f}'


def _metric(head_cfg, pred, labels):
    """validation metric of predictions (head outputs) against the file labels"""
    if head_cfg['task'] == 'regression':
        rho = [spearman(pred[:, c], labels[:, c]) for c in range(pred.shape[1])]
        return 'spearman ' + ' '.join(f'{r:.4f}' for r in rho)
    index = {c: i for i, c in enumerate(head_cfg['classes'])}
    truth = np.array([index[c] for c in labels])
    return f'accuracy {float((pred.argmax(-1) == truth).mean()):.4f}'


def _residue_rows(seqs, labels, head_cfg, seq_len, path):
    """collate rows and per-position targets of a residue-level file, without the sequences that keep no labelled
    residue within seq_len - 1 (a micro-batch needs one)"""
    try:
        targets = residue_targets(labels, head_cfg, seq_len)
    except ProgenError as e:
        raise click.ClickException(f'{path}: {e}')
    keep = ~np.isnan(targets).all(1) if head_cfg['task'] == 'regression' else (targets >= 0).any(1)
    if not keep.any():
        raise click.ClickException(f'{path}: no labelled residue within the first {seq_len - 1} of any sequence')
    if not keep.all():
        print(f'{path}: skipping {int((~keep).sum())} sequences without a labelled residue')
    return collate([s for s, k in zip(seqs, keep) if k], seq_len), targets[keep]


@click.group()
def cli():
    pass


@cli.command()
@click.option('--init_checkpoint', default=None, help='folder whose newest checkpoint is the frozen base')
@click.option('--train', 'train_path', required=True, help='labelled sequences, `sequence<TAB>value...` per line')
@click.option('--valid', 'valid_path', default=None, help='labelled sequences for the per-epoch validation metric')
@click.option('--task', type=click.Choice(['regression', 'classification']), default=None)
@click.option('--level', type=click.Choice(LEVELS), default=None,
              help='labels per sequence (default) or per residue (`sequence<TAB>labels`, one label per residue)')
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
@click.option('--recompute', default=False, is_flag=True,
              help='recompute activations in the backward pass: one residual checkpoint per layer (less memory, more time)')
def train(init_checkpoint, train_path, valid_path, task, level, lora_rank, lora_alpha, checkpoint_path, learning_rate,
          weight_decay, max_grad_norm, batch_size, grad_accum_every, epochs, seed, checkpoint_keep_n, mixed_precision,
          cuda_graph, recompute):
    if batch_size < 1 or grad_accum_every < 1 or epochs < 1:
        raise click.UsageError('--batch_size, --grad_accum_every and --epochs must be >= 1')
    _, get_last_checkpoint, save_checkpoint = get_checkpoint_fns(checkpoint_path)
    last = get_last_checkpoint()
    if last is not None:
        # a resumed run keeps its base, task and adapter settings: flags that would change them are refused
        if 'head' not in last:
            raise click.UsageError(f'{checkpoint_path} holds no property-head package; train into another --checkpoint_path')
        head_cfg, lora_cfg, base_file = last['head'], last['lora'], last['base_checkpoint']
        for flag, got, want in (('--task', task, head_cfg['task']), ('--level', level, head_level(head_cfg)),
                                ('--lora_rank', lora_rank, lora_cfg['rank']),
                                ('--lora_alpha', None if lora_alpha is None else float(lora_alpha), lora_cfg['alpha'])):
            if got is not None and got != want:
                raise click.UsageError(f'{flag} {got}: {checkpoint_path} holds a run with {want}')
        if init_checkpoint is not None and last_checkpoint_file(init_checkpoint) != base_file:
            raise click.UsageError(f'--init_checkpoint {init_checkpoint}: its newest checkpoint is not {base_file}, the base '
                                   f'of the run in {checkpoint_path}')
        task, level = head_cfg['task'], head_level(head_cfg)
    else:
        if init_checkpoint is None or task is None or lora_rank is None:
            raise click.UsageError('a new run needs --init_checkpoint, --task and --lora_rank')
        base_file = last_checkpoint_file(init_checkpoint)
        if base_file is None:
            raise click.ClickException(f'no checkpoints found at {init_checkpoint}')
        level = level or 'sequence'
    seqs, labels = _read(train_path, task, level)
    base = load_checkpoint_file(base_file)
    params, model_kwargs = base['params'], base['model_config']
    seq_len = model_kwargs['seq_len']
    model = ProGen(**{**model_kwargs, 'mixed_precision': mixed_precision}, recompute=recompute)
    if last is not None:
        if count_params(params) != last['num_params']:
            raise click.ClickException(f'base checkpoint {base_file} has changed')
        adapters, head, optim_state, start = last['adapters'], last['head']['params'], last['optim_state'], int(last['next_index'])
    else:
        if level == 'residue':
            try:
                head_cfg = residue_head_cfg(labels, task)
            except ProgenError as e:
                raise click.ClickException(f'{train_path}: {e}')
        elif task == 'regression':
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
    valid = None
    if level == 'residue':
        rows, targets = _residue_rows(seqs, labels, head_cfg, seq_len, train_path)
        if valid_path is not None:
            v_seqs, v_labels = _read(valid_path, task, level)
            valid = _residue_rows(v_seqs, v_labels, head_cfg, seq_len, valid_path)
    else:
        rows, targets = collate(seqs, seq_len), _targets(labels, head_cfg, train_path)
        if valid_path is not None:
            v_seqs, v_labels = _read(valid_path, task)
            _targets(v_labels, head_cfg, valid_path)            # the same checks as the training file
            valid = (collate(v_seqs, seq_len), v_labels)
    trainer = model.trainer(params, adapters=adapters, head=head, task=task, lora_alpha=lora_cfg['alpha'],
                            learning_rate=learning_rate, weight_decay=weight_decay, max_grad_norm=max_grad_norm,
                            grad_accum_every=grad_accum_every, optim_state=optim_state, data_parallel=False,
                            cuda_graph=cuda_graph)
    N = len(rows)
    print(f"{N} sequences, {level} level, task {task}, {head_cfg['num_outputs']} outputs, adapters: rank {lora_cfg['rank']}, alpha "
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
        step = trainer.residue_step if level == 'residue' else trainer.property_step
        losses.append(float(step(rows[idx], targets[idx]).item()))
        k += len(idx)
        if k % N == 0:
            msg = f'epoch {epoch}: train loss {np.mean(losses):.6f}'
            if valid is not None:
                merged = model.merge_adapters(params, trainer.adapters(), lora_alpha=lora_cfg['alpha'])
                fn = model.predict_residues if level == 'residue' else model.predict
                pred = fn(merged, trainer.head(), valid[0], batch_size=max(batch_size, 64))['prediction']
                trainer.eng.load_params(params)              # the engine's base again (predict loaded the merged weights)
                model._loaded = None
                if level == 'residue':
                    msg += f', valid {residue_metric(head_cfg, pred, valid[1])}'
                else:
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
@click.option('--output', default='preds.tsv', help='TSV: index, residues, then the values or the class and its '
              'probabilities; at residue level one line per residue: index, residue number, residue, value or class')
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
    if head_level(head_cfg) == 'residue':
        _write_residues(model, params, head_cfg, seqs, seq_len, batch_size, output)
        return
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


def _write_residues(model, params, head_cfg, seqs, seq_len, batch_size, output):
    """one TSV line per residue with a representation: sequence index, 1-based residue number, residue, then the value
    (regression) or the class and its probabilities"""
    res = model.predict_residues(params, head_cfg['params'], collate(seqs, seq_len), batch_size=batch_size)
    pred, mask = res['prediction'], res['mask']
    reg = head_cfg['task'] == 'regression'
    with open(output, 'w') as f:
        if reg:
            f.write('index\tresidue_number\tresidue\tvalue\n')
        else:
            f.write('index\tresidue_number\tresidue\tclass\t' + '\t'.join(f'p_{c}' for c in head_cfg['classes']) + '\n')
        lines = 0
        for i, s in enumerate(seqs):
            res_bytes = s.encode()
            for t in np.flatnonzero(mask[i]):
                ch = chr(res_bytes[t - 1])
                if reg:
                    v = float(destandardize(pred[i, t, :1], head_cfg['target_mean'], head_cfg['target_std'])[0])
                    f.write(f'{i}\t{t}\t{ch}\t{v:.9g}\n')
                else:
                    prob = softmax(pred[i, t])
                    f.write(f'{i}\t{t}\t{ch}\t{head_cfg["classes"][int(prob.argmax())]}\t' +
                            '\t'.join(f'{p:.6g}' for p in prob) + '\n')
                lines += 1
    print(f'wrote {output}: {lines} residues of {len(seqs)} sequences')


if __name__ == '__main__':
    cli()
