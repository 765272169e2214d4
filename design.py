"""design.py — move a generator toward sequences a property head scores well, while it stays close to the model it
started from, on one GPU: on-policy reinforcement learning with a group-relative policy gradient and an exact KL penalty
(DESIGN.md §3.14).

    python design.py --init_checkpoint ./ckpts --reward_checkpoint ./ckpts_fit --reward_output 0 \\
        --prompt "[Tax=Mammalia] #" --prompts_per_step 8 --group_size 8 --max_length 512 --lora_rank 16 \\
        --beta 0.04 --learning_rate 1e-5 --iterations 200 --checkpoint_path ./ckpts_design

Each iteration:
  1. draws --group_size samples for each of --prompts_per_step prompts (taken in turn from --prompt / --prompts_file)
     with Trainer.generate, from the weights being trained;
  2. scores them with ProGen.predict of the fitness.py package in --reward_checkpoint (a sequence-level head):
     the de-standardized output --reward_output k of a regression head, or log p(class --reward_class c) of a
     classification head;
  3. turns the rewards into advantages per prompt (policy.group_advantages: reward minus the group mean, over the group
     std);
  4. takes one Trainer.policy_step over all rows (--grad_accum_every micro-steps of at most --batch_size rows when the
     rows exceed --batch_size), with beta * KL(policy || reference) per generated position, the reference being the
     --init_checkpoint model;
  5. logs the mean, max and std of the reward, the mean KL, the mean length and the finished fraction.

The estimator is on-policy only when the samples come from the policy itself: temperature 1 and no --top_k, --top_p,
--alphabet or --min_new_tokens.  Those options are allowed, but they make the samples come from another distribution
than the policy's, and the step is then a biased estimate; the run prints a note when they are set.

--lora_rank R trains low-rank adapters on the frozen --init_checkpoint (which must then be a plain package); otherwise
every parameter trains.  Checkpoints are train.py's packages (adapter packages with --lora_rank) with next_iteration and
design = {reference_checkpoint, reward_checkpoint, beta}, so generate.py and score.py run the result through
checkpoint.package_params, and a run resumes from the newest package in --checkpoint_path at its next_iteration."""
import click
import numpy as np

from progen_b200.checkpoint import count_params, get_checkpoint_fns, last_checkpoint_file, load_checkpoint_file
from progen_b200.checkpoint import package_params
from progen_b200.lib import ProgenError

OFF_POLICY_NOTE = ('note: temperature != 1, --top_k, --top_p, --alphabet or --min_new_tokens make the samples come from '
                   'another distribution than the policy: the policy gradient is then a biased estimate')


def iteration_prompts(prompts, iteration, per_step):
    """the prompts of one iteration: per_step prompts taken in turn from the list, continuing where the last one ended"""
    return [prompts[(iteration * per_step + j) % len(prompts)] for j in range(per_step)]


def iteration_seed(seed, iteration):
    """the generation seed of one iteration"""
    return int(np.random.default_rng([seed, iteration]).integers(0, 2 ** 62))


def micro_batches(num_rows, batch_size):
    """[(start, stop)] of the micro-steps of one iteration: chunks of at most batch_size rows"""
    return [(a, min(num_rows, a + batch_size)) for a in range(0, num_rows, batch_size)]


def reward_fn(pkg, reward_output, reward_class):
    """(head params, f(prediction [N, C]) -> float64 rewards [N]) of a fitness.py sequence-level package"""
    from progen_b200.property import destandardize
    head = pkg['head']
    if head.get('level', 'sequence') != 'sequence':
        raise click.UsageError('--reward_checkpoint: a residue-level head gives no sequence reward')
    if head['task'] == 'regression':
        if reward_class is not None or reward_output is None:
            raise click.UsageError('--reward_checkpoint holds a regression head: pass --reward_output k')
        if not 0 <= reward_output < head['num_outputs']:
            raise click.UsageError(f"--reward_output {reward_output}: the head has {head['num_outputs']} outputs")
        return head['params'], lambda p: destandardize(p, head['target_mean'], head['target_std'])[:, reward_output]
    if reward_output is not None or reward_class is None:
        raise click.UsageError('--reward_checkpoint holds a classification head: pass --reward_class c')
    if reward_class not in head['classes']:
        raise click.UsageError(f"--reward_class {reward_class!r}: the head's classes are {head['classes']}")
    c = head['classes'].index(reward_class)

    def log_p(pred):
        z = np.asarray(pred, np.float64)
        m = z.max(-1, keepdims=True)
        return (z - m - np.log(np.exp(z - m).sum(-1, keepdims=True)))[:, c]
    return head['params'], log_p


@click.command(help=__doc__.split('\n\n', 1)[1])
@click.option('--init_checkpoint', default=None, help='folder whose newest package is the start and the KL reference')
@click.option('--reward_checkpoint', required=True, help='folder whose newest package is a fitness.py sequence head')
@click.option('--reward_output', default=None, type=int, help='regression head: the output that is the reward')
@click.option('--reward_class', default=None, help='classification head: the class whose log-probability is the reward')
@click.option('--prompt', 'prompts', multiple=True, help='prompt text (repeatable)')
@click.option('--prompts_file', default=None, help='text file, one prompt per line')
@click.option('--prompts_per_step', default=8, help='prompts per iteration')
@click.option('--group_size', default=8, help='samples per prompt: one advantage group')
@click.option('--max_length', default=None, type=int, help='BOS + prompt + generated tokens (default: seq_len)')
@click.option('--min_new_tokens', default=0, help='generated tokens before EOS may be drawn (off-policy when > 0)')
@click.option('--alphabet', default=None, help='the only residue characters that may be drawn (off-policy)')
@click.option('--temperature', default=1.0, help='sampling temperature (on-policy only at 1)')
@click.option('--top_k', default=None, type=int, help='top-k filter (off-policy)')
@click.option('--top_p', default=None, type=float, help='nucleus filter (off-policy)')
@click.option('--beta', default=0.04, help='weight of the KL to the --init_checkpoint model (>= 0)')
@click.option('--iterations', default=100, help='iterations of the run, counted from 0 across resumes')
@click.option('--batch_size', default=64, help='rows per policy micro-step')
@click.option('--grad_accum_every', default=None, type=int,
              help='micro-steps per update (default: the micro-steps one iteration needs at --batch_size)')
@click.option('--learning_rate', default=1e-5)
@click.option('--weight_decay', default=0.0)
@click.option('--lora_rank', default=None, type=int, help='train low-rank adapters of this rank on the frozen base')
@click.option('--lora_alpha', default=None, type=float, help='adapter scale alpha (s = alpha / rank; default: the rank)')
@click.option('--checkpoint_path', default='./ckpts_design')
@click.option('--checkpoint_every', default=10, help='iterations between checkpoints (and one at the end)')
@click.option('--checkpoint_keep_n', default=500)
@click.option('--seed', default=0)
@click.option('--mixed_precision', default=False, is_flag=True, help='bf16 tensor-core engine and bf16 decoder weights')
def main(init_checkpoint, reward_checkpoint, reward_output, reward_class, prompts, prompts_file, prompts_per_step,
         group_size, max_length, min_new_tokens, alphabet, temperature, top_k, top_p, beta, iterations, batch_size,
         grad_accum_every, learning_rate, weight_decay, lora_rank, lora_alpha, checkpoint_path, checkpoint_every,
         checkpoint_keep_n, seed, mixed_precision):
    from progen_b200 import ProGen
    from progen_b200.policy import check_beta, group_advantages, samples_to_rows
    for name, v in (('--prompts_per_step', prompts_per_step), ('--group_size', group_size), ('--iterations', iterations),
                    ('--batch_size', batch_size), ('--checkpoint_every', checkpoint_every)):
        if v < 1:
            raise click.UsageError(f'{name} must be >= 1')
    if grad_accum_every is not None and grad_accum_every < 1:
        raise click.UsageError('--grad_accum_every must be >= 1')
    try:
        beta = check_beta(beta, '--beta')
    except ProgenError as e:
        raise click.UsageError(str(e))
    if (reward_output is None) == (reward_class is None):
        raise click.UsageError('pass exactly one of --reward_output (regression head) and --reward_class '
                               '(classification head)')
    if lora_alpha is not None and lora_rank is None:
        raise click.UsageError('--lora_alpha needs --lora_rank')
    prompts = list(prompts)
    if prompts_file is not None:
        with open(prompts_file) as f:
            prompts += [l.rstrip('\n') for l in f if l.strip()]
    if not prompts:
        prompts = ['']

    _, get_last_checkpoint, save_checkpoint = get_checkpoint_fns(checkpoint_path)
    last = get_last_checkpoint()
    if last is not None:
        if 'next_iteration' not in last:
            raise click.UsageError(f'{checkpoint_path} holds no design.py package; write into another --checkpoint_path')
        lora = 'adapters' in last
        if lora_rank is not None and (not lora or lora_rank != last['lora']['rank']):
            raise click.UsageError(f'--lora_rank {lora_rank}: {checkpoint_path} holds '
                                   + (f"adapters of rank {last['lora']['rank']}" if lora else 'a full-parameter package'))
        ref_file = last['design']['reference_checkpoint']
        start = int(last['next_iteration'])
    else:
        if init_checkpoint is None:
            raise click.UsageError('a new run needs --init_checkpoint')
        ref_file = last_checkpoint_file(init_checkpoint)
        if ref_file is None:
            raise click.ClickException(f'no checkpoints found at {init_checkpoint}')
        lora, start = lora_rank is not None, 0
    ref_pkg = load_checkpoint_file(ref_file)
    if lora and 'adapters' in ref_pkg:
        raise click.UsageError(f'--lora_rank: {ref_file} is an adapter package; train adapters on a plain package')
    try:
        ref_params = package_params(ref_pkg)
        reward_pkg = get_checkpoint_fns(reward_checkpoint)[1]()
        if reward_pkg is None or 'head' not in reward_pkg:
            raise click.ClickException(f'no property-head package found at {reward_checkpoint}')
        reward_params = package_params(reward_pkg)
    except ProgenError as e:
        raise click.ClickException(str(e))
    head_params, reward_of = reward_fn(reward_pkg, reward_output, reward_class)

    model_kwargs = ref_pkg['model_config']
    n = model_kwargs['seq_len']
    if reward_pkg['model_config']['seq_len'] < n:
        raise click.UsageError(f"--reward_checkpoint: its seq_len ({reward_pkg['model_config']['seq_len']}) is below the "
                               f"generator's ({n})")
    model = ProGen(**{**model_kwargs, 'mixed_precision': mixed_precision})
    reward_model = ProGen(**{**reward_pkg['model_config'], 'mixed_precision': mixed_precision})
    reference = ProGen(**{**model_kwargs, 'mixed_precision': mixed_precision}) if beta > 0 else None
    bias = None
    if alphabet is not None:
        from generate import alphabet_bias
        bias = alphabet_bias(alphabet, model.config['num_tokens'])
    if temperature != 1.0 or top_k is not None or top_p is not None or alphabet is not None or min_new_tokens > 0:
        print(OFF_POLICY_NOTE)

    N = prompts_per_step * group_size
    chunks = micro_batches(N, batch_size)
    every = len(chunks) if grad_accum_every is None else grad_accum_every
    if last is not None and lora:
        params, adapters, lora_cfg = ref_params, last['adapters'], last['lora']
    elif last is not None:
        params, adapters, lora_cfg = last['params'], None, None
    else:
        params = ref_params
        adapters = model.init_adapters(seed, lora_rank, alpha=lora_alpha) if lora else None
        lora_cfg = dict(rank=lora_rank, alpha=float(lora_rank if lora_alpha is None else lora_alpha)) if lora else None
    trainer = model.trainer(params, learning_rate=learning_rate, weight_decay=weight_decay, grad_accum_every=every,
                            optim_state=None if last is None else last['optim_state'], data_parallel=False,
                            adapters=adapters, lora_alpha=None if lora_cfg is None else lora_cfg['alpha'],
                            reference=reference, reference_params=ref_params if beta > 0 else None)
    design = dict(reference_checkpoint=str(ref_file), reward_checkpoint=str(reward_checkpoint), beta=beta)
    print(f'{N} samples per iteration ({prompts_per_step} prompts x {group_size}), {len(chunks)} micro-steps, '
          f'beta {beta}, ' + (f"adapters rank {lora_cfg['rank']}" if lora else 'all parameters') +
          f', starting at iteration {start}')

    def save(next_iteration):
        package = {'next_seq_index': 0, 'next_iteration': next_iteration, 'optim_state': trainer.optim_state(),
                   'model_config': model_kwargs, 'run_id': None, 'design': design}
        if lora:
            package.update(adapters=trainer.adapters(), lora=lora_cfg, base_checkpoint=str(ref_file),
                           num_params=count_params(ref_params))
        else:
            package['params'] = trainer.params()
        save_checkpoint(package, checkpoint_keep_n)
        print(f'checkpoint to start at iteration {next_iteration}')

    for it in range(start, iterations):
        samples = trainer.generate(iteration_prompts(prompts, it, prompts_per_step), num_samples=group_size,
                                   temperature=temperature, top_k=top_k, top_p=top_p, max_length=max_length,
                                   seed=iteration_seed(seed, it), logit_bias=bias, min_new_tokens=min_new_tokens)
        rows, span = samples_to_rows(samples)
        scored = np.zeros((N, reward_model.config['seq_len'] + 1), np.int32)
        scored[:, :rows.shape[1]] = rows
        reward = reward_of(reward_model.predict(reward_params, head_params, scored)['prediction'])
        adv = group_advantages(reward, group_size)
        kl, loss = [], 0.0
        for a, b in chunks:
            loss += float(trainer.policy_step(rows[a:b], span[a:b], adv[a:b], beta).item()) * (b - a) / N
            kl.append(trainer.policy_stats()['kl'])
        print(f'iteration {it}: reward mean {reward.mean():.6g} max {reward.max():.6g} std {reward.std():.6g} '
              f'kl {np.concatenate(kl).mean():.6g} length {samples["length"].mean():.1f} '
              f'finished {samples["finished"].mean():.3f} loss {loss:.6g}')
        if (it + 1) % checkpoint_every == 0 or it + 1 == iterations:
            save(it + 1)
    if start >= iterations:
        print(f'nothing to do: the run is at iteration {start} of {iterations}')


if __name__ == '__main__':
    main()
