"""generate.py — sample many sequences per prompt from the newest checkpoint with the standard sampler.

    python generate.py --checkpoint_path ./ckpts --prompt "[Tax=Mammalia] #" [--prompt ... | --prompts_file f.txt]
        --num_samples 100 --temperature 1.0 [--top_k K] [--top_p 0.95] --seed 0 --batch_size 64 [--max_length L]
        [--alphabet ACDEFGHIKLMNPQRSTVWY] [--min_new_tokens N] [--repetition_penalty 1.2 --repetition_window 16]
        [--fix 12=H,57=D,102=S] [--position_bias bias.npy] [--mixed_precision] [--prefill forward] --output samples.fasta

Runs ProGen.generate: each prompt is laid out like training data (BOS, prompt), every sequence stops at its own EOS,
temperature / top-k / nucleus (top-p) filtering happen in the persistent decode kernel.  --alphabet restricts every
draw to those residues and EOS, --min_new_tokens forbids EOS for the first N generated tokens, and --repetition_penalty
penalises the residues present in the last --repetition_window positions (0: the whole sequence); these act on the
logits in the kernel and leave the reported log-likelihood that of the unconstrained model.  --fix K=R,... makes
generated residue K (1-based) of every sequence R, and no sequence ends before its last fixed residue; --position_bias
adds row j of a float32 [T, V] .npy array to the logits of generated token j + 1 (-inf bans an id there).  A
contradiction between these constraints (a fixed residue outside --alphabet, say) stops with the library's error
message before anything runs.  --prefill forward fills
the decoder's caches for the prompt with one forward pass per distinct prompt instead of one decode step per prompt
position (faster for long prompts; bf16 models then differ from the default by round-off).  Unlike sample.py (the reference
drop-in, one sequence, top_k=25 with the reference's quirks), the result of a row depends only on the seed and the row.
The FASTA has one record per row (row = prompt index * num_samples + sample index):
    >{row} prompt={i} sample={j} log_likelihood={sum of log p of the generated tokens, EOS included} length={...} eos={0|1}
    <generated residues, without the EOS; characters outside printable ASCII are written as '?'>"""
import time

import click
import numpy as np

from progen_b200 import ProGen
from progen_b200.checkpoint import get_checkpoint_fns, package_params
from progen_b200.data import decode_tokens, encode_tokens
from progen_b200.lib import ProgenError


def fasta_safe(residues):
    """one character per token: anything outside printable ASCII (line breaks included) and a leading '>' become '?', so
    every record stays two lines"""
    s = ''.join(ch if ' ' <= ch <= '~' else '?' for ch in residues)
    return '?' + s[1:] if s.startswith('>') else s


def alphabet_bias(alphabet, num_tokens):
    """logit bias that leaves EOS and the characters of `alphabet` (encoded like training text) as the only candidates"""
    ids = np.asarray(encode_tokens(alphabet), np.int64)
    if ids.size == 0 or ids.min() < 1 or ids.max() >= num_tokens:
        bad = [ch for ch in alphabet if not 1 <= ord(ch) + 1 < num_tokens]
        raise ProgenError(f'--alphabet: characters outside the {num_tokens}-token vocabulary: {bad!r}' if bad else
                          '--alphabet: empty')
    bias = np.full(num_tokens, -np.inf, np.float32)
    bias[0] = 0.0
    bias[ids] = 0.0
    return bias


def parse_fix(text):
    """--fix '12=H,57=D' -> {12: 'H', 57: 'D'}: 1-based generated offsets and one residue character each"""
    out = {}
    for item in text.split(','):
        k, sep, res = item.strip().partition('=')
        if not sep or not k.strip().isdigit() or len(res.strip()) != 1:
            raise ProgenError(f'--fix: expected OFFSET=RESIDUE items separated by commas (e.g. 12=H,57=D), got {item!r}')
        k = int(k)
        if k in out:
            raise ProgenError(f'--fix: offset {k} given twice')
        out[k] = res.strip()
    return out


def load_position_bias(path):
    """--position_bias: a [T, V] float32 array from a .npy file"""
    try:
        a = np.load(path, allow_pickle=False)
    except (OSError, ValueError) as e:
        raise ProgenError(f'--position_bias: cannot read {path}: {e}') from None
    if a.dtype != np.float32 or a.ndim != 2:
        raise ProgenError(f'--position_bias: {path} must hold a float32 [T, V] array, got {a.dtype} {a.shape}')
    return a


@click.command()
@click.option('--checkpoint_path', default='./ckpts')
@click.option('--prompt', 'prompts', multiple=True, help='prompt text (repeatable)')
@click.option('--prompts_file', default=None, help='text file, one prompt per line')
@click.option('--num_samples', default=1, help='samples per prompt')
@click.option('--temperature', default=1.0, help='softmax temperature; 0 = greedy')
@click.option('--top_k', default=None, type=int, help='keep the k largest logits (ties kept)')
@click.option('--top_p', default=None, type=float, help='nucleus: smallest set of tokens whose probability reaches top_p')
@click.option('--seed', default=0)
@click.option('--batch_size', default=64, help='sequences per kernel launch (<= 64)')
@click.option('--max_length', default=None, type=int, help='BOS + prompt + generated tokens (default: seq_len)')
@click.option('--alphabet', default=None, help='the only residue characters that may be drawn (EOS is always allowed)')
@click.option('--min_new_tokens', default=0, help='generated tokens before EOS may be drawn')
@click.option('--repetition_penalty', default=1.0, help='divide positive / multiply negative logits of recent ids (1 = off)')
@click.option('--repetition_window', default=0, help='positions the repetition penalty looks back (0 = the whole sequence)')
@click.option('--fix', default=None, help='fixed residues by 1-based generated offset, e.g. 12=H,57=D,102=S')
@click.option('--position_bias', default=None, help='.npy float32 [T, V]: row j is added to the logits of generated token j+1')
@click.option('--mixed_precision', default=False, is_flag=True, help='bf16 weights in the decode kernel')
@click.option('--prefill', default='decode', type=click.Choice(['decode', 'forward']),
              help='prompt positions: one decode step each, or one forward pass per distinct prompt')
@click.option('--output', default='samples.fasta')
def main(checkpoint_path, prompts, prompts_file, num_samples, temperature, top_k, top_p, seed, batch_size, max_length,
         alphabet, min_new_tokens, repetition_penalty, repetition_window, fix, position_bias, mixed_precision, prefill,
         output):
    _, get_last_checkpoint, _ = get_checkpoint_fns(checkpoint_path)
    last_checkpoint = get_last_checkpoint()
    if last_checkpoint is None:
        exit(f'no checkpoints found at {checkpoint_path}')
    params = package_params(last_checkpoint)             # plain params, or base + merged adapters
    model_kwargs = last_checkpoint['model_config']
    model = ProGen(**{**model_kwargs, 'mixed_precision': mixed_precision})
    bias = None if alphabet is None else alphabet_bias(alphabet, model.config['num_tokens'])
    try:
        fixed = None if fix is None else parse_fix(fix)
        pbias = None if position_bias is None else load_position_bias(position_bias)
    except ProgenError as e:
        exit(f'ProgenError: {e}')
    prompts = list(prompts)
    if prompts_file is not None:
        with open(prompts_file) as f:
            prompts += [l.rstrip('\n') for l in f if l.strip()]
    if not prompts:
        prompts = ['']
    print(f'sequence length: {model_kwargs["seq_len"]}')
    t0 = time.perf_counter()
    kw = dict(num_samples=num_samples, temperature=temperature, top_k=top_k, top_p=top_p, max_length=max_length, seed=seed,
              batch_size=batch_size, logit_bias=bias, min_new_tokens=min_new_tokens, repetition_penalty=repetition_penalty,
              repetition_window=repetition_window, prefill=prefill)
    if fixed is None and pbias is None:
        res = model.generate(params, prompts, **kw)
    else:
        try:                                             # contradictory constraints: the library's message, no traceback
            res = model.generate(params, prompts, position_bias=pbias, fixed=fixed, **kw)
        except ProgenError as e:
            exit(f'ProgenError: {e}')
    secs = time.perf_counter() - t0
    N = len(res['length'])
    with open(output, 'w') as f:
        for row in range(N):
            s, ln, fin = int(res['start'][row]), int(res['length'][row]), bool(res['finished'][row])
            body = fasta_safe(decode_tokens(res['tokens'][row, s:s + ln - int(fin)]))
            f.write(f'>{row} prompt={row // num_samples} sample={row % num_samples} '
                    f'log_likelihood={res["log_likelihood"][row]:.6f} length={ln} eos={int(fin)}\n{body}\n')
    gen = int(res['length'].sum())
    print(f'{N} sequences, {gen} generated tokens, {int(res["finished"].sum())} ended with EOS')
    print(f'{N / secs:.2f} sequences/s, {gen / secs:.0f} generated tokens/s (wall clock, including setup)')
    print(f'wrote {output}')


if __name__ == '__main__':
    main()
