"""variants.py — zero-shot variant effects against a wild type under the newest checkpoint.

    python variants.py --checkpoint_path ./ckpts --wild_type MKTAYIAK... --mutations sets.txt --output variants.tsv
    python variants.py --checkpoint_path ./ckpts --wild_type MKTAYIAK... --scan [--positions 1-120] --output dms.tsv

--mutations is a text file with one mutation set per line ('A23G', 'A23G:K45R'; a blank line is the wild type itself), or
a CSV with a `mutant` column (ProteinGym's substitution files).  Positions are 1-based over the residues of --wild_type,
not over --prefix (an optional tag such as '[Tax=Mammalia] #' placed before them).  Each row is scored by
ProGen.score_variants: delta = log p(variant) - log p(wild type), summed in float64 over the positions.  The TSV has one
row per set, in input order: mutant, delta, log_likelihood, num_tokens.

--scan scores every single substitution at --positions (default: every residue) to each of the 20 amino acids
(ProGen.mutational_scan) and writes the matrix: one row per position (position, wild-type letter, then delta per letter)."""
import csv

import click
import numpy as np

from progen_b200 import ProGen
from progen_b200.checkpoint import get_checkpoint_fns, package_params
from progen_b200.variants import AMINO_ACIDS, parse_positions


def read_mutations(path):
    with open(path, newline='') as f:
        text = f.read()
    lines = text.splitlines()
    head = [c.strip() for c in lines[0].split(',')] if lines else []
    if 'mutant' in head:
        return [r['mutant'].strip() for r in csv.DictReader(lines)]
    return [l.strip() for l in lines]


@click.command()
@click.option('--checkpoint_path', default='./ckpts')
@click.option('--wild_type', required=True, help='wild-type residue string')
@click.option('--prefix', default='', help='prompt / tag placed before the residues')
@click.option('--mutations', 'mutations_path', default=None, help='one mutation set per line, or a CSV with a mutant column')
@click.option('--scan', is_flag=True, default=False, help='score every single substitution (deep mutational scan)')
@click.option('--positions', default=None, help='--scan positions, 1-based, e.g. 1-120 or 5,9,20-30 (default: all)')
@click.option('--output', default='variants.tsv')
@click.option('--batch_size', default=64, help='sequences per forward pass')
@click.option('--mixed_precision', default=False, is_flag=True, help='bf16 tensor-core engine')
def main(checkpoint_path, wild_type, prefix, mutations_path, scan, positions, output, batch_size, mixed_precision):
    if scan == (mutations_path is not None):
        raise click.UsageError('give exactly one of --mutations FILE and --scan')
    _, get_last_checkpoint, _ = get_checkpoint_fns(checkpoint_path)
    last_checkpoint = get_last_checkpoint()
    if last_checkpoint is None:
        exit(f'no checkpoints found at {checkpoint_path}')
    params = package_params(last_checkpoint)             # plain params, or base + merged adapters
    model_kwargs = last_checkpoint['model_config']
    model = ProGen(**{**model_kwargs, 'mixed_precision': mixed_precision})
    print(f'sequence length: {model_kwargs["seq_len"]}, wild type: {len(wild_type)} residues')
    if scan:
        pos = None if positions is None else parse_positions(positions, len(wild_type))
        res = model.mutational_scan(params, wild_type, positions=pos, prefix=prefix, batch_size=batch_size)
        with open(output, 'w') as f:
            f.write('position\twild_type\t' + '\t'.join(AMINO_ACIDS) + '\n')
            for i, p in enumerate(res['positions']):
                f.write(f'{p}\t{wild_type[p - 1]}\t' + '\t'.join(f'{v:.9g}' for v in res['delta'][i]) + '\n')
        print(f'wild type log_likelihood {res["wt_log_likelihood"]:.9g}; {len(res["positions"])} positions x '
              f'{len(AMINO_ACIDS)} letters')
    else:
        sets = read_mutations(mutations_path)
        res = model.score_variants(params, wild_type, sets, prefix=prefix, batch_size=batch_size)
        with open(output, 'w') as f:
            f.write('mutant\tdelta\tlog_likelihood\tnum_tokens\n')
            for i, m in enumerate(sets):
                f.write(f'{m}\t{res["delta"][i]:.17g}\t{res["log_likelihood"][i]:.9g}\t{res["num_tokens"][i]}\n')
        print(f'wild type log_likelihood {res["wt_log_likelihood"]:.9g}; {len(sets)} mutation sets, '
              f'mean delta {float(np.mean(res["delta"])):.6g}')
    print(f'wrote {output}')


if __name__ == '__main__':
    main()
