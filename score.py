"""score.py — log-likelihood (and optionally embeddings) of protein sequences under the newest checkpoint.

    python score.py --checkpoint_path ./ckpts --input seqs.txt --output scores.tsv [--embeddings emb.npy]

--input is a text file with one sequence per line (the format of train.py --text_file; blank lines are skipped).  Each
sequence is tokenized like training data (data.collate: BOS, bytes + 1, truncated to seq_len, zero padded) and scored by
ProGen.score: the counted positions are the BOS and every residue (the labels of the loss, end-of-sequence included), so
mean_nll is the per-sequence cross entropy of the training loss and perplexity = exp(mean_nll).  The TSV has one row per
input sequence, in input order."""
import click
import numpy as np

from progen_b200 import ProGen
from progen_b200.checkpoint import get_checkpoint_fns, package_params
from progen_b200.data import collate


@click.command()
@click.option('--checkpoint_path', default='./ckpts')
@click.option('--input', 'input_path', required=True, help='text file, one sequence per line')
@click.option('--output', default='scores.tsv', help='TSV: index, residues, log_likelihood, num_tokens, mean_nll, perplexity')
@click.option('--embeddings', default=None, help='also write the per-sequence embeddings (N, dim) to this .npy file')
@click.option('--batch_size', default=64, help='sequences per forward pass')
@click.option('--mixed_precision', default=False, is_flag=True, help='bf16 tensor-core engine')
def main(checkpoint_path, input_path, output, embeddings, batch_size, mixed_precision):
    _, get_last_checkpoint, _ = get_checkpoint_fns(checkpoint_path)
    last_checkpoint = get_last_checkpoint()
    if last_checkpoint is None:
        exit(f'no checkpoints found at {checkpoint_path}')
    params = package_params(last_checkpoint)             # plain params, or base + merged adapters
    model_kwargs = last_checkpoint['model_config']
    model = ProGen(**{**model_kwargs, 'mixed_precision': mixed_precision})
    seq_len = model_kwargs['seq_len']
    with open(input_path) as f:
        seqs = [l.strip() for l in f if l.strip()]
    lengths = [len(s.encode()) for s in seqs]
    truncated = sum(1 for n in lengths if n > seq_len)
    print(f'sequence length: {seq_len}')
    print(f'{len(seqs)} sequences, {truncated} truncated to {seq_len} residues')
    res = model.score(params, collate(seqs, seq_len), batch_size=batch_size, return_embeddings=embeddings is not None)
    ll, cnt = res['log_likelihood'].astype(np.float64), res['num_tokens']
    mean_nll = -ll / np.maximum(cnt, 1)
    with open(output, 'w') as f:
        f.write('index\tresidues\tlog_likelihood\tnum_tokens\tmean_nll\tperplexity\n')
        for i in range(len(seqs)):
            f.write(f'{i}\t{min(lengths[i], seq_len)}\t{res["log_likelihood"][i]:.9g}\t{cnt[i]}\t{mean_nll[i]:.9g}\t'
                    f'{np.exp(mean_nll[i]):.9g}\n')
    print(f'wrote {output}')
    if embeddings is not None:
        np.save(embeddings, res['embedding'])
        print(f'wrote {embeddings} {res["embedding"].shape}')


if __name__ == '__main__':
    main()
