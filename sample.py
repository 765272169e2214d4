"""sample.py — drop-in for the reference CLI (lucidrains/progen sample.py:23-26: --seed, --checkpoint_path, --prime),
plus --greedy (zero Gumbel noise: the deterministic mode the parity tests use).  Loads the newest checkpoint, rebuilds
the model from its `model_config`, samples with top_k=25, add_bos=True (sample.py:70) and prints from prime_length on."""
import click
import numpy as np

from progen_b200 import ProGen
from progen_b200.checkpoint import get_checkpoint_fns, package_params
from progen_b200.data import decode_tokens, encode_tokens
from progen_b200.utils import sample


@click.command()
@click.option('--seed', default=42)
@click.option('--checkpoint_path', default='./ckpts')
@click.option('--prime', default='')
@click.option('--greedy', default=False, is_flag=True)
@click.option('--mixed_precision', default=False, is_flag=True, help='bf16 weights in the decode kernels')
@click.option('--no_kv_cache', default=False, is_flag=True, help="reference-style loop: full re-forward per token")
def main(seed, checkpoint_path, prime, greedy, mixed_precision, no_kv_cache):
    _, get_last_checkpoint, _ = get_checkpoint_fns(checkpoint_path)
    last_checkpoint = get_last_checkpoint()
    if last_checkpoint is None:
        exit(f'no checkpoints found at {checkpoint_path}')
    params = package_params(last_checkpoint)             # plain params, or base + merged adapters
    num_seqs = max(last_checkpoint['next_seq_index'], 0)
    model_kwargs = last_checkpoint['model_config']
    model = ProGen(**{**model_kwargs, 'mixed_precision': mixed_precision})
    seq_len = model_kwargs['seq_len']
    print(f'params: {sum(a.size for d in params.values() for a in d.values())}')
    print(f'sequence length: {seq_len}')
    print(f'trained for {num_seqs} sequences')
    prime_tokens = encode_tokens(prime)
    prime_length = len(prime_tokens) + 1
    prime_tensor = np.array(prime_tokens, dtype=np.uint16)
    if no_kv_cache:
        sampled = sample(seed, model.apply, params, prime_tensor, seq_len, top_k=25, add_bos=True, greedy=greedy)
    else:
        import torch
        from progen_b200.decode import BatchDecoder
        # one persistent kernel generates the whole sequence (csrc/decode_persist.cu).  With the reference's default
        # --prime '' the reference draws position 0 from logits[-1] of the all-pad sequence; the cached decoder keeps the
        # pad there (use --no_kv_cache for that exact behaviour).
        dec = BatchDecoder(model.config, params, batch=1, weights_dtype=torch.bfloat16 if mixed_precision else torch.float32)
        sampled, steps, secs = dec.sample(prime_tensor, top_k=25, add_bos=True, greedy=greedy, seed=seed)
        print(f'decoded {steps} tokens at {steps / max(secs, 1e-9):.0f} tokens/s (device time, KV-cached persistent kernel)')
    print('\n', prime, '\n', '*' * 40, '\n', decode_tokens(sampled[prime_length:]))


if __name__ == '__main__':
    main()
