"""Variant scoring on the cut forward: ProGen.score_variants / mutational_scan against `score` on the explicitly mutated
full-length rows (bitwise), against the float64 oracle, across batch sizes and chunkings, and the attention forward
with a partial last window that the cut forward runs on."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from test_gpu_elementwise import attn_ref

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
AA = 'ACDEFGHIKLMNPQRSTVWY'
PREFIX = '[Tax=Mammalia] #'
BASE = dict(num_tokens=256, dim=128, depth=2, heads=2, dim_head=64, global_mlp_depth=1)
MODELS = {
    'glu_sgu_w128': dict(BASE, seq_len=512, window_size=128),
    'gelu_sgu_w256': dict(BASE, seq_len=512, window_size=256, ff_glu=False),           # cuts at 128 / 384: partial windows
    'all_glu_w64': dict(BASE, seq_len=256, window_size=64, global_mlp_depth=0),
    'noshift_w256': dict(BASE, seq_len=512, window_size=256, shift_tokens=False),
    'cfg2_width': dict(num_tokens=256, dim=512, seq_len=1024, depth=2, heads=8, dim_head=64, window_size=256,
                       global_mlp_depth=1),
    'cfg3_width': dict(num_tokens=256, dim=1024, seq_len=2048, depth=3, heads=16, dim_head=64, window_size=512,
                       global_mlp_depth=2),
}


@functools.lru_cache(maxsize=None)
def _params(name):
    from oracle import progen_ref as O
    kw = MODELS[name]
    seed = 7 * kw['dim'] + kw['seq_len']
    return O.randomize_params(O.init_params(O.make_config(**kw), seed), seed + 1)


@functools.lru_cache(maxsize=None)
def _model(name, mp):
    from progen_b200 import ProGen
    return ProGen(**MODELS[name], mixed_precision=mp)


def _wild_type(length, seed):
    return ''.join(np.random.default_rng(seed).choice(list(AA), size=length))


def _mutate(wt, s):
    r = list(wt)
    for sub in filter(None, s.split(':')):
        r[int(sub[1:-1]) - 1] = sub[-1]
    return ''.join(r)


def _sets(wt, kept, seed):
    """the wild type, an identity, substitutions at the first and the last residue that fits, and a double"""
    rng = np.random.default_rng(seed)
    other = lambda p: [a for a in AA if a != wt[p - 1]][int(rng.integers(19))]
    mid = max(1, kept // 2)
    return ['', f'{wt[mid - 1]}{mid}{wt[mid - 1]}', f'{wt[0]}1{other(1)}', f'{wt[kept - 1]}{kept}{other(kept)}',
            f'{wt[0]}1{other(1)}:{wt[mid - 1]}{mid}{other(mid)}' if mid > 1 else f'{wt[0]}1{other(1)}']


def _check_against_score(model, params, wt, sets, prefix, batch_size=64):
    """score_variants == score on the explicitly mutated full-length rows, bit for bit; delta is the float64 sum of the
    token differences; returns the score_variants result"""
    from progen_b200.data import collate
    n = model.config['seq_len']
    res = model.score_variants(params, wt, sets, prefix=prefix, batch_size=batch_size, return_tokens=True)
    rows = collate([prefix + wt] + [prefix + _mutate(wt, s) for s in sets], n)
    ref = model.score(params, rows, batch_size=batch_size, return_tokens=True)
    np.testing.assert_array_equal(res['log_likelihood'], ref['log_likelihood'][1:])
    np.testing.assert_array_equal(res['num_tokens'], ref['num_tokens'][1:])
    np.testing.assert_array_equal(res['token_logp'], ref['token_logp'][1:])
    assert res['wt_log_likelihood'] == ref['log_likelihood'][0]
    lp = ref['token_logp'].astype(np.float64)
    np.testing.assert_array_equal(res['delta'], (lp[1:] - lp[0]).sum(-1))
    for i, s in enumerate(sets):
        if _mutate(wt, s) == wt:
            assert res['delta'][i] == 0.0, (s, res['delta'][i])           # '' and identities: exact zeros
    assert res['delta'].dtype == np.float64
    return res


# need = counted positions of a row = len(prefix + residues) + 1 (BOS ... EOS); n + 1 is a row longer than seq_len
NEEDS = [127, 128, 129, 'n-1', 'n', 'n+1']
CASES = [(name, mp) for name in MODELS for mp in (False, True)]


@pytest.mark.parametrize('prefix', ['', PREFIX])
@pytest.mark.parametrize('name, mp', CASES)
def test_score_variants_is_score_bitwise(name, mp, prefix):
    """at row lengths that need 127, 128, 129, n - 1, n counted positions and a row longer than n (no cut)"""
    from progen_b200.engine import cut_length
    from progen_b200.data import collate
    model, params = _model(name, mp), _params(name)
    n = model.config['seq_len']
    for k, need in enumerate(NEEDS):
        need = eval(need, {'n': n}) if isinstance(need, str) else need
        residues = need - 1 - len(prefix)
        wt = _wild_type(residues, 11 * need + len(prefix))
        kept = min(residues, n - len(prefix))
        sets = _sets(wt, kept, need)
        L = cut_length(collate([prefix + wt], n)[:, 1:])
        assert L == min(n, -(-min(need, n) // 128) * 128)
        _check_against_score(model, params, wt, sets, prefix, batch_size=4 if k % 2 else 64)


@pytest.mark.parametrize('mp', [False, True])
def test_results_do_not_depend_on_batch_or_company(mp):
    """a variant's bits are the same at batch_size 1, 7 and 64 and next to different other variants"""
    model, params = _model('gelu_sgu_w256', mp), _params('gelu_sgu_w256')
    wt = _wild_type(300, 3)
    rng = np.random.default_rng(4)
    pool = [f'{wt[p - 1]}{p}{a}' for p in rng.choice(np.arange(1, 301), 20, replace=False) for a in 'GW' if a != wt[p - 1]]
    probe = pool[:3]
    runs = [model.score_variants(params, wt, probe, batch_size=bs, return_tokens=True) for bs in (1, 7, 64)]
    runs.append({k: (v[-3:] if np.ndim(v) else v) for k, v in
                 model.score_variants(params, wt, pool[5:15] + probe, batch_size=7, return_tokens=True).items()})
    runs.append({k: (v[::2] if np.ndim(v) else v) for k, v in
                 model.score_variants(params, wt, [probe[0], pool[20], probe[1], pool[21], probe[2]], return_tokens=True).items()})
    for r in runs[1:]:
        for key in runs[0]:
            np.testing.assert_array_equal(r[key], runs[0][key], err_msg=key)


def test_delta_against_float64():
    """fp32 engine, small model: |delta - delta_ref| <= 2e-5 * num_tokens with delta_ref from the float64 oracle"""
    from oracle import progen_ref as O
    from oracle import progen_torch as T
    from progen_b200.data import collate
    name = 'glu_sgu_w128'
    model, params = _model(name, False), _params(name)
    cfg = O.make_config(**MODELS[name])
    wt = _wild_type(200, 21)
    sets = ['', 'M1A' if wt[0] == 'M' else f'{wt[0]}1M', f'{wt[99]}100W', f'{wt[9]}10P:{wt[149]}150G', f'{wt[199]}200K']
    res = model.score_variants(params, wt, sets, prefix=PREFIX)
    rows = collate([PREFIX + wt] + [PREFIX + _mutate(wt, s) for s in sets], cfg['seq_len']).astype(np.int64)
    with torch.no_grad():
        logits = T.forward(T.to_torch(params, torch.float64, device='cuda'), torch.as_tensor(rows[:, :-1]), cfg, device='cuda')
        labels = torch.as_tensor(rows[:, 1:], device='cuda')
        nll = T.cross_entropy(logits, labels)
        mask = labels != 0
        count = (mask | (((~mask).cumsum(-1) == 1) & ~mask)).sum(-1)
        ll = (-nll * count).cpu().numpy()
    ref = ll[1:] - ll[0]
    err = np.abs(res['delta'] - ref)
    print(f'delta vs float64: max abs err {err.max():.3e}, bound {2e-5 * res["num_tokens"].max():.3e}')
    assert (err <= 2e-5 * res['num_tokens']).all(), (err, res['num_tokens'])
    np.testing.assert_array_equal(res['num_tokens'], count[1:].cpu().numpy())


@pytest.mark.parametrize('mp', [False, True])
def test_mutational_scan_is_score_variants(mp):
    """the scan matrix equals score_variants over the same sets, with exact zeros at the wild-type letter"""
    model, params = _model('all_glu_w64', mp), _params('all_glu_w64')
    wt = _wild_type(150, 5)
    positions = [1, 2, 77, 150]
    scan = model.mutational_scan(params, wt, positions=positions, prefix=PREFIX, batch_size=16)
    assert scan['delta'].shape == (4, 20) and scan['delta'].dtype == np.float64
    np.testing.assert_array_equal(scan['positions'], positions)
    sets = [f'{wt[p - 1]}{p}{a}' for p in positions for a in AA]
    res = model.score_variants(params, wt, sets, prefix=PREFIX, batch_size=5)
    np.testing.assert_array_equal(scan['delta'], res['delta'].reshape(4, 20))
    for i, p in enumerate(positions):
        assert scan['delta'][i, AA.index(wt[p - 1])] == 0.0
    assert scan['wt_log_likelihood'] == res['wt_log_likelihood']
    assert (scan['delta'] != 0).sum() == 4 * 19


def test_cut_forward_adds_no_memory():
    """score_variants allocates the same inference activation set that score allocates at the same batch_size"""
    name = 'cfg2_width'
    added = {}
    for how in ('score', 'variants'):
        from progen_b200 import ProGen
        from progen_b200.data import collate
        model = ProGen(**MODELS[name], mixed_precision=True)
        params = _params(name)
        model._ensure_loaded(params)
        wt = _wild_type(300, 8)
        sets = [f'{wt[p - 1]}{p}{"W" if wt[p - 1] != "W" else "G"}' for p in range(1, 128)]
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        if how == 'score':
            model.score(params, collate([wt] + [_mutate(wt, s) for s in sets], 1024), batch_size=64)
        else:
            model.score_variants(params, wt, sets, batch_size=64)
        torch.cuda.synchronize()
        added[how] = torch.cuda.max_memory_allocated() - base
        del model
    print(f'score adds {added["score"] / 2**20:.1f} MiB, score_variants adds {added["variants"] / 2**20:.1f} MiB')
    assert added['variants'] <= added['score'], added


# ------------------------------------------------------------------------------------------------ attention kernels
@pytest.mark.parametrize('kernel', ['tc', 'simt'])
@pytest.mark.parametrize('cfg', [(2, 512, 256, 2, 320), (1, 1024, 512, 3, 640), (3, 512, 256, 2, 128), (2, 256, 128, 2, 192)])
def test_attention_forward_with_a_partial_last_window(kernel, cfg):
    """the forward at a per-sequence count cut (a multiple of 64, not of the window) is bitwise the first cut rows of the
    full-length forward, and within the existing attention tests' bound (2e-2) of float64"""
    from progen_b200 import lib as L
    L.require_device()
    B, n, w, h, cut = cfg
    dh, I = 64, h * 64
    g = torch.Generator(device='cuda').manual_seed(n + cut)
    qkv = (torch.randn(B * n, 3 * I, generator=g, device='cuda') * 1.5).bfloat16()
    qkv_cut = qkv.view(B, n, 3 * I)[:, :cut].contiguous().view(B * cut, 3 * I)

    def fwd(x, seq_len):
        out = torch.full((B * seq_len, I), float('nan'), device='cuda', dtype=torch.bfloat16)
        lse = torch.full((B * seq_len, h), float('nan'), device='cuda')
        if kernel == 'tc':
            L.check(L.load().progen_local_attn_fwd_tc(x.data_ptr(), out.data_ptr(), lse.data_ptr(), B, seq_len, w, h, dh, L.stream()))
        else:
            L.check(L.load().progen_local_attn_fwd_simt(x.data_ptr(), out.data_ptr(), lse.data_ptr(), L.BF16, B, seq_len, w, h, dh,
                                                        L.stream()))
        torch.cuda.synchronize()
        return out.view(B, seq_len, I), lse.view(B, seq_len, h)

    out, lse = fwd(qkv, n)
    out_c, lse_c = fwd(qkv_cut, cut)
    assert torch.equal(out_c, out[:, :cut]) and torch.equal(lse_c, lse[:, :cut])
    ref = attn_ref(qkv.double(), B, n, w, h, dh).view(B, n, I)[:, :cut]
    err = (out_c.double() - ref).abs().max().item()
    assert err < 2e-2, err


def test_simt_attention_forward_takes_any_count():
    """the CUDA-core forward takes a count that is not a multiple of 64 (fp32 operands: bitwise the full forward's rows)"""
    from progen_b200 import lib as L
    B, n, w, h, dh, cut = 2, 256, 128, 2, 32, 100
    I = h * dh
    g = torch.Generator(device='cuda').manual_seed(5)
    qkv = torch.randn(B * n, 3 * I, generator=g, device='cuda')
    qkv_cut = qkv.view(B, n, 3 * I)[:, :cut].contiguous().view(B * cut, 3 * I)
    outs = []
    for x, m in ((qkv, n), (qkv_cut, cut)):
        out, lse = torch.empty(B * m, I, device='cuda'), torch.empty(B * m, h, device='cuda')
        L.check(L.load().progen_local_attn_fwd_simt(x.data_ptr(), out.data_ptr(), lse.data_ptr(), L.F32, B, m, w, h, dh, L.stream()))
        outs.append((out.view(B, m, I), lse.view(B, m, h)))
    assert torch.equal(outs[1][0], outs[0][0][:, :cut]) and torch.equal(outs[1][1], outs[0][1][:, :cut])


@pytest.mark.parametrize('kernel', ['tc', 'simt'])
def test_attention_backward_still_needs_whole_windows(kernel):
    """training never cuts: the backward entry points reject a partial last window before launching anything"""
    from progen_b200 import lib as L
    B, n, w, h, dh = 1, 320, 256, 2, 64
    I = h * dh
    qkv = torch.zeros(B * n, 3 * I, device='cuda', dtype=torch.bfloat16)
    out, dout, dqkv = torch.zeros(B * n, I, device='cuda', dtype=torch.bfloat16), torch.zeros(B * n, I, device='cuda', dtype=torch.bfloat16), torch.zeros_like(qkv)
    lse, delta = torch.zeros(B * n, h, device='cuda'), torch.zeros(B * n, h, device='cuda')
    lib = L.load()
    if kernel == 'tc':
        rc = lib.progen_local_attn_bwd_tc(qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), dqkv.data_ptr(),
                                          delta.data_ptr(), 0, 0, B, n, w, h, dh, L.stream())
    else:
        rc = lib.progen_local_attn_bwd_simt(qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), dqkv.data_ptr(),
                                            delta.data_ptr(), L.BF16, B, n, w, h, dh, L.stream())
    assert rc == -2, rc                                   # PROGEN_ERR_ARG
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ CLI
def test_variants_cli(tmp_path):
    """variants.py on a checkpoint: the TSV is model.score_variants of the same sets (one set per line and a ProteinGym
    CSV), and --scan writes the mutational_scan matrix"""
    from progen_b200 import ProGen
    from progen_b200.checkpoint import file_save_checkpoint
    from oracle import progen_ref as O
    kwargs = dict(num_tokens=256, dim=128, seq_len=128, depth=2, window_size=64, global_mlp_depth=1, heads=2, dim_head=64)
    params = O.randomize_params(O.init_params(O.make_config(**kwargs), 91), 92)
    (tmp_path / 'ckpts').mkdir()
    file_save_checkpoint(tmp_path / 'ckpts', dict(next_seq_index=0, params=params, optim_state=None, model_config=kwargs,
                                                  run_id=None))
    wt = _wild_type(60, 93)
    sets = ['', f'{wt[0]}1A', f'{wt[4]}5W:{wt[59]}60K', f'{wt[9]}10{wt[9]}']
    (tmp_path / 'sets.txt').write_text('\n'.join(sets) + '\n')
    (tmp_path / 'sets.csv').write_text('mutant,DMS_score\n' + ''.join(f'{s},0.5\n' for s in sets))
    env = dict(os.environ, PYTHONPATH=ROOT)

    def run(*args):
        r = subprocess.run([sys.executable, os.path.join(ROOT, 'variants.py'), '--checkpoint_path', str(tmp_path / 'ckpts'),
                            '--wild_type', wt, '--prefix', '#', *args], cwd=str(tmp_path), env=env, capture_output=True,
                           text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        return [l.split('\t') for l in (tmp_path / args[args.index('--output') + 1]).read_text().splitlines()]

    ref = ProGen(**kwargs).score_variants(params, wt, sets, prefix='#')
    for src in ('sets.txt', 'sets.csv'):
        lines = run('--mutations', src, '--output', f'{src}.tsv')
        assert lines[0] == ['mutant', 'delta', 'log_likelihood', 'num_tokens']
        assert [l[0] for l in lines[1:]] == sets
        for i, l in enumerate(lines[1:]):
            assert float(l[1]) == ref['delta'][i] and np.float32(float(l[2])) == ref['log_likelihood'][i]
            assert int(l[3]) == ref['num_tokens'][i]
    lines = run('--scan', '--positions', '1-3,60', '--output', 'scan.tsv')
    scan = ProGen(**kwargs).mutational_scan(params, wt, positions=[1, 2, 3, 60], prefix='#')
    assert lines[0] == ['position', 'wild_type'] + list(AA)
    for i, l in enumerate(lines[1:]):
        assert int(l[0]) == scan['positions'][i] and l[1] == wt[scan['positions'][i] - 1]
        np.testing.assert_allclose([float(v) for v in l[2:]], scan['delta'][i], rtol=1e-8, atol=0)
