"""Parameters in a trained model's numerical regime, and the metrics that say they are in it.

`oracle.progen_ref.randomize_params` perturbs biases, LayerNorm scales and the SGU matrices but leaves every weight matrix
at its initialisation, so a model built from it has soft attention (scores of std ~1), logits within ~+-4, GELU inputs
near 0 and a residual stream of unit scale.  A trained checkpoint drives the same kernels much further: near one-hot
softmaxes, confident logits, saturated GELUs and a residual stream with outlier channels.  `sharpen` rescales a
randomized parameter set on the host, deterministically, until the float64 oracle shows that regime; `regime_metrics`
measures it, and THRESHOLDS is what a sharpened model must reach (tests/test_trained_regime_cpu.py checks both, and that
plain `randomize_params` reaches none of the attention, logit and GELU thresholds).

The gains below are the means; the thresholds are the contract."""
import numpy as np
import torch

from oracle.progen_ref import P, layer_kinds

QK_GAIN = 10.0           # q and k columns: attention scores of std ~15-25 after the outlier channel compresses the LayerNorm output
HEAD_GAIN = 14.0         # the logits head
GATE_GAIN = 6.0          # GELU inputs (the GLU gate half, every column of a GELU / gMLP layer's first linear)
EMBED_OFFSET = 40.0      # one embedding channel carried through the whole residual stream
BIAS_OUTLIER = 200.0     # added to one channel of the first layer's feed-forward output bias
SPATIAL_GAIN = 4.0       # SGU spatial weights

# metric -> the value sharpened parameters must reach (at least; and above 0 for the share of phantom-dominated rows)
THRESHOLDS = {
    'attn_max_prob_median': 0.9,      # min over layers of the median over (query, head) of the row's largest probability
    'phantom_dominated_share': 0.0,   # share of window-0 rows whose w zero keys (quirk Q1) hold > 0.5 of the mass (> 0)
    'top1_prob_median': 0.7,          # median over positions of the largest softmax(logits) probability
    'logit_absmax': 30.0,             # max |logit|
    'gelu_saturated_share': 0.05,     # share of GELU inputs with |u| >= 5
    'resid_outlier_ratio': 50.0,      # max |x| / median |x| of the stream entering the final LayerNorm
}


def sharpen(params, cfg, seed=0):
    """randomize_params output -> new float32 parameters in the trained regime (deterministic in seed)"""
    rng = np.random.default_rng(seed)
    d = cfg['dim']
    inner = cfg['heads'] * cfg['dim_head']
    out = {m: {k: np.array(v, np.float32, copy=True) for k, v in dd.items()} for m, dd in params.items()}
    ch = int(rng.integers(0, d))                                   # the outlier channel
    out[P + 'embed']['embeddings'][:, ch] += EMBED_OFFSET
    for i, kind in enumerate(layer_kinds(cfg)):
        w = out[P + f'attn{i}/~/linear']['w']
        w[:, :2 * inner] *= QK_GAIN
        f = P + f'ff{i}/~/'
        w = out[f + 'linear']['w']
        if kind == 'glu':
            w[:, w.shape[1] // 2:] *= GATE_GAIN
            out[f + 'linear']['b'][w.shape[1] // 2:] *= GATE_GAIN
        else:
            w *= GATE_GAIN
        if kind == 'sgu':
            out[f + 'sgu']['spatial_weights'] *= SPATIAL_GAIN
        if i == 0:
            out[f + 'linear_1']['b'][ch] += BIAS_OUTLIER
    out[P + 'linear']['w'] *= HEAD_GAIN
    return out


def regime_metrics(params, ids, cfg, device=None):
    """the metrics of THRESHOLDS for the float64 oracle forward of ids (B, n) -> dict of floats"""
    from oracle import progen_torch as T
    probe = {}
    with torch.no_grad():
        prm = T.to_torch(params, torch.float64, device=device)
        logits = T.forward(prm, torch.as_tensor(np.asarray(ids, np.int64)), cfg, device=device, probe=probe)
    w = cfg['window_size']
    attn_med = min(float(a.amax(-1).median()) for a in probe['attn'])
    phantom = torch.cat([a[:, :, 0, :, :w].sum(-1).flatten() for a in probe['attn']])
    top1 = torch.softmax(logits, -1).amax(-1)
    u = torch.cat([g.flatten() for g in probe['gelu_in']])
    x = probe['resid'][-1].abs()
    return dict(attn_max_prob_median=attn_med,
                phantom_dominated_share=float((phantom > 0.5).double().mean()),
                top1_prob_median=float(top1.median()),
                logit_absmax=float(logits.abs().max()),
                gelu_saturated_share=float((u.abs() >= 5).double().mean()),
                resid_outlier_ratio=float(x.max() / x.median()))


def unmet(metrics):
    """names of the thresholds the metrics do not reach"""
    return [k for k, t in THRESHOLDS.items() if metrics[k] < t or metrics[k] <= 0]
