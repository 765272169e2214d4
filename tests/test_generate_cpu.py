"""ProGen.generate argument checks: every invalid call raises ProgenError before anything needs a device."""
import numpy as np
import pytest

KW = dict(num_tokens=256, dim=64, seq_len=64, depth=2, window_size=16, global_mlp_depth=1, heads=2, dim_head=32)


@pytest.mark.parametrize('prompts,kwargs', [
    ('#' * 63, {}),                                     # BOS + 63 ids reach seq_len: nothing left to generate
    ('abcd', dict(max_length=5)),                       # len + 1 >= max_length
    ('', dict(max_length=65)),                          # max_length > seq_len
    ('', dict(max_length=1)),
    ([np.array([1, 2, 256])], {}),                      # ids outside [1, V)
    ([np.array([0, 5])], {}),                           # 0 is BOS / EOS, not a prompt id
    ([np.array([[1, 2]])], {}),                         # not 1-D
    ([np.array([1.5])], {}),                            # not integer
    ([], {}),
    (5, {}),
    ('a', dict(temperature=-0.1)),
    ('a', dict(temperature=float('inf'))),
    ('a', dict(temperature=float('nan'))),
    ('a', dict(temperature='hot')),
    ('a', dict(top_k=0)),
    ('a', dict(top_k=257)),
    ('a', dict(top_k=2.5)),
    ('a', dict(top_p=0.0)),
    ('a', dict(top_p=1.01)),
    ('a', dict(top_p=float('nan'))),
    ('a', dict(num_samples=0)),
    ('a', dict(num_samples=True)),
    ('a', dict(batch_size=0)),
    ('a', dict(batch_size=65)),
    ('a', dict(seed=-1)),
    ('a', dict(seed=1 << 64)),
])
def test_generate_rejects_invalid_arguments_without_a_device(prompts, kwargs):
    from progen_b200 import ProGen
    from progen_b200.lib import ProgenError
    model = ProGen(**KW)
    with pytest.raises(ProgenError):
        model.generate({}, prompts, **kwargs)
    assert model._engine is None and model._gen_decoder is None


@pytest.mark.parametrize('prompts,kwargs', [
    ('a', dict(temperature=-0.1)), ('a', dict(temperature=float('nan'))), ('a', dict(temperature='hot')),
    ('a', dict(top_k=0)), ('a', dict(top_k=257)), ('a', dict(top_k=2.5)), ('a', dict(top_k=True)),
    ('a', dict(top_p=0.0)), ('a', dict(top_p=1.01)), ('a', dict(seed=-1)), ('a', dict(seed=1 << 64)), ('a', dict(seed=1.0)),
    ('a', dict(logit_bias=np.zeros(255))), ('a', dict(logit_bias='abc')), ('a', dict(logit_bias=np.full(256, np.nan))),
    ('a', dict(logit_bias=np.full(256, 1e300))),
    ('a', dict(repetition_penalty=0.0)), ('a', dict(repetition_penalty='high')), ('a', dict(repetition_window=65)),
    ('a', dict(repetition_window=1.5)),
    ([np.array([1, 2, 256])], {}), ([np.array([0, 5])], {}), ([np.array([[1, 2]])], {}), ([np.array([1.5])], {}),
    ([np.arange(1, 64)], {}), ([np.arange(1, 5)], dict(max_length=5)),
])
def test_generate_and_the_decoder_refuse_alike(prompts, kwargs):
    """ProGen.generate and BatchDecoder share one check of the sampler settings (Sampling.check) and of the prompt ids
    (prompt_ids): the same refusal, with the same message, whichever the value reaches"""
    from progen_b200 import ProGen
    from progen_b200.decode import Sampling, prompt_ids
    from progen_b200.lib import ProgenError
    with pytest.raises(ProgenError) as via_model:
        ProGen(**KW).generate({}, prompts, **kwargs)
    settings = dict(kwargs)
    max_length = settings.pop('max_length', 64)
    with pytest.raises(ProgenError) as via_decoder:
        prompt_ids([np.array([66])] if prompts == 'a' else prompts, 256, max_length)      # 'a' encodes to [66]
        Sampling.check(256, 64, 64, False, **settings)                                    # BatchDecoder's limits
    assert str(via_model.value) == str(via_decoder.value)


def test_min_new_tokens_bound_and_all_banned_logit_bias():
    """the two rules the callers of Sampling.check set: ProGen.generate bounds min_new_tokens by max_length - 2 and keeps
    an id of [1, V) allowed; BatchDecoder takes the kernel's limits, min_new_tokens up to seq_len and any bans"""
    from progen_b200 import ProGen
    from progen_b200.decode import Sampling
    from progen_b200.lib import ProgenError
    model = ProGen(**KW)
    for kwargs, limit in ((dict(min_new_tokens=63), 62), (dict(min_new_tokens=9, max_length=10), 8)):
        with pytest.raises(ProgenError, match=rf'min_new_tokens must be an integer in \[0, {limit}\]'):
            model.generate({}, 'a', **kwargs)
    assert Sampling.check(256, 64, 62, True, min_new_tokens=62).min_new_tokens == 62
    assert Sampling.check(256, 64, 64, False, min_new_tokens=64).min_new_tokens == 64
    with pytest.raises(ProgenError, match=r'min_new_tokens must be an integer in \[0, 64\], got 65'):
        Sampling.check(256, 64, 64, False, min_new_tokens=65)
    only_eos = np.full(256, -np.inf, np.float32)
    only_eos[0] = 0.0
    with pytest.raises(ProgenError, match=r'bans every id in \[1, V\)'):
        model.generate({}, 'a', logit_bias=only_eos)
    with pytest.raises(ProgenError, match=r'bans every id in \[1, V\)'):
        Sampling.check(256, 64, 62, True, logit_bias=only_eos)
    s = Sampling.check(256, 64, 64, False, logit_bias=np.full(256, -np.inf))
    assert s.logit_bias.dtype == np.float32 and (s.logit_bias == -np.inf).all()
    assert model._engine is None and model._gen_decoder is None
