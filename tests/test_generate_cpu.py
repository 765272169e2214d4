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
