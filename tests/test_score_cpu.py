"""ProGen.score input checks that run before any device work (no GPU needed)."""
import numpy as np
import pytest


@pytest.mark.parametrize('shape', [(2, 64), (2, 66), (65,), (1, 2, 65)])
def test_score_rejects_rows_of_the_wrong_width(shape):
    """rows must be (B, seq_len + 1): ids = data[:, :-1], labels = data[:, 1:] (Q12: no silent resize)"""
    from progen_b200 import ProGen
    from progen_b200.lib import ProgenError
    model = ProGen(num_tokens=256, dim=64, seq_len=64, depth=2, window_size=16, global_mlp_depth=1, heads=2, dim_head=32)
    with pytest.raises(ProgenError):
        model.score({}, np.zeros(shape, np.uint16))
    assert model._engine is None
