"""ProGen.score_variants / mutational_scan input checks and row building, which run before any device work (no GPU
needed), and the cut length of the scoring forward."""
import numpy as np
import pytest

KW = dict(num_tokens=256, dim=64, seq_len=128, depth=2, window_size=64, global_mlp_depth=1, heads=2, dim_head=32)
WT = 'MKTAYIAKQR'


def _model():
    from progen_b200 import ProGen
    return ProGen(**KW)


@pytest.mark.parametrize('mutations, match', [
    ([], 'non-empty'),
    ('A4G', 'non-empty'),
    (['A4G', 5], r"mutation set 1 \(5\).*string"),
    (['K4G'], r"mutation set 0 \('K4G'\).*has 'A' at position 4"),
    (['', 'M0A'], r"mutation set 1 \('M0A'\).*out of range"),
    (['R11A'], r"mutation set 0 \('R11A'\).*out of range"),
    (['A4G:A4C'], r"mutation set 0 \('A4G:A4C'\).*twice"),
    (['A4'], r"mutation set 0 \('A4'\).*printable"),
    (['A4GG'], r"mutation set 0 \('A4GG'\).*printable"),
    (['A4\x07'], r"mutation set 0 .*printable"),
    (['A4é'], r"mutation set 0 .*printable"),
    (['4G'], r"mutation set 0 \('4G'\).*letter"),
    (['A4G:'], r"mutation set 0 \('A4G:'\)"),
])
def test_score_variants_rejects(mutations, match):
    from progen_b200.lib import ProgenError
    model = _model()
    with pytest.raises(ProgenError, match=match):
        model.score_variants({}, WT, mutations)
    assert model._engine is None


def test_position_cut_off_by_seq_len():
    """collate keeps the first seq_len tokens of prefix + residues: a residue beyond them cannot be scored"""
    from progen_b200.lib import ProgenError
    model = _model()
    wt = 'A' * 130
    prefix = '[tag] #'                                   # 7 characters: residues 1..121 fit in 128 tokens
    with pytest.raises(ProgenError, match=r"mutation set 1 \('A122G'\).*cut off by seq_len 128"):
        model.score_variants({}, wt, ['A121G', 'A122G'], prefix=prefix)
    with pytest.raises(ProgenError, match='cut off'):
        model.score_variants({}, wt, ['A129G'])
    with pytest.raises(ProgenError, match='cut off'):
        model.mutational_scan({}, wt, positions=[129])
    assert model._engine is None


def test_wild_type_and_prefix_must_be_ascii():
    from progen_b200.lib import ProgenError
    model = _model()
    with pytest.raises(ProgenError, match='wild_type'):
        model.score_variants({}, 'MKé', [''])
    with pytest.raises(ProgenError, match='prefix'):
        model.score_variants({}, WT, [''], prefix='é')


def test_mutational_scan_rejects():
    from progen_b200.lib import ProgenError
    model = _model()
    for kw in (dict(positions=[]), dict(positions=[0]), dict(positions=[11]), dict(positions=[2, 2]), dict(positions=[1.0]),
               dict(alphabet=''), dict(alphabet='AA'), dict(alphabet='Aé')):
        with pytest.raises(ProgenError):
            model.mutational_scan({}, WT, **kw)
    assert model._engine is None


def test_rows_are_collate_of_the_mutated_strings():
    """the wild type first, then each variant, as data.collate([prefix + residues]) of the explicitly mutated string;
    identity substitutions and '' give the wild-type row"""
    from progen_b200.data import collate
    from progen_b200.variants import parse_mutations, variant_rows
    sets = ['', 'M1A', 'A4G:K2R', 'Q9Q', 'R10W']
    subs = parse_mutations(WT, sets, 128, '# ')
    assert subs == [{}, {0: 'A'}, {3: 'G', 1: 'R'}, {8: 'Q'}, {9: 'W'}]
    rows = variant_rows(WT, subs, 128, '# ')
    expect = collate(['# ' + s for s in (WT, WT, 'AKTAYIAKQR', 'MRTGYIAKQR', WT, 'MKTAYIAKQW')], 128)
    np.testing.assert_array_equal(rows, expect)


def test_scan_sets():
    from progen_b200.variants import scan_sets, check_scan
    pos = check_scan(WT, [1, 4], 'AMG')
    sets, index = scan_sets(WT, pos, 'AMG')
    assert sets == ['M1A', 'M1G', 'A4M', 'A4G']
    np.testing.assert_array_equal(index, [[0, -1, 1], [-1, 2, 3]])
    np.testing.assert_array_equal(check_scan(WT, None, 'A'), np.arange(1, 11))


def test_parse_positions():
    from progen_b200.lib import ProgenError
    from progen_b200.variants import parse_positions
    assert parse_positions('1-3,7, 9-10', 10) == [1, 2, 3, 7, 9, 10]
    for bad in ('0-3', '5-4', '11', 'a', '1-2-3'):
        with pytest.raises(ProgenError):
            parse_positions(bad, 10)


@pytest.mark.parametrize('n', [128, 256, 1024])
def test_cut_length(n):
    """the counted positions are the non-pad labels and the first pad (quirk Q8); the cut rounds them up to 128"""
    from progen_b200.engine import counted_length, cut_length
    from progen_b200.data import collate
    for residues, need in ((0, 1), (1, 2), (126, 127), (127, 128), (128, 129), (n - 2, n - 1), (n - 1, n), (n, n),
                           (n + 5, n)):
        labels = collate(['A' * residues], n)[:, 1:]
        need = min(need, n)
        assert counted_length(labels)[0] == need, (residues, need)
        assert cut_length(labels) == min(n, -(-need // 128) * 128)
    labels = np.zeros((2, n), np.int64)
    labels[0, 5] = 3                                      # a non-pad label after pads still counts
    np.testing.assert_array_equal(counted_length(labels), [6, 1])
    assert cut_length(labels) == min(n, 128)
