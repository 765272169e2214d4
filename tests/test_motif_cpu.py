"""Motif constraints on the host (progen_b200/motif.py): the PROSITE parser and its refusals, the state machine against an
independent translation to Python `re`, the required pattern's lookahead against brute-force enumeration, refusals of
`ProGen.generate(require=, avoid=)` and generate.py before anything needs a device, and the descriptor's C layout."""
import itertools
import os
import re
import shutil
import subprocess
import sys
import zlib

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KW = dict(num_tokens=256, dim=64, seq_len=64, depth=2, window_size=16, global_mlp_depth=1, heads=2, dim_head=32)

ZINC_FINGER = 'C-x(2,4)-C-x(3)-[LIVMFYWC]-x(8)-H-x(3,5)-H'     # PS00028
P_LOOP = '[AG]-x(4)-G-K-[ST]'                                 # PS00017
GLYCOSYLATION = 'N-{P}-[ST]-{P}'


def to_regex(pattern):
    """the independent translation: x -> ., {..} -> [^..], (n,m) -> {n,m}, < / > -> ^ / $ (letters are characters)"""
    p = pattern.strip()
    p = p[:-1] if p.endswith('.') else p
    out = ''
    for el in p.split('-'):
        pre = '^' if el.startswith('<') else ''
        post = '$' if el.endswith('>') else ''
        el = el.strip('<>')
        m = re.match(r'^(x|[A-Z]|\[[A-Z]+\]|\{[A-Z]+\})(?:\((\d+)(?:,(\d+))?\))?$', el)
        sym = {'x': '.'}.get(m[1], m[1])
        if sym.startswith('{'):
            sym = '[^' + sym[1:-1] + ']'
        rep = '' if m[2] is None else ('{%s}' % m[2] if m[3] is None else '{%s,%s}' % (m[2], m[3]))
        out += pre + sym + rep + post
    return re.compile(out, re.DOTALL)


def enc(s):
    return np.array([ord(ch) + 1 for ch in s], np.int64)


@pytest.mark.parametrize('text', [ZINC_FINGER, P_LOOP, GLYCOSYLATION, '<M-x(3)-[KR]', 'G(2,3)-x(0,2)-C>', 'C-x(2,4)-C.'])
def test_parser_accepts_prosite_patterns(text):
    from progen_b200.motif import Pattern
    p = Pattern(text, 256)
    assert p.m <= 64 and not p.optional.all()
    assert p.anchored_start == ('<' in text) and p.anchored_end == ('>' in text)


def test_parser_expands_repeats():
    from progen_b200.motif import Pattern
    p = Pattern(ZINC_FINGER, 256)
    assert p.m == 1 + 4 + 1 + 3 + 1 + 8 + 1 + 5 + 1
    assert p.optional.sum() == 4 and p.optional[3] and p.optional[4] and p.optional[-2] and p.optional[-3]
    assert p.classes[0].sum() == 1 and p.classes[1].sum() == 255 and not p.classes[1][0]
    g = Pattern(GLYCOSYLATION, 256)
    assert g.classes[1].sum() == 254 and not g.classes[1][ord('P') + 1]


@pytest.mark.parametrize('text,words', [
    ('C-[G>]', 'inside brackets'),
    ('C-{A>}-G', 'inside brackets'),
    ('C-<G', 'anchors'),
    ('C>-G', 'anchors'),
    ('A-x(3,2)', 'n > m'),
    ('A-x(0)', 'zero'),
    ('x(0,3)', 'mandatory'),
    ('A-b-C', 'element'),
    ('A--C', 'element'),
    ('', 'empty'),
    ('[]-A', 'element'),
    ('x(65)', 'positions'),
])
def test_parser_refusals_name_the_pattern_and_reason(text, words):
    from progen_b200.motif import Pattern
    from progen_b200.lib import ProgenError
    with pytest.raises(ProgenError) as e:
        Pattern(text, 256)
    assert repr(text) in str(e.value) and words in str(e.value), str(e.value)


def test_letters_outside_the_vocabulary():
    from progen_b200.motif import Pattern
    from progen_b200.lib import ProgenError
    with pytest.raises(ProgenError, match='vocabulary'):
        Pattern('A-W', 70)                               # 'W' encodes to 88
    Pattern('A-B', 70)


MATCHER_PATTERNS = ['A-x(2,4)-C', 'A-[CG]-x(0,2)-A', '<C-x(3)-[AG]', 'G(2,3)-x(0,2)-C>', '<A-x(1,3)-C>', 'A-{C}-[AG]-{A}',
                    'C-x(2,4)-C.', '[AC]-x(0,3)-G-x(1,2)-A', 'x(0,2)-A-C', 'A-C-x(0,1)', '<x(0,2)-G-A', 'C-G-A-C-G',
                    '{A}(2,3)-A>']


@pytest.mark.parametrize('text', MATCHER_PATTERNS)
def test_matcher_agrees_with_python_re(text):
    """10^4 random strings per pattern over small alphabets (matches are common), with and without the pattern"""
    from progen_b200.motif import Motif
    rx = to_regex(text)
    rng = np.random.default_rng(zlib.crc32(text.encode()))
    alphabet = np.array(list('ACG'))
    strings = [''.join(rng.choice(alphabet, int(rng.integers(0, 14)))) for _ in range(10000)]
    rows = [enc(s) for s in strings]
    want = np.array([rx.search(s) is not None for s in strings])
    assert 0.01 < want.mean() < 0.99, want.mean()
    np.testing.assert_array_equal(Motif(text, None, 256).matches(rows), want)
    np.testing.assert_array_equal(Motif(None, text, 256).matches(rows), ~want)


def test_required_and_avoided_together():
    from progen_b200.motif import Motif
    m = Motif('C-x(2,4)-C', ['N-{P}-[ST]-{P}', 'W-W'], 256)
    got = m.matches([enc(s) for s in ('AACAACAA', 'CAAAAAC', 'CAACNASA', 'CAACWW', 'CAACNAS', '')])
    np.testing.assert_array_equal(got, [True, False, False, False, True, False])


LOOKAHEAD_PATTERNS = ['A-x(1,3)-C', '<G-x(0,2)-A>', '[AC]-{G}-x(2)-G', 'C-x(0,2)-C-A', 'G(2,3)-x(0,2)-C>', 'x(0,2)-A-C']


@pytest.mark.parametrize('text', LOOKAHEAD_PATTERNS)
def test_lookahead_equals_brute_force(text):
    """for random prefixes and budgets r over a short alphabet: some completion of <= r residues gives a string that
    satisfies the requirement  <=>  the state's lookahead <= r"""
    from progen_b200.motif import Motif
    V = 256
    alphabet = 'ACG'
    bias = np.full(V, -np.inf, np.float32)
    bias[0] = 0.0
    bias[enc(alphabet)] = 0.0
    m = Motif(text, None, V, bias)
    p = m.patterns[0]
    rx = to_regex(text)
    rng = np.random.default_rng(zlib.crc32(text.encode()))
    ok_count = checked = 0
    for _ in range(150):
        prefix = ''.join(rng.choice(list(alphabet), int(rng.integers(0, 7))))
        D, met = np.uint64(0), False
        for j, ch in enumerate(prefix):
            D = p.step(D, enc(ch)[0], j == 0)
            hit = bool(D & p.last)
            met = (met and not p.anchored_end) or hit
        assert met == (rx.search(prefix) is not None), prefix
        la = p.lookahead(m.need, D, met, len(prefix) == 0)
        for r in range(5):
            some = any(rx.search(prefix + ''.join(c)) is not None
                       for k in range(r + 1) for c in itertools.product(alphabet, repeat=k))
            assert some == (la <= r), (prefix, r, la)
            ok_count += some
            checked += 1
    assert 0 < ok_count < checked


def test_need_uses_the_logit_bias_bans():
    from progen_b200.motif import Motif, MAX_POSITIONS
    from progen_b200.lib import ProgenError
    bias = np.zeros(256, np.float32)
    bias[ord('W') + 1] = -np.inf
    m = Motif('A-[CW]-x(0,2)-G', None, 256, bias)
    assert m.shortest == 3 and m.need[MAX_POSITIONS] == 3
    with pytest.raises(ProgenError, match='mandatory position 2'):
        Motif('A-W-G', None, 256, bias)
    Motif(None, 'A-W-G', 256, bias)                      # an avoided pattern that cannot occur is harmless


@pytest.mark.parametrize('kwargs', [
    dict(require='C-x(2,4)-C', avoid=['A'] * 9),         # more than 8 avoided patterns
    dict(require=['C-x(2,4)-C', 'A']),                   # several required patterns
    dict(require='C-[G>]'),
    dict(avoid='C-<G'),
    dict(require='A-x(3,2)'),
    dict(require=5),
    dict(require='x(60)-A', max_length=40),              # longer than any row
    dict(require='x(30)-A', max_length=33),              # fits the empty prompt (32 positions), not 'MK' (30)
    dict(require='A-W-C', logit_bias=np.where(np.arange(256) == ord('W') + 1, -np.inf, 0).astype(np.float32)),
])
def test_motif_refusals_without_a_device(kwargs):
    from progen_b200 import ProGen
    from progen_b200.lib import ProgenError
    model = ProGen(**KW)
    with pytest.raises(ProgenError):
        model.generate({}, ['', 'MK'], **kwargs)
    assert model._engine is None and model._gen_decoder is None


def test_reach_refusal_names_the_prompt():
    from progen_b200 import ProGen
    from progen_b200.lib import ProgenError
    with pytest.raises(ProgenError, match='prompt 1'):
        ProGen(**KW).generate({}, ['', 'MKVLA'], require='x(10)-A', max_length=16)


@pytest.fixture(scope='module')
def ckpt(tmp_path_factory):
    from progen_b200.checkpoint import file_save_checkpoint
    from progen_b200 import ProGen
    d = tmp_path_factory.mktemp('motif_ckpt') / 'ckpts'
    d.mkdir()
    file_save_checkpoint(d, dict(next_seq_index=0, params=ProGen(**KW).init(1), optim_state=None, model_config=KW,
                                 run_id=None))
    return d


@pytest.mark.parametrize('args,words', [
    (['--require', 'C-[G>]'], 'inside brackets'),
    (['--require', 'A-x', '--require', 'C-x'], '--require'),
    (['--avoid', 'A-x(3,2)'], 'n > m'),
    (['--require', 'x(70)'], 'positions'),
    (['--require', 'A-W', '--alphabet', 'ACDEFG'], 'mandatory position 2'),
])
def test_cli_refuses_bad_patterns(ckpt, tmp_path, args, words):
    out = tmp_path / 'x.fasta'
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'generate.py'), '--checkpoint_path', str(ckpt),
                        '--output', str(out)] + args,
                       cwd=str(tmp_path), env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=600)
    assert r.returncode != 0
    assert 'ProgenError' in r.stderr and words in r.stderr and 'Traceback' not in r.stderr, r.stderr[-2000:]
    assert not out.exists()


def test_motif_descriptor_matches_the_header_layout(tmp_path):
    """the ctypes mirrors of progen_motif_t / progen_motif_pattern_t have gcc's size and field offsets"""
    import ctypes as C
    from progen_b200 import decode as D
    if shutil.which('gcc') is None:
        pytest.skip('no gcc')
    pairs = [('progen_motif_pattern_t', D.MotifPattern), ('progen_motif_t', D.MotifDesc),
             ('progen_decode_run_t', D.DecodeRun)]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "progen_b200.h"', 'int main(void) {']
    for cname, cls in pairs:
        lines.append(f'  printf("{cname} size %zu\\n", sizeof({cname}));')
        for fname, _ in cls._fields_:
            lines.append(f'  printf("{cname} {fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ['  return 0;', '}']
    src = tmp_path / 'layout.c'
    src.write_text('\n'.join(lines))
    exe = tmp_path / 'layout'
    subprocess.run(['gcc', '-std=c11', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)], check=True)
    want = {}
    for ln in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.strip().splitlines():
        c, f, v = ln.split()
        want[(c, f)] = int(v)
    for cname, cls in pairs:
        assert C.sizeof(cls) == want[(cname, 'size')], cname
        for fname, _ in cls._fields_:
            assert getattr(cls, fname).offset == want[(cname, fname)], (cname, fname)
    assert D.DecodeRun.motif.offset == C.sizeof(D.DecodeRun) - 8


def test_descriptor_arrays():
    from progen_b200.motif import Motif
    m = Motif('<M-x(0,2)-K', ['G-G>'], 256)
    mask, pat, need = m.descriptor_arrays()
    assert mask.shape == (2, 256) and mask.dtype == np.uint64
    assert mask[0, ord('M') + 1] & 1 and mask[0, ord('K') + 1] == (2 | 4 | 8) and mask[0, 0] == 0
    assert [int(v) for v in pat[0]] == [0b0110, 0, 1 << 3, 1] and [int(v) for v in pat[1]] == [0, 0, 2, 2]
    assert need.dtype == np.int32 and need[64] == 2 and need[0] == 1 and need[3] == 0
