"""Sequence motifs for `ProGen.generate(require=, avoid=)`: PROSITE patterns compiled to the bit-parallel state machine
that the standard sampler of csrc/decode_persist.cu runs per row (`progen_motif_t` in include/progen_b200.h,
DESIGN.md §3.3 "Motif constraints").

A pattern is a sequence of up to MAX_POSITIONS positions, each a set of ids (its class) and mandatory or optional.  A
row's state per pattern is a bitset D: bit i is set when positions 0..i match a suffix of the generated tokens read so far
(optional positions may be skipped).  This is the shift-and automaton with character classes and optional positions of
Navarro & Raffinot (J. Comput. Biol. 10(6), 2003), which was designed for PROSITE.  Reading id c:

    z   = the start state is active: always, or only at the first generated token for a '<'-anchored pattern
    D'  = closure((((D | (lead if z)) << 1) | z) & mask[c])

where lead is the closure of the start state (its leading optional positions) and closure(X) repeats
X |= (X << 1) & optional until nothing changes.  The pattern has matched when the bit of its last position is set; for a
'>'-anchored pattern only after the row's last token counts."""
import re

import numpy as np

from . import lib as L

MAX_POSITIONS = 64                 # positions of one pattern after expanding repeats: one uint64 bitset
MAX_AVOID = 8
INF = 1 << 30                      # the lookahead of a state that cannot complete the required pattern
_U64 = np.uint64
_ELEMENT = re.compile(r'^(x|[A-Z]|\[[A-Z]+\]|\{[A-Z]+\})(?:\((\d+)(?:,(\d+))?\))?$')


class Pattern:
    """One parsed PROSITE pattern: classes [m, V] bool, optional [m] bool, anchored_start / anchored_end."""

    def __init__(self, text, V):
        from .data import encode_tokens
        if not isinstance(text, str):
            raise L.ProgenError(f'motif {text!r}: a pattern must be a string')
        self.text = text
        fail = lambda why: L.ProgenError(f'motif {text!r}: {why}')
        body = text.strip()
        if body.endswith('.'):
            body = body[:-1]
        self.anchored_start = body.startswith('<')
        self.anchored_end = body.endswith('>')
        body = body[1 if self.anchored_start else 0:len(body) - (1 if self.anchored_end else 0)]
        if not body:
            raise fail('empty pattern')
        if re.search(r'\[[^\]]*>|\{[^}]*>', text):
            raise fail("'>' inside brackets is not supported")
        if '<' in body or '>' in body:
            raise fail("anchors '<' and '>' may only start and end the pattern")
        classes, optional = [], []
        for el in body.split('-'):
            m = _ELEMENT.match(el)
            if m is None:
                raise fail(f'element {el!r} is not a letter, x, [..] or {{..}} with an optional (n) or (n,m) repeat')
            sym, lo = m.group(1), m.group(2)
            n = 1 if lo is None else int(lo)
            hi = n if m.group(3) is None else int(m.group(3))
            if n > hi:
                raise fail(f'element {el!r} has n > m in its repeat')
            if hi == 0:
                raise fail(f'element {el!r} repeats zero times')
            cls = np.zeros(V, bool)
            letters = sym.strip('[]{}') if sym != 'x' else ''
            ids = encode_tokens(letters)
            bad = [ch for ch, c in zip(letters, ids) if not 1 <= c < V]
            if bad:
                raise fail(f'letters {bad!r} are outside the {V}-token vocabulary')
            if sym == 'x':
                cls[1:] = True
            elif sym.startswith('{'):
                cls[1:] = True
                cls[ids] = False
            else:
                cls[ids] = True
            classes += [cls] * hi
            optional += [False] * n + [True] * (hi - n)
        if len(classes) > MAX_POSITIONS:
            raise fail(f'{len(classes)} positions after expanding repeats (at most {MAX_POSITIONS})')
        self.classes = np.stack(classes)
        self.optional = np.asarray(optional, bool)
        if self.optional.all():
            raise fail('the pattern needs at least one mandatory position')
        self.m = len(classes)
        bits = _U64(1) << np.arange(self.m, dtype=_U64)
        self.mask = (self.classes.T.astype(_U64) * bits[None, :]).sum(axis=1, dtype=_U64)    # [V]: positions id c matches
        self.opt_bits = _U64(int((self.optional.astype(_U64) * bits).sum(dtype=_U64)))
        j = int(np.argmin(self.optional))                                                     # first mandatory position
        self.lead = _U64((1 << j) - 1)
        self.last = _U64(1 << (self.m - 1))

    def closure(self, X):
        X = np.asarray(X, _U64)
        while True:
            Y = X | ((X << _U64(1)) & self.opt_bits)
            if np.array_equal(Y, X):
                return Y
            X = Y

    def step(self, D, c, first):
        """next states after ids c (arrays over rows); first: c is the row's first generated token"""
        z = np.logical_or(not self.anchored_start, first)
        act = np.asarray(D, _U64) | np.where(z, self.lead, _U64(0))
        return self.closure(((act << _U64(1)) | z.astype(_U64)) & self.mask[np.asarray(c, np.int64)])

    def need(self, allowed):
        """[65] int64: the fewest residues (ids of `allowed`, a [V] bool mask) that complete the pattern from the state
        of bit i (need[64]: from the start state alone), INF where none do.  It never increases along the pattern, so
        the lookahead of a state D is need[msb(D)]."""
        nonempty = (self.classes & allowed[None, :]).any(axis=1)
        out = np.full(MAX_POSITIONS + 1, INF, np.int64)
        s = 0                                              # from the state after the last position (bit m - 1)
        out[self.m - 1] = 0
        for i in range(self.m - 1, -1, -1):               # the state before position i: bit i - 1, or the start
            s = min(s if self.optional[i] else INF, s + 1 if nonempty[i] else INF, INF)
            out[i - 1 if i > 0 else MAX_POSITIONS] = s
        return out

    def lookahead(self, need, D, met, first):
        """fewest residues after the current state (D, met) that satisfy the pattern; first: no token generated yet"""
        if met:
            return 0
        D = int(D)
        if D:
            return int(need[D.bit_length() - 1])
        return int(need[MAX_POSITIONS]) if (first or not self.anchored_start) else INF


class Motif:
    """The compiled patterns of one generate call: pattern 0 is the required one when `required`, the rest are
    avoided.  `descriptor_arrays` gives what the kernel reads; `matches` replays the rows on the host."""

    def __init__(self, require, avoid, V, logit_bias=None):
        if isinstance(avoid, str):
            avoid = [avoid]
        avoid = [] if avoid is None else list(avoid)
        if len(avoid) > MAX_AVOID:
            raise L.ProgenError(f'generate: at most {MAX_AVOID} avoided patterns, got {len(avoid)}')
        self.required = require is not None
        self.patterns = ([Pattern(require, V)] if self.required else []) + [Pattern(a, V) for a in avoid]
        self.V = V
        allowed = np.ones(V, bool)
        if logit_bias is not None:
            allowed = np.isfinite(np.asarray(logit_bias, np.float32))
        allowed[0] = False
        self.need = np.full(MAX_POSITIONS + 1, INF, np.int64)
        if self.required:
            p = self.patterns[0]
            empty = [i for i in range(p.m) if not p.optional[i] and not (p.classes[i] & allowed).any()]
            if empty:
                raise L.ProgenError(f'motif {p.text!r}: mandatory position {empty[0] + 1} has no residue left once '
                                    'logit_bias (the alphabet) is applied')
            self.need = p.need(allowed)

    @property
    def shortest(self):
        """residues in the shortest completion of the required pattern (0 without one)"""
        return int(self.need[MAX_POSITIONS]) if self.required else 0

    def check_reach(self, starts, max_length):
        """ProgenError naming the first prompt whose generated positions (max_length - start) cannot hold the
        required pattern"""
        for i, s in enumerate(starts):
            if self.shortest > max_length - int(s):
                raise L.ProgenError(f'generate: prompt {i} leaves {max_length - int(s)} positions before max_length '
                                    f'{max_length}, fewer than the {self.shortest} residues of the shortest match of '
                                    f'{self.patterns[0].text!r}')

    def descriptor_arrays(self):
        """-> (mask [P, V] uint64, per-pattern [P, 4] uint64 = (optional, lead, last, anchors), need [65] int32)"""
        mask = np.stack([p.mask for p in self.patterns])
        pat = np.array([[int(p.opt_bits), int(p.lead), int(p.last), int(p.anchored_start) | int(p.anchored_end) << 1]
                        for p in self.patterns], _U64)
        return mask, pat, np.minimum(self.need, INF).astype(np.int32)

    def initial_state(self):
        """a row's state before its first generated token: (D of every pattern, required pattern met)"""
        return [_U64(0)] * len(self.patterns), False

    def _next(self, state, ids, first):
        """[P, len(ids)] next bitsets and [len(ids)] met flags after each id of `ids`"""
        D, met = state
        X = np.stack([p.step(np.full(len(ids), D[k], _U64), ids, first) for k, p in enumerate(self.patterns)])
        new_met = np.zeros(len(ids), bool)
        if self.required:
            p = self.patterns[0]
            new_met = (met and not p.anchored_end) | ((X[0] & p.last) != 0)
        return X, new_met

    def banned(self, state, first, left):
        """[V] bool: the ids the kernel bans for a row in `state` whose draw is its first generated token (`first`) and
        leaves `left` positions after it before max_length"""
        ids = np.arange(self.V)
        X, met = self._next(state, ids, first)
        ban = np.zeros(self.V, bool)
        for k, p in enumerate(self.patterns):
            hit = (X[k] & p.last) != 0
            if k == 0 and self.required:
                msb = np.full(self.V, -1, np.int64)
                for i in range(p.m):
                    msb = np.where((X[0] >> _U64(i)) & _U64(1) != 0, i, msb)
                la = np.where(msb >= 0, self.need[np.maximum(msb, 0)], INF if p.anchored_start else self.need[MAX_POSITIONS])
                ban |= ~met & (la > left)
            else:
                ban |= hit & ((not p.anchored_end) or left == 0)
        D, met0 = state
        ban[0] = (self.required and not met0) or any(p.anchored_end and (D[k] & p.last) != 0 for k, p in
                                                     enumerate(self.patterns) if not (k == 0 and self.required))
        return ban

    def advance(self, state, c, first):
        """the state after a row draws residue c"""
        X, met = self._next(state, np.array([c]), first)
        return [X[k, 0] for k in range(len(self.patterns))], bool(met[0])

    def matches(self, rows):
        """rows: a list of 1-D id arrays, each a row's generated tokens t_1..t_L (no EOS).  -> [N] bool: the required
        pattern occurs and no avoided one does"""
        N = len(rows)
        Lmax = max((len(r) for r in rows), default=0)
        lens = np.array([len(r) for r in rows], np.int64)
        tok = np.zeros((N, Lmax), np.int64)
        for i, r in enumerate(rows):
            tok[i, :len(r)] = r
        ok = np.ones(N, bool)
        for k, p in enumerate(self.patterns):
            D = np.zeros(N, _U64)
            hit = np.zeros(N, bool)
            for j in range(Lmax):
                live = j < lens
                Dn = p.step(D, tok[:, j], j == 0)
                D = np.where(live, Dn, D)
                done = live & ((Dn & p.last) != 0)
                hit |= done & ((j == lens - 1) | (not p.anchored_end))
            ok &= hit if (k == 0 and self.required) else ~hit
        return ok
