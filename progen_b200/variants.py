"""Variant sets against a wild type: parsing and row building for `ProGen.score_variants` / `ProGen.mutational_scan`.

A mutation set is ProteinGym's `mutant` notation: substitutions `<wild-type letter><1-based position><new letter>` joined
by ':' (`"A23G"`, `"A23G:K45R"`), or `""` for the wild type itself.  Positions count residues of the wild type, not the
prefix in front of it.  Everything here runs on the host and raises ProgenError, naming the set, before any device work."""
import re

import numpy as np

from .data import collate
from .lib import ProgenError

AMINO_ACIDS = 'ACDEFGHIKLMNPQRSTVWY'
_SUB = re.compile(r'^(.)(\d+)(.*)$', re.S)


def _printable(c):
    return isinstance(c, str) and len(c) == 1 and c.isascii() and c.isprintable()


def check_sequence(s, what):
    """wild types and prefixes are ASCII strings: one byte, one token, one position"""
    if not isinstance(s, str) or not s.isascii():
        raise ProgenError(f'{what} must be an ASCII string, got {s!r}')
    return s


def parse_mutations(wild_type, mutations, seq_len, prefix=''):
    """-> list of {position (0-based residue index): new letter}, one per set, in order.  Rejects: an empty list, a set
    that is not a string, a substitution that does not parse, a wild-type letter that does not match, a position out of
    range or cut off by seq_len (collate keeps the first seq_len tokens of prefix + residues), the same position twice
    in one set, a new letter that is not one printable ASCII character.  Identity substitutions (A23A) are allowed."""
    check_sequence(wild_type, 'wild_type')
    check_sequence(prefix, 'prefix')
    if isinstance(mutations, str) or not isinstance(mutations, (list, tuple)) or len(mutations) == 0:
        raise ProgenError('mutations must be a non-empty list of mutation sets ("A23G", "A23G:K45R" or "" for the wild type)')
    kept = min(len(wild_type), seq_len - len(prefix))        # residues that fit in the row
    out = []
    for i, m in enumerate(mutations):
        where = f'mutation set {i} ({m!r})'
        if not isinstance(m, str):
            raise ProgenError(f'{where}: must be a string')
        subs = {}
        for sub in (m.strip().split(':') if m.strip() else []):
            match = _SUB.match(sub.strip())
            if not match:
                raise ProgenError(f'{where}: {sub!r} is not <wild-type letter><position><new letter>')
            old, pos, new = match.group(1), int(match.group(2)), match.group(3)
            if not 1 <= pos <= len(wild_type):
                raise ProgenError(f'{where}: position {pos} is out of range 1..{len(wild_type)}')
            if pos > kept:
                raise ProgenError(f'{where}: position {pos} is cut off by seq_len {seq_len} (prefix of {len(prefix)} '
                                  f'characters: residues 1..{kept} fit)')
            if wild_type[pos - 1] != old:
                raise ProgenError(f'{where}: the wild type has {wild_type[pos - 1]!r} at position {pos}, not {old!r}')
            if not _printable(new):
                raise ProgenError(f'{where}: the new residue {new!r} is not one printable ASCII character')
            if pos - 1 in subs:
                raise ProgenError(f'{where}: position {pos} is mutated twice')
            subs[pos - 1] = new
        out.append(subs)
    return out


def variant_rows(wild_type, subs, seq_len, prefix=''):
    """rows (1 + len(subs), seq_len + 1) uint16: the wild type, then each variant, as `collate([prefix + residues])`"""
    seqs = [prefix + wild_type]
    for s in subs:
        r = list(wild_type)
        for p, c in s.items():
            r[p] = c
        seqs.append(prefix + ''.join(r))
    return collate(seqs, seq_len)


def scan_sets(wild_type, positions, alphabet):
    """the single substitutions of a mutational scan -> (sets, index): sets in (position, letter) order without the
    identities, and index [P, |alphabet|] of each set's entry (-1 at the wild-type letter)"""
    index = np.full((len(positions), len(alphabet)), -1, np.int64)
    sets = []
    for i, p in enumerate(positions):
        for j, a in enumerate(alphabet):
            if a != wild_type[p - 1]:
                index[i, j] = len(sets)
                sets.append(f'{wild_type[p - 1]}{p}{a}')
    return sets, index


def check_scan(wild_type, positions, alphabet):
    """-> positions as a 1-based int64 array (default: every residue)"""
    check_sequence(wild_type, 'wild_type')
    if not isinstance(alphabet, str) or not alphabet or not all(_printable(c) for c in alphabet) \
            or len(set(alphabet)) != len(alphabet):
        raise ProgenError(f'alphabet must be a non-empty string of distinct printable ASCII characters, got {alphabet!r}')
    if positions is None:
        positions = range(1, len(wild_type) + 1)
    pos = list(positions)
    if not pos or not all(isinstance(p, (int, np.integer)) and not isinstance(p, (bool, np.bool_)) for p in pos):
        raise ProgenError('positions must be a non-empty list of 1-based residue positions')
    if len(set(int(p) for p in pos)) != len(pos):
        raise ProgenError('positions must not repeat')
    for p in pos:
        if not 1 <= p <= len(wild_type):
            raise ProgenError(f'position {p} is out of range 1..{len(wild_type)}')
    return np.asarray(pos, np.int64)


def parse_positions(spec, length):
    """'1-120,150,200-210' -> [1..120, 150, 200..210] (1-based, inclusive ranges)"""
    out = []
    for part in str(spec).split(','):
        part = part.strip()
        m = re.fullmatch(r'(\d+)(?:-(\d+))?', part)
        if not m:
            raise ProgenError(f'positions: {part!r} is not a position or a range a-b')
        a, b = int(m.group(1)), int(m.group(2) or m.group(1))
        if not 1 <= a <= b <= length:
            raise ProgenError(f'positions: {part!r} is not within 1..{length}')
        out.extend(range(a, b + 1))
    return out
