"""CPU-side checks of the drop-in boundary: the C-ABI library builds, loads, and exports exactly the entry points that
include/progen_b200.h declares (no compute is launched without a GPU)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def lib():
    from progen_b200 import lib as L
    if not os.path.exists(L.LIB_PATH):
        import __graft_entry__ as G
        G.build()
    return L


def header_functions():
    src = open(os.path.join(ROOT, 'include', 'progen_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return set(re.findall(r'\b(progen_[a-z0-9_]+)\s*\(', src))


def test_library_exports_every_declared_symbol(lib):
    handle = lib.load()
    declared = header_functions()
    assert declared, 'no declarations parsed from include/progen_b200.h'
    for name in declared:
        assert hasattr(handle, name), f'{name} declared in the header but not exported by the .so'
    assert declared == set(lib.PROTOTYPES), (declared ^ set(lib.PROTOTYPES))


def test_version_and_error_text(lib):
    assert 'sm_90a' in lib.version()
    assert lib.load().progen_last_error() is not None


def test_product_has_no_oracle_or_cpu_fallback():
    """The product path must not import the oracle and must fail loudly without a GPU."""
    import torch
    pkg = os.path.join(ROOT, 'progen_b200')
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith('.py'):
                text = open(os.path.join(dirpath, f)).read()
                assert not re.search(r'^\s*(from|import)\s+\.*oracle', text, flags=re.M), f'{f} imports the oracle'
                assert 'progen_ref' not in text and 'progen_torch' not in text, f'{f} references the oracle'
    if not torch.cuda.is_available():
        from progen_b200 import lib as L
        with pytest.raises(L.ProgenError):
            L.require_device()


def test_ctypes_mirrors_match_the_header_layout(tmp_path):
    """Every ctypes mirror of a C-ABI struct has the size and the field offsets gcc gives the declaration in
    include/progen_b200.h (a field added on one side only would shift every pointer after it)."""
    import ctypes as C
    import shutil
    import subprocess
    from progen_b200 import lib as L
    from progen_b200 import decode as D
    if shutil.which('gcc') is None:
        pytest.skip('no gcc')
    pairs = [('progen_gemm_t', L.GemmDesc), ('progen_decode_layer_t', D.DecodeLayer), ('progen_decode_run_t', D.DecodeRun)]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "progen_b200.h"', 'int main(void) {']
    for cname, cls in pairs:
        lines.append(f'  printf("{cname} size %zu\\n", sizeof({cname}));')
        for fname, _ in cls._fields_:
            lines.append(f'  printf("{cname} {fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ['  return 0;', '}']
    src = tmp_path / 'layout.c'
    src.write_text('\n'.join(lines))
    exe = tmp_path / 'layout'
    inc = os.path.join(ROOT, 'include')
    subprocess.run(['gcc', '-std=c11', '-I', inc, str(src), '-o', str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    want = {}
    for ln in out.strip().splitlines():
        c, f, v = ln.split()
        want[(c, f)] = int(v)
    for cname, cls in pairs:
        assert C.sizeof(cls) == want[(cname, 'size')], cname
        for fname, _ in cls._fields_:
            assert getattr(cls, fname).offset == want[(cname, fname)], (cname, fname)
