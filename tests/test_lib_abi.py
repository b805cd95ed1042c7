"""The C-ABI shared library: builds for sm_90a, loads without a GPU, exports every symbol include/quadswarm.h
declares, and the ctypes mirror of QsConfig matches the C layout.  No compute calls (CPU-only)."""
import ctypes
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, 'include', 'quadswarm.h')


@pytest.fixture(scope='module')
def lib():
    sys.path.insert(0, ROOT)
    import __graft_entry__ as g
    g.build()
    from quad_swarm_rl_b200 import _lib
    return _lib


def declared_symbols():
    text = open(HEADER).read()
    text = re.sub(r'/\*.*?\*/', '', text, flags=re.S)
    return sorted(set(re.findall(r'\b(qs_[a-z_]+)\s*\(', text)))


def test_library_exports_every_declared_symbol(lib):
    l = lib.load()
    names = declared_symbols()
    assert len(names) >= 20
    for n in names:
        assert hasattr(l, n), f'{n} declared in include/quadswarm.h but not exported'
        assert n in lib.EXPORTS, f'{n} has no ctypes prototype'


def test_qsconfig_layout_matches_c(lib, tmp_path):
    src = tmp_path / 'sz.c'
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "quadswarm.h"\nint main(){printf("%zu %zu %zu %zu\\n", '
                   'sizeof(QsConfig), offsetof(QsConfig, obst_size), offsetof(QsConfig, env_id_offset), offsetof(QsConfig, seed));return 0;}\n')
    exe = tmp_path / 'sz'
    subprocess.run(['gcc', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    c = lib.QsConfig
    assert [int(x) for x in out] == [ctypes.sizeof(c), c.obst_size.offset, c.env_id_offset.offset, c.seed.offset]


def test_error_path_without_gpu(lib):
    """qs_create validates its arguments before touching CUDA; a bad config must fail with a message, not crash."""
    l = lib.load()
    cfg = lib.QsConfig()
    cfg.num_envs, cfg.num_agents = 4, 33          # > QS_MAX_AGENTS
    h = ctypes.c_void_p()
    rc = l.qs_create(ctypes.byref(cfg), 0, ctypes.byref(h))
    assert rc == -2 and b'32' in l.qs_last_error()
    cfg.num_agents, cfg.neighbor_visible_num = 8, 9
    assert l.qs_create(ctypes.byref(cfg), 0, ctypes.byref(h)) == -1
    assert b'neigbors' in l.qs_last_error()


def test_product_never_imports_the_oracle():
    """The oracle is test infrastructure: nothing under quad_swarm_rl_b200/ may import it."""
    pkg = os.path.join(ROOT, 'quad_swarm_rl_b200')
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith('.py'):
                text = open(os.path.join(dirpath, f)).read()
                assert not re.search(r'^\s*(from|import)\s+oracle\b', text, flags=re.M), f


def test_integration_doc_binding_matches_the_header():
    """The ctypes stub shown in INTEGRATION.md must list QsConfig's fields in the header's order (a stale stub would
    silently shift every field after the change)."""
    import re
    from quad_swarm_rl_b200 import _lib as L
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    md = open(os.path.join(root, 'INTEGRATION.md')).read()
    block = md[md.index('class QsConfig(C.Structure)'):]
    block = block[:block.index(']\n') + 1]
    doc_fields = re.findall(r'\("(\w+)",', block)
    assert doc_fields == [f[0] for f in L.QsConfig._fields_]
    hdr = open(os.path.join(root, 'include', 'quadswarm.h')).read()
    struct = hdr[hdr.index('typedef struct QsConfig {'):hdr.index('} QsConfig;')]
    hdr_fields = re.findall(r'^\s+(?:int32_t|float|uint64_t)\s+(\w+)', struct, flags=re.M)
    assert hdr_fields == doc_fields
