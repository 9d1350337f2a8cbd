"""CPU: which need set each interaction layer's receptor <- receptor group is restricted to (CGModel._need_levels), and the
ctypes bindings of the need-set and edge-selection entry points against their declarations in include/diffdock_b200.h."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("L,shared,want", [
    (6, False, [5, 4, 3, 2, 1, None]),
    (6, True, [None, 4, 3, 2, 1, None]),        # layer 0 keeps the messages shared across copies of a receptor
    (3, False, [2, 1, None]),
    (2, False, [1, None]),
    (2, True, [None, None]),
    (1, False, [None]),                          # the only layer is the last one: it has no receptor <- receptor group
])
def test_need_levels(L, shared, want):
    from diffdock_b200.cg_model import CGModel
    assert CGModel._need_levels(None, L, shared) == want


@pytest.mark.parametrize("name", ['ddb200_crop_select_edges', 'ddb200_receptor_need'])
def test_bindings_match_header(name):
    from diffdock_b200._lib import SIGNATURES
    with open(os.path.join(ROOT, 'include', 'diffdock_b200.h')) as f:
        text = f.read()
    decl = re.search(r'int ' + name + r'\(([^)]*)\);', text)
    assert decl, name
    params = [p.strip() for p in decl.group(1).split(',')]
    argtypes = SIGNATURES[name][1]
    assert len(params) == len(argtypes)
    for p, a in zip(params, argtypes):
        kind = 'ptr' if '*' in p else ('i64' if p.startswith('int64_t') else 'i32')
        assert a.__name__ == {'ptr': 'c_void_p', 'i64': 'c_long', 'i32': 'c_int'}[kind] or \
            (kind == 'i64' and a.__name__ == 'c_longlong'), (p, a)
