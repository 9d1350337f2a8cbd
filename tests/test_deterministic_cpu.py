"""CPU: the deterministic (fixed-point) convolutions.  Their header (include/diffdock_b200_fixed.h) against the ctypes
table (diffdock_b200/_lib.py:FIXED_SIGNATURES) and the library's exports; their machine code (tools/sass_histogram.py):
the fixed-point fused instantiations keep one wgmma chain per staged k-block and reduce into the sums with 64-bit integer
REDs only; and a restatement of the conversion, saturation and epilogue arithmetic, which tests/test_deterministic_gpu.py
uses as its oracle."""
import os
import re
import shutil
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tools'))

SCALE = 2.0 ** 32
I64_MAX = 2 ** 63 - 1
EPS = np.float32(1.1920928955078125e-07)


# ------------------------------------------------------------------------------------------ restated arithmetic
def to_fixed(v):
    """int64 fixed point of fp32 values: round half to even of v * 2^32 (exact in float64); |v| >= 2^31 and non-finite
    values saturate to +-(2^63 - 1) (NaN: 0).  Returns (q, saturated?)."""
    v = np.asarray(v, dtype=np.float32).astype(np.float64) * SCALE
    bad = ~(np.abs(v) < 2.0 ** 63)
    q = np.rint(np.where(bad, 0.0, v)).astype(np.int64)
    q = np.where(bad & (v > 0), I64_MAX, np.where(bad & (v < 0), -I64_MAX, q))
    return q, bool(bad.any())


def restated_fixed_sum(m, tgt, n_out):
    """The int64 sums [n_out, d] of per-edge fp32 messages m [E, d] scattered to tgt [E] (wrapping, as the device adds)."""
    q, _ = to_fixed(m)
    out = np.zeros((n_out, q.shape[1]), dtype=np.int64)
    np.add.at(out, np.asarray(tgt, dtype=np.int64), q)
    return out


def restated_finalize(s, cnt, mean, scale, shift, residual):
    """ddb200_tpconv_finalize_fixed: (double) sum * 2^-32 (/ max(cnt, eps)) rounded once to fp32, then fmaf(v, scale,
    shift) and the residual added in fp32."""
    v = np.asarray(s, dtype=np.int64).astype(np.float64) / SCALE
    if mean:
        v = v / np.maximum(np.asarray(cnt, dtype=np.float32), EPS).astype(np.float64)[:, None]
    v = v.astype(np.float32)
    if scale is not None:
        v = (v.astype(np.float64) * np.asarray(scale, np.float32) + np.asarray(shift, np.float32)).astype(np.float32)
    if residual is not None:
        r = np.asarray(residual, np.float32)
        v[:, :r.shape[1]] = v[:, :r.shape[1]] + r
    return v


def test_conversion_rounds_to_nearest_even_and_saturates():
    q, sat = to_fixed([0.0, 1.0, -1.0, 2.0 ** -33, 3 * 2.0 ** -33, -(2.0 ** -33), 2.0 ** 31 - 128, 0.5])
    assert not sat
    assert q.tolist() == [0, 2 ** 32, -(2 ** 32), 0, 2, 0, (2 ** 31 - 128) * 2 ** 32, 2 ** 31]
    for bad in (2.0 ** 31, -(2.0 ** 31), np.inf, np.nan, 1e30):
        q, sat = to_fixed([bad])
        assert sat and abs(int(q[0])) in (I64_MAX, 0)


def test_integer_sums_do_not_depend_on_order_but_float_sums_do():
    g = np.random.default_rng(0)
    m = (g.standard_normal((4000, 3)) * np.exp(g.uniform(-8, 8, (4000, 1)))).astype(np.float32)
    tgt = g.integers(0, 7, 4000)
    perm = g.permutation(4000)
    assert np.array_equal(restated_fixed_sum(m, tgt, 7), restated_fixed_sum(m[perm], tgt[perm], 7))
    f = lambda mm, tt: np.stack([np.cumsum(mm[tt == k], 0, dtype=np.float32)[-1] for k in range(7)])
    assert not np.array_equal(f(m, tgt), f(m[perm], tgt[perm]))        # why the float scatter is not reproducible
    exact = np.zeros((7, 3))
    np.add.at(exact, tgt, m.astype(np.float64))
    assert np.abs(restated_fixed_sum(m, tgt, 7) / SCALE - exact).max() <= 4000 * 2.0 ** -33


def test_epilogue_rounds_once():
    s = np.array([[3 * 2 ** 32 + 1, -(2 ** 40)]], dtype=np.int64)
    got = restated_finalize(s, np.array([3.0], np.float32), True, None, None, None)
    assert got.dtype == np.float32
    assert got[0, 0] == np.float32((3 * 2 ** 32 + 1) / SCALE / 3) and got[0, 1] == np.float32(-(2.0 ** 8) / 3)
    got = restated_finalize(s, np.array([0.0], np.float32), True, None, None, None)      # no edge: max(cnt, eps)
    assert got[0, 0] == np.float32((3 * 2 ** 32 + 1) / SCALE / np.float64(EPS))


# ------------------------------------------------------------------------------------------------------- C ABI
def test_header_declares_the_ctypes_table(built_lib):
    import ctypes as C
    from diffdock_b200 import _lib
    hdr = open(os.path.join(ROOT, 'include', 'diffdock_b200_fixed.h')).read()
    decls = {m.group(1): m.group(2) for m in re.finditer(r'\bint\s+(ddb200_\w+)\s*\(([^;]*)\)\s*;', hdr)}
    assert sorted(decls) == sorted(_lib.FIXED_SIGNATURES)
    ctype = {'int64_t': C.c_int64, 'int': C.c_int, 'int32_t': C.c_int32}
    for name, params in decls.items():
        args = [a.strip() for a in params.replace('\n', ' ').split(',')]
        res, want = _lib.FIXED_SIGNATURES[name]
        assert res is C.c_int and len(args) == len(want), name
        for a, w in zip(args, want):
            t = ' '.join(a.split()[:-1])
            assert (w is C.c_void_p) if '*' in t else ctype[t.replace('const ', '')] is w, (name, a)
        assert getattr(built_lib, name) is not None
    main = open(os.path.join(ROOT, 'include', 'diffdock_b200.h')).read()
    assert not set(decls) & set(re.findall(r'\b(ddb200_\w+)\s*\(', main))
    assert not set(decls) & set(_lib.SIGNATURES)


# ---------------------------------------------------------------------------------------------------------- SASS
@pytest.fixture(scope='module')
def sass(built_lib):
    if shutil.which('cuobjdump') is None:
        pytest.skip('cuobjdump not on PATH')
    import sass_histogram as sh
    return sh.kernels(os.path.join(ROOT, 'diffdock_b200', 'libdiffdock_b200.so'), operands=True)


def _kernel(sass, name):
    hits = [v for k, v in sass.items() if re.search(rf'\d{name}E', k)]          # mangled: <length><name>E<params>
    assert len(hits) == 1, name
    return hits[0]


FUSED = ('fused_conv_kernel', 'fused_conv_kernel_so', 'fused_conv_fixed_kernel', 'fused_conv_fixed_kernel_so')


@pytest.mark.parametrize('name', FUSED)
def test_every_fused_instantiation_issues_one_chain_per_k_block(sass, name):
    from tests.test_fused_chain_sass_cpu import _chains, _is_mma
    runs = _chains(_kernel(sass, name))
    assert runs
    for r in runs:
        body = r['body'][:max(k for k, i in enumerate(r['body']) if _is_mma(i)) + 1]
        mmas = [i for i in body if _is_mma(i)]
        assert sum(i.startswith('WARPGROUP.ARRIVE') for i in r['lead']) == 1, r
        assert not any(i.startswith('WARPGROUP') for i in body), body
        assert all('gsb0' not in i for i in mmas[:-1]) and 'gsb0' in mmas[-1], mmas
    assert max(sum(_is_mma(i) for i in r['body']) for r in runs) == 8


def _reds(ins):
    ops = [i.split()[0] for i in ins if i.startswith('REDG')]
    return sum(o.startswith('REDG.E.ADD.F32') for o in ops), sum(o.startswith('REDG.E.ADD.64') for o in ops)


@pytest.mark.parametrize('name', ['fused_conv_fixed_kernel', 'fused_conv_fixed_kernel_so'])
def test_fixed_fused_kernels_reduce_with_64_bit_integer_reds(sass, name):
    """the only f32 RED left is the edge count (one per 64-edge half); the float instantiation has one per flush"""
    f32, i64 = _reds(_kernel(sass, name))
    f32_float, i64_float = _reds(_kernel(sass, name.replace('_fixed', '')))
    assert i64 > 0 and f32 == 1, (f32, i64)
    assert i64_float == 0 and f32_float > 1


def test_fixed_streaming_kernel_reduces_with_64_bit_integer_reds(sass):
    """the float kernel has a sum and a count RED at each of its two row flushes; the fixed one keeps the counts only"""
    f32, i64 = _reds(_kernel(sass, 'tpconv_accumulate_fixed_kernel'))
    f32_float, i64_float = _reds(_kernel(sass, 'tpconv_accumulate_kernel'))
    assert i64 > 0 and i64_float == 0 and f32 == f32_float // 2, (f32, i64, f32_float)


FIXED_FUSED = ('fused_conv_fixed_kernel', 'fused_conv_fixed_kernel_so')


def test_fixed_fused_kernels_have_no_stack(built_lib):
    """as tests/test_fused_chain_sass_cpu.py requires of the float instantiations: no local-memory spills"""
    import subprocess
    if shutil.which('cuobjdump') is None:
        pytest.skip('cuobjdump not on PATH')
    out = subprocess.run(['cuobjdump', '-res-usage', os.path.join(ROOT, 'diffdock_b200', 'libdiffdock_b200.so')],
                         capture_output=True, text=True, check=True).stdout.splitlines()
    for name in FIXED_FUSED:
        usage = [out[k + 1] for k, l in enumerate(out[:-1])
                 if re.search(rf'\d{name}E', l) and l.lstrip().startswith('Function')]
        assert len(usage) == 1, name
        m = re.search(r'STACK:(\d+)', usage[0])
        assert m and int(m.group(1)) == 0, usage[0]


def test_ptxas_keeps_the_wgmma_pipeline_of_the_fixed_kernels(built_lib, tmp_path):
    """ptxas neither serialises nor fences the fixed-point instantiations' wgmmas (C7514 / C7517 / C7519)"""
    import subprocess
    import __graft_entry__ as g
    cmd = [g._nvcc()] + [f for f in g.NVCC_FLAGS if f not in ('-Xcompiler', '-fPIC')] + [
        '-Xptxas', '-v', '-cubin', '-o', str(tmp_path / 'fused_conv.cubin'),
        os.path.join(ROOT, 'diffdock_b200', 'csrc', 'fused_conv.cu')]
    log = subprocess.run(cmd, capture_output=True, text=True, check=True, cwd=ROOT)
    log = log.stdout + log.stderr
    assert all(n in log for n in FIXED_FUSED)
    bad = [l for l in log.splitlines() if re.search(r'\(C75(14|17|19)\)', l) and 'fixed_kernel' in l]
    assert not bad, bad
