"""CPU: the fused kernel issues the MMAs of one staged k-block as ONE wgmma chain - a single register fence
(WARPGROUP.ARRIVE) in front of the first MMA and the group's scoreboard (gsb0) on the last one only - and ptxas neither
injects fences / waits around its wgmmas nor serialises them (C7514 / C7517 / C7519).  A chain that ptxas breaks up waits
for every MMA to complete before issuing the next one."""
import os
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tools'))


@pytest.fixture(scope='module')
def fused_sass(built_lib):
    if shutil.which('cuobjdump') is None:
        pytest.skip('cuobjdump not on PATH')
    import sass_histogram as sh
    body = sh.kernels(os.path.join(ROOT, 'diffdock_b200', 'libdiffdock_b200.so'), operands=True)
    return next(v for k, v in body.items() if 'fused_conv_kernel' in k)


def _is_mma(ins):
    return ins.startswith('HGMMA') and '.BF16' in ins.split()[0]


def _chains(ins):
    """maximal runs of bf16 HGMMA separated only by the glue of tools/sass_histogram.py, each with the instructions
    between the previous non-glue instruction and the run's first MMA"""
    import sass_histogram as sh
    glue = lambda i: i.split()[0] in sh.GLUE or i.split()[0].split('.')[0] in sh.GLUE
    runs, cur, lead = [], None, []
    for i in ins:
        if _is_mma(i):
            if cur is None:
                cur = {'lead': lead, 'body': []}
            cur['body'].append(i)
        elif glue(i):
            (cur['body'] if cur is not None else lead).append(i)
        else:
            if cur is not None:
                runs.append(cur)
            cur, lead = None, []
    if cur is not None:
        runs.append(cur)
    return runs


def test_each_k_block_is_one_chain(fused_sass):
    runs = _chains(fused_sass)
    assert runs
    for r in runs:
        body = r['body']
        last = max(k for k, i in enumerate(body) if _is_mma(i))
        body = body[:last + 1]                  # glue after the last MMA belongs to what follows
        mmas = [i for i in body if _is_mma(i)]
        assert sum(i.startswith('WARPGROUP.ARRIVE') for i in r['lead']) == 1, r
        assert not any(i.startswith('WARPGROUP') for i in body), body
        assert all('gsb0' not in i for i in mmas[:-1]) and 'gsb0' in mmas[-1], mmas
    assert max(sum(_is_mma(i) for i in r['body']) for r in runs) == 8


def test_fused_kernel_has_no_stack(built_lib):
    """two accumulator sets (192 registers) and the consumer's contraction state fit in 255 registers: no local-memory
    spills in the hot loops"""
    if shutil.which('cuobjdump') is None:
        pytest.skip('cuobjdump not on PATH')
    out = subprocess.run(['cuobjdump', '-res-usage', os.path.join(ROOT, 'diffdock_b200', 'libdiffdock_b200.so')],
                         capture_output=True, text=True, check=True).stdout.splitlines()
    usage = [out[k + 1] for k, l in enumerate(out[:-1]) if 'fused_conv_kernel' in l and l.lstrip().startswith('Function')]
    assert usage, 'fused_conv_kernel not in the resource usage'
    for u in usage:
        m = re.search(r'STACK:(\d+)', u)
        assert m and int(m.group(1)) == 0, u


def test_ptxas_keeps_the_wgmma_pipeline(built_lib, tmp_path):
    import __graft_entry__ as g
    cmd = [g._nvcc()] + [f for f in g.NVCC_FLAGS if f not in ('-Xcompiler', '-fPIC')] + [
        '-Xptxas', '-v', '-cubin', '-o', str(tmp_path / 'fused_conv.cubin'),
        os.path.join(ROOT, 'diffdock_b200', 'csrc', 'fused_conv.cu')]
    out = subprocess.run(cmd, capture_output=True, text=True, check=True, cwd=ROOT)
    log = out.stdout + out.stderr
    assert 'fused_conv_kernel' in log
    bad = [l for l in log.splitlines() if re.search(r'\(C75(14|17|19)\)', l) and 'fused_conv_kernel' in l]
    assert not bad, bad
