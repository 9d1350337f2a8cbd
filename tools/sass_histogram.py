#!/usr/bin/env python
"""Static instruction histogram of the built library (cuobjdump -sass): one row per kernel with the counts of the mnemonics
that show what the code runs on - warpgroup MMAs (HGMMA), their register fences (WARPGROUP), bulk / TMA copies (UBLKCP /
UTMALDG), mbarrier operations (SYNCS), reductions to global memory (REDG) - and of the legacy ones it must not contain (HMMA =
mma.sync).  Also the longest run of bf16 HGMMA separated only by uniform-datapath / move instructions (no wgmma wait,
barrier or memory access in between): the size of the fused kernel's MMA issue block, one chain per staged k-block.
    mkdir -p build/profiles && python tools/sass_histogram.py [lib.so] > build/profiles/sass_histogram.csv"""
import os
import re
import subprocess
import sys
from collections import Counter, OrderedDict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COLS = ['HGMMA', 'WARPGROUP', 'UBLKCP', 'UTMALDG', 'SYNCS', 'ELECT', 'REDG', 'ATOMG', 'HMMA', 'FFMA', 'LDS', 'STS',
        'LDG', 'STG', 'SHFL', 'MUFU', 'UCGABAR', 'BAR']
VARIANTS = ('HGMMA', 'WARPGROUP', 'UBLKCP', 'REDG')
# instructions allowed between two MMAs of one issue block: the descriptor moves (uniform / register->uniform moves, adds,
# predicate setup).  A warpgroup register fence (WARPGROUP.ARRIVE) does not end the block either, so that one injected by
# ptxas inside a chain is seen as part of it (tests/test_fused_chain_sass_cpu.py rejects that).  Anything else - the wgmma
# wait (WARPGROUP.DEPBAR), a barrier, a memory access - ends the block.
GLUE = ('UMOV', 'R2UR', 'UISETP', 'IMAD', 'IADD3', 'NOP', 'UIADD3', 'LOP3', 'SHF', 'ISETP', 'P2R', 'MOV', 'PLOP3', 'BRA',
        'VOTEU', 'WARPGROUP.ARRIVE')


def kernels(lib, operands=False):
    """kernel -> its instructions' mnemonics (with `operands`: mnemonic and operands, e.g. 'HGMMA.64x192x16.F32.BF16 R24,
    gdesc[UR4], R24, gsb0')."""
    out = subprocess.run(['cuobjdump', '-sass', lib], capture_output=True, text=True, check=True).stdout
    cur, body = None, OrderedDict()
    for line in out.splitlines():
        m = re.search(r'Function : (\S+)', line)
        if m:
            cur = m.group(1)
            body[cur] = []
            continue
        m = re.match(r'\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Za-z0-9_.]*)([^;]*)', line)
        if m and cur is not None:
            body[cur].append(m.group(1) + m.group(2).rstrip() if operands else m.group(1))
    return body


def demangle(names):
    try:
        out = subprocess.run(['cu++filt'] + list(names), capture_output=True, text=True, check=True).stdout.splitlines()
        clean = [re.sub(r'\(anonymous namespace\)::|<unnamed>::|\((?:int|bool|unsigned int)\)', '', o) for o in out]
        return [c.split('(')[0][:70] for c in clean]
    except Exception:
        return list(names)


def longest_mma_run(ops):
    best = run = 0
    for op in ops:
        base = op.split('.')[0]
        if base == 'HGMMA' and '.BF16' in op:        # the project's MMAs (the compiler also emits an empty F16 HGMMA)
            run += 1
            best = max(best, run)
        elif base not in GLUE and op not in GLUE:
            run = 0
    return best


def rows(lib):
    body = kernels(lib)
    names = demangle(body.keys())
    for name, ops in zip(names, body.values()):
        c = Counter(op.split('.')[0] for op in ops)
        var = Counter(op for op in ops if op.split('.')[0] in VARIANTS)
        yield name, len(ops), [c.get(k, 0) for k in COLS], longest_mma_run(ops), ';'.join(f'{k}={v}' for k, v in sorted(var.items()))


if __name__ == '__main__':
    lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, 'diffdock_b200', 'libdiffdock_b200.so')
    print('# cuobjdump -sass diffdock_b200/libdiffdock_b200.so, instruction counts per kernel (static code, not executed counts);'
          ' mma_block = longest run of HGMMA with only move / uniform glue in between')
    print('kernel,instructions,' + ','.join(COLS) + ',mma_block,variants')
    for name, n, counts, block, var in sorted(rows(lib), key=lambda r: -r[1]):
        print(f'"{name}",{n},' + ','.join(map(str, counts)) + f',{block},"{var}"')
