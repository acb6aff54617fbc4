"""Static SASS opcode counts of csrc/libb2ins.so per kernel family (all instantiations summed):
evidence that the bulk-copy / mbarrier path is there (UBLKCP, SYNCS) and that the path has no
tensor-core opcodes.  Needs cuobjdump only (no GPU).
    python tools/sass_opcodes.py > profiles/sass_opcodes_r02.txt"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, 'gnss_ins_sim_b200', 'csrc', 'libb2ins.so')
COLS = ['UBLKCP', 'SYNCS', 'BAR', 'DFMA', 'DMUL', 'DADD', 'DSETP', 'MUFU', 'IMAD', 'SHFL', 'LDS', 'STS', 'LDG',
        'STG', 'ATOM', 'RED', 'HMMA', 'UTCHMMA', 'UTCMMA']


def main():
    out = subprocess.run(['cuobjdump', '-sass', LIB], capture_output=True, text=True).stdout
    fam, counts, inst = None, collections.defaultdict(collections.Counter), collections.Counter()
    for line in out.split('\n'):
        m = re.search(r'Function : (\S+)', line)
        if m:
            name = m.group(1)
            d = re.search(r'b2ins\d+([a-z_0-9]+?_kernel)', name)      # _ZN5b2ins14mc_spec_kernelILi...
            fam = d.group(1) if d else name
            inst[fam] += 1
            continue
        m = re.match(r'\s+/\*[0-9a-f]{4,5}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)', line)
        if m and fam:
            counts[fam][m.group(1)] += 1
    print('# Static SASS opcode counts of csrc/libb2ins.so (cuobjdump -sass, sm_90a), per kernel family '
          '(all instantiations summed); tools/sass_opcodes.py.')
    print('# UBLKCP = cp.async.bulk (1-D TMA copy), SYNCS = mbarrier ops; no tensor-core opcodes (HMMA / UTC*MMA) '
          'anywhere: the path has no contraction.')
    print('%-26s %7s' % ('kernel family', 'inst') + ''.join(' %7s' % c for c in COLS))
    tot = collections.Counter()
    for f in sorted(counts):
        print('%-26s %7d' % (f, inst[f]) + ''.join(' %7d' % counts[f][c] for c in COLS))
        tot.update(counts[f])
    print('%-26s %7d' % ('total', sum(inst.values())) + ''.join(' %7d' % tot[c] for c in COLS))


if __name__ == '__main__':
    sys.exit(main())
