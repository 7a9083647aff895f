"""Per-kernel SASS opcode table of libnnconv_b200.so (evidence that the hot kernels are wgmma / TMA code):
    python scripts/sass_table.py > sass_opcodes.md
Runs on the build container (cuobjdump only needs the .so)."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, 'graph_pde_b200', 'libnnconv_b200.so')
OPS = ['HGMMA', 'WARPGROUP', 'UTMALDG', 'UTMASTG', 'UBLKRED', 'SYNCS', 'REDG', 'ATOMG', 'STG', 'LDG', 'ELECT', 'HMMA', 'FFMA']


def main():
    sass = subprocess.run(['cuobjdump', '-sass', SO], stdout=subprocess.PIPE, text=True, check=True).stdout
    dem = {}
    counts = collections.OrderedDict()
    cur = None
    for line in sass.splitlines():
        m = re.match(r'\s*Function : (\S+)', line)
        if m:
            cur = m.group(1)
            counts[cur] = collections.Counter()
            continue
        m = re.match(r'\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)', line)
        if m and cur:
            counts[cur][m.group(1).split('.')[0]] += 1
            counts[cur]['_total'] += 1
    names = list(counts)
    out = subprocess.run(['c++filt'] + names, stdout=subprocess.PIPE, text=True).stdout.splitlines()
    for n, d in zip(names, out):
        d = d.replace('(anonymous namespace)::', '').replace('nnc::', '').replace('void ', '')
        d = re.sub(r'\(.*', '', d)
        dem[n] = d
    print('# SASS opcode counts per kernel of libnnconv_b200.so (cuobjdump -sass, sm_90a)\n')
    print('HGMMA = wgmma.mma_async, WARPGROUP = wgmma fence / arrive / wait, UTMALDG / UTMASTG = TMA tensor load / '
          'store, UBLKRED = cp.reduce.async.bulk, SYNCS = mbarrier ops, REDG = red.global (fp32 scatter atomics).  '
          'HMMA (mma.sync) must be absent.\n')
    print('| kernel | instr | ' + ' | '.join(OPS) + ' |')
    print('|---|---|' + '---|' * len(OPS))
    for n in names:
        c = counts[n]
        if c['_total'] == 0:
            continue
        print('| `%s` | %d | ' % (dem[n], c['_total']) + ' | '.join(str(c[o]) if c[o] else '' for o in OPS) + ' |')


if __name__ == '__main__':
    sys.exit(main())
