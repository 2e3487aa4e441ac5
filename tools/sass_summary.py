#!/usr/bin/env python
"""tools/sass_summary.py -- what the shipped binary contains: per kernel of libl3c_b200.so the count of
the SASS mnemonics that show the Hopper path (wgmma.mma_async -> HGMMA, wgmma fences -> WARPGROUP,
TMA -> UTMALDG/UTMASTG/UBLKCP, mbarrier -> SYNCS) next to the legacy warp-level tensor path (HMMA) and
the plain FFMA count.

    python tools/sass_summary.py
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, 'l3c_pytorch_b200', 'libl3c_b200.so')
PATTERNS = ['HGMMA', 'WARPGROUP', 'UTMALDG', 'UTMASTG', 'UBLKCP', 'SYNCS', 'HMMA', 'FFMA', 'MUFU', 'REDUX', 'LDGSTS']


def main():
    sass = subprocess.run(['cuobjdump', '-sass', SO], capture_output=True, text=True, check=True).stdout
    git = subprocess.run(['git', '-C', ROOT, 'rev-parse', '--short', 'HEAD'], capture_output=True, text=True).stdout.strip()
    arch = sorted(set(re.findall(r'arch = (sm_\w+)', sass)))
    per = collections.OrderedDict()
    cur = None
    for line in sass.splitlines():
        m = re.match(r'\s*Function : (\S+)', line)
        if m:
            cur = m.group(1)
            per[cur] = collections.Counter()
            continue
        if cur is None:
            continue
        m = re.match(r'\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)', line)
        if m:
            op = m.group(1)
            per[cur]['_all'] += 1
            for p in PATTERNS:
                if op.startswith(p):
                    per[cur][p] += 1
    demangle = subprocess.run(['c++filt'] + list(per), capture_output=True, text=True).stdout.splitlines()
    print('# SASS summary of l3c_pytorch_b200/libl3c_b200.so (cuobjdump -sass), built from the tree at/after commit %s' % git)
    print('# target:', ', '.join(arch))
    print('# columns: instructions | ' + ' '.join(PATTERNS))
    tot = collections.Counter()
    for (name, c), dn in zip(per.items(), demangle):
        short = re.sub(r'\(.*', '', dn)
        print('%-70s %6d | %s' % (short[:70], c['_all'], ' '.join('%s=%d' % (p, c[p]) for p in PATTERNS if c[p])))
        tot.update(c)
    print('%-70s %6d | %s' % ('TOTAL', tot['_all'], ' '.join('%s=%d' % (p, tot[p]) for p in PATTERNS if tot[p])))
    return 0


if __name__ == '__main__':
    sys.exit(main())
