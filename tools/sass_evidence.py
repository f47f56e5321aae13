"""Counts the SASS mnemonics that identify the Hopper paths per kernel of the shipped library:
    cuobjdump -sass one-2-3-45_b200/lib/libo2345_sm90.so | python tools/sass_evidence.py > sass_evidence.txt
HGMMA = wgmma.mma_async, WARPGROUP = wgmma fence / wait, UTMALDG = TMA (cp.async.bulk.tensor), SYNCS = mbarrier, UCGABAR = cluster
barrier, HMMA = mma.sync, LDSM / STSM = ldmatrix / stmatrix, LDGSTS = cp.async."""
import collections
import re
import subprocess
import sys

OPS = ('HGMMA', 'WARPGROUP', 'UTMALDG', 'UTMASTG', 'UBLKCP', 'SYNCS', 'HMMA', 'LDGSTS', 'LDSM', 'STSM', 'REDG',
       'UCGABAR_ARV', 'UCGABAR_WAIT')
cur, counts, n = None, collections.defaultdict(collections.Counter), collections.Counter()
for line in sys.stdin:
    m = re.search(r'Function : (\S+)', line)
    if m:
        cur = m.group(1)
        continue
    if cur is None:
        continue
    m = re.search(r'^\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)', line)
    if m:
        op = m.group(1).split('.')[0]
        n[cur] += 1
        if op in OPS:
            counts[cur][op] += 1
names = subprocess.run(['c++filt'], input="\n".join(n), capture_output=True, text=True).stdout.split("\n")
agg = collections.defaultdict(lambda: [0, collections.Counter(), 0])
for k, name in zip(n, names):
    name = re.sub(r'o2345::\(anonymous namespace\)::', '', name)
    base = re.sub(r'^void ', '', re.sub(r'\(.*$', '', name))
    key = re.sub(r'gemm_tc_kernel<(\d+), (\d+), (\d+)>', r'gemm_tc_kernel<BN, STAGES, MODE=\3>', base)
    a = agg[key]
    a[0] += 1
    a[1].update(counts[k])
    a[2] = max(a[2], n[k])
print("cuobjdump -sass one-2-3-45_b200/lib/libo2345_sm90.so | python tools/sass_evidence.py   (sm_90a; instantiations merged: 'xN' of them,")
print("counts summed over them, instruction count of the largest)\n")
for key, (ni, c, mx) in sorted(agg.items(), key=lambda kv: -sum(kv[1][1].values())):
    if c:
        print(f"{key:62s} x{ni:<3d} {mx:6d} instr  " + "  ".join(f"{o} {v}" for o, v in sorted(c.items())))
print("\nkernels without any of these mnemonics (plain HBM / L2 kernels): " + ", ".join(sorted(k for k, (ni, c, mx) in agg.items() if not c)))
