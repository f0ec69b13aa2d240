"""SASS mnemonic counts per kernel of the built library (cuobjdump -sass): the static evidence that TMA bulk copies (UBLKCP), mbarriers
(SYNCS) and warpgroup MMAs (HGMMA = wgmma.mma_async) are in the kernels that claim them.  usage: python scripts/sass_evidence.py"""
import collections
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = os.path.join(ROOT, "lightgaussian_b200", "_lib", "liblgrast.so")
out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
KEYS = ["HGMMA", "UBLKCP", "SYNCS", "LDG.E.128", "REDG", "ATOMS", "MUFU", "LDS.128", "VOTE", "FFMA"]
cur, counts, total = None, collections.OrderedDict(), {}
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = m.group(1)
        counts[cur] = collections.Counter()
        total[cur] = 0
        continue
    if cur is None:
        continue
    m = re.search(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]*)", line)
    if m:
        op = m.group(1)
        total[cur] += 1
        for k in KEYS:
            if op.startswith(k):
                counts[cur][k] += 1
print("# SASS mnemonic counts per kernel (cuobjdump -sass, sm_90a): HGMMA = wgmma.mma_async, UBLKCP = cp.async.bulk (TMA bulk copy),")
print("# SYNCS = mbarrier, REDG = fire-and-forget global reductions")
for name, c in counts.items():
    short = re.sub(r"^_ZN\d+_GLOBAL__N__[0-9a-f]+_\d+_lgrast_cu_[0-9a-f]+", "", name)[:72]
    print(f"{short:72s} " + " ".join(f"{k} {c[k]:3d}" for k in KEYS) + f" total {total[name]:5d}")
