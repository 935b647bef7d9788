"""cuobjdump -sass of libkbo.so -> per-kernel counts of the tensor-core / TMA / mbarrier / FP64-tensor / SFU mnemonics.
   python tools/sass_summary.py > sass_summary.txt"""
import collections, os, re, subprocess, sys

LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "kubeflow_b200", "libkbo.so")
KEEP = re.compile(r"^(HGMMA|WARPGROUP|UTMA|DMMA|DFMA|MUFU|F2FP|STG\.E\.ENL2|SYNCS|UCGABAR|REDUX|SHFL|BAR|LDGSTS|ATOM|RED\.)")
txt = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
print("cuobjdump -sass kubeflow_b200/libkbo.so (sm_90a) — instruction counts per kernel, tensor-core / TMA / mbarrier / FP64-tensor mnemonics")
print("(HGMMA = wgmma.mma_async; WARPGROUP.ARRIVE / DEPBAR = wgmma.fence / wait_group; UTMALDG = cp.async.bulk.tensor; SYNCS = mbarrier;")
print(" DMMA = mma.sync f64; MUFU = SFU)\n")
name, counts, total = None, None, 0
def flush():
    if name and any(k for k in counts if k.startswith(("UTC", "UTMA", "LDTM", "DMMA", "MUFU", "DFMA"))):
        print(f"{name}  [{total} instructions]")
        for k in sorted(counts):
            print(f"    {k:34s} {counts[k]}")
        print()
for line in txt.splitlines():
    m = re.match(r"\s*Function : (\S+)", line)
    if m:
        flush()
        name, counts, total = m.group(1), collections.Counter(), 0
        continue
    m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Za-z0-9_.]+)", line)
    if m and name:
        total += 1
        op = m.group(1)
        if KEEP.match(op):
            counts[op] += 1
flush()
