"""Instruction mix of the hot kernels from the SASS of the built library:
  python profiles/sass_mix.py raven_b200/libraven_b200.so > profiles/r02_sass_mix.txt
(static counts per kernel; shows what the kernels are made of - integer ALU, shuffles,
votes, shared/global memory - and that no tensor-core or TMA instruction is on the path)"""
import collections
import re
import subprocess
import sys

HOT = ["SketchFastKernel", "OnesweepPass", "RadixHistogramKernel", "TierScatterKernel",
       "GroupCountKernel", "IndexTableKernel", "MicromizeKernel", "JoinSweepKernel",
       "ExpandJoinKernel", "SplitKernel", "GroupChainKernel", "PairChainKernel",
       "ColumnsWarpKernel", "LeafKernel", "BandedMyersKernel", "PoaKernelFast",
       "PileRegionsKernel"]
out = subprocess.run(["cuobjdump", "-sass", sys.argv[1]], capture_output=True, text=True).stdout
name, mix, total = None, None, {}
kernels = {}
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        name = m.group(1)
        kernels[name] = collections.Counter()
        continue
    m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_]*)", line)
    if m and name:
        kernels[name][m.group(1)] += 1
special = ("UTMA", "UTC", "TCGEN", "HMMA", "IMMA", "UBLKCP", "LDGSTS", "MATCH", "VOTE", "SHFL",
           "ATOMS", "ATOMG", "RED", "LDG", "STG", "LDS", "STS", "BAR", "POPC", "LOP3", "IADD3",
           "SHF", "VIMNMX", "LDL", "STL")
for hot in HOT:
    for k, c in kernels.items():
        if hot not in k or not c:
            continue
        n = sum(c.values())
        short = re.sub(r"^_ZN3rvn\d+_GLOBAL__N__[0-9a-f_]+cu_[0-9a-f]+", "", k)[:70]
        top = ", ".join(f"{op} {v}" for op, v in c.most_common(9))
        flags = ", ".join(f"{s}:{sum(v for op, v in c.items() if op.startswith(s))}"
                          for s in ("UTMA", "UTC", "HMMA", "IMMA", "MATCH", "VOTE", "SHFL", "ATOMS",
                                    "LDL", "STL") if any(op.startswith(s) for op in c))
        print(f"{short}\n    {n} instructions; {top}\n    of note: {flags or '-'}")
