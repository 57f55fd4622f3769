"""SASS opcode summary of the shipped kernels (cuobjdump -sass of co_snarks_b200/libcosnarks_gpu.so), per kernel:
instruction count, the dominant opcodes, local-memory traffic (LDL / STL = spills or stack arrays) and the
Blackwell / Hopper-era mnemonics the profiling recipe names (UBLKCP = cp.async.bulk, SYNCS = mbarrier, UTMALDG /
UTMASTG = tensor-map TMA, DFMA, IMAD.WIDE).  usage: sass_summary.py [lib.so] > sass_summary.md"""
import collections
import re
import subprocess
import sys

LIB = sys.argv[1] if len(sys.argv) > 1 else "co_snarks_b200/libcosnarks_gpu.so"
out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
kern = collections.OrderedDict()
cur = None
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = m.group(1)
        kern[cur] = collections.Counter()
        continue
    if cur is None:
        continue
    m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]*)", line)
    if m:
        kern[cur][m.group(1)] += 1
demangle = subprocess.run(["c++filt"], input="\n".join(kern), capture_output=True, text=True).stdout.splitlines()
WATCH = ("UBLKCP", "SYNCS", "UTMALDG", "UTMASTG", "DFMA", "SHFL", "LDL", "STL", "ATOMG", "RED", "LDGSTS")
print("# SASS summary of %s (sm_90a)\n" % LIB)
print("Opcode classes counted per kernel body incl. its out-of-line device functions; `local` = LDL + STL.\n")
print("| kernel | instr | IMAD.WIDE* | IMAD* other | DFMA+DADD | ALU (IADD3/LOP3/SHF/SEL/..) | local | TMA/mbarrier | top opcodes |")
print("|---|---|---|---|---|---|---|---|---|")
tot = collections.Counter()
for (name, c), dn in zip(kern.items(), demangle):
    n = sum(c.values())
    if n < 40:
        continue
    short = re.sub(r"\(.*", "", dn)
    short = re.sub(r"cs::", "", short)
    wide = sum(v for k, v in c.items() if k.startswith("IMAD.WIDE"))
    imad = sum(v for k, v in c.items() if k.startswith("IMAD")) - wide
    f64 = sum(v for k, v in c.items() if k.startswith(("DFMA", "DADD", "DMUL")))
    alu = sum(v for k, v in c.items() if k.startswith(("IADD3", "LOP3", "SHF", "SEL", "ISETP", "VIADD", "MOV", "PRMT", "LEA")))
    local = sum(v for k, v in c.items() if k.startswith(("LDL", "STL")))
    tma = ", ".join("%s x%d" % (k, v) for k, v in sorted(c.items()) if k.startswith(("UBLKCP", "SYNCS", "UTMA")))
    top = ", ".join("%s %d" % kv for kv in c.most_common(4))
    print("| `%s` | %d | %d | %d | %d | %d | %d | %s | %s |" % (short[:90], n, wide, imad, f64, alu, local, tma or "-", top))
    for k, v in c.items():
        for w in WATCH:
            if k.startswith(w):
                tot[w] += v
print("\nWhole library: " + ", ".join("%s %d" % (w, tot[w]) for w in WATCH))
