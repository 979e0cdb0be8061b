"""SASS evidence for the shipped library: per kernel family the count of the tensor-core / TMA / cluster opcodes
(cuobjdump -sass of anakin_b200/lib/libb200saber.so; runs without a GPU).
  python tools/sass_histogram.py
HGMMA = wgmma (sm_90a), WARPGROUP = wgmma fence / wait (ARRIVE, DEPBAR), UTMALDG = TMA load (tiled / im2col),
UTMASTG = TMA store, SYNCS = mbarrier, UCGABAR = cluster barrier, LDGSTS = cp.async."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "anakin_b200", "lib", "libb200saber.so")
OPS = ["HGMMA", "WARPGROUP", "UTMALDG", "UTMASTG", "UTMAPF", "SYNCS", "UCGABAR",
       "LDGSTS", "UBLKCP", "ACQBULK", "IDP", "HMMA", "IMMA", "REDG", "ATOMG"]


def main():
    out = subprocess.run(["cuobjdump", "-sass", LIB], stdout=subprocess.PIPE, text=True).stdout
    fam = None
    counts = collections.OrderedDict()
    variants = collections.Counter()
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = subprocess.run(["c++filt", m.group(1)], stdout=subprocess.PIPE, text=True).stdout.strip()
            fam = re.sub(r"<.*", "", re.sub(r"\(.*", "", name)).replace("void ", "").replace("b200::", "")
            variants[fam] += 1
            counts.setdefault(fam, collections.Counter())
            continue
        m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)((?:\.[A-Z0-9_]+)*)", line)
        if m and fam:
            op = m.group(1)
            if op.startswith("UCGABAR"):
                op = "UCGABAR"
            if op in OPS:
                key = op + (".IM2COL" if ".IM2COL" in m.group(2) else "")
                key = key + (".MULTICAST" if "MULTICAST" in m.group(2) else "")
                counts[fam][key] += 1
            counts[fam]["(all instructions)"] += 1
    print("cuobjdump -sass anakin_b200/lib/libb200saber.so (sm_90a): opcode counts per kernel family, summed over its template instances")
    for f, c in counts.items():
        ops = ", ".join("%s x%d" % (k, v) for k, v in sorted(c.items()) if k != "(all instructions)")
        print("%-28s %3d instance(s) %7d instr | %s" % (f, variants[f], c["(all instructions)"], ops or "-"))


if __name__ == "__main__":
    main()
