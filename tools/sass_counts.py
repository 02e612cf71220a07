#!/usr/bin/env python
"""Per-kernel SASS evidence: which of the mnemonics the design relies on each kernel of
pire_b200/libpire_b200.so really contains (cuobjdump -sass; no GPU needed).

    python tools/sass_counts.py > sass_counts.txt
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pire_b200", "libpire_b200.so")
WATCH = [
    ("UBLKCP", r"\bUBLKCP"),                     # cp.async.bulk (1-D TMA): table staging
    ("SYNCS", r"\bSYNCS"),                       # mbarrier arrive / try_wait
    ("LDGSTS", r"\bLDGSTS"),                     # cp.async 16 B: staging ring of the CSR kernels
    ("LDG.128", r"\bLDG\.E\.[A-Z0-9.]*128"),       # streaming loads of the uniform kernels, two per 32 bytes
    ("LDS.U8", r"\bLDS\.U8"),                    # the table walk
    ("@P LDS.U8", r"@!?P\d\s+LDS\.U8"),          # predicated walk (exit filter / look-ahead)
    ("LDS.128", r"\bLDS\.128"),
    ("IDP.4A", r"\bIDP\.4A"),                    # byte extraction on the FMA pipe
    ("PRMT", r"\bPRMT"),
    ("SHF", r"\bSHF\."),
    ("SHF.R.U64", r"\bSHF\.R\.U64"),             # 64-slot filter probe
    ("LOP3", r"\bLOP3"),
    ("IMAD", r"\bIMAD\b(?!\.MOV|\.U32 R\d+, RZ)"),
    ("VOTE", r"\bVOTE"),
    ("STL/LDL", r"\b(STL|LDL)"),                 # spills
    ("HMMA/UTCMMA", r"\b(HMMA|IMMA|UTC\w*MMA)"), # tensor cores: none expected (no contraction on this path)
]


def main():
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    kernels = collections.OrderedDict()
    name = None
    arch = set()
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip() or m.group(1)
            name = re.sub(r"pire_b200::\(anonymous namespace\)::|pire_b200::<unnamed>::", "", name)
            name = re.sub(r"\(pire_b200::ScanArgs\)|\(ScanArgs\)", "", name)
            kernels[name] = []
            continue
        m = re.search(r"arch = (sm_\w+)", line)
        if m:
            arch.add(m.group(1))
        if name and re.match(r"\s+/\*[0-9a-f]{4}\*/", line):
            kernels[name].append(line)
    print("# SASS mnemonic counts per kernel of pire_b200/libpire_b200.so (cuobjdump -sass), cubin arch: %s" % ", ".join(sorted(arch)))
    print("# columns: instructions, then", ", ".join(k for k, _ in WATCH))
    for kname, lines in kernels.items():
        if "cub::" in kname or not lines:
            continue
        text = "\n".join(lines)
        counts = [len(re.findall(pat, text)) for _, pat in WATCH]
        print("%-62s %5d  %s" % (kname[:62], len(lines), " ".join("%s=%d" % (k, c) for (k, _), c in zip(WATCH, counts) if c)))


if __name__ == "__main__":
    sys.exit(main())
