#!/usr/bin/env python
"""Per-kernel SASS opcode histogram of the product library.

    python tools/sass_hist.py [lib.so] [--filter SUBSTR] [--top N] [--all]

Runs `cuobjdump -sass` on the library, demangles nothing (the mangled names carry the template
arguments), and prints for every kernel: instruction count, registers are NOT in SASS (see
`cuobjdump -res-usage`), and the opcode histogram collapsed to the mnemonic before the first '.'.
The lines that matter for the north_star claims are marked: UTMALDG / UBLKCP (TMA), SYNCS (mbarrier),
LDGSTS (cp.async), HGMMA (warpgroup MMA), ATOMS / ATOMG / RED.
"""
from __future__ import annotations

import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MARK = ("UTMALDG", "UTMASTG", "UBLKCP", "SYNCS", "LDGSTS", "HGMMA", "WARPGROUP", "ATOMS", "ATOMG", "RED", "HMMA", "ELECT")


def histogram(lib):
    txt = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    kernels = collections.OrderedDict()
    cur = None
    ins = re.compile(r"^\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_]*)")
    for ln in txt.splitlines():
        if "Function :" in ln:
            cur = ln.split("Function :")[1].strip()
            kernels[cur] = collections.Counter()
            continue
        if cur is None:
            continue
        m = ins.match(ln)
        if m:
            kernels[cur][m.group(1)] += 1
    return kernels


def short(name):
    """_ZN3psb51_GLOBAL__N__..._18march_level_kernelILi13ELb0ELb0EEEv... -> march_level_kernel<13,0,0>"""
    m = re.search(r"\d+([a-z_0-9]+_kernel[a-z_0-9]*)(I[^v]*?E)?Ev", name)
    if not m:
        return name[:60]
    base, targs = m.group(1), m.group(2) or ""
    args = re.findall(r"L[ib](\d+)E|([fh])(?=E|L|$)", targs)
    flat = [a or {"f": "float", "h": "u8"}.get(b, b) for a, b in args]
    return base + ("<" + ",".join(flat) + ">" if flat else "")


def main(argv):
    lib = os.path.join(ROOT, "popsift_b200", "lib", "libpopsift_b200.so")
    flt, top, show_all = None, 14, False
    i = 0
    while i < len(argv):
        a = argv[i]
        if a == "--filter":
            flt = argv[i + 1]; i += 1
        elif a == "--top":
            top = int(argv[i + 1]); i += 1
        elif a == "--all":
            show_all = True
        else:
            lib = a
        i += 1
    ks = histogram(lib)
    print("# cuobjdump -sass %s : %d kernels" % (os.path.relpath(lib, ROOT), len(ks)))
    tot = collections.Counter()
    for name, c in ks.items():
        tot.update(c)
    print("# library totals of the marked opcodes: " + "  ".join("%s %d" % (m, tot[m]) for m in MARK if tot[m]))
    for name, c in ks.items():
        s = short(name)
        if flt and flt not in s and flt not in name:
            continue
        n = sum(c.values())
        marks = "  ".join("%s %d" % (m, c[m]) for m in MARK if c[m])
        print("%-52s %6d instr   %s" % (s, n, marks))
        if show_all or flt:
            print("      " + "  ".join("%s %d" % (o, k) for o, k in c.most_common(top)))


if __name__ == "__main__":
    main(sys.argv[1:])
