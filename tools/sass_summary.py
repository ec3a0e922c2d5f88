"""Per-kernel counts of the SASS mnemonics that show which hardware path a kernel uses
(warpgroup MMA = HGMMA, TMA = UTMALDG / UTMASTG / UBLKCP / UTMAPF, mma.sync tensor path =
HMMA), from `cuobjdump -sass` of the in-tree library.  Runs without a GPU.

    python tools/sass_summary.py
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "opendwm_b200", "libdwm_b200.so")
PATTERNS = ["HGMMA", "WARPGROUP.ARRIVE", "UTMALDG", "UTMASTG", "UTMAPF", "UBLKCP", "UBLKPF",
            "SYNCS", "USETMAXREG", "HMMA", "LDSM", "LDGSTS", "MUFU.EX2", "RED.", "ATOM"]


def main():
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    kernels = collections.OrderedDict()
    name = None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = subprocess.run(["c++filt", m.group(1)], capture_output=True,
                                  text=True).stdout.strip()
            name = re.sub(r"\(.*", "", name).replace("void dwm::", "").replace("dwm::", "")
            kernels[name] = collections.Counter()
            continue
        if name is None:
            continue
        ins = re.search(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
        if not ins:
            continue
        op = ins.group(1)
        for p in PATTERNS:
            if p.endswith("."):
                hit = op.startswith(p)
            elif "." in p:
                hit = op.startswith(p.split(".")[0]) and p.split(".", 1)[1] in op
            else:
                hit = op.split(".")[0] == p
            if hit:
                kernels[name][p] += 1
    print("SASS mnemonic counts per kernel of opendwm_b200/libdwm_b200.so (cuobjdump -sass, "
          "sm_90a)\n")
    cols = [p for p in PATTERNS if any(k[p] for k in kernels.values())]
    width = max(len(n) for n in kernels) + 2
    print("kernel".ljust(width) + "".join(c.rjust(max(9, len(c) + 1)) for c in cols))
    total = collections.Counter()
    for n, c in kernels.items():
        if not any(c[p] for p in cols):
            continue
        print(n.ljust(width) + "".join(str(c[p] or ".").rjust(max(9, len(p) + 1)) for p in cols))
        total.update(c)
    print("\nTOTAL".ljust(width + 1) + "".join(str(total[p]).rjust(max(9, len(p) + 1)) for p in cols))
    print("\nHGMMA = wgmma.mma_async, WARPGROUP.ARRIVE = wgmma.fence, USETMAXREG = setmaxnreg; "
          "UTMALDG/UTMASTG = cp.async.bulk.tensor load/store (TMA), UTMAPF = TMA L2 prefetch, "
          "UBLKCP/UBLKPF = cp.async.bulk copy / prefetch; HMMA + LDSM = mma.sync path "
          "(gathered attention kernel for short / separate-KV sequences only).")


if __name__ == "__main__":
    sys.exit(main())
