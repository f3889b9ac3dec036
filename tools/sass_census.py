#!/usr/bin/env python3
"""SASS census of kernels in libluaradio_b200.so (runs on a machine without a GPU: cuobjdump only).

    python tools/sass_census.py 'polyphase_crcf_kernel<5, 26, true, true' 'rs_poly_kernel<float2, 2, 1, 8>' > profiles/rNN_sass.txt

For every kernel whose demangled name contains one of the patterns: register count, instruction count, the mnemonic
histogram of the whole kernel and of its hottest loop (the backward branch whose body holds the most FFMA2 / FFMA), and the
first lines of that loop's body as an excerpt."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "luaradio_b200", "libluaradio_b200.so")


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    return dict(zip(names, out))


def main():
    pats = sys.argv[1:] or ["polyphase_crcf_kernel<5, 26"]
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True).stdout
    regs = {}
    cur = None
    for line in res.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            cur = m.group(1)
        m = re.search(r"REG:(\d+)", line)
        if m and cur:
            regs[cur] = int(m.group(1))
    funcs = re.split(r"\n\s*Function : ", sass)[1:]
    names = [f.split("\n", 1)[0].strip() for f in funcs]
    dm = demangle(names)
    for f, name in zip(funcs, names):
        d = dm.get(name, name)
        if not any(p in d for p in pats):
            continue
        ins = []
        for line in f.splitlines():
            m = re.match(r"\s+/\*([0-9a-f]{4,})\*/\s+(.*?);", line)
            if m:
                ins.append((int(m.group(1), 16), m.group(2).strip()))
        mnem = lambda t: re.sub(r"^@!?U?P\d+\s+", "", t).split()[0].split(".")[0]
        hist = collections.Counter(mnem(t) for _, t in ins)
        addr_index = {a: i for i, (a, _) in enumerate(ins)}
        best = None
        for i, (a, t) in enumerate(ins):
            m = re.search(r"\bBRA(?:\.U)?\s+(?:!?U?P\d+,\s*)?0x([0-9a-f]+)", t)
            if m and int(m.group(1), 16) <= a and int(m.group(1), 16) in addr_index:
                j = addr_index[int(m.group(1), 16)]
                body = ins[j:i + 1]
                fma = sum(1 for _, x in body if mnem(x) in ("FFMA2", "FFMA"))
                if best is None or fma > best[0]:
                    best = (fma, j, i)
        print("=" * 120)
        print("kernel:", d)
        print("registers:", regs.get(name, "?"), " instructions:", len(ins))
        print("whole kernel:", ", ".join("%s %d" % kv for kv in hist.most_common(14)))
        if best and best[0] > 0:
            fma, j, i = best
            body = ins[j:i + 1]
            h = collections.Counter(mnem(t) for _, t in body)
            print("hottest loop: %d instructions at 0x%04x-0x%04x, FFMA2+FFMA %d = %.1f %% of its issue slots" %
                  (len(body), ins[j][0], ins[i][0], fma, 100.0 * fma / len(body)))
            print("  loop mix:", ", ".join("%s %d" % kv for kv in h.most_common(14)))
            # the loop body between its barriers (static counts): for the persistent tile loop that is staging | compute |
            # epilogue, give or take where the loop's back edge falls
            cuts = [k for k, (_, x) in enumerate(body) if mnem(x) == "BAR"]
            for k0, k1 in zip([0] + [c + 1 for c in cuts], cuts + [len(body)]):
                seg = body[k0:k1]
                if seg:
                    hs = collections.Counter(mnem(x) for _, x in seg)
                    print("  region 0x%04x-0x%04x: %d instructions: %s" % (seg[0][0], seg[-1][0], len(seg),
                                                                        ", ".join("%s %d" % kv for kv in hs.most_common(10))))
            print("  excerpt (first 48 instructions of the loop body):")
            for a, t in body[:48]:
                print("    /*%04x*/ %s" % (a, t))
    return 0


if __name__ == "__main__":
    sys.exit(main())
