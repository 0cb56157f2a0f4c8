"""Audit the SASS of every kernel for memory accesses that precede `griddepcontrol.wait` (SASS: ACQBULK).

Under programmatic dependent launch a kernel starts while its predecessor is still running; everything the predecessor
produces must be read after the wait.  `asm volatile(... ::: "memory")` does NOT pin `ld.global.nc` loads (the compiler
treats `const __restrict__` data as immutable for the whole kernel and may hoist them above the wait -- observed on an
RMSNorm variant whose token-id loads moved up and read the previous tree level's ids).  This script makes the property
checkable: per kernel it lists global loads / stores / atomics issued before the first ACQBULK.  Allowed before the wait:
TMA weight loads of the GEMM producers (UTMALDG / UBLKCP) and constant-bank reads.

    python tools/audit_pdl_sass.py [libeagle_b200.so | objdir]      # exit code 1 if a kernel violates the rule
"""
import glob
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BAD = re.compile(r"\b(LDG|LD|LDGSTS|STG|ST|ATOM|ATOMG|RED|REDG)(\.|\s)")


def audit(target):
    bad = {}
    n_kernels = 0
    objs = sorted(glob.glob(os.path.join(target, "*.o"))) if os.path.isdir(target) else [target]
    for obj in objs:
        out = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
        fn, seen_wait, hits = None, False, []

        def flush():
            if fn is not None and hits and has_wait[0]:
                bad[fn] = list(hits)

        has_wait = [False]
        for line in out.splitlines():
            m = re.match(r"\s*Function : (\S+)", line)
            if m:
                flush()
                fn, seen_wait, hits = m.group(1), False, []
                has_wait = [False]
                n_kernels += 1
                continue
            ins = re.match(r"\s*/\*[0-9a-f]+\*/\s+(.*?);", line)
            if not ins or fn is None:
                continue
            text = ins.group(1)
            if "ACQBULK" in text:
                seen_wait = True
                has_wait[0] = True
            elif not seen_wait:
                t = re.sub(r"^@!?U?P\d+\s+", "", text)
                if BAD.match(t) and not t.startswith(("LDC", "LDCU", "LDS", "LDSM", "LDL", "STS", "STL")):
                    hits.append(text.strip())
        flush()
    return n_kernels, bad


def main():
    target = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "eagle_b200", "libeagle_b200.so")
    n, bad = audit(target)
    print(f"{n} kernels audited in {target}")
    for fn, hits in bad.items():
        name = subprocess.run(["c++filt", fn], capture_output=True, text=True).stdout.strip()[:110]
        print(f"BEFORE THE WAIT in {name}:")
        for h in hits[:8]:
            print("    ", h)
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
