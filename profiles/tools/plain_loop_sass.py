"""Diagnostic: size and local-memory traffic of the plain ADMM inner loop of a Kp3 kernel, from its SASS.

  cuobjdump -sass pqp_k3_17_6_4_17.o > k.sass   (or a .cubin; one kernel per translation unit)
  python profiles/tools/plain_loop_sass.py k.sass [more.sass ...]

The plain inner loop is taken as the innermost loop (backward branch to loop head) whose body holds at least four
barriers: every other loop of a Kp3 kernel (Ruiz sweeps, refactorisation, epilogue) has fewer.  Prints per file the
loop's instruction count, barriers, and LDL / STL (local-memory loads / stores, i.e. spill traffic in the hot loop)."""
import re
import sys


def parse(path):
    ins = []
    with open(path) as f:
        for line in f:
            m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s*(.*?);", line)
            if m:
                ins.append((int(m.group(1), 16), m.group(2)))
    return ins


def plain_loop(ins):
    best = None
    for a, t in ins:
        if "BRA" not in t:
            continue
        m = re.search(r"0x([0-9a-f]+)", t.split("BRA", 1)[1])
        if not m:
            continue
        head = int(m.group(1), 16)
        if head >= a:
            continue
        body = [x for b, x in ins if head <= b <= a]
        bars = sum("BAR.SYNC" in x or "BAR.RED" in x for x in body)
        if bars >= 4 and (best is None or a - head < best[0]):
            best = (a - head, body, bars)
    if best is None:
        return None
    _, body, bars = best
    return {"instructions": len(body), "barriers": bars, "LDL": sum("LDL" in x for x in body),
            "STL": sum("STL" in x for x in body)}


if __name__ == "__main__":
    for p in sys.argv[1:]:
        print(p, plain_loop(parse(p)))
