#!/usr/bin/env python
"""Static opcode histogram of the longest loop (the widest backward branch) of every kernel in a cubin, executable or shared
library built for sm_90a, from `cuobjdump -sass`.  No GPU and no profiler needed: for unrolled step bodies such as the
fill kernel's 8-step loop this is the instruction mix per loop body.

    python tools/loop_sass.py FILE [NAME_SUBSTRING ...]     # e.g. libssw.so 'ssw_fill_kernel<8, 19, 1, 2'
"""
import re
import subprocess
import sys
from collections import Counter


def functions(path):
    """(demangled name, [(address, instruction text)]) per kernel."""
    sass = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    out, name, ins = [], None, []
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name:
                out.append((name, ins))
            name, ins = m.group(1), []
            continue
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?);", line)
        if m and name:
            ins.append((int(m.group(1), 16), m.group(2).strip()))
    if name:
        out.append((name, ins))
    names = subprocess.run(["c++filt"], input="\n".join(n for n, _ in out), capture_output=True, text=True).stdout.split("\n")
    return [(names[i] if i < len(names) and names[i] else n, ins) for i, (n, ins) in enumerate(out)]


def loop_histogram(ins):
    """Opcodes (predicate guards stripped) between the target and the source of the widest backward branch."""
    span = None
    for a, t in ins:
        m = re.search(r"BRA\b.*0x([0-9a-f]+)", t)
        if m and int(m.group(1), 16) < a and (span is None or a - int(m.group(1), 16) > span[1] - span[0]):
            span = (int(m.group(1), 16), a)
    if span is None:
        return 0, Counter()
    body = [re.sub(r"^@!?U?P\w+\s+", "", t) for a, t in ins if span[0] <= a <= span[1]]
    return len(body), Counter(t.split()[0] for t in body)


def main():
    path, keys = sys.argv[1], sys.argv[2:]
    for name, ins in functions(path):
        if keys and not any(k in name for k in keys):
            continue
        n, hist = loop_histogram(ins)
        print("%s\n  loop body: %d instructions: %s" % (name, n, ", ".join("%s %d" % kv for kv in hist.most_common())))


if __name__ == "__main__":
    main()
