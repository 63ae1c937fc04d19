#!/usr/bin/env python3
"""Address-ordered SASS of one kernel with source-line labels: python tools/sass_dump.py <lib.so> <kernel-substr> > out.txt"""
import os, re, subprocess, sys, tempfile


def sass(lib, pat):
    """Yield (address, "file:line", instruction) for every instruction of the kernels whose name contains `pat`, and
    (None, None, label) for every branch-target label, in address order."""
    d = tempfile.mkdtemp()
    subprocess.run(["cuobjdump", "-xelf", "all", os.path.abspath(lib)], cwd=d, capture_output=True)
    cub = [f for f in os.listdir(d) if f.endswith(".cubin") and "ingest" not in f][0]
    out = subprocess.run(["nvdisasm", "-g", "-c", os.path.join(d, cub)], capture_output=True, text=True).stdout
    infn, cur = False, ""
    for l in out.split("\n"):
        m = re.match(r"\s*\.text\.(\S+):", l) or re.match(r"\s*//-+ \.text\.(\S+)", l)
        if m:
            infn = pat in m.group(1); continue
        if not infn: continue
        m = re.search(r'//## File "([^"]+)", line (\d+)(.*)', l)
        if m:
            cur = os.path.basename(m.group(1))[:14] + ":" + m.group(2); continue
        m = re.match(r"\s+/\*([0-9a-f]{4,5})\*/\s+(.*?);", l)
        if m: yield int(m.group(1), 16), cur, m.group(2)
        elif re.match(r"\s*\.L_x?_?\w+:", l): yield None, None, l.strip()


if __name__ == "__main__":
    for a, cur, text in sass(sys.argv[1], sys.argv[2]):
        print(text if a is None else f"{a:04x} {cur:22s} {text}")
