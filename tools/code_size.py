#!/usr/bin/env python
"""SASS size of the light kernels under a set of extra nvcc flags (no GPU needed).
usage: tools/code_size.py [-DHK_MINB_INDIRECT=12 ...]
Compiles bevy_hikari_b200/csrc/kernels_light.cu with the build's flags + the given ones into a scratch object and prints
instructions / KB / registers / spill bytes per kernel."""
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bevy_hikari_b200 import build as B  # noqa: E402

src = os.path.join(B.HERE, sys.argv[1] if len(sys.argv) > 1 and sys.argv[1].endswith(".cu") else "csrc/kernels_light.cu")
flags = [a for a in sys.argv[1:] if not a.endswith(".cu")]
with tempfile.TemporaryDirectory() as d:
    obj = os.path.join(d, "k.o")
    r = subprocess.run([B.NVCC] + B.NVCC_FLAGS + ["-Xptxas", "-v"] + flags + ["-c", src, "-o", obj], capture_output=True, text=True)
    if r.returncode:
        sys.exit(r.stderr)
    info = {}
    cur = None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            info.setdefault(cur, {})["spill"] = (int(m.group(2)), int(m.group(3)), int(m.group(1)))
        m = re.search(r"Used (\d+) registers", line)
        if m and cur:
            info.setdefault(cur, {})["regs"] = int(m.group(1))
    sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
cnt = collections.Counter()
name = None
for l in sass.splitlines():
    m = re.search(r"Function : (\S+)", l)
    if m:
        name = m.group(1); continue
    if re.match(r"\s+/\*[0-9a-f]{4,6}\*/\s+\S", l):
        cnt[name] += 1
for n, c in sorted(cnt.items(), key=lambda x: x[1]):
    i = info.get(n, {})
    dem = subprocess.run(["c++filt", n], capture_output=True, text=True).stdout.strip()
    print(f"{c:6d} instr {c * 16 / 1024:6.1f} KB  regs {i.get('regs', '?'):>3}  spill st/ld/stack {i.get('spill', '?')}  {dem[:70]}")
