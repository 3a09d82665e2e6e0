#!/usr/bin/env python3
"""Per-kernel resources of libtavec.so from ``cuobjdump --dump-resource-usage`` (registers, stack, local
memory), and the kernels whose figures differ between two builds.  Runs without a GPU.

    python tools/kernel_resources.py NEW.so                # one line per kernel
    python tools/kernel_resources.py OLD.so NEW.so         # only what changed, was added or went away

To compare against the parent commit: ``git worktree add /tmp/parent HEAD~1``, ``python
/tmp/parent/typeagent-py_b200/build.py``, then pass ``/tmp/parent/typeagent-py_b200/libtavec.so`` as OLD.  Spill
stores and loads per kernel are in ``typeagent-py_b200/build_ptxas.log`` (ptxas -v), written by every build.
"""

from __future__ import annotations

import os
import re
import shutil
import subprocess
import sys


def resources(lib: str) -> dict[str, str]:
    """demangled kernel name -> "REG:.. STACK:.. LOCAL:.." of one library."""
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    out = subprocess.run([cuobjdump, "--dump-resource-usage", lib], capture_output=True, text=True, check=True).stdout
    found, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1)
        elif name and "REG:" in line:
            fields = dict(re.findall(r"(\w+):(\d+)", line))
            found[name] = f"REG:{fields['REG']} STACK:{fields['STACK']} LOCAL:{fields['LOCAL']}"
            name = None
    filt = shutil.which("c++filt")
    if filt and found:
        names = subprocess.run([filt], input="\n".join(found), capture_output=True, text=True).stdout.splitlines()
        found = dict(zip(names, found.values()))
    return found


def main(argv):
    if len(argv) == 1:
        for name, res in sorted(resources(argv[0]).items()):
            print(f"{res}  {name}")
        return 0
    if len(argv) != 2 or not all(os.path.exists(p) for p in argv):
        print(__doc__)
        return 2
    old, new = resources(argv[0]), resources(argv[1])
    same = sum(1 for k in old if new.get(k) == old[k])
    print(f"{len(old)} kernels before, {len(new)} after, {same} with the same name and the same figures")
    for k in sorted(set(old) | set(new)):
        if old.get(k) != new.get(k):
            print(f"{old.get(k, '(absent)'):<28} -> {new.get(k, '(absent)'):<28} {k}")
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
