"""Recipe for ``oracle/_ref/``: copy the reference's lookup-path modules, unmodified, from
``/root/reference`` so that the GPU box (which has no ``/root/reference``) can run the REAL
``VectorBase`` as the timed CPU comparator and as the ``install()`` integration target.

    python oracle/vendor_ref.py

``oracle/_ref/`` is git-ignored (reference sources never enter the history); like the built ``.so``
it travels with a copy of the working tree to a GPU machine without the reference.  The reference is pure
Python, so there is nothing to compile: "building" it is this copy.  Files are copied byte for
byte; ``oracle/_ref/MANIFEST.json`` records their sha256 so a test can check nothing was edited.

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).
"""

from __future__ import annotations

import hashlib
import json
import os
import shutil

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = "/root/reference/src/typeagent"
DST = os.path.join(HERE, "_ref", "typeagent")

# the hot path (aitools/vectorbase.py), its wrapper, and the index classes that call it, plus
# the modules those import; storage/ and knowpro/ are small pure-Python trees
FILES_AND_DIRS = [
    "aitools/vectorbase.py",
    "aitools/embeddings.py",
    "knowpro",
    "storage/memory",
    "storage/sqlite",
]
EXTRA = {
    # the reference's own micro-benchmark of the path (BASELINE.json configs[0])
    "/root/reference/tools/benchmark_vectorbase.py": os.path.join(HERE, "_ref", "tools", "benchmark_vectorbase.py"),
}


def _sha(path: str) -> str:
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def vendor() -> str | None:
    """Copy the files; returns the destination, or None when /root/reference is absent (the
    GPU box: the copy made in the build container is used as is)."""
    if not os.path.isdir(SRC):
        return None
    if os.path.isdir(os.path.join(HERE, "_ref")):
        shutil.rmtree(os.path.join(HERE, "_ref"))
    manifest = {}
    for rel in FILES_AND_DIRS:
        src = os.path.join(SRC, rel)
        dst = os.path.join(DST, rel)
        if os.path.isdir(src):
            for dirpath, _dirs, files in os.walk(src):
                for name in files:
                    if not name.endswith(".py"):
                        continue
                    s = os.path.join(dirpath, name)
                    d = os.path.join(dst, os.path.relpath(s, src))
                    os.makedirs(os.path.dirname(d), exist_ok=True)
                    shutil.copyfile(s, d)
                    manifest[os.path.relpath(d, os.path.join(HERE, "_ref"))] = _sha(d)
        else:
            os.makedirs(os.path.dirname(dst), exist_ok=True)
            shutil.copyfile(src, dst)
            manifest[os.path.relpath(dst, os.path.join(HERE, "_ref"))] = _sha(dst)
    for src, dst in EXTRA.items():
        if os.path.isfile(src):
            os.makedirs(os.path.dirname(dst), exist_ok=True)
            shutil.copyfile(src, dst)
            manifest[os.path.relpath(dst, os.path.join(HERE, "_ref"))] = _sha(dst)
    with open(os.path.join(HERE, "_ref", "MANIFEST.json"), "w") as f:
        json.dump({"source": SRC, "files": manifest}, f, indent=1, sort_keys=True)
    return DST


if __name__ == "__main__":
    print(vendor())
