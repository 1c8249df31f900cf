"""Stage the unmodified pulser-core (the reference's input layer) under ``oracle/_ref``.

The facade tests build real pulser Sequences and compare what the emulator makes of them with the reference's own
results.  pulser-core is pure Python, so "building" it is a copy of its package and of the VERSION.txt its
``_version.py`` reads (two directories up).  The source checkout of Pulser is looked for in ``$PULSER_SOURCE``, then
in ``/root/reference``; when neither is readable nothing is staged and the pulser-dependent tests skip.
``oracle/_ref`` is git-ignored.
"""
from __future__ import annotations

import os
import shutil

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.join(HERE, "_ref")
CORE = os.path.join(REF, "pulser-core")   # what pulser_b200._compat puts on sys.path


def source_root() -> str | None:
    for root in (os.environ.get("PULSER_SOURCE"), "/root/reference"):
        if not root:
            continue
        try:
            if os.path.isdir(os.path.join(root, "pulser-core", "pulser")) and os.access(
                    os.path.join(root, "VERSION.txt"), os.R_OK):
                return root
        except OSError:
            continue
    return None


def build() -> bool:
    """Copy pulser-core into ``oracle/_ref``; returns whether a staged copy exists afterwards."""
    src = source_root()
    if src is None:
        return os.path.isdir(os.path.join(CORE, "pulser"))
    tmp = REF + ".tmp"
    shutil.rmtree(tmp, ignore_errors=True)
    try:
        shutil.copytree(os.path.join(src, "pulser-core", "pulser"), os.path.join(tmp, "pulser-core", "pulser"),
                        ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
        shutil.copy2(os.path.join(src, "VERSION.txt"), os.path.join(tmp, "VERSION.txt"))
    except OSError:
        shutil.rmtree(tmp, ignore_errors=True)
        return os.path.isdir(os.path.join(CORE, "pulser"))
    shutil.rmtree(REF, ignore_errors=True)
    os.replace(tmp, REF)
    return True


if __name__ == "__main__":
    print(REF if build() else "no Pulser source found: nothing staged")
