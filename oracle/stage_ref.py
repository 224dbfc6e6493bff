"""Stages the reference implementation for the comparison legs of bench.py (baseline/run_reference.py).

The reference is a script tree without setup.py / pyproject (nothing for pip to install), so its "build" is a copy of its Python
packages and its tree file into the git-ignored `oracle/_ref/`, where baseline/run_reference.py imports them from.  The
reference root is $TRIFORCE_REFERENCE_ROOT (default as in oracle/ref_harness.py); where it is absent an earlier staging is kept.
"""
from __future__ import annotations

import os
import shutil

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DST = os.path.join(REPO, "oracle", "_ref")


def stage_reference(src: str = None) -> str:
    if src is None:
        from oracle.ref_harness import REF_ROOT as src
    if not os.path.isdir(os.path.join(src, "models")):
        return "oracle/_ref present" if os.path.isfile(os.path.join(DST, "utils", "decoding.py")) else "reference not available here"
    for sub in ("models", "utils"):
        shutil.copytree(os.path.join(src, sub), os.path.join(DST, sub), dirs_exist_ok=True,
                        ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
    os.makedirs(os.path.join(DST, "tree"), exist_ok=True)
    if os.path.isfile(os.path.join(src, "tree", "512.pt")):
        shutil.copy2(os.path.join(src, "tree", "512.pt"), os.path.join(DST, "tree", "512.pt"))
    return f"staged oracle/_ref from {src}"
