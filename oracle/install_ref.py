#!/usr/bin/env python
"""Install the UNMODIFIED reference (facebookresearch/flashy) into oracle/_ref.

    python oracle/install_ref.py [REFERENCE_CHECKOUT]

The checkout is the argument, else ``$FLASHY_REFERENCE``, else ``/root/reference``.  ``oracle/_ref`` is
git-ignored (never committed); the solver drop-in tests and ``benchmarks/gan_step.py`` import the
reference's ``flashy`` package from it and skip / fail with a clear message where it is absent.  The
reference's own dependencies ``dora_search`` and ``colorlog`` are not installed (``--no-deps``, no package
index); the solver tests provide minimal stand-ins for the two (tests/shims/, test-only).  The checkout
may be read-only, so the build runs from a copy in a temporary directory.  Prints one line with the
outcome.
"""
import os
import shutil
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
DEST = ROOT / "oracle" / "_ref"


def reference_checkout(arg: str = "") -> Path:
    return Path(arg or os.environ.get("FLASHY_REFERENCE") or "/root/reference")


def install(src_dir: str = "") -> str:
    if (DEST / "flashy" / "solver.py").exists():
        return f"already installed: {DEST}"
    ref = reference_checkout(src_dir)
    try:
        readable = (ref / "setup.py").is_file() and os.access(ref / "flashy", os.R_OK | os.X_OK)
    except OSError:
        readable = False
    if not readable:
        return f"unavailable: no readable reference checkout at {ref}"
    with tempfile.TemporaryDirectory() as tmp:
        src = Path(tmp) / "reference"
        shutil.copytree(ref, src, ignore=shutil.ignore_patterns(".git"))
        for p in (src, *src.rglob("*")):                       # the build writes its metadata into the copy
            p.chmod(p.stat().st_mode | 0o200)
        cmd = [sys.executable, "-m", "pip", "install", "--no-index", "--no-build-isolation", "--no-deps",
               "--no-cache-dir", "--disable-pip-version-check", "--target", str(DEST), str(src)]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            return "failed: " + (res.stderr.strip().splitlines() or ["pip error"])[-1]
    return f"installed {DEST} (pip --no-deps)"


if __name__ == "__main__":
    print(install(sys.argv[1] if len(sys.argv) > 1 else ""))
