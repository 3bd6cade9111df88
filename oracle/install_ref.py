"""Recipe for oracle/_ref: the UNMODIFIED reference (sample-factory 2.1.3) pip-installed next to the oracle, for the
reference arm of bench.py, its cpu_baseline leg and the example-script test (tests/test_boundary.py).  oracle/_ref is
git-ignored and travels with the tree.  The reference checkout is SF_REFERENCE_DIR when set, else the default location
DEFAULT_REFERENCE_DIR; build() installs it whenever such a checkout exists.
--no-deps because the reference's third-party dependencies (gymnasium, signal-slot-mp, faster-fifo, tensorboardX, colorlog)
are not needed: oracle/ref_shims.py stands in for them at import time."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
DEFAULT_REFERENCE_DIR = "/root/reference"


def reference_dir() -> str | None:
    """The reference checkout (a directory with sample_factory/ and setup.py), or None when there is none."""
    ref = os.environ.get("SF_REFERENCE_DIR") or DEFAULT_REFERENCE_DIR
    return ref if os.path.isfile(os.path.join(ref, "sample_factory", "__init__.py")) else None


def install(reference_src: str | None = None) -> None:
    ref = reference_src or reference_dir()
    if not ref:
        return
    if os.path.isfile(os.path.join(REF_DIR, "sample_factory", "algo", "learning", "learner.py")):
        return
    with tempfile.TemporaryDirectory() as tmp:     # the checkout may be read-only and setuptools writes build/ next to setup.py
        src = os.path.join(tmp, "ref_src")
        shutil.copytree(ref, src, symlinks=True)
        for d, dirs, files in os.walk(src):   # copytree keeps the checkout's read-only modes; setuptools writes build/ here
            for name in [""] + files:
                path = os.path.join(d, name)
                if not os.path.islink(path):
                    os.chmod(path, os.stat(path).st_mode | 0o200)
        res = subprocess.run([sys.executable, "-m", "pip", "install", "--no-index", "--no-build-isolation", "--no-deps",
                              "--target", REF_DIR, src], capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write("installing the reference into oracle/_ref failed (the bench falls back to the oracle port):\n"
                         + res.stdout[-1500:] + res.stderr[-1500:] + "\n")
