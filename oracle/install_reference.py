"""Install the UNMODIFIED reference package (beat_this) into oracle/_ref/, for bench.py's reference arms.

    python oracle/install_reference.py [<beat_this source tree>]

The source tree is the argument, else $BEAT_THIS_REFERENCE, else /root/reference.  `__graft_entry__.build()` runs
this when such a tree exists and oracle/_ref/ does not hold the package yet.  The install is `pip install --no-deps
--target oracle/_ref` from a temporary copy (the build writes egg-info into the source tree).  `--no-deps` because
`soxr`, `rotary-embedding-torch`, `soundfile` and `madmom` are not installable offline; the two of them the reference
imports at module import time come from oracle/shims/.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, "_ref")


def default_source() -> str:
    return os.environ.get("BEAT_THIS_REFERENCE") or "/root/reference"


def installed() -> bool:
    return os.path.isdir(os.path.join(REF_DIR, "beat_this"))


def install(source: str | None = None) -> str:
    """Install the reference from `source` into oracle/_ref/.  Returns a one-line status; never raises."""
    source = source or default_source()
    if installed():
        return "oracle/_ref: already installed"
    if not os.path.isdir(os.path.join(source, "beat_this")):
        return f"oracle/_ref: no reference source tree at {source}; bench.py falls back to the oracle port"
    with tempfile.TemporaryDirectory() as td:
        try:
            src = shutil.copytree(source, os.path.join(td, "reference"))
            for d, _, files in os.walk(src):  # the copy keeps the modes of a read-only tree; the build writes into it
                os.chmod(d, 0o755)
                for f in files:
                    os.chmod(os.path.join(d, f), 0o644)
        except OSError as e:
            return f"oracle/_ref: cannot copy {source}: {e}"
        r = subprocess.run([sys.executable, "-m", "pip", "install", "--no-index", "--no-build-isolation", "--no-deps",
                            "--no-cache-dir", "--target", REF_DIR, src], capture_output=True, text=True)
    if r.returncode != 0 or not installed():
        return "oracle/_ref: install failed: " + " | ".join((r.stderr or r.stdout).strip().splitlines()[-3:])
    return "oracle/_ref: installed the unmodified reference"


if __name__ == "__main__":
    print(install(sys.argv[1] if len(sys.argv) > 1 else None))
