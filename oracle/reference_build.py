"""Compiled copy of the reference dmosopt package, for the tests that run the reference's own controller code.

``build_reference()`` (called by ``__graft_entry__.build()``) byte-compiles every module of a dmosopt checkout into
``oracle/_ref/dmosopt/`` as sourceless ``.pyc`` files (git-ignored, never committed; importable by the interpreter that
compiled them).  The checkout is taken from ``$DMOSOPT_REF`` or, failing that, from ``DEFAULT_CHECKOUT``, where the
project's build environment mounts it read-only.  Without a checkout nothing is built and those tests skip.
"""

import os
import py_compile
import shutil

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "oracle", "_ref")
DEFAULT_CHECKOUT = "/root/reference"


def _checkout():
    for p in (os.environ.get("DMOSOPT_REF"), DEFAULT_CHECKOUT):
        if p and os.path.isfile(os.path.join(p, "dmosopt", "MOASMO.py")) and os.access(os.path.join(p, "dmosopt"), os.R_OK | os.X_OK):
            return p
    return None


def build_reference(verbose=True):
    """Compile the reference package into oracle/_ref/dmosopt.  Returns the output directory, or None without a checkout."""
    src_root = _checkout()
    if src_root is None:
        return None
    pkg = os.path.join(src_root, "dmosopt")
    dst_pkg = os.path.join(OUT, "dmosopt")
    tmp = dst_pkg + ".tmp"
    shutil.rmtree(tmp, ignore_errors=True)
    n = 0
    for dirpath, dirnames, filenames in os.walk(pkg):
        dirnames[:] = [d for d in dirnames if d != "__pycache__"]
        rel = os.path.relpath(dirpath, pkg)
        for f in filenames:
            if f.endswith(".py"):
                dst = os.path.join(tmp, rel, f[:-3] + ".pyc")
                os.makedirs(os.path.dirname(dst), exist_ok=True)
                py_compile.compile(os.path.join(dirpath, f), cfile=dst, dfile=os.path.join("dmosopt", rel, f), doraise=True)
                n += 1
    shutil.rmtree(dst_pkg, ignore_errors=True)
    os.replace(tmp, dst_pkg)
    if verbose:
        print(f"[oracle] compiled {n} reference modules into {dst_pkg}", flush=True)
    return OUT


def reference_path():
    """Directory holding an importable ``dmosopt`` reference package: $DMOSOPT_REF, oracle/_ref or baseline/_ref."""
    for p in (os.environ.get("DMOSOPT_REF"), OUT, os.path.join(ROOT, "baseline", "_ref")):
        if p and os.path.isdir(os.path.join(p, "dmosopt")):
            return p
    return None
