"""Builds oracle/_ref/: the reference's `polyfuzz` package as sourceless byte code (TEST INFRASTRUCTURE).

The drop-in tests hand this package's matchers to the unmodified PolyFuzz orchestrator.  The reference source is
only present where the project is built, so build() compiles it into oracle/_ref/ (kept out of git), which travels
with the other build products; where the reference is not readable nothing is built and those tests skip."""
import os
import py_compile
import shutil
import warnings

from . import ref_shim

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")


def build():
    src = os.path.join(ref_shim.REFERENCE_ROOT, "polyfuzz")
    if not os.path.isdir(src) or not os.access(src, os.R_OK | os.X_OK):
        return None
    dst = os.path.join(OUT, "polyfuzz")
    tmp = dst + ".tmp"
    shutil.rmtree(tmp, ignore_errors=True)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", SyntaxWarning)                 # the reference's own regex literals
        for d, _, files in os.walk(src):
            rel = os.path.relpath(d, src)
            for f in files:
                if f.endswith(".py"):
                    os.makedirs(os.path.join(tmp, rel), exist_ok=True)
                    py_compile.compile(os.path.join(d, f), cfile=os.path.join(tmp, rel, f[:-3] + ".pyc"),
                                       dfile=os.path.join("polyfuzz", rel, f), doraise=True)
    shutil.rmtree(dst, ignore_errors=True)
    os.replace(tmp, dst)
    return OUT
