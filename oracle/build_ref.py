"""Install the unmodified reference (torchnmf 0.3.5, pure Python) into oracle/_ref for the benchmark's reference lines
and for regenerating the golden fixtures:

    TORCHNMF_REFERENCE_SRC=<reference source tree> python oracle/build_ref.py

The reference's `torchnmf` package is copied as it is into oracle/_ref/torchnmf (git-ignored; never part of the
repository).  Without a source tree nothing is installed and bench.py reports its reference lines as unavailable.
"""
import os
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DST = os.path.join(ROOT, "oracle", "_ref")


def build(src=None):
    """Returns the install directory, or None when no reference source tree is given."""
    src = src or os.environ.get("TORCHNMF_REFERENCE_SRC")
    if not src:
        return None
    pkg = os.path.join(src, "torchnmf")
    if not os.path.isfile(os.path.join(pkg, "__init__.py")):
        raise RuntimeError(f"{src} holds no torchnmf package")
    if not os.path.isdir(os.path.join(DST, "torchnmf")):
        os.makedirs(DST, exist_ok=True)
        tmp = os.path.join(DST, "torchnmf.partial")
        shutil.rmtree(tmp, ignore_errors=True)
        shutil.copytree(pkg, tmp, ignore=shutil.ignore_patterns("__pycache__"))
        os.replace(tmp, os.path.join(DST, "torchnmf"))
    return DST


if __name__ == "__main__":
    print(build(sys.argv[1] if len(sys.argv) > 1 else None))
