"""Install the UNMODIFIED reference package (lucidrains/muse-maskgit-pytorch) into oracle/_ref/ for the reference arm of bench.py.

The reference is pure Python, so installing it is copying its package directory `muse_maskgit_pytorch/` byte for byte (no pip, no
build step).  Its third-party requirements are not installed: four of them are stood in for by tests/golden/_shims at import time
(baseline/ref_loader.py), the others come from the environment.

The checkout is looked up in $MUSE_MASKGIT_REFERENCE, else in DEFAULT_SOURCE.  Without a readable one the install is skipped:
oracle/_ref/ is git-ignored and travels with the working tree to where the benchmark runs.

  python -m oracle.reference_install        (also run by __graft_entry__.build())
"""
import os
import shutil
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEST = os.path.join(ROOT, "oracle", "_ref")
PACKAGE = "muse_maskgit_pytorch"
DEFAULT_SOURCE = "/root/reference"


def source_dir():
    src = os.environ.get("MUSE_MASKGIT_REFERENCE", DEFAULT_SOURCE)
    return src if os.path.isfile(os.path.join(src, PACKAGE, "__init__.py")) else None


def installed():
    return os.path.isfile(os.path.join(DEST, PACKAGE, "__init__.py"))


def install():
    """Returns DEST when the reference is installed there (now or earlier), None when no checkout was found."""
    if installed():
        return DEST
    src = source_dir()
    if src is None:
        return None
    os.makedirs(DEST, exist_ok=True)
    # copy next to the target and rename, so that an interrupted install never leaves a partial package behind
    tmp = tempfile.mkdtemp(prefix=".install_", dir=DEST)
    try:
        staged = os.path.join(tmp, PACKAGE)
        shutil.copytree(os.path.join(src, PACKAGE), staged, ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
        for d, _, files in os.walk(staged):                    # the checkout may be read-only; the copy is owned and writable here
            os.chmod(d, 0o755)
            for f in files:
                os.chmod(os.path.join(d, f), 0o644)
        os.replace(staged, os.path.join(DEST, PACKAGE))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return DEST


if __name__ == "__main__":
    print(install())
