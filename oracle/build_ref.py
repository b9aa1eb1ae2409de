"""Recipe for ``oracle/_ref``: the unmodified reference Pyro (1.9.1) that the binding tests
(tests/test_bind_pyro.py) and the reference arm of bench.py import.

Pyro is pure Python, so "building" it is copying its ``pyro`` package out of a reference checkout; the
checkout is found at ``$PYRO_REFERENCE`` (default ``/root/reference``).  Its one dependency that is not
installed here, ``opt_einsum``, is covered by the stand-in under tests/golden/opt_einsum_standin.
``oracle/_ref`` is git-ignored and nothing in it is edited.  Without a checkout nothing is built, and
whatever needs the reference skips (tests) or falls back to the oracle port (bench.py reference arm)."""
import os
import shutil

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")


def source():
    return os.environ.get("PYRO_REFERENCE", "/root/reference")


def build():
    """Copy the reference ``pyro`` package into oracle/_ref (once).  Returns the path, or None when no
    reference checkout is available."""
    if os.path.isdir(os.path.join(REF_DIR, "pyro")):
        return REF_DIR
    src = os.path.join(source(), "pyro")
    if not os.path.isfile(os.path.join(src, "__init__.py")):
        return None
    tmp = REF_DIR + ".tmp"
    shutil.rmtree(tmp, ignore_errors=True)
    shutil.copytree(src, os.path.join(tmp, "pyro"), ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
    # an oracle/_ref without pyro/ inside (an interrupted copy, stray files) is stale: os.replace cannot
    # rename over a non-empty directory
    shutil.rmtree(REF_DIR, ignore_errors=True)
    os.replace(tmp, REF_DIR)
    return REF_DIR


if __name__ == "__main__":
    print(build())
