"""Installs the unmodified upstream `normflows` package into oracle/_ref/ (git-ignored) for the reference arms of
bench.py (`--impl reference`, `--impl reference-eager`, the `cpu_baseline` and `reference_eager` keys).

The upstream project is pure Python (numpy + torch): installing it is a verbatim copy of its `normflows` package
directory, without upstream's own unit tests (`*_test.py`: pytest run from this repository's root would collect them).
It is taken from $NORMFLOWS_REFERENCE (a checkout of the upstream repository), else from a checkout named `reference`
next to this repository.  When neither exists nothing is installed, an existing copy is left as it is, and the
reference arms report themselves unavailable."""
import os
import shutil

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEST = os.path.join(ROOT, "oracle", "_ref")


def source():
    """The upstream `normflows` package directory, or None."""
    checkout = os.environ.get("NORMFLOWS_REFERENCE") or os.path.join(os.path.dirname(ROOT), "reference")
    pkg = os.path.join(checkout, "normflows")
    return pkg if os.path.isfile(os.path.join(pkg, "__init__.py")) else None


def installed():
    return os.path.isfile(os.path.join(DEST, "normflows", "__init__.py"))


def install():
    """Copy the upstream package to oracle/_ref/normflows; returns whether a copy is installed afterwards."""
    src = source()
    if src is not None:
        dst = os.path.join(DEST, "normflows")
        os.makedirs(DEST, exist_ok=True)
        shutil.rmtree(dst, ignore_errors=True)
        shutil.copytree(src, dst, ignore=shutil.ignore_patterns("__pycache__", "*.pyc", "*_test.py", "test_*.py"))
    return installed()
