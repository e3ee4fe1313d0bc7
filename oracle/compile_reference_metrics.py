"""Byte-compile the reference's `moge/test/metrics.py` and the `moge/utils` modules it imports into oracle/_ref/ (git-ignored)
as the package `reference_moge`: the comparator of tools/bench_metrics.py, which times it on the same GPU as the engine.  Another
top-level name keeps its relative imports resolving and leaves the repository's `moge` alias unshadowed.

Runs from `__graft_entry__.build()`.  MOGE_REFERENCE names a checkout of the reference (microsoft/MoGe); without it there is
nothing to compile and the benchmark reports the comparator as not measured.  The sources are not copied: only their bytecode is
written, next to the build products.
"""
import importlib
import os
import py_compile
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
PACKAGE = "reference_moge"
MODULES = ("__init__", "test/__init__", "test/metrics", "utils/__init__", "utils/alignment", "utils/geometry_torch",
           "utils/geometry_numpy", "utils/tools")


def main() -> None:
    ref = os.environ.get("MOGE_REFERENCE")
    if not ref or not os.path.isfile(os.path.join(ref, "moge", "test", "metrics.py")):
        print("oracle/_ref: MOGE_REFERENCE does not name a reference checkout; the metrics comparator is not built")
        return
    for m in MODULES:
        py_compile.compile(os.path.join(ref, "moge", m + ".py"), cfile=os.path.join(REF_DIR, PACKAGE, m + ".pyc"), doraise=True)
    print("oracle/_ref: compiled", os.path.join(REF_DIR, PACKAGE))


def load_metrics():
    """The reference's `moge.test.metrics` from oracle/_ref/reference_moge, or None when it was not built.  Its `import utils3d`
    resolves to the stand-in under oracle/utils3d_shim with the metrics' two functions installed (oracle/utils3d_metrics.py)."""
    if not os.path.isfile(os.path.join(REF_DIR, PACKAGE, "test", "metrics.pyc")):
        return None
    from oracle.utils3d_metrics import install
    install()
    if REF_DIR not in sys.path:
        sys.path.append(REF_DIR)
    return importlib.import_module(PACKAGE + ".test.metrics")


if __name__ == "__main__":
    main()
