"""Byte-compile the reference's modules that the tools/bench_*.py comparators time into oracle/_ref/ (git-ignored), as the
package `reference_moge`: `moge/utils/alignment.py` (tools/bench_align.py), `moge/test/metrics.py` (tools/bench_metrics.py),
`moge/utils/panorama.py` (tools/bench_panorama.py) and `moge/train/losses.py` (tools/bench_losses.py), with the `moge/utils`
modules they import.  Another top-level name keeps their relative imports resolving and leaves the repository's `moge` alias
unshadowed.

Runs from `__graft_entry__.build()`.  MOGE_REFERENCE names a checkout of the reference (microsoft/MoGe); without it there is
nothing to compile and the benchmarks report the comparators as not measured.  The sources are not copied: only their bytecode
is written, next to the build products.  Each `load_*` returns its module, or None when it was not built.  The modules'
`import utils3d` resolves to the stand-in under oracle/utils3d_shim, with the functions they call added by
oracle/utils3d_metrics.py or oracle/utils3d_panorama.py.
"""
import importlib
import os
import py_compile
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
PACKAGE = "reference_moge"
MODULES = ("__init__", "utils/__init__", "utils/alignment", "utils/geometry_torch", "utils/geometry_numpy", "utils/tools",
           "utils/panorama", "test/__init__", "test/metrics", "train/__init__", "train/losses")


def main() -> None:
    ref = os.environ.get("MOGE_REFERENCE")
    if not ref or not all(os.path.isfile(os.path.join(ref, "moge", m + ".py")) for m in MODULES):
        print("oracle/_ref: MOGE_REFERENCE does not name a reference checkout; the comparators are not built")
        return
    for m in MODULES:
        py_compile.compile(os.path.join(ref, "moge", m + ".py"), cfile=os.path.join(REF_DIR, PACKAGE, m + ".pyc"), doraise=True)
    print("oracle/_ref: compiled", os.path.join(REF_DIR, PACKAGE))


def _load(module: str, stand_in: str):
    """`module` of the compiled package after `oracle.<stand_in>.install()` has added the utils3d functions it calls."""
    if not os.path.isfile(os.path.join(REF_DIR, PACKAGE, module + ".pyc")):
        return None
    importlib.import_module("oracle." + stand_in).install()
    if REF_DIR not in sys.path:
        sys.path.append(REF_DIR)
    return importlib.import_module(PACKAGE + "." + module.replace("/", "."))


def load_alignment():
    """The reference's `moge.utils.alignment` (the solvers call no utils3d function)."""
    return _load("utils/alignment", "utils3d_metrics")


def load_metrics():
    """The reference's `moge.test.metrics`."""
    return _load("test/metrics", "utils3d_metrics")


def load_panorama():
    """The reference's `moge.utils.panorama`; None also when cv2, SciPy or tqdm are missing."""
    try:
        import cv2  # noqa: F401
        import scipy.sparse.linalg  # noqa: F401
        import tqdm  # noqa: F401
    except ImportError:
        return None
    return _load("utils/panorama", "utils3d_panorama")


def load_losses():
    """The reference's `moge.train.losses`."""
    return _load("train/losses", "utils3d_metrics")


if __name__ == "__main__":
    main()
