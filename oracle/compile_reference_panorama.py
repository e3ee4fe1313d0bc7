"""Byte-compile the reference's `moge/utils/panorama.py` into oracle/_ref/ (git-ignored) as `reference_panorama.pyc`: the host
comparator of tools/bench_panorama.py (cv2 split, SciPy LSMR merge).  Follows oracle/compile_reference_metrics.py.

Runs from `__graft_entry__.build()`.  MOGE_REFERENCE names a checkout of the reference (microsoft/MoGe); without it there is
nothing to compile and the benchmark reports the comparator as not measured.  The source is not copied: only its bytecode is
written, next to the build products.
"""
import importlib.util
import os
import py_compile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
PYC = os.path.join(REF_DIR, "reference_panorama.pyc")


def main() -> None:
    ref = os.environ.get("MOGE_REFERENCE")
    src = os.path.join(ref, "moge", "utils", "panorama.py") if ref else ""
    if not ref or not os.path.isfile(src):
        print("oracle/_ref: MOGE_REFERENCE does not name a reference checkout; the panorama comparator is not built")
        return
    py_compile.compile(src, cfile=PYC, doraise=True)
    print("oracle/_ref: compiled", PYC)


def load_panorama():
    """The reference's panorama module from oracle/_ref, or None when it was not built or cv2 / SciPy / tqdm are missing.  Its
    `import utils3d` resolves to the stand-in with `utils3d.np` installed (oracle/utils3d_panorama.py)."""
    if not os.path.isfile(PYC):
        return None
    try:
        import cv2  # noqa: F401
        import scipy.sparse.linalg  # noqa: F401
        import tqdm  # noqa: F401
    except ImportError:
        return None
    from oracle.utils3d_panorama import install
    install()
    spec = importlib.util.spec_from_file_location("reference_panorama", PYC)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    main()
