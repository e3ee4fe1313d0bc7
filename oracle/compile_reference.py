"""Byte-compile the reference's `moge/utils/alignment.py` into oracle/_ref/ (git-ignored) as the comparator of
tools/bench_align.py, which times it on the same GPU as the engine's solvers.

Runs from `__graft_entry__.build()`.  MOGE_REFERENCE names a checkout of the reference (microsoft/MoGe); without it there is
nothing to compile and the benchmark reports the comparator as not measured.  The source is not copied: only its bytecode is
written, next to the build products.
"""
import os
import py_compile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
ALIGNMENT_PYC = os.path.join(REF_DIR, "reference_alignment.pyc")


def main() -> None:
    ref = os.environ.get("MOGE_REFERENCE")
    src = os.path.join(ref, "moge", "utils", "alignment.py") if ref else None
    if not src or not os.path.isfile(src):
        print("oracle/_ref: MOGE_REFERENCE does not name a reference checkout; the alignment comparator is not built")
        return
    os.makedirs(REF_DIR, exist_ok=True)
    py_compile.compile(src, cfile=ALIGNMENT_PYC, doraise=True)
    print("oracle/_ref: compiled", ALIGNMENT_PYC)


def load_alignment():
    """The reference's alignment module from oracle/_ref/, or None when it was not built.  Its `import utils3d` resolves to
    the stand-in under oracle/utils3d_shim (the solvers do not call it)."""
    if not os.path.isfile(ALIGNMENT_PYC):
        return None
    import importlib.machinery
    import importlib.util
    import sys
    shim = os.path.join(ROOT, "oracle", "utils3d_shim")
    if shim not in sys.path:
        sys.path.append(shim)
    loader = importlib.machinery.SourcelessFileLoader("reference_alignment", ALIGNMENT_PYC)
    spec = importlib.util.spec_from_loader("reference_alignment", loader)
    mod = importlib.util.module_from_spec(spec)
    loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    main()
