"""Compare the machine code of two builds of libmoge_b200 kernel by kernel.

    python tools/compare_sass.py OLD_BUILD_DIR NEW_BUILD_DIR [unit ...]

Each BUILD_DIR is a moge_b200/csrc/build directory (the objects and the `-Xptxas -v` logs build.sh writes), for example one of a
`git worktree` of the parent commit and one of the working tree.  For every unit (default: the op libraries and elementwise) the
`cuobjdump -sass` of each kernel and its ptxas register, spill and shared-memory lines are compared.  Kernels are matched by name
with the anonymous-namespace tag stripped: it hashes the source file, so it changes with any edit of the file.  Prints one line
per unit and exits non-zero when any kernel differs.
"""
import os
import re
import subprocess
import sys

UNITS = ("align", "metrics", "mesh", "panorama", "losses", "elementwise")
CUOBJDUMP = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
ANON = re.compile(r"\d+_GLOBAL__N__[0-9a-f]{8}_\d+_\w+?_cu_[0-9a-f]{8}")


def sass(obj):
    """{kernel: SASS text} of one object file.  Runs of blanks are collapsed: cuobjdump pads its columns to the object's widest
    instruction, so the padding changes with the other kernels of the unit."""
    out = subprocess.run([CUOBJDUMP, "-sass", obj], check=True, capture_output=True, text=True).stdout
    kernels, name = {}, None
    for line in ANON.sub("ANON", out).splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            kernels[name] = []
        elif name is not None:
            kernels[name].append(re.sub(r"[ \t]+", " ", line.strip()))
    return {k: "\n".join(v).strip() for k, v in kernels.items()}


def resources(log):
    """{kernel: ptxas resource lines} of one build log."""
    res, name = {}, None
    with open(log) as f:
        for line in ANON.sub("ANON", f.read()).splitlines():
            m = re.search(r"Compiling entry function '(\S+)'", line)
            if m:
                name = m.group(1)
                res[name] = []
            elif name is not None and re.search(r"registers|spill|smem", line):
                res[name].append(line.split(":", 1)[-1].strip())
    return res


def main(argv):
    if len(argv) < 2:
        sys.exit(__doc__)
    old_dir, new_dir, units = argv[0], argv[1], argv[2:] or UNITS
    differ = False
    for u in units:
        a, b = sass(os.path.join(old_dir, u + ".o")), sass(os.path.join(new_dir, u + ".o"))
        ra, rb = resources(os.path.join(old_dir, u + ".log")), resources(os.path.join(new_dir, u + ".log"))
        bad = sorted(k for k in set(a) | set(b) if a.get(k) != b.get(k) or ra.get(k) != rb.get(k))
        differ |= bool(bad)
        print(f"{u}: {len(a)} kernels, " + ("identical" if not bad else f"{len(bad)} differ: " + ", ".join(bad)))
    sys.exit(1 if differ else 0)


if __name__ == "__main__":
    main(sys.argv[1:])
