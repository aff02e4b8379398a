"""Recipe for oracle/_ref: the UNMODIFIED reference, byte-compiled (test / baseline infrastructure, never product).

The reference is a Python repo without packaging (no setup.py / pyproject: `pip install /root/reference` has nothing to
build), so "building" it means compiling its modules to sourceless .pyc files under oracle/_ref/ (git-ignored: no
reference source enters the history).
`__graft_entry__.build()` runs this where a reference checkout exists; elsewhere the tests that need it skip.  Consumers: bench.py's reference arm / cpu_baseline (kind "reference"), tests/test_dropin_reference.py.
Loader with the third-party stubs: oracle/ref_loader.py.
"""
import os
import py_compile
import sys

REF_ROOT = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
# everything the training / editing entry points import (data preparation and visualisation tools are not needed)
TOP_FILES = ["train.py"]
PACKAGES = ["models", "utils", "datasets", "render_tools"]


def build(ref_root=REF_ROOT, out=OUT, quiet=True):
    if not os.path.isdir(ref_root):
        return False
    n = 0
    jobs = [(f, f) for f in TOP_FILES]
    for pkg in PACKAGES:
        for fn in sorted(os.listdir(os.path.join(ref_root, pkg))):
            if fn.endswith(".py"):
                jobs.append((os.path.join(pkg, fn), os.path.join(pkg, fn)))
    for src_rel, dst_rel in jobs:
        src = os.path.join(ref_root, src_rel)
        dst = os.path.join(out, dst_rel[:-3] + ".pyc")
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        # dfile: the path tracebacks show (cites the reference file, as the oracle's comments do)
        py_compile.compile(src, cfile=dst, dfile=os.path.join("reference", src_rel), doraise=True)
        n += 1
    with open(os.path.join(out, "BUILD_INFO"), "w") as f:
        f.write(f"compiled {n} modules of {ref_root} with python {sys.version.split()[0]}\n")
    if not quiet:
        print(f"oracle/_ref: {n} modules")
    return True


if __name__ == "__main__":
    ok = build(quiet=False)
    sys.exit(0 if ok else 1)
