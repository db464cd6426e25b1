"""Recipe for oracle/_ref/: the reference's OWN Python files, byte for byte, as a build product.

The reference is pure Python (SURVEY.md §0: no native code, nothing to compile), so "building the reference" means
placing the unmodified files of a reference checkout (IGMC_REFERENCE_DIR) where the tree can import them:

    python oracle/make_ref.py            # $IGMC_REFERENCE_DIR -> oracle/_ref/{util_functions.py, Main.py}

oracle/_ref/ is git-ignored: no reference source enters the history.  Users: oracle/ref_shim.py, bench.py's CPU arm
(extraction = the reference's own subgraph_extraction_labeling + construct_pyg_graph,
`cpu_baseline.extraction_kind = "reference"`), tests/golden/make_golden.py, and tests/test_gpu_main_script.py (runs
the unmodified Main.py on the drop-in modules).  __graft_entry__.build() calls this; without a readable reference
checkout it does nothing.
"""
import hashlib
import os
import shutil
import sys

SRC = os.environ.get("IGMC_REFERENCE_DIR", "/root/reference")
DST = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")
FILES = ("util_functions.py", "Main.py")


def make(verbose=False):
    if not os.path.isfile(os.path.join(SRC, FILES[0])):
        return False
    os.makedirs(DST, exist_ok=True)
    lines = []
    for f in FILES:
        shutil.copyfile(os.path.join(SRC, f), os.path.join(DST, f))
        with open(os.path.join(DST, f), "rb") as fh:
            lines.append("%s  %s" % (hashlib.sha256(fh.read()).hexdigest(), f))
    with open(os.path.join(DST, "SHA256SUMS"), "w") as fh:
        fh.write("\n".join(lines) + "\n")
    if verbose:
        print("\n".join(lines))
    return True


if __name__ == "__main__":
    ok = make(verbose=True)
    sys.exit(0 if ok else 1)
