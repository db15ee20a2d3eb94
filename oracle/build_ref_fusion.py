"""ORACLE - TEST INFRASTRUCTURE ONLY.  Adds the reference's misc/fusion.py (one Python file; nothing to compile) to the
git-ignored oracle/_ref/ that oracle/build_ref.py makes, so that a machine without the reference sources can still time
and check the reference's own depth-map fusion functions (tools/bench_fusion.py `kind: "reference"`,
tests/test_fusion_cpu.py).  Run after build_ref, which recreates oracle/_ref/; a no-op where the reference is absent.

  python oracle/build_ref_fusion.py
"""
import os
import shutil
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle.build_ref import DST, SRC  # noqa: E402


def build_ref_fusion():
    src = os.path.join(SRC, "misc", "fusion.py")
    dst = os.path.join(DST, "misc", "fusion.py")
    if os.path.isfile(src):
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        shutil.copy2(src, dst)
    return os.path.isfile(dst)


if __name__ == "__main__":
    print("oracle/_ref/misc/fusion.py:", "present" if build_ref_fusion() else "absent")
