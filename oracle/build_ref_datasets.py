"""ORACLE - TEST INFRASTRUCTURE ONLY.  Adds the reference's eval loader, datasets/general_eval.py and datasets/data_io.py
(Python files; nothing to compile), to the git-ignored oracle/_ref/ that oracle/build_ref.py makes, so that a machine
without the reference sources can still time the reference's own loader and file writers (tools/bench_scene.py's
reference arm).  Run after build_ref, which recreates oracle/_ref/; a no-op where the reference is absent.  Nothing in the
package imports them.

  python oracle/build_ref_datasets.py
"""
import os
import shutil
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle.build_ref import DST, SRC  # noqa: E402

FILES = ("general_eval.py", "data_io.py")


def build_ref_datasets():
    for name in FILES:
        src = os.path.join(SRC, "datasets", name)
        if os.path.isfile(src):
            os.makedirs(os.path.join(DST, "datasets"), exist_ok=True)
            shutil.copy2(src, os.path.join(DST, "datasets", name))
    return all(os.path.isfile(os.path.join(DST, "datasets", n)) for n in FILES)


if __name__ == "__main__":
    print("oracle/_ref/datasets:", "present" if build_ref_datasets() else "absent")
