"""BASELINE INFRASTRUCTURE ONLY -- a verbatim, git-ignored copy of the UNMODIFIED reference next to the oracle.

    python -m oracle.vendor_ref        (also run by __graft_entry__.build() when /root/reference is mounted)

Copies the reference's Python sources (mikwieczorek/centroids-reid, /root/reference, read-only) verbatim into
``oracle/_ref/``.  That directory is listed in .gitignore -- reference sources never enter this repository's history.
Where the reference tree itself is absent, ``oracle/ref_import.py`` imports this copy (through the same
pytorch_lightning / yacs / mlflow stubs) so that

  * ``bench.py --impl reference`` times the reference's own ``backbone -> bn`` forward and its own
    ``CTLModel.training_step`` on the host cores (``cpu_baseline.kind == "reference"``), and
  * ``python -m oracle.make_golden --only bench_autocast`` can run the reference's own trunk under CUDA fp16 autocast on
    a GPU to regenerate tests/golden/bench_autocast_*.npz.

No test needs it: the tests compare against the committed goldens.

Nothing under centroids-reid_b200/ imports oracle/ or oracle/_ref.
"""
from __future__ import annotations

import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.environ.get("CTL_REFERENCE_SRC", "/root/reference")
DST = os.path.join(HERE, "_ref")
SKIP_DIRS = {".git", "scripts", "train_scripts", "configs", "__pycache__"}


def vendor(src: str = SRC, dst: str = DST) -> int:
    if not os.path.isfile(os.path.join(src, "train_ctl_model.py")):
        return 0
    n = 0
    for root, dirs, files in os.walk(src):
        dirs[:] = [d for d in dirs if d not in SKIP_DIRS]
        rel = os.path.relpath(root, src)
        for f in files:
            if not f.endswith(".py"):
                continue
            out_dir = os.path.join(dst, rel) if rel != "." else dst
            os.makedirs(out_dir, exist_ok=True)
            shutil.copyfile(os.path.join(root, f), os.path.join(out_dir, f))
            n += 1
    with open(os.path.join(dst, "VENDORED_FROM"), "w") as fh:
        fh.write(f"{src}\n{n} python files copied verbatim by oracle/vendor_ref.py\n")
    return n


if __name__ == "__main__":
    k = vendor()
    print(f"vendored {k} reference files into {DST}" if k else f"no reference tree at {SRC}: nothing vendored")
    sys.exit(0)
