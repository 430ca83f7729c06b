"""Stage the UNMODIFIED reference model files into oracle/_ref/ (git-ignored) at build time.

The reference has no setup.py / pyproject; this does what `pip install --target oracle/_ref <reference>` would have done: a
verbatim copy of the importable Python sources (the `models` package, loss.py, Dataloader.py).  The staged copy is what

  * `bench.py --impl reference` times on the host cores (`cpu_baseline.kind == "reference"`), and
  * the boundary tests import: the reference's own `models/image_inpainting.py` / `models/text_segmentation.py` on top of this
    repo's layer library (INTEGRATION.md section 1).

Source directory: $PCB_REFERENCE (default /root/reference).  Tests and the benchmark only ever read the staged copy.
Nothing under oracle/_ref is imported by the product package."""
import filecmp
import os
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.environ.get("PCB_REFERENCE", "/root/reference")
DST = os.path.join(ROOT, "oracle", "_ref")
ITEMS = ["models", "loss.py", "Dataloader.py"]


def stage(verbose=False):
    """Returns the staged directory, or None when the reference is not available here and nothing was staged before."""
    if not os.path.isdir(os.path.join(SRC, "models")):
        return DST if os.path.isdir(os.path.join(DST, "models")) else None
    os.makedirs(DST, exist_ok=True)
    for item in ITEMS:
        s, d = os.path.join(SRC, item), os.path.join(DST, item)
        if not os.path.exists(s):
            continue
        if os.path.isdir(s):
            for dirpath, dirnames, filenames in os.walk(s):
                dirnames[:] = [x for x in dirnames if x != "__pycache__"]
                rel = os.path.relpath(dirpath, s)
                os.makedirs(os.path.join(d, rel), exist_ok=True)
                for f in filenames:
                    if f.endswith(".py") or f.endswith(".md"):
                        a, b = os.path.join(dirpath, f), os.path.join(d, rel, f)
                        if not (os.path.exists(b) and filecmp.cmp(a, b, shallow=False)):
                            shutil.copyfile(a, b)
        elif not (os.path.exists(d) and filecmp.cmp(s, d, shallow=False)):
            shutil.copyfile(s, d)
    if verbose:
        print("reference staged at", DST)
    return DST


def reference_dir():
    """The staged copy of the unmodified reference (None when build() found nothing to stage)."""
    return DST if os.path.isdir(os.path.join(DST, "models")) else None


if __name__ == "__main__":
    print(stage(verbose=True))
    sys.exit(0)
