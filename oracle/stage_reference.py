"""TEST / BASELINE INFRASTRUCTURE ONLY — stages the UNMODIFIED reference (ultralytics/yolov3, the read-only checkout at ``SRC``
where it exists) under the git-ignored ``oracle/_ref/`` so that a machine without the original checkout can still run it.  Nothing
under ``yolov3_b200/`` ever imports it; the only consumers are ``bench.py --impl reference`` / ``bench.py``'s ``cpu_baseline``
and ``gpu_library_baseline`` legs (the reference's own ``Model`` / ``non_max_suppression``), which fall back to the oracle
port when nothing is staged.  The tests never need it: what they compare against is stored under ``tests/golden/``.

A file copy, not ``pip install``: the reference's pyproject.toml declares no ``version`` and its layout is a flat script tree
(``models/``, ``utils/``, ``detect.py`` at top level), so it is meant to be run from a clone; a clone of the needed files is
what this makes.  Files are copied byte for byte, never edited, and never enter this repository's history.

    python oracle/stage_reference.py            # no-op when the original is absent or unreadable, or already staged
"""
from __future__ import annotations

import shutil
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
SRC = Path("/root/reference")
DST = ROOT / "oracle" / "_ref"
# what the hot path's callers import: the model/graph code, the utils they pull in, the three loop scripts, YAMLs, the two
# sample images of BASELINE config 1 and the hyper-parameter files ComputeLoss reads
TOP_FILES = ["detect.py", "val.py", "train.py", "hubconf.py", "export.py", "LICENSE"]
TREES = ["models", "utils", "data/hyps", "data/images"]
DATA_FILES = ["data/coco128.yaml", "data/coco.yaml"]


def readable(p: Path) -> bool:
    """exists and may be read by this user (who may lack the permission to look inside the directory that holds it)"""
    try:
        with open(p, "rb"):
            return True
    except OSError:
        return False


def staged() -> bool:
    return readable(DST / "models" / "yolo.py")


def stage(force: bool = False) -> Path | None:
    if not readable(SRC / "models" / "yolo.py"):
        return DST if staged() else None
    if staged() and not force:
        return DST
    if DST.exists():
        shutil.rmtree(DST)
    DST.mkdir(parents=True)
    ignore = shutil.ignore_patterns("__pycache__", "*.pyc", "*.ipynb", "docker", "aws", "google_app_engine", "flask_rest_api")
    for t in TREES:
        if (SRC / t).exists():
            shutil.copytree(SRC / t, DST / t, ignore=ignore)
    for f in TOP_FILES + DATA_FILES:
        if (SRC / f).exists():
            (DST / f).parent.mkdir(parents=True, exist_ok=True)
            shutil.copy2(SRC / f, DST / f)
    (DST / "STAGED_FROM").write_text(f"{SRC} (ultralytics/yolov3 @ 97b87b1), byte-for-byte copy by oracle/stage_reference.py\n")
    return DST


if __name__ == "__main__":
    p = stage(force="--force" in sys.argv)
    print(p if p else "reference not available here and nothing staged")
