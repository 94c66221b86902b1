"""Compiles the reference's own Python modules behind `Scene(traindata, gaussians, opt)` to bytecode, from the sources
where they lie under the reference checkout, into oracle/_ref/pyref_scene/ (git-ignored like every other
oracle/_ref output). No reference source text enters the repository.

Test infrastructure only (tests/test_scene_gpu.py): the test imports these modules sourceless and runs the
reference's Scene unchanged beside luciddreamer_b200.scene.build_scene. They live in a directory of their own,
with their own copy of the `scene` and `utils` packages, because the reference's `scene/__init__` imports cv2 and
the camera and dataset modules; putting it into oracle/_ref/pyref would make every import of
`scene.gaussian_model` there (tests/test_dropin_gpu.py) need them too.

    package in pyref_scene/       compiled from (under the reference checkout)
    scene/__init__                scene/__init__.py                 (Scene)
    scene/{dataset_readers,cameras,colmap_loader,gaussian_model}
    utils/{__init__,general,system,graphics,sh,loss,trajectory}
    arguments                     arguments.py                      (GSParams)
"""
import os
import py_compile
import sys

REF = os.environ.get("GS_REFERENCE", "/root/reference")
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref", "pyref_scene")

MODULES = ["scene/__init__.py", "scene/dataset_readers.py", "scene/cameras.py", "scene/colmap_loader.py",
           "scene/gaussian_model.py", "utils/__init__.py", "utils/general.py", "utils/system.py",
           "utils/graphics.py", "utils/sh.py", "utils/loss.py", "utils/trajectory.py", "arguments.py"]


def main() -> int:
    if not os.path.isdir(REF):
        print(f"reference not mounted: {REF}")
        return 1
    for src in MODULES:
        s, d = os.path.join(REF, src), os.path.join(OUT, src + "c")
        os.makedirs(os.path.dirname(d), exist_ok=True)
        # dfile: the traceback path points back at the reference checkout, not into this repo
        py_compile.compile(s, cfile=d, dfile=s, doraise=True)
    print(f"compiled {len(MODULES)} reference modules -> {OUT}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
