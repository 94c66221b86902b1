"""Writes preset_cameras.json: the reference's `utils.trajectory.get_camerapaths()` output as data, so that tests of
luciddreamer_b200.scene can pass LucidDreamer's three preset camera paths without the reference checkout.

Run from the repository root with the reference checkout at REF (default /root/reference). Floats are written with
Python's shortest round-trip repr, so json.load gives back the reference's float64 values exactly.
"""
import json
import os
import sys

REF = os.environ.get("REF", "/root/reference")
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, REF)
from utils.trajectory import get_camerapaths  # noqa: E402


def main():
    presets = get_camerapaths()
    with open(os.path.join(HERE, "preset_cameras.json"), "w") as f:
        json.dump(presets, f, separators=(",", ":"))
    print({k: len(v["frames"]) for k, v in presets.items()})


if __name__ == "__main__":
    main()
