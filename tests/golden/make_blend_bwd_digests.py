"""Digests of the deterministic backward's gradients on the scenes and routes of tests/test_blend_bwd_gpu.py, which checks
that the current build reproduces them bit for bit; for a route also the backward kernel slots that launched.  Each
scene or route runs in a process of its own (test_blend_bwd_gpu._run).  Run on an H100 with the package built:

    python tests/golden/make_blend_bwd_digests.py [out.json] [--routes]

(default out.json: tests/golden/blend_bwd_digests.json).  --routes recomputes the routes only and keeps the scenes of the
file as they are.  The scenes are generated from CPU seeds and their strip / block choice is the same for every H100 SM
count, so the digests hold on any H100.
"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
TEST = os.path.join(ROOT, "tests", "test_blend_bwd_gpu.py")


def _child(name, tmp):
    """Runs scene or route `name` in a process of its own; returns the path of its saved gradients."""
    out = os.path.join(tmp, f"{name}.npz")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    subprocess.run([sys.executable, "-s", TEST, name, out], env=env, check=True, timeout=900)
    return out


def _digests(path):
    g = np.load(path)
    return {k: {"shape": list(g[k].shape), "dtype": str(g[k].dtype),
                "sha256": hashlib.sha256(g[k].tobytes()).hexdigest()} for k in sorted(g.files)}


def digests(scene):
    """{case/gradient index: {shape, dtype, sha256 of the bytes}} of every non-empty gradient of `scene`."""
    with tempfile.TemporaryDirectory() as tmp:
        return _digests(_child(scene, tmp))


def route_record(route):
    """{"digests": {route/gradient name: digest}, "launched": sorted backward kernel slots that launched} of `route`."""
    with tempfile.TemporaryDirectory() as tmp:
        out = _child(route, tmp)
        with open(out + ".json") as f:
            return {"digests": _digests(out), "launched": json.load(f)}


if __name__ == "__main__":
    import torch
    args = [a for a in sys.argv[1:] if a != "--routes"]
    path = args[0] if args else os.path.join(HERE, "blend_bwd_digests.json")
    sys.path.insert(0, os.path.dirname(TEST))
    from test_blend_bwd_gpu import ROUTES, SCENES
    card = torch.cuda.get_device_name(0)
    if "--routes" in sys.argv:
        with open(os.path.join(HERE, "blend_bwd_digests.json")) as f:
            gold = json.load(f)
        assert gold["card"] == card, (gold["card"], card)
    else:
        gold = {"card": card, "scenes": {s: digests(s) for s in SCENES}}
    gold["routes"] = {r: route_record(r) for r in ROUTES}
    with open(path, "w") as f:
        json.dump(gold, f, indent=1, sort_keys=True)
    n = sum(len(v) for v in gold["scenes"].values()) + sum(len(v["digests"]) for v in gold["routes"].values())
    print(f"{n} gradients on {gold['card']} -> {path}")
