"""Digests of the deterministic backward's gradients on the scenes of tests/test_blend_bwd_gpu.py, which checks that
the current build reproduces them bit for bit.  Each scene runs in a process of its own (test_blend_bwd_gpu._run).
Run on an H100 with the package built:

    python tests/golden/make_blend_bwd_digests.py [out.json]      (default: tests/golden/blend_bwd_digests.json)

The scenes are generated from CPU seeds and their strip / block choice is the same for every H100 SM count, so the
digests hold on any H100.
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


def digests(scene):
    """{case/gradient index: {shape, dtype, sha256 of the bytes}} of every non-empty gradient of `scene`."""
    with tempfile.TemporaryDirectory() as tmp:
        out = os.path.join(tmp, f"{scene}.npz")
        env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
        subprocess.run([sys.executable, "-s", TEST, scene, out], env=env, check=True, timeout=900)
        g = np.load(out)
        return {k: {"shape": list(g[k].shape), "dtype": str(g[k].dtype),
                    "sha256": hashlib.sha256(g[k].tobytes()).hexdigest()} for k in sorted(g.files)}


if __name__ == "__main__":
    import torch
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "blend_bwd_digests.json")
    sys.path.insert(0, os.path.dirname(TEST))
    from test_blend_bwd_gpu import SCENES
    gold = {"card": torch.cuda.get_device_name(0), "scenes": {s: digests(s) for s in SCENES}}
    with open(path, "w") as f:
        json.dump(gold, f, indent=1, sort_keys=True)
    print(f"{sum(len(v) for v in gold['scenes'].values())} gradients on {gold['card']} -> {path}")
