"""ms per densify on LucidDreamer-shaped scenes: the reference's GaussianModel.densify_and_prune (bytecode from
oracle/_ref/pyref) against densify.densify_and_prune, and the first TrainStep.run() after each (the re-capture, which
both arms pay).

The scene is synthetic.make_frustum_scene at each size, SH degree 3; about 100 TrainStep iterations (CUDA graph,
FusedAdam) first make the gradient statistics real. Every round copies that trained model once per arm and densifies
it with LucidDreamer's arguments (0.0002, 0.005, cameras_extent, None) from the same seed; the arms alternate, and the
two results are checked equal. One untimed warm-up round first (library loading, allocator growth); then medians over
rounds, with the min and max beside them.

Traffic model of the device densify: each output row reads and writes its 59 parameter floats and, for the groups
with Adam state, 118 moment floats once: 1 416 bytes per row. The achieved rate is that over the whole call (plan,
count read, map, torch.normal, gather), so it is a lower bound of the gather's own rate; it is given for the median and
for the best round.

    python tools/densify_bench.py --sizes 1000000 2000000 --rounds 5 --out /tmp/densify_bench.json
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import train_bench as TB  # noqa: E402  (puts the repository and the reference bytecode on sys.path)

ROW_BYTES = 4 * 2 * (59 + 118)


def _copy(ref, src):
    """An independent GaussianModel with src's parameters, FusedAdam state and statistics."""
    from luciddreamer_b200 import optim
    gm = ref.GaussianModel(src.max_sh_degree)
    gm.active_sh_degree, gm.percent_dense, gm.spatial_lr_scale = src.active_sh_degree, src.percent_dense, src.spatial_lr_scale
    gm.xyz_scheduler_args = src.xyz_scheduler_args
    attr = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity",
            "scaling": "_scaling", "rotation": "_rotation"}
    groups, state = [], {}
    for g in src.optimizer.param_groups:
        p = nn.Parameter(g["params"][0].detach().clone())
        setattr(gm, attr[g["name"]], p)
        groups.append(dict(g, params=[p]))
        st = src.optimizer.state.get(g["params"][0])
        if st is not None:
            state[p] = {k: v.clone() for k, v in st.items()}
    d = src.optimizer.defaults
    gm.optimizer = optim.FusedAdam(groups, lr=d["lr"], betas=d["betas"], eps=d["eps"])
    for p, st in state.items():
        gm.optimizer.state[p] = st
    for n in ("xyz_gradient_accum", "denom", "max_radii2D"):
        setattr(gm, n, getattr(src, n).clone())
    return gm


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[1_000_000, 2_000_000])
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--train-iters", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("densify_bench needs a GPU")
    from luciddreamer_b200 import densify, optim, train
    dev = torch.device("cuda:0")
    ref = TB._refmods()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    result = dict(gpu=smi, res=a.res, train_iters=a.train_iters, rounds=a.rounds, row_bytes=ROW_BYTES, scenes=[])
    bg = torch.zeros(3, device=dev)
    for P in a.sizes:
        model, cams, opt = TB._scene(ref, P, a.res, a.res, 8, 7, dev)
        base = model()
        optim.attach(base)
        ts = train.TrainStep(base, cams, bg, opt)
        for it in range(1, a.train_iters + 1):
            ts.run(it, it % len(cams))
        ts.check()
        ts.close()
        del ts
        extent = 1.0                                         # the scene's cameras_extent (create_from_pcd(pcd, 1.0))
        args = (0.0002, 0.005, extent, None)
        it0 = a.train_iters + 1
        times = {"reference": [], "device": []}
        recap = {"reference": [], "device": []}
        counts = None
        for r in range(-a.warmup, a.rounds):              # rounds r < 0 warm up both arms and are not recorded
            outs = {}
            for arm in (("reference", "device") if r % 2 == 0 else ("device", "reference")):
                gm = _copy(ref, base)
                if arm == "device":
                    densify.attach(gm)
                step = train.TrainStep(gm, cams, bg, opt)
                torch.cuda.synchronize()
                torch.manual_seed(1234 + r % 1000)
                t0 = time.perf_counter()
                c = gm.densify_and_prune(*args)
                torch.cuda.synchronize()
                if r >= 0:
                    times[arm].append((time.perf_counter() - t0) * 1e3)
                if arm == "device":
                    counts = c
                outs[arm] = [t.detach().clone() for t in (gm._features_rest, gm._opacity, gm._scaling)]
                t0 = time.perf_counter()
                step.run(it0, 1)                             # captures on the densified model
                torch.cuda.synchronize()
                if r >= 0:
                    recap[arm].append((time.perf_counter() - t0) * 1e3)
                step.check()
                step.close()
                del step, gm
            same = [x.shape == y.shape and torch.equal(x, y) for x, y in zip(outs["reference"], outs["device"])]
            assert all(same), ("arms differ", counts, same, [tuple(x.shape) for x in outs["reference"]])
            del outs
            torch.cuda.empty_cache()
        med = {k: float(np.median(v)) for k, v in times.items()}
        best = {k: float(min(v)) for k, v in times.items()}
        row = dict(P=P, counts=counts, densify_ms=med, densify_min_max={k: (min(v), max(v)) for k, v in times.items()},
                   recapture_ms={k: float(np.median(v)) for k, v in recap.items()},
                   recapture_min_max={k: (min(v), max(v)) for k, v in recap.items()},
                   model_bytes=ROW_BYTES * counts["P"],
                   achieved_GBps_whole_call=ROW_BYTES * counts["P"] / (med["device"] * 1e-3) / 1e9,
                   achieved_GBps_whole_call_best=ROW_BYTES * counts["P"] / (best["device"] * 1e-3) / 1e9)
        print(json.dumps(row), flush=True)
        result["scenes"].append(row)
        del base
        torch.cuda.empty_cache()
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(result, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
