"""One LucidDreamer training iteration (luciddreamer.py:283-327) on the reference's own GaussianModel, replayed as one CUDA
graph.

    optim.attach(gm)                                   # gm.optimizer becomes a FusedAdam over the same state
    step = TrainStep(gm, cameras, background, opt)     # cameras: the reference's Camera objects, opt: GSParams
    step.run(iteration, cam_index)                     # one graph replay: activate -> rasterize -> L1 + SSIM loss ->
                                                       # backward -> densification statistics -> scheduled Adam
    step.check()                                       # raises if a replay overflowed the pair capacity

The graph reads the raw parameters, the optimiser state and gm.xyz_gradient_accum / denom / max_radii2D in place.  The
reference's densify_and_prune and reset_opacity (scene/gaussian_model.py:210-401) run between iterations, as they are
or on the device after densify.attach(gm) (luciddreamer_b200/densify.py, the same results); either replaces those
tensors, and the next run() re-captures.  So does a change of gm.active_sh_degree.

Iterations that edit the model run with step=False: statistics without the optimiser.  After the edit, step_unchanged()
steps the groups whose Parameter survived it, which is what the reference's optimizer.step() does (every replaced
Parameter has no .grad): nothing after a densify, everything but the opacity after an opacity reset.
"""
from __future__ import annotations

import math
from typing import Optional

import torch

from . import _native as N
from . import graphs
from . import multiview as MV
from . import optim
from . import rasterizer as R

_NAMES = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")


def lr_schedule(schedule, last: int, first: int = 0) -> list:
    """[schedule(i) for i in first..last] as Python floats (doubles): the xyz learning-rate table, taken from the
    model's own scheduler (gm.xyz_scheduler_args), i.e. exactly what update_learning_rate(i) sets."""
    return [float(schedule(i)) for i in range(first, last + 1)]


class TrainStep:
    def __init__(self, gm, cameras, bg: torch.Tensor, opt, pair_capacity: Optional[int] = None, headroom: float = 1.25):
        if not isinstance(gm.optimizer, optim.FusedAdam):
            raise RuntimeError("TrainStep needs gm.optimizer to be an optim.FusedAdam: call optim.attach(gm) first")
        names = [g.get("name") for g in gm.optimizer.param_groups]
        if sorted(names) != sorted(_NAMES):
            raise RuntimeError(f"TrainStep: parameter groups {names} are not GaussianModel.training_setup's")
        self.gm, self.opt, self.cameras = gm, opt, list(cameras)
        self.dev = gm._xyz.device
        self.idx = self.dev.index if self.dev.index is not None else torch.cuda.current_device()
        c0 = self.cameras[0]
        self.W, self.H = int(c0.image_width), int(c0.image_height)
        self.tanfovx, self.tanfovy = math.tan(c0.FoVx * 0.5), math.tan(c0.FoVy * 0.5)
        for c in self.cameras:      # the graph bakes the image size and the field of view in
            if (int(c.image_width), int(c.image_height), math.tan(c.FoVx * 0.5), math.tan(c.FoVy * 0.5)) != \
                    (self.W, self.H, self.tanfovx, self.tanfovy):
                raise RuntimeError("TrainStep: every camera must have the same image size and field of view")
        d, H, W = self.dev, self.H, self.W
        self.bg = bg.detach().to(device=d, dtype=torch.float32).contiguous().clone()
        # static inputs, written in stream order before every replay
        self.viewmatrix = torch.empty(4, 4, device=d)
        self.projmatrix = torch.empty(4, 4, device=d)
        self.campos = torch.empty(3, device=d)
        self.gt = torch.empty(3, H, W, device=d)
        self.iteration = torch.zeros(1, dtype=torch.int32, device=d)
        self.loss3 = torch.zeros(3, device=d)                # [loss, l1, ssim] of the last iteration
        self.dimage = torch.empty(3, H, W, device=d)
        self.loss_scratch = torch.empty(N.lib().gs_photometric_scratch_bytes(H, W), dtype=torch.uint8, device=d)
        o = gm.optimizer                                     # made here, not inside a capture
        o.scratch(d)
        optim.bias_tables(*o.param_groups[0]["betas"], d)
        self.pair_capacity_arg, self.headroom = pair_capacity, float(headroom)
        self.lr_host: list = []
        self.lr_table = None
        self._extend_lr_table(int(getattr(opt, "iterations", 0)))
        self._P = None
        self._graph: Optional[graphs.GraphedStep] = None
        self._key = None
        self._pending = None
        self.captures = 0

    # ---- schedule -----------------------------------------------------------------------------------------------------
    def _extend_lr_table(self, last: int) -> None:
        """xyz learning rate of every iteration 0..last from gm.xyz_scheduler_args itself, i.e. exactly what
        update_learning_rate(iteration) sets (scene/gaussian_model.py:171-177)."""
        n0 = len(self.lr_host)
        if last < n0:
            return
        self.lr_host += lr_schedule(self.gm.xyz_scheduler_args, last, n0)
        self.lr_table = torch.tensor(self.lr_host, dtype=torch.float64, device=self.dev)

    # ---- static buffers -----------------------------------------------------------------------------------------------
    def _ensure_buffers(self) -> None:
        gm = self.gm
        P, M = gm._xyz.shape[0], 1 + gm._features_rest.shape[1]
        if self._P == (P, M):
            return
        d = self.dev
        self.shs = torch.empty(P, M, 3, device=d)
        self.opacities = torch.empty(P, 1, device=d)
        self.scales = torch.empty(P, 3, device=d)
        self.rotations = torch.empty(P, 4, device=d)
        self.bucket = MV.GradBucket(P, M, d)
        self.dm2 = torch.zeros(P, 3, device=d)
        self._P = (P, M)

    def _signature(self, stats: bool):
        gm, o = self.gm, self.gm.optimizer
        ptrs = []
        for g in o.param_groups:
            p = g["params"][0]
            st = o._state(p)
            ptrs += [p.data_ptr(), st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr(), st["step"].data_ptr(),
                     None if g["name"] == "xyz" else float(g["lr"])]
        return (gm._xyz.shape[0], gm.active_sh_degree, bool(stats), R.is_deterministic(self.idx), tuple(ptrs),
                gm._features_dc.data_ptr(), gm._features_rest.data_ptr(), gm._opacity.data_ptr(), gm._scaling.data_ptr(),
                gm._rotation.data_ptr(), gm.xyz_gradient_accum.data_ptr(), gm.denom.data_ptr(),
                gm.max_radii2D.data_ptr(), self.lr_table.data_ptr())

    # ---- one iteration ------------------------------------------------------------------------------------------------
    def _frame(self):
        gm = self.gm
        return R._Frame(self.bg, gm._xyz.detach(), None, self.opacities, self.scales, self.rotations, 1.0, None,
                        self.viewmatrix, self.projmatrix, self.tanfovx, self.tanfovy, self.H, self.W, self.shs,
                        gm.active_sh_degree, self.campos)

    def _activate(self) -> None:
        gm, (P, M) = self.gm, self._P
        N.check(N.lib().gs_activate(R._ctx(self.idx), P, M, gm._features_dc.data_ptr(),
                                    gm._features_rest.data_ptr() if M > 1 else None, gm._opacity.data_ptr(),
                                    gm._scaling.data_ptr(), gm._rotation.data_ptr(), self.shs.data_ptr(),
                                    self.opacities.data_ptr(), self.scales.data_ptr(), self.rotations.data_ptr(),
                                    R._raw_stream(self.idx)))

    def _body(self, stats: bool, step: bool):
        """activate -> forward -> loss -> backward [-> statistics] [-> Adam], all stream work.  Returns the forward's
        (image buffer, pair capacity): the guard of the state updates."""
        gm, L, idx = self.gm, N.lib(), self.idx
        ctx, s = R._ctx(idx), R._raw_stream(idx)
        P = self._P[0]
        self._activate()
        frame = self._frame()
        fwd = R._forward(*frame, False, False)
        img, cap = fwd.img, fwd.pair_capacity
        N.check(L.gs_photometric_loss_backward(ctx, fwd.color.data_ptr(), self.gt.data_ptr(), self.H, self.W,
                                               float(self.opt.lambda_dssim), self.loss_scratch.data_ptr(),
                                               self.dimage.data_ptr(), self.loss3.data_ptr(), s))
        b = self.bucket
        R._backward(frame, fwd, self.dimage, dm3=b.means3D, dm2=self.dm2, dop=b.opacities, dsh=b.shs, dsc=b.scales,
                    drot=b.rotations)
        if stats:
            N.check(L.gs_densify_stats_guarded(ctx, P, fwd.radii.data_ptr(), self.dm2.data_ptr(),
                                               gm.xyz_gradient_accum.data_ptr(), gm.denom.data_ptr(),
                                               gm.max_radii2D.data_ptr(), img.data_ptr(), self.W, self.H, cap, s))
        if step:
            self._adam(_NAMES, (img, self.W, self.H, cap))
        return img, cap

    def _adam(self, names, guard) -> None:
        self.gm.optimizer.step_activated(self.bucket, names=names, lr_tables={"xyz": self.lr_table},
                                         iteration=self.iteration, guard=guard)

    def _pair_capacity(self) -> int:
        """Pairs of the largest view over all cameras (one forward each) x headroom, unless given."""
        if self.pair_capacity_arg is not None:
            return int(self.pair_capacity_arg)
        peak = 0
        frame = self._frame()
        for c in self.cameras:
            view = frame._replace(viewmatrix=c.world_view_transform, projmatrix=c.full_proj_transform,
                                  campos=c.camera_center)
            peak = max(peak, int(R._forward(*view, False, False).num_pairs))
        return R._binding().pair_capacity(peak, headroom=self.headroom)

    def _capture(self, stats: bool) -> None:
        self._key = None
        self.close()                         # reports an overflow of the last replay, frees the graph, its pool and slots
        with R._guard(self.idx):
            self._activate()                 # the activated values the capacity sweep renders
            cap = self._pair_capacity()

        def fn():
            # GraphedStep warms up by running fn eagerly: only the capture may carry the state updates
            capturing = torch.cuda.is_current_stream_capturing()
            self._body(stats and capturing, capturing)

        self._graph = graphs.GraphedStep(fn, pair_capacity=cap, warmup=2, device=self.idx)
        self.captures += 1

    def _load(self, iteration: int, cam_index: int) -> None:
        self._extend_lr_table(iteration)
        for g in self.gm.optimizer.param_groups:
            if g["name"] == "xyz":
                g["lr"] = self.lr_host[iteration]          # what update_learning_rate(iteration) sets
        c = self.cameras[cam_index]
        self.viewmatrix.copy_(c.world_view_transform)
        self.projmatrix.copy_(c.full_proj_transform)
        self.campos.copy_(c.camera_center)
        self.gt.copy_(c.original_image)
        self.iteration.fill_(int(iteration))

    def run(self, iteration: int, cam_index: int, stats: bool = True, step: bool = True) -> None:
        """One iteration on camera `cam_index`: forward, loss, backward, then the densification statistics (stats) and
        the optimiser step (step).  step=False runs the iteration eagerly without the optimiser; call step_unchanged()
        after editing the model (or nothing, on the last iteration, luciddreamer.py:325)."""
        if iteration < 0:
            raise ValueError("iteration must be >= 0")
        with R._guard(self.idx):
            self._pending = None
            self._ensure_buffers()
            self._load(iteration, cam_index)
            if not step:
                params = {g["name"]: g["params"][0] for g in self.gm.optimizer.param_groups}
                self._pending = (self._body(stats, False), params)
                return
            key = self._signature(stats)
            if key != self._key or self._graph is None:
                self._capture(stats)
                self._key = key
            self._graph.replay()

    def step_unchanged(self) -> None:
        """The optimiser step of the last run(step=False), for the groups whose Parameter is still the one that was
        rendered (the reference's optimizer.step() skips every Parameter replaced since the backward: grad is None)."""
        if self._pending is None:
            raise RuntimeError("step_unchanged() follows run(..., step=False)")
        guard, params = self._pending
        self._pending = None
        o = self.gm.optimizer
        keep = [g["name"] for g in o.param_groups if g["params"][0] is params[g["name"]]]
        if keep:
            with R._guard(self.idx):
                self._adam(keep, (guard[0], self.W, self.H, guard[1]))

    def close(self) -> None:
        """Checks the last replay (raises if it overflowed, after the release), then destroys the captured graph and
        returns its memory pool and status slots.  run() captures again when it is called next."""
        old, self._graph = self._graph, None
        if old is not None:
            try:
                old.check()
            finally:
                old.release()

    def __del__(self):
        try:
            if self._graph is not None:
                self._graph.release()
        except Exception:           # interpreter shutdown: the library or the device may already be gone
            pass

    def check(self) -> dict:
        """Synchronises and verifies the most recent replay (raises if its frame overflowed the pair capacity, in which
        case that iteration left the model unchanged); returns its counts."""
        if self._graph is None:
            torch.cuda.synchronize(self.idx)
            return {}
        return self._graph.check()
