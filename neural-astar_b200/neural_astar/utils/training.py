"""Training helpers with the reference's interface (/root/reference/src/neural_astar/utils/training.py).

`PlannerModule` derives from `pytorch_lightning.LightningModule` when Lightning is importable (then
scripts/train.py runs unchanged) and from `nn.Module` otherwise — this image has no Lightning, so a small
`fit()` loop is included.  Optimiser / loss / metrics follow the reference (:42-87): RMSprop(lr),
L1(histories, opt_trajs), and p_opt / p_exp / h_mean measured against VanillaAstar.
"""
from __future__ import annotations

import glob
import random
import re

import numpy as np
import torch
import torch.nn as nn

from .. import _native
from ..planner.astar import VanillaAstar

try:  # pragma: no cover - optional dependency
    import pytorch_lightning as pl
except ImportError:
    pl = None
_ModuleBase = nn.Module if pl is None else pl.LightningModule


def set_global_seeds(seed: int) -> None:
    """Seed torch / numpy / random and make cuDNN deterministic (reference :90-106)."""
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed_all(seed)
        torch.backends.cudnn.benchmark = False
        torch.backends.cudnn.deterministic = True


def load_from_ptl_checkpoint(checkpoint_path: str) -> dict:
    """State dict of the planner inside the newest Lightning *.ckpt below `checkpoint_path`: entries whose key
    mentions 'planner', with everything up to 'planner.' removed (reference :20-39)."""
    newest = sorted(glob.glob(f"{checkpoint_path}/**/*.ckpt", recursive=True))[-1]
    print(f"load {newest}")
    full = torch.load(newest, map_location="cpu", weights_only=False)["state_dict"]
    return {re.split("planner.", name)[-1]: tensor for name, tensor in full.items() if "planner" in name}


def planner_metrics(outputs, va_outputs):
    """(p_opt, p_exp, h_mean) of a planner against vanilla A*, reduced on the device.

    p_opt: share of maps whose path is as long as A*'s; p_exp: mean relative saving in explored nodes
    (clipped at 0); h_mean: their harmonic mean (reference :71-85 does this in NumPy after host copies).
    """
    len_ref, len_out = va_outputs.paths.sum((1, 2, 3)), outputs.paths.sum((1, 2, 3))
    exp_ref = va_outputs.histories.sum((1, 2, 3)).double()
    exp_out = outputs.histories.sum((1, 2, 3)).double()
    p_opt = (len_ref == len_out).double().mean()
    p_exp = ((exp_ref - exp_out) / exp_ref).clamp_min(0.0).mean()
    h_mean = 2.0 / (1.0 / (p_opt + 1e-10) + 1.0 / (p_exp + 1e-10))
    return float(p_opt), float(p_exp), float(h_mean)


def planner_metrics_from_counts(n_closed: torch.Tensor, path_len: torch.Tensor):
    """(p_opt, p_exp, h_mean) from the per-map counts a NASTAR_FWD_PAIR launch wrote: entries [0,B) belong to the
    learned-cost search, [B,2B) to vanilla A* on the same problems (the same formulas as planner_metrics /
    reference :71-85, without reducing the B x H x W masks again)."""
    B = n_closed.numel() // 2
    exp_out, exp_ref = n_closed[:B].double(), n_closed[B:].double()
    p_opt = (path_len[:B] == path_len[B:]).double().mean()
    p_exp = ((exp_ref - exp_out) / exp_ref).clamp_min(0.0).mean()
    h_mean = 2.0 / (1.0 / (p_opt + 1e-10) + 1.0 / (p_exp + 1e-10))
    vals = torch.stack((p_opt, p_exp, h_mean)).tolist()    # one device->host read for the three scalars
    return vals[0], vals[1], vals[2]


def path_cost_metrics(paths: torch.Tensor, cost_maps: torch.Tensor, opt_path_costs: torch.Tensor, rtol: float = 1e-5):
    """(p_opt, cost_ratio) of paths on cost maps against their optimal path costs, reduced on the device.

    paths / cost_maps: [B,...] masks and costs of the same shape (e.g. a planner's `paths` and the true cost maps);
    opt_path_costs: [B], e.g. shortest_path_maps' path_costs.  A path's cost is the fp64 sum of the costs of its
    cells (mask != 0).  p_opt: share of maps whose path costs at most opt * (1 + rtol) -- the fp32 optimum is a
    rounded fold, so an optimal path may sum a few ulps away from it; cost_ratio: mean of path cost / optimum.
    Keep maps with a finite, positive optimum: others give inf or NaN ratios.  One device->host read."""
    B = paths.shape[0]
    mask = paths.detach().reshape(B, -1) != 0
    cost = torch.where(mask, cost_maps.detach().reshape(B, -1).double(), 0.0).sum(1)
    opt = opt_path_costs.detach().reshape(B).double()
    p_opt = (cost <= opt * (1.0 + rtol)).double().mean()
    ratio = (cost / opt).mean()
    vals = torch.stack((p_opt, ratio)).tolist()
    return vals[0], vals[1]


def chamfer_distances(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """Directed Chamfer distances between the cell sets of two masks, on the GPU (include/nastar_b200.h,
    nastar_b200_chamfer; DESIGN.md §23).  a, b: CUDA tensors of one shape, [B,1,H,W] or [B,H,W], of any real,
    integer or bool dtype; a cell belongs to a set iff its value != 0.  Returns fp64 [B,2]: the mean, over A's cells, of
    the Euclidean distance in cells to the nearest cell of B, and the same from B to A.  A map where either set is
    empty gets NaN in both columns.  Exact squared distances, correctly rounded square roots and a fixed summation
    order make the result the same from run to run.  H, W <= 1024.  A metric: no autograd."""
    if a.shape != b.shape:
        raise ValueError(f"chamfer_distances: masks of one shape expected (got {tuple(a.shape)} and {tuple(b.shape)})")
    if a.ndim == 4 and a.shape[1] == 1:
        a, b = a[:, 0], b[:, 0]
    if a.ndim != 3:
        raise ValueError(f"chamfer_distances: masks are [B,1,H,W] or [B,H,W] (got {tuple(a.shape)})")
    if not (a.is_cuda and b.is_cuda) or a.device != b.device:
        raise RuntimeError("chamfer_distances runs on CUDA tensors of one device (there is no CPU fallback)")
    if a.shape[1] > _native.CHAMFER_MAX_SIDE or a.shape[2] > _native.CHAMFER_MAX_SIDE:
        raise ValueError(f"chamfer_distances: H, W <= {_native.CHAMFER_MAX_SIDE} (got {tuple(a.shape[1:])})")
    if a.shape[0] == 0 or a.shape[1] == 0 or a.shape[2] == 0:
        return torch.full((a.shape[0], 2), float("nan"), dtype=torch.float64, device=a.device)
    a, b = a.detach(), b.detach()
    masks = (a != 0).to(torch.uint8) | ((b != 0).to(torch.uint8) << 1)
    return _native.chamfer(masks)


def chamfer_distance(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """The Chamfer distance d(A -> B) + d(B -> A) per map, fp64 [B] (chamfer_distances summed): how far a planned
    path lies from a trajectory, the metric of Neural A*'s raw-image (Stanford Drone) experiment."""
    return chamfer_distances(a, b).sum(1)


class GraphedTrainStep:
    """One training step of scripts/train.py (forward, L1 loss on histories, backward through the search kernels
    and the encoder, RMSprop update; reference utils/training.py:52-61) captured ONCE as a CUDA graph and replayed.

    An eager step issues ~150 small launches from Python (train-mode convs + BatchNorms, their backward, the two
    search kernels, the optimiser's foreach kernels) and is CPU-launch bound at b=100 / 32x32; the replay is one
    launch.  Same arithmetic as the eager step (same kernels, same order).  Fixed batch shape.  Below `g_ratio` 0.5 the
    captured search couples the batch with T_batch decided on the device (`_native.forward_coupled`) where the eager
    step decides it on the host; outputs and gradients are the same.

        step = GraphedTrainStep(module, example_batch)        # module: PlannerModule, in train() mode, on CUDA
        for batch in loader:
            loss = step(batch)                                # device scalar; float(loss) synchronises
    """

    def __init__(self, module, example_batch, warmup: int = 3):
        planner = module.planner
        if not module.training:
            raise ValueError("GraphedTrainStep captures the training step: call module.train() first")
        self.module = module
        dev = next(planner.parameters()).device
        self.optimizer = torch.optim.RMSprop(planner.parameters(), module.config.params.lr, capturable=True)
        self._batch = [torch.empty(x.shape, dtype=x.dtype, device=dev) for x in example_batch]
        for dst, src in zip(self._batch, example_batch):
            dst.copy_(torch.as_tensor(src))
        # warm-up on a side stream (cuDNN autotuning, lazy initialisation, optimiser state), then capture; the
        # parameters are restored afterwards so that constructing the step does not train the model
        saved = [p.detach().clone() for p in planner.parameters()]
        bufs = [b.detach().clone() for b in planner.buffers()]
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(max(1, warmup)):
                self._one_step()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self.optimizer.zero_grad(set_to_none=True)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self._loss = self._one_step(zero=False)
        with torch.no_grad():
            for p, q in zip(planner.parameters(), saved):
                p.copy_(q)
            for b, q in zip(planner.buffers(), bufs):
                b.copy_(q)
        self.optimizer = self._reset_optimizer_state()
        self.replays = 0

    def _one_step(self, zero: bool = True):
        if zero:
            self.optimizer.zero_grad(set_to_none=True)
        loss, _ = self.module._loss(self._batch)
        loss.backward()
        self.optimizer.step()
        return loss

    def _reset_optimizer_state(self):
        # the captured graph updates the optimiser state tensors in place: zero them instead of replacing them
        for st in self.optimizer.state.values():
            for v in st.values():
                if torch.is_tensor(v):
                    v.zero_()
        return self.optimizer

    def __call__(self, batch) -> torch.Tensor:
        for dst, src in zip(self._batch, batch):
            dst.copy_(torch.as_tensor(src), non_blocking=True)
        self.graph.replay()
        self.replays += 1
        return self._loss


class PlannerModule(_ModuleBase):
    def __init__(self, planner, config):
        super().__init__()
        self.planner = planner
        # the validation baseline searches the planner's neighbourhood (forward_pair's vanilla half does too)
        astar = getattr(planner, "astar", None)
        self.vanilla_astar = VanillaAstar(mechanism=getattr(astar, "mechanism", "moore"))
        self.config = config

    # -- Lightning hooks (same names as the reference) ---------------------------------------------
    def forward(self, map_designs, start_maps, goal_maps):
        return self.planner(map_designs, start_maps, goal_maps)

    def configure_optimizers(self) -> torch.optim.Optimizer:
        return torch.optim.RMSprop(self.planner.parameters(), self.config.params.lr)

    def training_step(self, train_batch, batch_idx):
        loss, _ = self._loss(train_batch)
        self._record("metrics/train_loss", loss)
        return loss

    def validation_step(self, val_batch, batch_idx):
        map_designs, start_maps, goal_maps, opt_trajs = val_batch
        pair = None
        if map_designs.shape[1] == 1 and hasattr(self.planner, "forward_pair") and not torch.is_grad_enabled():
            # SURVEY 8(f)-2: the learned-cost search and the vanilla baseline of this batch in ONE launch, metrics
            # from the per-map counts the kernel wrote (reference :63-87 runs two planners and reduces in NumPy)
            pair = self.planner.forward_pair(map_designs, start_maps, goal_maps,
                                             vanilla_g_ratio=self.vanilla_astar.g_ratio)
        if pair is not None:
            outputs, _, counts = pair
            loss = nn.functional.l1_loss(outputs.histories, opt_trajs)
            self._record("metrics/val_loss", loss)
            metrics = planner_metrics_from_counts(*counts)
        else:
            loss, outputs = self._loss(val_batch)
            self._record("metrics/val_loss", loss)
            metrics = None
            if map_designs.shape[1] == 1:  # single-channel maps = shortest-path problems with an A* baseline
                metrics = planner_metrics(outputs, self.vanilla_astar(map_designs, start_maps, goal_maps))
        if metrics is not None:
            for name, value in zip(("p_opt", "p_exp", "h_mean"), metrics):
                self._record(f"metrics/{name}", value)
        return loss

    # -- helpers -----------------------------------------------------------------------------------
    def _loss(self, batch):
        map_designs, start_maps, goal_maps, opt_trajs = batch
        outputs = self.forward(map_designs, start_maps, goal_maps)
        return nn.functional.l1_loss(outputs.histories, opt_trajs), outputs

    def _record(self, name, value):
        if pl is not None:
            self.log(name, value)
        else:
            self.__dict__.setdefault("logged", {})[name] = float(value.detach() if torch.is_tensor(value) else value)

    def fit(self, train_loader, val_loader=None, num_epochs: int = 1, device="cuda"):
        """Plain-PyTorch stand-in for pl.Trainer.fit, driving the same step functions."""
        self.to(device)
        optimiser = self.configure_optimizers()
        curve = []
        for _ in range(num_epochs):
            self.train()
            for i, batch in enumerate(train_loader):
                optimiser.zero_grad(set_to_none=True)
                loss = self.training_step([torch.as_tensor(x).to(device) for x in batch], i)
                loss.backward()
                optimiser.step()
                curve.append(float(loss))
            if val_loader is not None:
                self.eval()
                with torch.no_grad():
                    for i, batch in enumerate(val_loader):
                        self.validation_step([torch.as_tensor(x).to(device) for x in batch], i)
        return curve
