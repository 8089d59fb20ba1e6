#!/usr/bin/env python
"""Time of the U-Net planner (NeuralAstar(encoder_arch="Unet"), encoder_depth 4, "m+" input, seeded weights) on an
H100, with the card's name and power limit read in the same run.

Workload: the 100 mazes_032 test problems (tests/golden/mazes032_neural_test.npz, with their
optimal paths for the training rows), b = 100, 32x32.  Rows:
  eager_plane_search   the eager module's cost plane (channels-last cuDNN, F.interpolate + torch.cat per decoder
                       block), then the search on that plane: the route an smp-built U-Net takes;
  fused_forward        planner(...) in eval / no-grad: folded plan, upsample-concat kernel, head products into the
                       search's NASTAR_COST_TAPS prologue;
  graphed_replay       GraphedPlanner.replay() of the same forward;
  upsample_concat      the decoder's four upsample + concat steps, kernel against F.interpolate + torch.cat;
  train_step_eager     one eager training step (PlannerModule, RMSprop, Tmax 0.25);
  train_step_graphed   the same step as a GraphedTrainStep replay.
Each row is the median of 5 windows of CUDA events around `--iters` calls after a warm-up.  The fused forward's launch
count per call comes from a torch.profiler trace of one call in steady state, taken in a separate pass.  Prints one
JSON object; --out also writes it.

    python tools/unet_bench.py [--out profiles/h100_unet_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "neural-astar_b200"), os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in q.split(","))
    return name, power


def _time(fn, iters, windows=5):
    """Median milliseconds per call over `windows` windows of `iters` calls, CUDA events around each window."""
    fn()
    torch.cuda.synchronize()
    per = []
    for _ in range(windows):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        e1.synchronize()
        per.append(e0.elapsed_time(e1) / iters)
    return float(np.median(per))


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out")
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args(argv)
    from golden_util import Golden
    from neural_astar import _native
    from neural_astar.planner import NeuralAstar, encoder
    from neural_astar.utils.inference import GraphedPlanner
    from neural_astar.utils.training import GraphedTrainStep, PlannerModule

    assert torch.cuda.is_available(), "unet_bench needs a GPU"
    dev = torch.device("cuda:0")
    name, power = _card()
    g = Golden("mazes032_neural_test")
    maps, starts, goals = (torch.from_numpy(x).to(dev) for x in (g.obst, g.start, g.goal))
    torch.manual_seed(0)
    planner = NeuralAstar(encoder_arch="Unet", encoder_depth=4, encoder_input="m+").to(dev).eval()
    rows = {}
    with torch.no_grad():
        x = _native.pack_inputs(maps, starts, goals)

        def eager_plane_search():
            planner.encoder.prepare_channels_last()
            cost = torch.sigmoid(planner.encoder.model(x.contiguous(memory_format=torch.channels_last)))
            cost = cost * planner.encoder.const
            return planner.perform_astar(cost, starts, goals, maps)

        rows["eager_plane_search_ms"] = _time(eager_plane_search, args.iters)
        rows["fused_forward_ms"] = _time(lambda: planner(maps, starts, goals), args.iters)
        graphed = GraphedPlanner(planner, maps, starts, goals)
        rows["graphed_replay_ms"] = _time(graphed.replay, args.iters)
        rows["graphed_native_launches_per_replay"] = graphed.native_launches_per_replay

        # the decoder's upsample + concat inputs of this batch: (dec, skip) per block, channels-last
        torch.manual_seed(1)
        shapes = [(512, 2, 512), (256, 4, 256), (128, 8, 128), (64, 16, 0)]    # (Cd, h, Cs) for depth 4 at 32x32
        pairs = []
        for cd, h, cs in shapes:
            dec = torch.randn(100, cd, h, h, device=dev).contiguous(memory_format=torch.channels_last)
            skip = (torch.randn(100, cs, 2 * h, 2 * h, device=dev).contiguous(memory_format=torch.channels_last)
                    if cs else None)
            pairs.append((dec, skip))

        def kernel():
            for dec, skip in pairs:
                _native.upsample_concat(dec, skip)

        def aten():
            for dec, skip in pairs:
                up = F.interpolate(dec, scale_factor=2, mode="nearest")
                if skip is not None:
                    torch.cat((up, skip), 1)

        rows["upsample_concat_kernel_us"] = 1000 * _time(kernel, args.iters)
        rows["upsample_concat_aten_us"] = 1000 * _time(aten, args.iters)
        moved = sum(d.numel() * 4 + (0 if s is None else s.numel() * 4) + 4 * d.numel() * 4
                    + (0 if s is None else s.numel() * 4) for d, s in pairs)
        rows["upsample_concat_bytes"] = moved

    # launches of one steady-state fused forward, from a torch.profiler trace (a separate pass: tracing slows the host)
    from torch.profiler import ProfilerActivity, profile

    with torch.no_grad():
        planner(maps, starts, goals)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            planner(maps, starts, goals)
            torch.cuda.synchronize()
    kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
               and not e.name.startswith(("Memcpy", "Memset"))]
    rows["fused_forward_launches"] = len(kernels)
    rows["fused_forward_kernels"] = sorted({e.name for e in kernels})

    batch = [maps, starts, goals, torch.from_numpy(g.bits("opt_bits").astype(np.float32)).to(dev)]

    def make():
        torch.manual_seed(1234)
        p = NeuralAstar(encoder_arch="Unet", encoder_depth=4, encoder_input="m+", Tmax=0.25)
        return PlannerModule(p, SimpleNamespace(params=SimpleNamespace(lr=1e-3))).to(dev).train()

    module = make()
    opt = module.configure_optimizers()

    def eager_step():
        opt.zero_grad()
        loss = module.training_step(batch, 0)
        loss.backward()
        opt.step()

    rows["train_step_eager_ms"] = _time(eager_step, max(1, args.iters // 5))
    step = GraphedTrainStep(make(), batch)
    rows["train_step_graphed_ms"] = _time(lambda: step(batch), max(1, args.iters // 5))

    result = {"card": name, "power_limit": power, "workload": "mazes_032 test, b=100, 32x32, Unet depth 4, m+",
              "encoder_tf32": encoder.ALLOW_TF32, **rows}
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as f:
            f.write(json.dumps(result) + "\n")


if __name__ == "__main__":
    main()
