#!/usr/bin/env python
"""BB-A*'s black-box backward against the closed-form backward, and BB-A* against Neural A* in training, with the
card's name and power limit read in the same run.

    python tools/bbastar_bench.py --out profiles/h100_bbastar_bench.json [--dataset planning.npz] [--train-steps N]

Rows (CUDA events, median of three trials of `--reps` calls each):
  backward   b = 100 mazes_032 maps (32x32, tests/golden/inputs_mazes032_all1000.npz) and 96 random 64x64 maps, costs
             from a seeded NeuralAstar encoder, training step bound int(0.25 * W * W), g_ratio 0.5, an L1-loss upstream
             gradient: nastar_b200_backward (closed form, given the forward's T_batch and t_solve) against
             nastar_b200_backward_blackbox (one launch), and against the same black-box backward written as PyTorch
             elementwise ops around a _native.forward (w' = cost + lam * g, the search, (y' - y) / lam).
  train      GraphedTrainStep steps/s of NeuralAstar and BBAstar (b = 100, 32x32, Tmax 0.25, CNN depth 4).
  quality    a short seeded training of NeuralAstar and of BBAstar at each --lambdas value (the same initial weights, batches and step count) and the test
             split's p_opt / p_exp / h_mean.  The maps are the 1000 mazes_032 maps of the golden inputs with their
             goals, labelled on the device by compute_opt_labels and sampled by DeviceMazeDataset.from_labels (first
             800 train, last 200 test), or the train / test splits of a planning-dataset .npz given with --dataset.
"""
import argparse
import json
import os
import subprocess
import sys
from types import SimpleNamespace

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, os.path.join(ROOT, "neural-astar_b200"), HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from labels_bench import power_limit_w, timed  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "inputs_mazes032_all1000.npz")


def card():
    """(name, power limit in W) of cuda:0, read now."""
    limit = power_limit_w(0)
    if limit is None:
        try:
            out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                                 capture_output=True, text=True, check=True).stdout
            limit = float(out.strip().splitlines()[0])
        except Exception:
            limit = None
    return torch.cuda.get_device_name(0), limit


def golden_maps(dev):
    """(maps [1000,1,32,32], start [1000,1,32,32], goal [1000,1,32,32]) of the golden mazes_032 inputs."""
    z = np.load(GOLDEN)
    n = z["obst_bits"].shape[0]
    maps = np.unpackbits(z["obst_bits"], axis=1)[:, :1024].reshape(n, 1, 32, 32).astype(np.float32)
    start = np.zeros_like(maps)
    goal = np.zeros_like(maps)
    start.reshape(n, -1)[np.arange(n), z["start_idx"]] = 1
    goal.reshape(n, -1)[np.arange(n), z["goal_idx"]] = 1
    return tuple(torch.from_numpy(x).to(dev) for x in (maps, start, goal))


def random_maps(B, H, W, dev, seed=0):
    rng = np.random.RandomState(seed)
    maps = (rng.rand(B, 1, H, W) > 0.25).astype(np.float32)
    start = np.zeros_like(maps)
    goal = np.zeros_like(maps)
    for b in range(B):
        s, g = rng.choice(H * W, 2, replace=False)
        maps[b, 0].flat[s] = maps[b, 0].flat[g] = 1
        start[b, 0].flat[s] = 1
        goal[b, 0].flat[g] = 1
    return tuple(torch.from_numpy(x).to(dev) for x in (maps, start, goal))


def backward_rows(maps, start, goal, lam, reps):
    """Times of the three backwards for one batch, plus how many cells the black-box gradient moves."""
    from neural_astar import _native
    from neural_astar.planner import NeuralAstar

    B, _, H, W = maps.shape
    torch.manual_seed(0)
    planner = NeuralAstar(Tmax=0.25).to(maps.device).eval()
    with torch.no_grad():
        cost = planner.encode(maps, start, goal).contiguous()
    T = int(0.25 * W * W)
    hist, _, t_solve, n_steps, _ = _native.forward(cost, start, goal, maps, 0.5, T)
    opt = (torch.rand(maps.shape, generator=torch.Generator(device=maps.device).manual_seed(1), device=maps.device)
           > 0.9).float()
    g = torch.sign(hist - opt) / hist.numel()              # d l1_loss(histories, opt) / d histories
    g = g.contiguous()
    T_batch = _native.batch_steps(t_solve, n_steps, T)

    def closed_form():
        return _native.backward(cost, start, goal, maps, g, T_batch, t_solve, 0.5)

    def blackbox():
        return _native.backward_blackbox(cost, start, goal, maps, hist, g, lam, 0.5, T)

    def torch_ops():
        w2 = cost + lam * g
        h2 = _native.forward(w2, start, goal, maps, 0.5, T)[0]
        return (h2 - hist) / lam

    assert torch.equal(blackbox(), torch_ops()), "the PyTorch restatement must give the same gradient"
    rows = {}
    for name, fn in (("closed_form_us", closed_form), ("blackbox_us", blackbox), ("torch_ops_us", torch_ops)):
        med, trials = timed(fn, reps)
        rows[name] = round(med * 1e3, 2)
        rows[name.replace("_us", "_trials_us")] = [round(t * 1e3, 2) for t in trials]
    gbb = blackbox()
    rows.update(B=B, H=H, W=W, T=T, lam=lam, engine=int(_native.lib().nastar_b200_engine_for(H, W)),
                cells_moved_per_map=float((gbb != 0).sum()) / B)
    return rows


def make_module(lam, lr, seed=1234):
    """PlannerModule of NeuralAstar (lam None) or of BBAstar with lambda = lam, from the same seeded weights."""
    from neural_astar.planner import BBAstar, NeuralAstar
    from neural_astar.utils.training import PlannerModule

    torch.manual_seed(seed)
    planner = NeuralAstar(Tmax=0.25, encoder_depth=4) if lam is None else BBAstar(Tmax=0.25, encoder_depth=4,
                                                                                bbastar_lambda=lam)
    return PlannerModule(planner, SimpleNamespace(params=SimpleNamespace(lr=lr))).cuda().train()


def datasets(path, dev):
    from neural_astar.utils.data import DeviceMazeDataset, compute_opt_labels

    if path:
        return DeviceMazeDataset(path, "train", device=dev), DeviceMazeDataset(path, "test", device=dev), path
    maps, _, goal = golden_maps(dev)
    pol, dist, _ = compute_opt_labels(maps, goal)
    make = lambda sl: DeviceMazeDataset.from_labels(maps[sl], goal[sl], pol[sl], dist[sl])   # noqa: E731
    return make(slice(0, 800)), make(slice(800, 1000)), "golden mazes_032 (800 train / 200 test)"


def train_rows(args, dev):
    """GraphedTrainStep steps/s, then a short seeded training and the test metrics, for both planners."""
    from neural_astar.utils.training import GraphedTrainStep, planner_metrics_from_counts

    train, test, source = datasets(args.dataset, dev)
    gen = torch.Generator(device=dev).manual_seed(7)
    n_batches = max(1, len(train) // args.batch)
    order = [torch.randperm(len(train), generator=gen, device=dev)[:n_batches * args.batch].reshape(n_batches, -1)
             for _ in range(-(-args.train_steps // n_batches))]
    batches = [o for perm in order for o in perm][:args.train_steps]
    draws = [torch.randint(-2 ** 31, 2 ** 31, (args.batch, 1, 2), dtype=torch.int32, device=dev, generator=gen)
             for _ in range(len(batches))]
    test_idx = torch.arange(len(test), device=dev)
    test_draws = torch.randint(-2 ** 31, 2 ** 31, (len(test), 1, 2), dtype=torch.int32, device=dev, generator=gen)
    test_batch = test.sample(test_idx, draws=test_draws)
    out = {"dataset": source, "train_steps": len(batches), "batch": args.batch, "lr": args.lr}
    for kind, lam in [("neural_astar", None)] + [(f"bbastar_lambda{lam:g}", lam) for lam in args.lambdas]:
        module = make_module(lam, args.lr)
        step = GraphedTrainStep(module, train.sample(batches[0], draws=draws[0]))
        # steps/s: replays of one fixed batch, the graph alone
        fixed = train.sample(batches[0], draws=draws[0])
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(5):
            step(fixed)
        a.record()
        for _ in range(args.rate_steps):
            step(fixed)
        b.record()
        torch.cuda.synchronize()
        rate = args.rate_steps / (a.elapsed_time(b) / 1e3)
        # the timing replays trained the model: start the seeded run from the same weights again
        module = make_module(lam, args.lr)
        step = GraphedTrainStep(module, train.sample(batches[0], draws=draws[0]))
        losses = []
        for idx, dr in zip(batches, draws):
            losses.append(step(train.sample(idx, draws=dr)).clone())   # the graph overwrites its loss tensor
        losses = torch.stack(losses).detach().cpu().numpy()
        module.eval()
        metrics = []
        with torch.no_grad():
            for s in range(0, len(test), args.batch):
                sl = slice(s, s + args.batch)
                pair = module.planner.forward_pair(test_batch[0][sl], test_batch[1][sl], test_batch[2][sl])
                metrics.append(planner_metrics_from_counts(*pair[2]))
        m = np.mean(np.array(metrics), 0)
        out[kind] = {"graphed_steps_per_s": round(rate, 1), "loss_first": float(losses[0]),
                     "loss_last_100_mean": float(losses[-100:].mean()),
                     "test_p_opt": round(float(m[0]), 4), "test_p_exp": round(float(m[1]), 4),
                     "test_h_mean": round(float(m[2]), 4)}
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", default=None)
    ap.add_argument("--dataset", default=None, help="planning-dataset .npz (train / test splits) instead of the golden maps")
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--batch", type=int, default=100)
    ap.add_argument("--lr", type=float, default=1e-3)
    ap.add_argument("--train-steps", type=int, default=2000)
    ap.add_argument("--rate-steps", type=int, default=200)
    ap.add_argument("--lambdas", type=float, nargs="+", default=[20.0, 5000.0], help="BBAstar's lambdas to train")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bbastar_bench: needs a CUDA device")
    dev = torch.device("cuda", 0)
    name, limit = card()
    torch.backends.cudnn.benchmark = True
    maps, start, goal = golden_maps(dev)
    res = {"device": name, "power_limit_w": limit, "backward": []}
    res["backward"].append(backward_rows(maps[:100], start[:100], goal[:100], 20.0, args.reps))
    res["backward"].append(backward_rows(*random_maps(96, 64, 64, dev), 20.0, args.reps))
    res["train"] = train_rows(args, dev)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
