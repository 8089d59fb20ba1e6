#!/usr/bin/env python
"""Training-batch sampling on the GPU (csrc/nastar_sampler.cuh, neural_astar.utils.data.DeviceMazeDataset) against the
host loader (create_dataloader / MazeDataset), with the card's name and power limit read in the same run.

Data, all built from what the repository carries: the 100 mazes_032 test maps with their shipped labels
(tests/golden/labels/mazes032_test.npz) and the 400 all_064 test maps (all064_test.npz), each written to a temporary
planning .npz with save_planning_dataset; 1024 Config-5 256x256 maps (tools/c5_data.py, seed 1234) labelled on the
GPU with compute_opt_labels.  Reports:
  * host_loader: create_dataloader(..., 100, shuffle=True) ms per 100-map batch at 32x32, host clock, this host;
  * sample: DeviceMazeDataset.sample alone, CUDA events around 20 back-to-back calls, median of 3 trials, at B = 100
    (32x32, 64x64) and B = 1024 (256x256);
  * prepare: the one-off preparation kernel (CUDA events) and the whole DeviceMazeDataset construction (host clock);
  * train: GraphedTrainStep steps/s over the same number of batches fed by each loader (batch 100, 32x32, Config-3
    planner), the two loaders alternated over 3 rounds in the same session.
Prints one JSON object; --out also writes it to a file.

    python tools/sampler_bench.py [--out profiles/h100_sampler_bench.json]
"""
import argparse
import json
import os
import sys
import tempfile
import time
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "neural-astar_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def timed(fn, reps=20):
    for _ in range(3):
        fn()
    trials = []
    for _ in range(3):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        trials.append(a.elapsed_time(b) / reps)
    return sorted(trials)[1], trials


def power_limit_w(index):
    try:
        import pynvml as nv

        nv.nvmlInit()
        return nv.nvmlDeviceGetEnforcedPowerLimit(nv.nvmlDeviceGetHandleByIndex(index)) / 1e3
    except Exception:
        return "not measured (NVML unavailable)"


def fixture_npz(name, tmp):
    import labels_golden
    from neural_astar.utils.data import save_planning_dataset

    maps, goal_idx, dists, action = labels_golden.load(name)
    B, H, W = maps.shape
    goals = np.zeros((B, 1, H, W), np.float32)
    goals.reshape(B, -1)[np.arange(B), goal_idx] = 1
    pol = np.zeros((B, 8, 1, H, W), np.float32)
    np.put_along_axis(pol, action[:, None, None].astype(np.int64), 1.0, axis=1)
    split = (maps, goals, pol, dists[:, None])
    path = os.path.join(tmp, name + ".npz")
    save_planning_dataset(path, split, split, split)
    return path


def host_loader_ms(path, batches=60):
    from neural_astar.utils.data import create_dataloader

    loader = create_dataloader(path, "train", 100, shuffle=True)
    np.random.seed(0)
    torch.manual_seed(0)
    for _ in loader:
        pass
    t0 = time.perf_counter()
    n = 0
    while n < batches:
        for _ in loader:
            n += 1
    return (time.perf_counter() - t0) * 1e3 / n


def sample_entry(ds, B, dev):
    g = torch.Generator(device=dev)
    g.manual_seed(0)
    idx = torch.randperm(len(ds), device=dev, generator=g)[:B] if B <= len(ds) else torch.randint(
        0, len(ds), (B,), device=dev, generator=g)
    ms, trials = timed(lambda: ds.sample(idx, generator=g))
    H, W = ds.map_designs.shape[-2:]
    out_bytes = 4 * B * H * W * (2 + 2 * ds.num_starts)
    return {"B": B, "grid": f"{H}x{W}", "num_starts": ds.num_starts, "sample_ms": ms, "sample_ms_trials": trials,
            "maps_per_s": B / (ms * 1e-3), "output_bytes": out_bytes, "output_GB_per_s": out_bytes / (ms * 1e-3) / 1e9}


def prepare_entry(make, inputs):
    """(dataset, record): construction on the host clock, then the preparation kernel alone on `inputs`."""
    from neural_astar import _native

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ds = make()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) * 1e3
    kms, _ = timed(lambda: _native.sampler_prepare(*inputs), reps=5)
    return ds, {"maps": len(ds), "prepare_kernel_ms": kms, "construct_ms_host_clock": wall}


def file_inputs(path, dev):
    from neural_astar.utils.data import _percentile_fractions

    with np.load(path) as f:
        _, g, p, d = (torch.from_numpy(f[f"arr_{j}"].astype(np.float32)).to(dev) for j in range(4))
    return d, p, g, _percentile_fractions([0.55, 0.70, 0.85, 1.0])


def train_entry(host_path, dev, steps=40, rounds=3):
    from neural_astar.planner import NeuralAstar
    from neural_astar.utils.data import create_dataloader, create_device_dataloader
    from neural_astar.utils.training import GraphedTrainStep, PlannerModule

    torch.manual_seed(1234)
    planner = NeuralAstar(encoder_input="m+", encoder_arch="CNN", encoder_depth=4, Tmax=0.25)
    module = PlannerModule(planner, SimpleNamespace(params=SimpleNamespace(lr=1e-3))).to(dev).train()
    host = create_dataloader(host_path, "train", 100, shuffle=True)
    g = torch.Generator(device=dev)
    g.manual_seed(0)
    device = create_device_dataloader(host_path, "train", 100, shuffle=True, generator=g)
    step = GraphedTrainStep(module, next(iter(device)))

    def run(loader):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        n = 0
        while n < steps:
            for batch in loader:
                step(batch)
                n += 1
                if n == steps:
                    break
        torch.cuda.synchronize()
        return steps / (time.perf_counter() - t0)

    run(host)
    run(device)
    res = {"host": [], "device": []}
    for _ in range(rounds):
        res["host"].append(run(host))
        res["device"].append(run(device))
    return {"what": "GraphedTrainStep, NeuralAstar m+ CNN depth 4, Tmax 0.25, batch 100 of the 100 mazes_032 test maps "
                    f"(shuffled), {steps} steps per measurement, host clock to a device synchronise, loaders alternated",
            "host_loader_steps_per_s": res["host"], "device_loader_steps_per_s": res["device"],
            "host_loader_steps_per_s_median": float(np.median(res["host"])),
            "device_loader_steps_per_s_median": float(np.median(res["device"]))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from c5_data import c5_maps
    from neural_astar.utils.data import DeviceMazeDataset, _percentile_fractions, compute_opt_labels

    assert torch.cuda.is_available(), "sampler_bench measures the GPU sampler: no GPU found"
    dev = torch.device("cuda:0")
    out = {"kernels": "nastar::sampler_prepare_kernel (once per dataset), nastar::sampler_sample_kernel (once per batch)",
           "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0),
           "timing": "CUDA events around 20 back-to-back calls, median of 3 trials, unless stated"}
    with tempfile.TemporaryDirectory() as tmp:
        p32 = fixture_npz("mazes032_test", tmp)
        p64 = fixture_npz("all064_test", tmp)
        out["host_loader"] = {"what": "create_dataloader(mazes_032 test maps as train split, batch 100, shuffle=True), "
                                      "host clock over 60 batches", "ms_per_batch": host_loader_ms(p32)}

        out["prepare"], out["sample"] = {}, {}
        for name, path in (("mazes_032_test", p32), ("all_064_test", p64)):
            ds, prep = prepare_entry(lambda: DeviceMazeDataset(path, "train", device=dev), file_inputs(path, dev))
            out["prepare"][name] = prep
            out["sample"][name] = sample_entry(ds, 100, dev)
        c5o, _, c5g = c5_maps(1024, 256, 256, 1234)
        md, gm = torch.from_numpy(c5o).to(dev), torch.from_numpy(c5g).to(dev)
        pol, d, _ = compute_opt_labels(md, gm)
        ds, prep = prepare_entry(lambda: DeviceMazeDataset.from_labels(md, gm, pol, d),
                                 (d, pol, gm, _percentile_fractions([0.55, 0.70, 0.85, 1.0])))
        out["prepare"]["c5_256x256"] = prep
        out["sample"]["c5_256x256"] = sample_entry(ds, 1024, dev)
        del ds, pol, d
        out["train"] = train_entry(p32, dev)
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
