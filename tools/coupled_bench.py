#!/usr/bin/env python
"""The batch-coupled search for g_ratio < 0.5: the host procedure (full-length trace search, host decision, search of
T_batch steps) against the device procedure (_native.forward_coupled), with the card's name and power limit read in
the same run.

    python tools/coupled_bench.py --out profiles/h100_coupled_bench.json

Rows (CUDA events, median of three trials, the two procedures measured alternately in one process on the same inputs):
  search     the 100 mazes_032 test problems with the shipped checkpoint's costs x 10 at g_ratio 0, 0.2 and 0.4, and 100
             all_064 test maps with random costs x 10; Moore and NEWS.  Besides the times: the selection steps the
             two procedures execute (host: B*T + B*T_batch; device: pass 1 + pass 2), which are counts.
  train      GraphedTrainStep steps/s at g_ratio 0.3 against the eager PlannerModule step at 0.3 and the graphed step
             at 0.5 (b = 100 mazes_032 training samples, Tmax 0.25).
--counts-only computes the step counts alone; they need a GPU too (the engine has no CPU path).
"""
import argparse
import ctypes
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, os.path.join(ROOT, "neural-astar_b200"), os.path.join(ROOT, "tests"), HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from labels_bench import power_limit_w, timed  # noqa: E402


def _host(cost, start, goal, obst, g_ratio, T, mech):
    from neural_astar import _native
    from neural_astar.planner.differentiable_astar import _coupled_steps

    T_batch, _ = _coupled_steps(cost, start, goal, obst, g_ratio, T, mech)
    return _native.forward(cost, start, goal, obst, g_ratio, T_batch, no_early_exit=True, mechanism=mech), T_batch


def _device_steps(cost, start, goal, obst, g_ratio, T, mech):
    """(pass-1 steps, pass-2 steps, T_batch): nastar_b200_forward_coupled called with a workspace this tool owns, so
    that pass 1's per-map step counts (the workspace's first B int32 words) can be read back."""
    from neural_astar import _native

    L = _native.lib()
    B, _, H, W = start.shape
    p = _native.FwdParams()
    keep = _native._set_planes(p, (("cost", cost), ("start", start), ("goal", goal), ("obst", obst)))
    p.B, p.H, p.W, p.T = B, H, W, T
    p.g_ratio, p.one_minus_g_ratio, _ = _native.host_scalars(g_ratio, W)
    p.flags = _native.FWD_NEWS if mech == "news" else 0
    nbytes = int(L.nastar_b200_forward_coupled_workspace_bytes(B, H, W, T))
    ws = torch.empty((nbytes,), dtype=torch.uint8, device=cost.device)
    hist = torch.empty((B, 1, H, W), device=cost.device)
    paths = torch.empty((B, 1, H, W), dtype=torch.int64, device=cost.device)
    cnt = torch.empty((3, B), dtype=torch.int32, device=cost.device)
    T_batch = torch.empty((1,), dtype=torch.int32, device=cost.device)
    p.histories, p.paths, p.t_solve, p.n_steps = hist.data_ptr(), paths.data_ptr(), cnt[0].data_ptr(), cnt[1].data_ptr()
    p.workspace, p.workspace_bytes = ws.data_ptr(), nbytes
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _native._check(L.nastar_b200_forward_coupled(ctypes.byref(p), T_batch.data_ptr(), cnt[2].data_ptr(), stream),
                   "nastar_b200_forward_coupled")
    torch.cuda.synchronize()
    del keep
    stop = ws[:4 * B].view(torch.int32).long()
    Tb = int(T_batch.item())
    rerun = stop > Tb
    return int(stop.sum()), int(cnt[1].long()[rerun].sum()), Tb


def _problems(dev):
    from golden_util import Golden
    from neural_astar.planner import NeuralAstar

    g = Golden("mazes032_vanilla_test")
    maps, start, goal = (torch.from_numpy(x).to(dev) for x in (g.obst, g.start, g.goal))
    state = np.load(os.path.join(ROOT, "tests", "golden", "mazes032_ckpt_planner_state.npz"))
    na = NeuralAstar(encoder_arch="CNN")
    na.load_state_dict({k: torch.from_numpy(state[k]) for k in state.files})
    with torch.no_grad():
        cost = na.to(dev).eval().encode(maps, start, goal) * 10
    out = {"mazes032_ckpt_cost_x10": (cost.contiguous(), start, goal, maps)}
    a = Golden("inputs_all064_test400")
    rs = np.random.RandomState(64)
    m64, s64, g64 = (torch.from_numpy(x[:100].copy()).to(dev) for x in (a.obst, a.start, a.goal))
    c64 = torch.from_numpy((rs.rand(100, 1, 64, 64) * 10).astype(np.float32)).to(dev)
    out["all064_random_cost_x10"] = (c64, s64, g64, m64)
    return out


def search_rows(dev, n_timed, counts_only):
    from neural_astar import _native

    rows = {}
    for name, (cost, start, goal, obst) in _problems(dev).items():
        B, W = start.shape[0], start.shape[-1]
        T = W * W
        for mech in ("moore", "news"):
            for g_ratio in (0.0, 0.2, 0.4):
                p1, p2, Tb = _device_steps(cost, start, goal, obst, g_ratio, T, mech)
                row = {"T": T, "T_batch": Tb, "host_steps": B * T + B * Tb, "device_steps": p1 + p2,
                       "device_pass1_steps": p1, "device_pass2_steps": p2}
                if not counts_only:
                    for proc in ("host", "device") * 2:   # alternate; the second pair is kept
                        fn = ((lambda: _host(cost, start, goal, obst, g_ratio, T, mech)) if proc == "host" else
                              (lambda: _native.forward_coupled(cost, start, goal, obst, g_ratio, T, mechanism=mech)))
                        ms, trials = timed(fn, n_timed)
                        row[proc] = {"ms": ms, "trials_ms": trials}
                    row["host_over_device"] = row["host"]["ms"] / row["device"]["ms"]
                rows[f"{name}/{mech}/g{g_ratio}"] = row
    return rows


def train_rows(dev, n_steps=20):
    from types import SimpleNamespace

    from golden_util import Golden
    from neural_astar.planner import NeuralAstar
    from neural_astar.utils.data import DeviceMazeDataset, compute_opt_labels
    from neural_astar.utils.training import GraphedTrainStep, PlannerModule

    g = Golden("mazes032_vanilla_test")
    maps, goal = (torch.from_numpy(x).to(dev) for x in (g.obst, g.goal))
    policies, dists, _ = compute_opt_labels(maps, goal)
    ds = DeviceMazeDataset.from_labels(maps, goal, policies, dists)
    batch = list(ds.sample(torch.arange(100, device=dev), generator=torch.Generator(device=dev).manual_seed(3)))

    def make(g_ratio):
        torch.manual_seed(1234)
        planner = NeuralAstar(g_ratio=g_ratio, encoder_input="m+", encoder_arch="CNN", encoder_depth=4, Tmax=0.25)
        return PlannerModule(planner, SimpleNamespace(params=SimpleNamespace(lr=1e-3))).to(dev).train()

    eager = make(0.3)
    opt = eager.configure_optimizers()

    def eager_step():
        opt.zero_grad()
        loss = eager.training_step(batch, 0)
        loss.backward()
        opt.step()

    graphed = {gr: GraphedTrainStep(make(gr), batch) for gr in (0.3, 0.5)}
    out = {}
    for key, fn in (("eager_g0.3", eager_step), ("graphed_g0.3", lambda: graphed[0.3](batch)),
                    ("graphed_g0.5", lambda: graphed[0.5](batch))) * 2:
        ms, trials = timed(fn, n_steps)
        out[key] = {"ms_per_step": ms, "steps_per_s": 1e3 / ms, "trials_ms": trials}
    out["graphed_over_eager_g0.3"] = out["eager_g0.3"]["ms_per_step"] / out["graphed_g0.3"]["ms_per_step"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    ap.add_argument("--counts-only", action="store_true", help="step counts only, no timing")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("coupled_bench measures the GPU search: no CUDA device")
    dev = torch.device("cuda:0")
    out = {"what": "batch-coupled search (g_ratio < 0.5): host procedure vs forward_coupled, CUDA events, median of 3",
           "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0)}
    out["search_B100"] = search_rows(dev, 20, args.counts_only)
    if not args.counts_only:
        out["train_B100"] = train_rows(dev)
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
