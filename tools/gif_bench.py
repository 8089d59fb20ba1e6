#!/usr/bin/env python
"""Time of search animations with the device GIF path (nastar_gif.cuh; utils.data.search_gifs) on an H100, with the
card's name and power limit read in the same run, next to the host route (store_intermediate_results, then
visualize_results per frame and Pillow's save(save_all=True), on one host core).

Workloads (committed fixtures or seeds):
  mazes_va_each   the 100 mazes_032 test problems (tests/golden/mazes032_vanilla_test.npz), VanillaAstar, one GIF per
                  problem, scale 4, 15 hold frames;
  mazes_na_each   the same with the shipped checkpoint's NeuralAstar (tests/golden/mazes032_ckpt_planner_state.npz);
  mazes_va_grid   one grid GIF of the 100 problems, VanillaAstar;
  c5_each         64 Config-5 256x256 maps (tools/c5_data.py, seed 1234), VanillaAstar, one GIF each, scale 1.
Per workload: the two GIF kernels (CUDA events around both launches, summed, median of 3 calls after a warm-up),
search_gifs end to end (host clock, the search included, median of 3), and the host route once.  The host route for
c5_each runs on the first 2 maps only, since its dense frame tensor is T_batch x 65536 floats per map; its time per
map is reported.  Prints one JSON object; --out also writes it.

    python tools/gif_bench.py [--out profiles/h100_gif_bench.json]
"""
import argparse
import io
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "neural-astar_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in q.split(","))
    return name, power


def _workloads(dev):
    from c5_data import c5_maps
    from golden_util import Golden
    from neural_astar.planner import NeuralAstar, VanillaAstar

    z = Golden("mazes032_vanilla_test")
    mazes = tuple(torch.from_numpy(x).to(dev) for x in (z.obst, z.start, z.goal))
    state = np.load(os.path.join(ROOT, "tests", "golden", "mazes032_ckpt_planner_state.npz"))
    na = NeuralAstar(encoder_arch="CNN")
    na.load_state_dict({k: torch.from_numpy(state[k]) for k in state.files})
    va = VanillaAstar().to(dev).eval()
    c5 = tuple(torch.from_numpy(x).to(dev) for x in c5_maps(64)[:3])
    return {
        "mazes_va_each": (va, mazes, dict(scale=4, hold=15, layout="each"), None),
        "mazes_na_each": (na.to(dev).eval(), mazes, dict(scale=4, hold=15, layout="each"), None),
        "mazes_va_grid": (va, mazes, dict(scale=4, hold=15, layout="grid"), None),
        "c5_each": (va, c5, dict(scale=1, hold=15, layout="each"), 2),
    }


def _host_route(planner, maps, starts, goals, scale, hold, layout, fps=30):
    from PIL import Image

    from neural_astar.utils.data import visualize_results

    problems = [(maps, starts, goals)] if layout == "grid" else [
        (maps[b:b + 1], starts[b:b + 1], goals[b:b + 1]) for b in range(len(maps))]
    total = 0
    for m, s, g in problems:
        out = planner(m, s, g, store_intermediate_results=True)
        frames = [Image.fromarray(visualize_results(m, f, scale)) for f in out.intermediate_results]
        frames += [frames[-1]] * hold
        buf = io.BytesIO()
        frames[0].save(buf, format="GIF", save_all=True, append_images=frames[1:], duration=round(1000 / fps), loop=0)
        total += buf.tell()
    return total


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out")
    args = ap.parse_args(argv)
    from neural_astar import _native
    from neural_astar.utils.data import search_gifs

    assert torch.cuda.is_available(), "gif_bench needs a GPU"
    dev = torch.device("cuda:0")
    name, power = _card()
    torch.set_num_threads(1)
    # CUDA events around the two GIF launches of every search_gifs call
    events = []
    plan, encode = _native.gif_plan, _native.gif_encode

    def timed(fn):
        def run(*a, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = fn(*a, **k)
            e1.record()
            events.append((e0, e1))
            return r
        return run

    _native.gif_plan, _native.gif_encode = timed(plan), timed(encode)
    result = {"card": name, "power_limit": power, "torch_threads": torch.get_num_threads(), "workloads": {}}
    with torch.no_grad():
        for key, (planner, (maps, starts, goals), kw, host_maps) in _workloads(dev).items():
            search_gifs(planner, maps, starts, goals, **kw)
            torch.cuda.synchronize()
            e2e, kern = [], []
            for _ in range(3):
                events.clear()
                t = time.perf_counter()
                gifs = search_gifs(planner, maps, starts, goals, **kw)
                e2e.append(time.perf_counter() - t)
                kern.append(sum(a.elapsed_time(b) for a, b in events) / 1000)
            n = len(maps) if host_maps is None else host_maps
            t = time.perf_counter()
            host_bytes = _host_route(planner, maps[:n], starts[:n], goals[:n], **kw)
            host = time.perf_counter() - t
            row = {"maps": len(maps), "gifs": len(gifs), "bytes": sum(map(len, gifs)),
                   "kernels_s": float(np.median(kern)), "search_gifs_s": float(np.median(e2e)),
                   "host_route_s": host, "host_route_maps": n, "host_route_bytes": host_bytes}
            if host_maps is not None:
                row["host_route_s_per_map"] = host / n
                row["search_gifs_s_per_map"] = row["search_gifs_s"] / len(maps)
            else:
                row["speedup_e2e"] = host / row["search_gifs_s"]
            result["workloads"][key] = row
            print(key, json.dumps(row), file=sys.stderr)
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as f:
            f.write(json.dumps(result) + "\n")


if __name__ == "__main__":
    main()
