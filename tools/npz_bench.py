#!/usr/bin/env python
"""Time of writing planning datasets with the device deflate (nastar_deflate.cuh; savez_compressed_device, reached
through save_planning_dataset) on an H100, with the card's name and power limit read in the same run, next to the host
path (.cpu() + np.savez_compressed on one host core).

Workloads (all from committed fixtures or seeds, labelled on the device: compute_opt_labels + draw_opt_policies):
  mp_032       the 1000 mazes_032 maps of tests/golden/inputs_mazes032_all1000.npz with their goals, split 800/100/100;
  tiled_064    3200/400/400 64x64 tiles of those maps (tile_maps, t = 2, seeded torch.Generator), goals from
               sample_device_goal_maps; float32, and the same arrays as float64 (tiled_064_f64);
  c5_256       1024 256x256 maps of tools/c5_data.py (seed 1234) with their goals, split 820/102/102.
Per workload: the kernel alone (one launch over the twelve arrays' bytes, CUDA events, median of 3 after warm-up),
save_planning_dataset with CUDA tensors (host clock, warm-up then median of 3), the host path once, and both file
sizes.  Prints one JSON object; --out also writes it to a file.  Files go to a temporary directory.

    python tools/npz_bench.py [--out profiles/h100_npz_bench.json]
"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "neural-astar_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "inputs_mazes032_all1000.npz")


def _label(maps, goals, gen):
    from neural_astar.utils.data import compute_opt_labels, draw_opt_policies

    _, dists, mask = compute_opt_labels(maps, goals)
    return maps, goals, draw_opt_policies(mask, generator=gen), dists


def _splits(arrays, sizes):
    out, a = [], 0
    for n in sizes:
        out.append(tuple(x[a:a + n] for x in arrays))
        a += n
    return out


def workloads(dev):
    """(name, [3 splits of (maps [N,H,W], goals, policies, dists)]) on `dev`, built in order from seeds."""
    from c5_data import c5_maps
    from neural_astar.utils.data import sample_device_goal_maps, tile_maps

    gen = torch.Generator(dev).manual_seed(1234)
    z = np.load(GOLDEN)
    maps = np.unpackbits(z["obst_bits"], axis=1)[:, :1024].reshape(1000, 32, 32).astype(np.float32)
    goal_idx = z["goal_idx"]
    if maps.reshape(1000, -1)[np.arange(1000), goal_idx].min() == 0:
        maps = 1 - maps
    goals = np.zeros((1000, 1, 32, 32), np.float32)
    goals.reshape(1000, -1)[np.arange(1000), goal_idx] = 1
    m32 = torch.from_numpy(maps).to(dev)
    mp = _label(m32, torch.from_numpy(goals).to(dev), gen)
    yield "mp_032", _splits(mp, (800, 100, 100))
    del mp
    t64 = tile_maps(m32, 2, generator=gen, num=4000)
    t64 = t64[:, 0] if t64.ndim == 4 else t64
    tiled = _label(t64, sample_device_goal_maps(t64, 0, generator=gen), gen)
    yield "tiled_064", _splits(tiled, (3200, 400, 400))
    yield "tiled_064_f64", _splits(tuple(x.double() for x in tiled), (3200, 400, 400))
    del tiled, t64
    obst, _, goal = c5_maps(1024, seed=1234)
    c5 = _label(torch.from_numpy(obst[:, 0]).to(dev), torch.from_numpy(goal).to(dev), gen)
    yield "c5_256", _splits(c5, (820, 102, 102))


def member_descriptors(tensors, dev):
    """Descriptors of the tensors' bytes as members with empty heads (the kernel-alone arm and the oracle checks)."""
    from neural_astar import _native

    flat = [t.detach().contiguous().reshape(-1).view(torch.uint8) for t in tensors]
    d = np.zeros(len(flat), _native.DEFLATE_DESC_DTYPE)
    d["data"] = [f.data_ptr() for f in flat]
    d["data_len"] = [f.numel() for f in flat]
    d["chunk0"] = np.concatenate([[0], np.cumsum(_native.deflate_chunk_counts(d["data_len"]))[:-1]])
    return d, torch.from_numpy(d.view(np.uint8).copy()).to(dev), flat


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from labels_bench import timed
    from neural_astar import _native
    from neural_astar.utils.data import save_planning_dataset
    from wlabels_bench import power_limit_w

    assert torch.cuda.is_available(), "npz_bench measures the GPU kernel: no GPU found"
    torch.set_num_threads(1)
    dev = torch.device("cuda:0")
    out = {"kernel": "nastar::deflate_kernel (256 KiB chunks, persistent CTAs, ordered look-back)",
           "timing": "kernel: CUDA events, median of 3 after warm-up; save_planning_dataset: host clock around the "
                     "call (file written and closed), warm-up then median of 3; host path: one call",
           "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0),
           "host_arm": ".cpu() of the 12 CUDA tensors + np.savez_compressed (zlib level 6), one host core"}
    tmp = tempfile.mkdtemp(prefix="npz_bench_")
    for name, splits in workloads(dev):
        tensors = [x for s in splits for x in s]
        raw = sum(t.numel() * t.element_size() for t in tensors)
        d, dd, keep = member_descriptors(tensors, dev)
        k_ms, k_trials = timed(lambda: _native.deflate(d, dd), 1)
        del keep, dd
        pdev, phost = os.path.join(tmp, name + "_dev.npz"), os.path.join(tmp, name + "_host.npz")
        save_planning_dataset(pdev, *splits)
        walls = []
        for _ in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            save_planning_dataset(pdev, *splits)
            walls.append((time.perf_counter() - t0) * 1e3)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        host = [tuple(x.cpu().numpy() for x in s) for s in splits]
        save_planning_dataset(phost, *host)
        host_ms = (time.perf_counter() - t0) * 1e3
        zd, zh = np.load(pdev), np.load(phost)
        assert all(np.array_equal(zd[k], zh[k]) and zd[k].dtype == zh[k].dtype for k in zh.files), name
        dev_ms = sorted(walls)[1]
        out[name] = {"shape": list(tensors[0].shape[1:]), "maps": sum(s[0].shape[0] for s in splits),
                     "dtype": str(tensors[0].dtype).replace("torch.", ""), "raw_bytes": raw,
                     "kernel_ms": k_ms, "kernel_ms_trials": k_trials, "kernel_raw_gb_per_s": raw / (k_ms * 1e6),
                     "device_save_ms": dev_ms, "device_save_ms_trials": walls, "host_save_ms": host_ms,
                     "speedup_end_to_end": host_ms / dev_ms,
                     "device_file_bytes": os.path.getsize(pdev), "host_file_bytes": os.path.getsize(phost),
                     "size_ratio_device_over_host": os.path.getsize(pdev) / os.path.getsize(phost)}
        print(name, json.dumps(out[name]), flush=True)
        os.remove(pdev)
        os.remove(phost)
        del splits, tensors, host, zd, zh
        torch.cuda.empty_cache()
    os.rmdir(tmp)
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
