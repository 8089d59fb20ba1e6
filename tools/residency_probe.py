#!/usr/bin/env python
"""Does the search run beside the fused 128->256 convolution + head kernel, or after it?

Flagship inputs (the 100 test maps of mazes_032, shipped checkpoint).  Three CUDA graphs, replayed alternately in one
process and timed with CUDA events:
  conv   _native.conv3x3_head_taps on the encoder's conv3 output (the kernel the step graph runs last);
  search the search the step graph launches (NeuralAstar.astar.search_from_taps on that kernel's taps);
  pair   both, the search enqueued first on a side stream, the convolution on the main stream, joined.
If the two kernels share the SMs, `pair` takes about max(conv, search); if a convolution CTA cannot start on an SM
that still holds a search CTA, it takes about conv + search.  Also records the card, its power limit and the SM clock
sampled while each case runs, and a digest of the taps computed alone and beside the search.  Prints one JSON line.

    python tools/residency_probe.py [--rounds 7] [--replays 200]
"""
import argparse
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "neural-astar_b200"), os.path.join(ROOT, "tests")]
import numpy as np  # noqa: E402
import torch  # noqa: E402

from golden_util import Golden  # noqa: E402
from neural_astar import _native  # noqa: E402
from neural_astar.planner import NeuralAstar, encoder as enc_mod  # noqa: E402


def nvml_handle(index):
    import pynvml as nv

    nv.nvmlInit()
    return nv, nv.nvmlDeviceGetHandleByIndex(index)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7, help="alternations of the three cases")
    ap.add_argument("--replays", type=int, default=200, help="graph replays per case and round")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the probe times kernels on a GPU"
    dev = torch.device("cuda", 0)
    nv, h = nvml_handle(0)

    g = Golden("mazes032_vanilla_test")
    maps, start, goal = (torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (g.obst, g.start, g.goal))
    state = np.load(os.path.join(ROOT, "tests", "golden", "mazes032_ckpt_planner_state.npz"))
    na = NeuralAstar(encoder_arch="CNN")
    na.load_state_dict({k: torch.from_numpy(state[k]) for k in state.files})
    na = na.to(dev).eval()
    enc = na.encoder
    with torch.no_grad():
        plan = enc._inference_plan(dev)
        with enc_mod._conv_flags():
            x = enc_mod._run_layers(plan.body[1:], _native.conv1_marks(maps, start, goal, *plan.conv1))
        x3 = x.contiguous(memory_format=torch.channels_last)
    w, b = plan.last.w, plan.last.b
    hw = plan.head_w
    bias, scale = plan.head_b, plan.const
    taps = torch.empty(tuple(maps.shape[:1]) + tuple(maps.shape[2:]) + (9,), device=dev)
    side = torch.cuda.Stream(device=dev)

    def conv():
        _native.conv3x3_head_taps(x3, w, b, hw, out=taps)

    search_taps = _native.conv3x3_head_taps(x3, w, b, hw)   # the search reads its own copy: no race with `conv`

    def search():
        return na.astar.search_from_taps(search_taps, bias, scale, start, goal, maps)

    def pair():
        main_s = torch.cuda.current_stream(dev)
        side.wait_stream(main_s)
        with torch.cuda.stream(side):
            out = search()
        conv()
        main_s.wait_stream(side)
        return out

    with torch.no_grad():
        for fn in (conv, search, pair):     # module loads, heuristic table, allocator pools: all before capture
            fn()
        torch.cuda.synchronize()
        graphs = {}
        for name, fn in (("conv", conv), ("search", search), ("pair", pair)):
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr):
                fn()
            graphs[name] = gr
        for gr in graphs.values():
            gr.replay()
        torch.cuda.synchronize()

    digests = {}
    graphs["conv"].replay()
    torch.cuda.synchronize()
    digests["conv"] = hashlib.sha256(taps.cpu().numpy().tobytes()).hexdigest()
    taps.zero_()
    graphs["pair"].replay()
    torch.cuda.synchronize()
    digests["pair"] = hashlib.sha256(taps.cpu().numpy().tobytes()).hexdigest()

    times = {k: [] for k in graphs}
    clocks = {k: [] for k in graphs}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(args.rounds):
        for name, gr in graphs.items():
            torch.cuda.synchronize()
            ev[0].record()
            for _ in range(args.replays):
                gr.replay()
            ev[1].record()
            clocks[name].append(int(nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM)))   # sampled while it runs
            torch.cuda.synchronize()
            times[name].append(ev[0].elapsed_time(ev[1]) * 1e3 / args.replays)

    med = {k: float(np.median(v)) for k, v in times.items()}
    c, s, p = med["conv"], med["search"], med["pair"]
    name = nv.nvmlDeviceGetName(h)
    line = {
        "gpu": name if isinstance(name, str) else name.decode(),
        "power_limit_w": nv.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0,
        "sm_clock_max_mhz": int(nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM)),
        "sm_clock_mhz_during": {k: int(np.median(v)) for k, v in clocks.items()},
        "lib": os.path.relpath(os.path.realpath(_native.LIB_PATH), ROOT),
        "workload": "b=100 32x32 mazes_032 test maps, shipped checkpoint; CUDA graphs, "
                    f"{args.rounds} alternating rounds x {args.replays} replays, median of rounds",
        "conv_us": round(c, 1), "search_us": round(s, 1), "pair_us": round(p, 1),
        "conv_plus_search_us": round(c + s, 1), "max_us": round(max(c, s), 1),
        # 0 when the pair costs max(conv, search) (the kernels share the SMs), 1 when it costs conv + search
        "serialised_fraction": round((p - max(c, s)) / min(c, s), 3),
        "rounds_us": {k: [round(t, 1) for t in v] for k, v in times.items()},
        "taps_sha256": digests["conv"],
        "taps_equal_beside_search": digests["conv"] == digests["pair"],
    }
    print(json.dumps(line))


if __name__ == "__main__":
    main()
