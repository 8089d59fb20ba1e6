#!/usr/bin/env python
"""Developer probe (round 2): timings of the new paths on one GPU.  Usage: python tools/quick_r2.py [c5|c2|all]"""
import json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "neural-astar_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]
import numpy as np, torch
from neural_astar import _native

what = sys.argv[1] if len(sys.argv) > 1 else "all"


def ev_time(fn, reps=5, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); out = fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(np.min(ts)), out


if what in ("c5", "all"):
    from c5_data import c5_maps
    H = W = 256
    n = int(os.environ.get("C5_MAPS", "1024"))
    t0 = time.time()
    obst, start, goal = c5_maps(n, H, W, 1234)
    gen_s = time.time() - t0
    o, s, g = (torch.from_numpy(x).cuda() for x in (obst, start, goal))
    med, mn, out = ev_time(lambda: _native.forward(o, s, g, o, 0.5, W * W))
    ns = out[3].cpu().numpy()
    print(json.dumps({"c5": {"maps": n, "ms_median": med, "ms_min": mn, "maps_per_s": n / (med * 1e-3),
                             "steps_mean": float(ns.mean()), "steps_max": int(ns.max()), "gen_s": gen_s,
                             "us_per_step_tail": med * 1e3 / ns.max(),
                             "bin16": os.environ.get("NASTAR_B200_BIN16", "1")}}))

if what in ("c2", "all"):
    from golden_util import Golden
    from neural_astar.planner import NeuralAstar
    from neural_astar.utils.inference import GraphedPlanner, PipelinedPlanner
    g_ = Golden("mazes032_vanilla_test")
    state = np.load(os.path.join(ROOT, "tests", "golden", "mazes032_ckpt_planner_state.npz"))
    na = NeuralAstar(encoder_arch="CNN"); na.load_state_dict({k: torch.from_numpy(state[k]) for k in state.files})
    na = na.cuda().eval()
    maps, start, goal = (torch.from_numpy(x).cuda() for x in (g_.obst, g_.start, g_.goal))
    res = {}
    with torch.no_grad():
        res["eager_ms"] = ev_time(lambda: na(maps, start, goal), reps=20, warm=5)[0]
        cost = na.encode(maps, start, goal)
        res["search_plane_us"] = ev_time(lambda: _native.forward(cost, start, goal, maps, 0.5, 1024), reps=20, warm=5)[0] * 1e3
        head = na._head_taps(maps, start, goal)
        res["search_taps_us"] = ev_time(lambda: _native.forward(head[0], start, goal, maps, 0.5, 1024, cost_kind=2, cost_bias=head[1], cost_scale=head[2]), reps=20, warm=5)[0] * 1e3
        res["pack_us"] = ev_time(lambda: _native.pack_inputs(maps, start, goal), reps=20, warm=5)[0] * 1e3
        x = _native.pack_inputs(maps, start, goal)
        res["encoder_to_taps_us"] = ev_time(lambda: na.encoder.head_taps(x), reps=20, warm=5)[0] * 1e3
    fast = GraphedPlanner(na, maps, start, goal)
    res["graph_ms"] = ev_time(lambda: fast.replay(), reps=50, warm=5)[0]
    res["graph_host_ms"] = ev_time(lambda: fast.replay_host(), reps=50, warm=5)[0]
    for host in (False, True):
        pipe = PipelinedPlanner(na, maps, start, goal, host=host)
        pipe.prepare()
        K = 200
        def loop():
            for _ in range(K):
                pipe.submit(maps, start, goal) if not host else pipe.submit()
            return pipe.drain()
        med, mn, _ = ev_time(loop, reps=5, warm=2)
        res["pipe_%s_ms_per_step" % ("host" if host else "dev")] = med / K
    print(json.dumps({"c2": res}))
