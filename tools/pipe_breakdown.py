#!/usr/bin/env python
"""Where does the pipelined step's time go?  Times (CUDA events, 200 replays each, inputs rotated through a ring
larger than L2) the three graph variants of PipelinedPlanner — encoder branch alone, search branch alone, both forked (late = before the last conv, and early = at the start of the step) —
plus each encoder kernel issued alone on the stream.  Prints one JSON line."""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "neural-astar_b200"), os.path.join(ROOT, "tests")]
import numpy as np, torch
from neural_astar import _native
from neural_astar.planner import NeuralAstar, encoder as enc_mod
from neural_astar.utils.inference import PipelinedPlanner
from golden_util import Golden

g_ = Golden("mazes032_vanilla_test")
state = np.load(os.path.join(ROOT, "tests", "golden", "mazes032_ckpt_planner_state.npz"))
na = NeuralAstar(encoder_arch="CNN"); na.load_state_dict({k: torch.from_numpy(state[k]) for k in state.files})
na = na.cuda().eval()
maps, start, goal = (torch.from_numpy(x).cuda() for x in (g_.obst, g_.start, g_.goal))
RING = 112
ring = torch.stack([torch.stack([t.roll(i, 0) for t in (maps, start, goal)]) for i in range(RING)])
pipe = PipelinedPlanner(na, maps, start, goal, fork="late")
pipe.prepare()
for k in range(5):
    pipe.submit_stacked(ring[k])
pipe.drain()
torch.cuda.synchronize()


def timed(fn, n=200):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for k in range(5):
        fn(k)
    torch.cuda.synchronize(); a.record()
    for k in range(n):
        fn(k)
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / n * 1e3


res = {}
def dev_step(pp, enc, search):
    def f(k):
        kk = 2 + (k & 1)
        if enc:
            pp._stacked[kk & 1].copy_(ring[k % RING], non_blocking=True)
        pp._graphs[pp._step_graph(kk, False, enc, search)].replay()
    return f
res["enc_graph_us"] = timed(dev_step(pipe, True, False))
res["search_graph_us"] = timed(dev_step(pipe, False, True))
res["full_graph_fork_late_us"] = timed(dev_step(pipe, True, True))
early = PipelinedPlanner(na, maps, start, goal, fork="early"); early.prepare()
for k in range(3): early.submit_stacked(ring[k])
early.drain()
res["full_graph_fork_early_us"] = timed(dev_step(early, True, True))
for fk in ("early", "late"):      # end-to-end variant: H2D(k) || encoder(k-1) || search(k-2) + D2H in each step's graph
    hp = PipelinedPlanner(na, maps, start, goal, host=True, fork=fk); hp.prepare()
    for k in range(4): hp.submit()
    hp.drain()
    res[f"host_step_fork_{fk}_us"] = timed(lambda k: hp._graphs[hp._step_graph(2 + k % 6, True, True, True)].replay())
res["copy_only_us"] = timed(lambda k: pipe._stacked[k & 1].copy_(ring[k % RING], non_blocking=True))

# encoder kernels one by one (eager, back to back on one stream; includes launch gaps when shorter than the CPU issue time)
plan = na.encoder._inference_plan(maps.device)
with torch.no_grad(), enc_mod._conv_flags():
    x0 = [_native.conv1_marks(ring[i][0], ring[i][1], ring[i][2], *plan.conv1).contiguous(memory_format=torch.channels_last) for i in range(4)]
    res["conv1_us"] = timed(lambda k: _native.conv1_marks(ring[k % RING][0], ring[k % RING][1], ring[k % RING][2], *plan.conv1))
    xs = x0
    for li, layer in enumerate(plan.body[1:] + [plan.last], 1):
        w, b, st, pad, dil, relu, pool = layer
        res[f"conv{li + 1}_us"] = timed(lambda k: torch.cudnn_convolution_relu(xs[k & 3], w, b, st, pad, dil, 1))
        xs = [torch.cudnn_convolution_relu(x, w, b, st, pad, dil, 1) for x in xs]
    res["head_us"] = timed(lambda k: _native.head_taps(xs[k & 3], plan.head_w))
    # conv4 immediately followed by the head (the head then finds part of conv4's output in L2)
    w, b, st, pad, dil, relu, pool = plan.last
    x3 = [enc_mod._run_layers(plan.body[1:], x) for x in x0]
    res["conv4_plus_head_us"] = timed(lambda k: _native.head_taps(torch.cudnn_convolution_relu(x3[k & 3], w, b, st, pad, dil, 1), plan.head_w))
    # the same two layers as the one fused kernel the eval path selects with TF32 on (csrc/nastar_convhead.cuh)
    res["conv4_head_fused_us"] = timed(lambda k: _native.conv3x3_head_taps(x3[k & 3], w, b, plan.head_w))
print(json.dumps({k: round(v, 1) for k, v in res.items()}))
