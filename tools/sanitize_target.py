"""Small workload for compute-sanitizer (memcheck / racecheck / synccheck): every engine, fwd + bwd."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "neural-astar_b200"), os.path.join(ROOT, "tests")]
import numpy as np, torch
from neural_astar import _native
rng = np.random.RandomState(0)
for (H, W, B) in ((32, 32, 6), (12, 12, 5), (7, 5, 3), (64, 64, 3), (40, 48, 2), (144, 136, 2), (80, 97, 3)):
    obst = (rng.rand(B, 1, H, W) > 0.2).astype(np.float32)
    start = np.zeros_like(obst); goal = np.zeros_like(obst)
    obst[:, 0, 0, 0] = obst[:, 0, -1, -1] = 1; start[:, 0, 0, 0] = 1; goal[:, 0, -1, -1] = 1
    cost = (obst * (0.5 + rng.rand(B, 1, H, W))).astype(np.float32)
    c, s, g, o = (torch.from_numpy(x).cuda() for x in (cost, start, goal, obst))
    for T in (W * W, max(1, (W * W) // 8)):
        hist, paths, ts, ns, tr = _native.forward(c, s, g, o, 0.5, T, True)
        Tb = _native.batch_steps(ts, ns, T)
        gc = _native.backward(c, s, g, o, torch.randn_like(c), Tb, ts, 0.5)
    hist2 = _native.forward(o, s, g, o, 0.5, W * W)[0]   # aliasing path (engine 5 above 64x64)
    pair = _native.forward(c, s, g, o, 0.5, W * W, pair=True, want_counts=True)   # validation pair + counts
    if H <= 64 and W <= 64:                               # fused encoder hand-off: logits / 9-tap products
        lg = torch.randn_like(c)
        _native.forward(lg, s, g, o, 0.5, W * W, cost_kind=_native.COST_LOGIT, cost_scale=10.0)
        taps = torch.randn((B, H, W, 9), device="cuda")
        _native.forward(taps, s, g, o, 0.5, W * W, cost_kind=_native.COST_TAPS, cost_scale=1.0, cost_bias=0.1)
        _native.cost_from_taps(taps, 0.1, 1.0)
    torch.cuda.synchronize()
    print(H, W, "ok", float(hist.sum()), float(gc.abs().sum()) > 0)
# glue kernels
x = torch.randn(3, 64, 12, 12, device="cuda").contiguous(memory_format=torch.channels_last)
_native.head_taps(x, np.ascontiguousarray(rng.randn(64, 9).astype(np.float32)))
m = torch.rand(3, 3, 96, 96, device="cuda"); st = torch.zeros(3, 1, 12, 12, device="cuda"); st[:, :, 0, 0] = 1
_native.pack_inputs(m, st, st)
mm = torch.rand(3, 1, 20, 27, device="cuda"); s1 = torch.zeros_like(mm); s1[:, :, 0, 0] = 1
_native.conv1_marks(mm, s1, s1, rng.randn(9, 2, 32).astype(np.float32), rng.randn(32).astype(np.float32))
torch.cuda.synchronize()
print("glue ok")
# the reference heap A* (nastar_pq.cuh): shared-memory and global-workspace state, unreachable and start == goal maps
for (H, W, B) in ((32, 32, 5), (1, 40, 3), (130, 120, 2), (41, 41, 6), (1, 2001, 3)):   # odd H*W: 8-byte slots
    obst = (rng.rand(B, 1, H, W) > 0.2).astype(np.float32)
    start = np.zeros_like(obst); goal = np.zeros_like(obst)
    obst[:, 0, 0, 0] = obst[:, 0, -1, -1] = 1; start[:, 0, 0, 0] = 1; goal[:, 0, -1, -1] = 1
    goal[1] = start[1]
    obst[0, 0, :, W // 2] = 0
    c, s, g, o = (torch.from_numpy(x).cuda() for x in (rng.rand(B, 1, H, W).astype(np.float32), start, goal, obst))
    _native.pq_astar(c, s, g, o, 0.5)
torch.cuda.synchronize()
print("pq ok")
