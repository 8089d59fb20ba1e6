"""NeuralAstar's U-Net encoder on the GPU against the reference's own NeuralAstar run in float64, stage by stage, on the
matrix of tests/test_unet_reference_cpu.py: depths 1 to 5, "m" and "m+" inputs on square, non-square and the smallest
legal grids, "rgb+", a learnable const with and without learn_obstacles, and 128 x 128 maps above TAPS_MAX_SIDE.

Every configuration runs its eval fast path with TF32 on (the default), off, and with the head kernel off.  Per case:
  graph     the fast path's recorded calls (pack_inputs, every folded conv, max pool, upsample_concat, head_taps<C> or
            torch.mm, cost_from_taps) are the reference's graph for the depth, and conv1_marks and conv3x3_head_taps
            never run;
  stages    the first conv's input is the reference's encoder input bit for bit, and every stage meets its bound
            (test_unet_reference_cpu.stage_ratios) evaluated in float64 on the GPU;
  forward   forward() with either mechanism equals perform_astar(encode()) bit for bit and the staged reference's fp32
            DifferentiableAstar on that cost (not at 128 x 128, where forward() does not hand the taps to the search and
            the reference's stored search frames would fill gigabytes); a GraphedPlanner replay equals it;
  cuDNN     the kernels every conv of the plan runs, from torch.profiler; those run as Winograd or FFT transforms,
            whose rounding the stage bound does not model, are listed apart.
The plan follows load_state_dict at depths 1 and 5.  head_taps and upsample_concat are also checked directly at the
pixel counts, channel counts and grid shapes the U-Net does not reach.  The worst |error| / bound of every configuration
and mode, and the cuDNN kernels each layer ran, are printed at teardown.
"""
import numpy as np
import pytest
import scipy.ndimage
import torch
import torch.nn.functional as F

import test_encoder_reference_cpu as er
import test_reference_parity_cpu as rp
import test_unet_reference_cpu as ur
from test_gpu_convhead import U_TF32
from test_gpu_reference_parity import _forward_matches
from test_gpu_unet import _decoder_shapes, _grid_cap_items
from test_unet_reference_cpu import CONFIGS, UConfig

pytestmark = pytest.mark.gpu

MODES = ("tf32", "fp32", "nohead")
CASES = [(c, m) for c in CONFIGS for m in MODES]
FORWARD = [(c, mech) for c in CONFIGS for mech in ("moore", "news")]
PROFILED = [(c, m) for c in CONFIGS if c.inp == "m+" and c.const is None for m in ("tf32", "fp32")]
INVALIDATION = [UConfig("m+", 1, (32, 96)), UConfig("m+", 5, (64, 64))]
WORST = {}          # (config id, mode) -> (worst |error| / bound, its stage)
KERNELS = {}        # (config id, mode) -> [(stage, cuDNN kernels)]
TRANSFORMS = []     # convs that cuDNN ran as a Winograd or FFT transform
_CACHE = {}         # config id -> (float64 reference on the GPU, its encoder input, NumPy inputs); the latest only


@pytest.fixture(scope="module")
def native():
    from neural_astar import _native

    _native.lib()
    return _native


@pytest.fixture(scope="module")
def ref_astar():
    mod = er.staged_encoder_reference()
    if mod is None:
        pytest.skip("the reference's astar.py / encoder.py are not staged in oracle/_ref/ (build() stages them)")
    return mod


@pytest.fixture(scope="module")
def search_ref():
    ref = rp.staged_reference()
    if ref is None:
        pytest.skip("the reference is not staged in oracle/_ref/")
    return ref


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for key in sorted(WORST):
        print(f"\n{key[0]} {key[1]}: worst |error| / bound {WORST[key][0]:.4f} ({WORST[key][1]})")
    for mode in sorted({k[1] for k in WORST}):
        print(f"\nworst over {mode}: {max(v[0] for k, v in WORST.items() if k[1] == mode):.4f}")
    for key in sorted(KERNELS):
        print(f"\ncuDNN kernels {key[0]} {key[1]}:")
        for stage, names in KERNELS[key]:
            print(f"  {stage}: {' + '.join(names)}")
    print(f"\nconvs run as a Winograd or FFT transform, which the stage bound does not model: {len(TRANSFORMS)}")
    for line in TRANSFORMS:
        print(f"  {line}")


def _cu(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _reference(ref_astar, cfg):
    """The configuration's float64 reference on the GPU, its encoder input and the NumPy inputs, built once for all
    the tests of a configuration in a row (never mutated)."""
    if cfg.id not in _CACHE:
        _CACHE.clear()
        ref = ur.build_reference(ref_astar, cfg, cfg.seed, device="cuda")
        maps, start, goal = er.inputs(cfg, cfg.seed)
        x, _ = er.encoder_input(ref, *(_cu(v).double() for v in (maps, start, goal)))
        _CACHE[cfg.id] = (ref, x, (maps, start, goal))
    return _CACHE[cfg.id]


def _set_mode(mp, mode):
    from neural_astar.planner import encoder as enc

    mp.setattr(enc, "ALLOW_TF32", mode != "fp32")
    mp.setattr(enc, "HEAD_KERNEL", mode != "nohead")


def _record(mp, native):
    """Record the fast path's calls, in order: names in `calls`, outputs in `outs`, (layer, input) of every conv in
    `convs`.  conv1_marks and conv3x3_head_taps fail the test."""
    from neural_astar.planner import encoder as enc

    calls, outs, convs = [], [], []

    def recorded(name, real):
        def call(*a, **k):
            y = real(*a, **k)
            calls.append(f"head_taps<{a[0].shape[1]}>" if name == "head_taps" else name)
            outs.append(y)
            if name == "conv":
                convs.append(a)
            return y
        return call

    mp.setattr(enc, "_conv", recorded("conv", enc._conv))
    mp.setattr(enc.F, "max_pool2d", recorded("pool", enc.F.max_pool2d))
    mp.setattr(torch, "mm", recorded("mm", torch.mm))
    for name, kind in (("pack_inputs", "pack"), ("upsample_concat", "upcat"), ("head_taps", "head_taps"),
                       ("cost_from_taps", "cost")):
        mp.setattr(native, name, recorded(kind, getattr(native, name)))
    for name in ("conv1_marks", "conv3x3_head_taps"):
        mp.setattr(native, name, lambda *a, _n=name, **k: pytest.fail(f"{_n} ran on the U-Net's fast path"))
    return calls, outs, convs


def expected_calls(ref, cfg, mode):
    """The reference's graph as the fast path's calls."""
    head = "mm" if mode == "nohead" else f"head_taps<{cfg.head_channels}>"
    names = {"conv": "conv", "pool": "pool", "upcat": "upcat", "taps": head, "cost": "cost"}
    graph = [names[n.kind] for n in ur.reference_graph(ref.encoder.model, fast=True)]
    return (["pack"] if "+" in cfg.inp else []) + graph


def _encode_recorded(na, native, cfg, mode, m, s, g):
    with pytest.MonkeyPatch.context() as mp:
        _set_mode(mp, mode)
        calls, outs, convs = _record(mp, native)
        with torch.no_grad():
            cost = na.encode(m, s, g)
        torch.cuda.synchronize()
    return calls, outs, convs, cost


def _check_stages(ref, x, cfg, mode, calls, outs, convs, key):
    assert calls == expected_calls(ref, cfg, mode), (key, calls)
    assert calls.count("upcat") == cfg.depth
    assert torch.equal(convs[0][1].double(), x), "the first conv's input is not the reference's encoder input"
    if calls[0] == "pack":
        assert torch.equal(outs[0].double(), x)
        outs = outs[1:]
    stages = ur.stage_ratios(ref, x, outs, fast=True, u_op=0.0 if mode == "fp32" else U_TF32)
    worst = max(stages, key=lambda st: st.ratio)
    WORST[key] = max(WORST.get(key, (0.0, "")), (worst.ratio, worst.name))
    bad = [st for st in stages if not st.ratio <= 1.0]
    assert not bad, (key, bad)


@pytest.mark.parametrize("cfg,mode", CASES, ids=[f"{c.id}-{m}" for c, m in CASES])
def test_fast_path_stages_match_reference(native, ref_astar, cfg, mode):
    ref, x, (maps, start, goal) = _reference(ref_astar, cfg)
    na = ur.build_product(ref, cfg).cuda()
    m, s, g = (_cu(v) for v in (maps, start, goal))
    calls, outs, convs, cost = _encode_recorded(na, native, cfg, mode, m, s, g)
    assert tuple(cost.shape) == (cfg.B, 1) + cfg.grid and outs[-1] is cost
    _check_stages(ref, x, cfg, mode, calls, outs, convs, (cfg.id, mode))


@pytest.mark.parametrize("cfg,mech", FORWARD, ids=[f"{c.id}-{m}" for c, m in FORWARD])
def test_forward_matches_encode_and_reference_search(native, ref_astar, search_ref, monkeypatch, cfg, mech):
    from neural_astar.utils.inference import GraphedPlanner

    ref, _, (maps, start, goal) = _reference(ref_astar, cfg)
    na = ur.build_product(ref, cfg, mechanism=mech).cuda()
    m, s, g = (_cu(v) for v in (maps, start, goal))
    searched = []
    real = na.astar.search_from_taps
    monkeypatch.setattr(na.astar, "search_from_taps", lambda *a, **k: searched.append(1) or real(*a, **k))
    passable = torch.ones_like(s) if cfg.learn_obstacles else m
    with torch.no_grad():
        out = na(m, s, g)
        cost = na.encode(m, s, g)
        unfused = na.perform_astar(cost, s, g, passable)
    small = max(cfg.grid) <= native.TAPS_MAX_SIDE
    assert searched == ([1] if small else []), "forward() handed the search the taps it cannot read, or did not"
    assert torch.equal(out.histories, unfused.histories) and torch.equal(out.paths, unfused.paths)
    hist, paths = out.histories.cpu().numpy(), out.paths.cpu().numpy()
    # the reference's NEWS heuristic (planning_datasets' mechanism) takes square maps only, and its backtrack fails on a
    # goal the search cannot reach: the inputs' goals lie in their start's 8-connected region, not always 4-connected
    keep = np.arange(cfg.B)
    if mech == "news":
        structure = np.array([[0, 1, 0], [1, 1, 1], [0, 1, 0]])
        passable_np = passable.cpu().numpy()[:, 0]
        labels = [scipy.ndimage.label(passable_np[b], structure=structure)[0] for b in range(cfg.B)]
        keep = np.array([b for b in keep if labels[b].flat[start[b, 0].argmax()] == labels[b].flat[goal[b, 0].argmax()]])
    if cfg.grid != (128, 128) and (mech == "moore" or cfg.grid[0] == cfg.grid[1]):
        p = rp.Problem(mech, 0.5, 1.0, False, cost.cpu().numpy()[keep], start[keep], goal[keep],
                       passable.cpu().numpy()[keep], np.zeros_like(start[keep]))
        _forward_matches(hist[keep], paths[keep], rp.run_reference(search_ref, p, torch.float32), p, (cfg.id, mech))
    if small:
        replay = GraphedPlanner(na, m, s, g).replay()
        assert torch.equal(replay.histories, out.histories) and torch.equal(replay.paths, out.paths)


@pytest.mark.parametrize("cfg,mode", PROFILED, ids=[f"{c.id}-{m}" for c, m in PROFILED])
def test_cudnn_kernels_recorded(native, ref_astar, cfg, mode):
    """Each conv of the plan, run again with the cuDNN settings of the fast path (its autotuned choice cached for the
    shape), under torch.profiler: the kernels it launches, printed at teardown.  The stage bound models a direct or
    implicit-GEMM convolution (every output a sum of 9 C_in products).  Winograd and FFT transforms round differently,
    and the autotuner may pick them (on an H100 80GB HBM3 it picked FFT for a 384 -> 64 conv on 8 x 8 maps
    with TF32 off): those convs are listed apart, and
    their stages are held to the same bound by test_fast_path_stages_match_reference, without a derivation for the
    transform."""
    from torch.profiler import ProfilerActivity, profile

    from neural_astar.planner import encoder as enc

    ref, _, (maps, start, goal) = _reference(ref_astar, cfg)
    na = ur.build_product(ref, cfg).cuda()
    m, s, g = (_cu(v) for v in (maps, start, goal))
    real_conv = enc._conv
    _, _, convs, _ = _encode_recorded(na, native, cfg, mode, m, s, g)
    names = [n.name for n in ur.reference_graph(ref.encoder.model, fast=True) if n.kind == "conv"]
    assert len(names) == len(convs)
    found = []
    with pytest.MonkeyPatch.context() as mp, torch.no_grad():
        _set_mode(mp, mode)
        for name, (layer, x) in zip(names, convs):
            kernels = []
            for _ in range(5):                  # a profiling session now and then records no device activity
                with enc._conv_flags():
                    with profile(activities=[ProfilerActivity.CUDA]) as prof:
                        real_conv(layer, x)
                        torch.cuda.synchronize()
                kernels = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
                if kernels:
                    break
            found.append((name, kernels))
    KERNELS[(cfg.id, mode)] = found
    assert sum(bool(kernels) for _, kernels in found) >= len(found) - 1, (cfg.id, mode, "no kernels recorded")
    for name, kernels in found:
        if any("winograd" in k.lower() or "fft" in k.lower() for k in kernels):
            TRANSFORMS.append(f"{cfg.id} {mode} {name}: {' + '.join(kernels)}")


@pytest.mark.parametrize("cfg", INVALIDATION, ids=[c.id for c in INVALIDATION])
def test_plan_follows_load_state_dict(native, ref_astar, cfg):
    """Weights loaded after the plan was built reach the next eval call: every stage meets its bound against the second
    reference."""
    ref, x, (maps, start, goal) = _reference(ref_astar, cfg)
    na = ur.build_product(ref, cfg).cuda()
    m, s, g = (_cu(v) for v in (maps, start, goal))
    with torch.no_grad():
        first = na.encode(m, s, g).clone()
    assert na.encoder._plan is not None
    second = ur.build_reference(ref_astar, cfg, cfg.seed + 1, device="cuda")
    result = na.load_state_dict(second.state_dict())
    assert not result.missing_keys and not result.unexpected_keys
    calls, outs, convs, cost = _encode_recorded(na, native, cfg, "tf32", m, s, g)
    assert not torch.equal(first, cost)
    _check_stages(second, x, cfg, "tf32", calls, outs, convs, (cfg.id, "load_state_dict"))


# ------------------------------------------------------------------------------------------------- the kernels alone
def _head_cap_pixels():
    # launch_head caps the grid at 16 CTAs of 4 warps per SM, each warp taking one 32-pixel group per turn
    return torch.cuda.get_device_properties(0).multi_processor_count * 16 * 4 * 32


@pytest.mark.parametrize("C", [16, 32, 64, 128, 256])
def test_head_taps_against_float64(native, C):
    """head_taps at ragged pixel counts (one pixel, one short of a 32-pixel group, one past it, and an odd count past
    two turns of the capped grid) against float64 under gamma_C, written into a NaN-filled buffer longer than P x 9
    that must keep its tail."""
    assert C in native.HEAD_CHANNELS
    g = torch.Generator(device="cuda").manual_seed(C)
    w = np.random.RandomState(C).randn(C, 9).astype(np.float32)
    wd = torch.from_numpy(w).double().cuda()
    for P in (1, 31, 33, 2 * _head_cap_pixels() + 69):
        x = torch.randn(P, C, device="cuda", generator=g)
        act = x.view(1, 1, P, C).permute(0, 3, 1, 2)                # [1, C, 1, P], channels-last
        assert act.is_contiguous(memory_format=torch.channels_last)
        out = torch.full((P * 9 + 37,), float("nan"), device="cuda")
        got = native.head_taps(act, w, out=out)
        assert got.data_ptr() == out.data_ptr()
        want = x.double() @ wd
        bound = er.gamma(C) * (x.double().abs() @ wd.abs())
        err = (out[:P * 9].view(P, 9).double() - want).abs()
        assert bool((err <= bound).all()), (C, P, float((err / bound).max()))
        assert bool(out[P * 9:].isnan().all()), (C, P, "head_taps wrote past P x 9")


PAIRS = sorted({(cd, cs) for d in (1, 2, 3, 4, 5) for _, cd, cs in _decoder_shapes(d, 32)})


@pytest.mark.parametrize("cd,cs", PAIRS, ids=[f"{cd}+{cs}" for cd, cs in PAIRS])
def test_upsample_concat_non_square(native, cd, cs):
    """upsample_concat bit-equal to cat(interpolate(dec, x2, nearest), skip) for every (Cd, Cs) of the five depths, on
    grids with h != w, with one map and with a batch past two turns of the capped grid."""
    g = torch.Generator(device="cuda").manual_seed(cd * 1000 + cs)
    for h, w in ((3, 5), (5, 3), (1, 7)):
        per_map = h * w * cd // 4 + 4 * h * w * cs // 4
        for B in (1, 2 * _grid_cap_items() // per_map + 1):
            dec = torch.randn(B, cd, h, w, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
            skip = None
            if cs:
                skip = torch.randn(B, cs, 2 * h, 2 * w, device="cuda", generator=g)
                skip = skip.contiguous(memory_format=torch.channels_last)
            got = native.upsample_concat(dec, skip)
            want = F.interpolate(dec, scale_factor=2, mode="nearest")
            if skip is not None:
                want = torch.cat((want, skip), 1)
            assert got.is_contiguous(memory_format=torch.channels_last)
            assert got.shape == want.shape and torch.equal(got, want), (cd, cs, h, w, B)
