"""NeuralAstar's encoder on the GPU against the reference's own NeuralAstar run in float64, on the matrix of
tests/test_encoder_reference_cpu.py: the "m+" CNN at depths 1 to 4 on square, non-square and tiny grids, the "m" CNN, a
learnable const with and without learn_obstacles, and CNNDownSize at depths 1 to 4 ("rgb+") and without marks ("rgb").

Every configuration runs with TF32 on (the default) and off, and one per depth with the head kernel off.  Per case:
  heads     which kernels the eval fast path reaches, counted: conv1_marks exactly for the "m+" CNN, conv3x3_head_taps
            exactly where the last body layer is an unpooled 128 -> 256 conv and TF32 is on, head_taps<C> otherwise
            (torch.mm with the head kernel off);
  encode    encode() under no_grad (the folded plan) is within the element-wise bound of the float64 reference's encode()
            for the mode's rounding, and so is encode() under autograd (the module path, cuDNN's default TF32);
  forward   forward() (the head's taps straight into the search) equals perform_astar(encode()) bit for bit, and the
            staged reference's fp32 DifferentiableAstar run on that cost with the obstacle plane the reference would
            use, up to the documented exp-collision, where it equals SPEC;
  graph     a GraphedPlanner replay equals the eager forward().
The folded plan follows load_state_dict and a train-mode batch's running statistics.  The worst |error| / bound of
every configuration and mode, and the kernels each reached, are printed at teardown.
"""
import numpy as np
import pytest
import torch

import test_encoder_reference_cpu as er
import test_reference_parity_cpu as rp
from test_encoder_reference_cpu import CONFIGS, _cnn, _down
from test_gpu_reference_parity import _forward_matches

pytestmark = pytest.mark.gpu

NOHEAD = [_cnn("m+", d, 20, 48) for d in (1, 2, 3, 4)]      # head kernel off: one configuration per depth
CASES = [(c, m) for c in CONFIGS for m in ("tf32", "fp32")] + [(c, "nohead") for c in NOHEAD]
INVALIDATION = [_cnn("m+", 1, 20, 48), _cnn("m+", 4, 48, 20), _cnn("m", 2, 32, 32), _down("rgb+", 3, 96)]
HEAD_KERNELS = ("conv1_marks", "conv3x3_head_taps", "head_taps")
WORST = {}          # (config id, mode) -> worst |error| / bound
SHARE = {}          # (config id, mode) -> median bound / median |cost - const / 2|
HEADS = {}          # (config id, mode) -> kernels the fast path reached
_REFERENCES = {}    # config id -> (float64 reference, inputs)


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
        heads = HEADS.get(key)
        print(f"\n{key[0]} {key[1]}: worst |error| / bound {WORST[key]:.4f}"
              + (f", median bound / spread {SHARE[key]:.4f}" if key in SHARE else "")
              + (f", kernels {'+'.join(heads) if heads else 'cuDNN only'}" if heads is not None else ""))
    if WORST:
        for mode in sorted({k[1] for k in WORST}):
            print(f"\nworst over {mode}: {max(v for k, v in WORST.items() if k[1] == mode):.4f}")


def _cu(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _reference(ref_astar, cfg):
    """The configuration's float64 reference and inputs, built once for all its modes (never mutated)."""
    if cfg.id not in _REFERENCES:
        _REFERENCES[cfg.id] = (er.build_reference(ref_astar, cfg, cfg.seed), er.inputs(cfg, cfg.seed))
    return _REFERENCES[cfg.id]


def _set_mode(monkeypatch, mode):
    from neural_astar.planner import encoder as enc

    monkeypatch.setattr(enc, "ALLOW_TF32", mode != "fp32")
    monkeypatch.setattr(enc, "HEAD_KERNEL", mode != "nohead")


def _count_heads(monkeypatch, native):
    """Record every call of the fast path's own kernels: names, with head_taps' channel count."""
    calls = []
    for name in HEAD_KERNELS:
        real = getattr(native, name)

        def counted(*a, _real=real, _name=name, **k):
            calls.append(f"head_taps<{a[0].shape[1]}>" if _name == "head_taps" else _name)
            return _real(*a, **k)

        monkeypatch.setattr(native, name, counted)
    return calls


def expected_heads(cfg, mode):
    want = ["conv1_marks"] if cfg.conv1_marks else []
    if cfg.fused and mode == "tf32":
        want.append("conv3x3_head_taps")
    elif mode != "nohead":
        want.append(f"head_taps<{cfg.head_channels}>")
    return want


def _within(got, walk, key):
    ratio = er.bound_ratio(got.detach().cpu().numpy(), walk)
    WORST[key] = max(WORST.get(key, 0.0), ratio)
    assert ratio <= 1.0, (key, ratio)
    return ratio


@pytest.mark.parametrize("cfg,mode", CASES, ids=[f"{c.id}-{m}" for c, m in CASES])
def test_fast_path_matches_reference(native, ref_astar, search_ref, monkeypatch, cfg, mode):
    from neural_astar.utils.inference import GraphedPlanner

    ref, (maps, start, goal) = _reference(ref_astar, cfg)
    _set_mode(monkeypatch, mode)
    na = er.build_product(ref, cfg).cuda()
    m, s, g = (_cu(v) for v in (maps, start, goal))
    calls = _count_heads(monkeypatch, native)
    with torch.no_grad():
        cost = na.encode(m, s, g)
    torch.cuda.synchronize()
    HEADS[(cfg.id, mode)] = list(calls)
    assert calls == expected_heads(cfg, mode), (cfg.id, mode, calls)
    assert tuple(cost.shape) == (cfg.B, 1) + cfg.grid

    # encode(): the folded plan, then the module path under autograd
    walk = er.reference_case(ref, cfg, maps, start, goal, mode)
    _within(cost, walk, (cfg.id, mode))
    frac = er.VACUOUS_FP32 if mode == "fp32" else er.VACUOUS_TF32
    SHARE[(cfg.id, mode)] = er.assert_not_vacuous(walk, er.const_of(cfg), (cfg.id, mode), frac)
    if mode == "tf32":
        slow = na.encode(m, s, g)
        assert slow.requires_grad
        _within(slow, er.reference_case(ref, cfg, maps, start, goal, "module"), (cfg.id, "module"))

    # forward(): the taps go straight into the search
    searched = []
    real = na.astar.search_from_taps
    monkeypatch.setattr(na.astar, "search_from_taps", lambda *a, **k: searched.append(1) or real(*a, **k))
    passable = torch.ones_like(s) if cfg.learn_obstacles else m
    with torch.no_grad():
        out = na(m, s, g)
        unfused = na.perform_astar(cost, s, g, passable)
    assert searched == [1], "forward() did not hand the taps to the search"
    assert torch.equal(out.histories, unfused.histories) and torch.equal(out.paths, unfused.paths)
    hist, paths = out.histories.cpu().numpy(), out.paths.cpu().numpy()
    p = rp.Problem("moore", 0.5, 1.0, False, cost.cpu().numpy(), start, goal, passable.cpu().numpy(),
                   np.zeros_like(start))
    _forward_matches(hist, paths, rp.run_reference(search_ref, p, torch.float32), p, (cfg.id, mode))

    # a CUDA-graph replay of the same batch
    replay = GraphedPlanner(na, m, s, g).replay()
    assert torch.equal(replay.histories, out.histories) and torch.equal(replay.paths, out.paths)


@pytest.mark.parametrize("cfg", INVALIDATION, ids=[c.id for c in INVALIDATION])
def test_plan_follows_load_state_dict(native, ref_astar, cfg):
    """Weights loaded after the plan was built reach the next eval call: it meets the bound against the second
    reference."""
    ref, (maps, start, goal) = _reference(ref_astar, cfg)
    na = er.build_product(ref, cfg).cuda()
    m, s, g = (_cu(v) for v in (maps, start, goal))
    with torch.no_grad():
        first = na.encode(m, s, g).clone()
    assert na.encoder._plan is not None
    second_ref = er.build_reference(ref_astar, cfg, cfg.seed + 1)
    result = na.load_state_dict(second_ref.state_dict())
    assert not result.missing_keys and not result.unexpected_keys
    with torch.no_grad():
        second = na.encode(m, s, g)
    assert not torch.equal(first, second)
    _within(second, er.reference_case(second_ref, cfg, maps, start, goal, "tf32"), (cfg.id, "load_state_dict"))


def _bn_stats(model):
    return {k: v.detach().double().cpu().clone() for k, v in model.state_dict().items()
            if k.endswith("running_mean") or k.endswith("running_var")}


@pytest.mark.parametrize("cfg", INVALIDATION, ids=[c.id for c in INVALIDATION])
def test_plan_follows_running_statistics(native, ref_astar, cfg):
    """One train-mode batch moves the running statistics; the next eval call uses them.  The product's fp32 statistics
    (its training forward runs cuDNN's TF32 convolutions) must agree with the float64 reference's, given the same
    batch, to 2 % of how far the batch moved them; the reference then takes the product's statistics, so that the eval
    call is held to the bound of its own arithmetic."""
    ref = er.build_reference(ref_astar, cfg, cfg.seed)
    maps, start, goal = er.inputs(cfg, cfg.seed)
    na = er.build_product(ref, cfg).cuda()
    m, s, g = (_cu(v) for v in (maps, start, goal))
    with torch.no_grad():
        before = na.encode(m, s, g).clone()
    old = _bn_stats(ref)
    batch = er.inputs(cfg, cfg.seed + 2)
    na.train()
    ref.train()
    with torch.no_grad():
        na.encode(*(_cu(v) for v in batch))
        ref.encode(*(torch.from_numpy(v).double() for v in batch))
    na.eval()
    ref.eval()
    got, want = _bn_stats(na), _bn_stats(ref)
    for k in want:
        moved = float((want[k] - old[k]).abs().max())
        assert moved > 0, k
        assert float((got[k] - want[k]).abs().max()) <= 0.02 * moved, k
    ref.load_state_dict(na.state_dict())
    with torch.no_grad():
        after = na.encode(m, s, g)
    assert not torch.equal(before, after)
    _within(after, er.reference_case(ref, cfg, maps, start, goal, "tf32"), (cfg.id, "train-batch"))
