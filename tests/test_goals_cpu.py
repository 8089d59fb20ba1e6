"""CPU tests of the GPU goal sampler's specification (no GPU needed): the NumPy oracle (tests/goals_oracle.py) draws
from exactly the cells sample_goal_maps hands to rng.choice, the C ABI rejects bad arguments before any launch, and the
binding refuses CPU tensors and malformed draws."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

import goals_oracle as go
import labels_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EINVAL, EUNSUPPORTED = 1, 2


@pytest.fixture(scope="module")
def built_lib():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "neural-astar_b200"), "-s", "all"])
    from neural_astar import _native

    return _native


class _RecordingRng:
    """stands in for random.Random: records every sequence given to choice and returns its first element"""

    def __init__(self):
        self.seen = []

    def choice(self, seq):
        self.seen.append(np.asarray(seq).copy())
        return seq[0]


def _edges(H, W):
    return (0, H // 4, (max(H, W) + 1) // 2, max(H, W) + 1)


def _assert_candidates_equal_host(maps):
    from neural_astar.utils.data import sample_goal_maps

    B, H, W = maps.shape
    for e in _edges(H, W):
        rng = _RecordingRng()
        sample_goal_maps(maps, edge_size=e, rng=rng)
        assert len(rng.seen) == B
        for i in range(B):
            assert np.array_equal(go.candidates(maps[i], e), rng.seen[i]), (i, e)


@pytest.mark.parametrize("name", labels_golden.NAMES)
def test_oracle_candidates_equal_sample_goal_maps_on_fixtures(name):
    maps = labels_golden.load(name)[0]
    keep = [i for i in range(len(maps)) if (maps[i] != 0).any()]
    _assert_candidates_equal_host(maps[keep])


@pytest.mark.parametrize("H,W", [(1, 1), (5, 40), (33, 31), (64, 64), (3, 100)])
@pytest.mark.parametrize("p", [0.2, 0.5])
def test_oracle_candidates_equal_sample_goal_maps_on_random_maps(H, W, p):
    rs = np.random.RandomState(H * 131 + W + int(p * 10))
    maps = np.where(rs.rand(12, H, W) < p, 0.0, rs.choice([1.0, 0.5, -1.0], size=(12, H, W))).astype(np.float32)
    maps[:, 0, 0] = 1.0   # at least one passable cell per map
    _assert_candidates_equal_host(maps)


def test_oracle_draw_mapping():
    for n in (1, 2, 7, 1000, 262144):
        assert go.pick(n, 0) == 0 and go.pick(n, -1) == n - 1 and go.pick(n, 2 ** 32 - 1) == n - 1
        for k in {0, 1 % n, n // 2, n - 1}:
            d = go.draw_for(k, n)
            assert 0 <= d < 2 ** 32 and go.pick(n, d) == k and (d == 0 or go.pick(n, d - 1) == k - 1)


def test_goals_abi_rejects_bad_arguments_without_a_gpu(built_lib):
    L = built_lib.lib()
    p = ctypes.c_void_p(256)   # never dereferenced: every call below fails validation before any launch
    n0 = built_lib.launch_count()

    def call(*, maps=p, stride=64, B=2, H=8, W=8, e=0, draws=p, gi=p, gm=p, st=p):
        return L.nastar_b200_sample_goals(maps, stride, B, H, W, e, draws, gi, gm, st, None)

    for k in ("maps", "draws", "gi", "gm", "st"):
        assert call(**{k: None}) == EINVAL, k
    assert call(B=0) == EINVAL and call(B=-1) == EINVAL
    assert call(H=0) == EINVAL and call(W=0) == EINVAL and call(H=-4) == EINVAL
    assert call(stride=63) == EINVAL and call(H=9) == EINVAL           # map stride < H*W
    assert call(e=-1) == EINVAL
    assert call(H=513, stride=513 * 8) == EUNSUPPORTED and call(W=513, stride=8 * 513) == EUNSUPPORTED
    assert built_lib.launch_count() == n0, "a rejected call must not launch"


def test_goals_binding_refuses_cpu_tensors_and_bad_draws(built_lib):
    from neural_astar.utils.data import sample_device_goal_maps

    maps = torch.ones(3, 1, 8, 8)
    with pytest.raises(RuntimeError, match="CUDA"):
        built_lib.sample_goals(maps, torch.zeros(3, dtype=torch.int32))
    with pytest.raises(RuntimeError, match="CUDA"):
        sample_device_goal_maps(maps)
    for bad in (torch.zeros(2, dtype=torch.int32), torch.zeros(3, 1, dtype=torch.int32), torch.zeros(3)):
        with pytest.raises(ValueError, match="draws"):
            built_lib.sample_goals(maps, bad)
