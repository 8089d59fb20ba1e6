"""CPU-only checks of the batch-coupled forward's C ABI (nastar_b200_forward_coupled): declared, exported, and every
rejected argument returns before any launch.  The device addresses are fake and never dereferenced."""
import ctypes
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EINVAL, EUNSUPPORTED, EWORKSPACE = 1, 2, 4
NEW_SYMBOLS = ("nastar_b200_forward_coupled", "nastar_b200_forward_coupled_workspace_bytes")


@pytest.fixture(scope="module")
def native():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "neural-astar_b200"), "-s", "all"])
    from neural_astar import _native

    return _native


@pytest.fixture
def no_launch(native):
    L = native.lib()
    before = L.nastar_b200_launch_count()
    yield L
    assert L.nastar_b200_launch_count() == before, "a rejected call launched something"


def test_symbols_declared_and_exported(native):
    header = open(os.path.join(ROOT, "include", "nastar_b200.h")).read()
    for s in NEW_SYMBOLS:
        assert re.search(r"\b" + s + r"\s*\(", header), s
        assert s in native.EXPORTS
        assert hasattr(native.lib(), s)


def _params(native, **kw):
    p = native.FwdParams()
    p.cost, p.start, p.goal, p.obst = 0x10000, 0x20000, 0x30000, 0x40000
    p.cost_stride = p.start_stride = p.goal_stride = p.obst_stride = 32 * 32
    p.histories, p.paths = 0x50000, 0x60000
    p.B, p.H, p.W, p.T = 4, 32, 32, 1024
    p.g_ratio, p.one_minus_g_ratio = 0.2, 0.8
    p.workspace = 0x70000
    p.workspace_bytes = native.lib().nastar_b200_forward_coupled_workspace_bytes(p.B, p.H, p.W, p.T)
    for k, v in kw.items():
        setattr(p, k, v)
    return p


@pytest.mark.parametrize("kw,outs,status", [
    (dict(), (None, 0x90000), EINVAL),                   # no T_batch
    (dict(), (0x80000, None), EINVAL),                   # no goal_clamp
    (dict(trace=0xA0000), (0x80000, 0x90000), EINVAL),
    (dict(flags=1), (0x80000, 0x90000), EINVAL),         # NASTAR_FWD_NO_EARLY_EXIT
    (dict(flags=2), (0x80000, 0x90000), EINVAL),         # NASTAR_FWD_PAIR
    (dict(flags=5), (0x80000, 0x90000), EINVAL),         # NEWS | NO_EARLY_EXIT
    (dict(B=0), (0x80000, 0x90000), EINVAL),
    (dict(T=0), (0x80000, 0x90000), EINVAL),
    (dict(cost_kind=3), (0x80000, 0x90000), EINVAL),
    (dict(H=96, W=96, cost_kind=2), (0x80000, 0x90000), EUNSUPPORTED),
    (dict(workspace=None), (0x80000, 0x90000), EWORKSPACE),
])
def test_rejected_before_any_launch(native, no_launch, kw, outs, status):
    p = _params(native, **kw)
    assert no_launch.nastar_b200_forward_coupled(ctypes.byref(p), outs[0], outs[1], None) == status


@pytest.mark.parametrize("H,W", [(32, 32), (64, 64), (100, 72), (144, 136)])
def test_workspace_smaller_than_the_query_is_rejected(native, no_launch, H, W):
    p = _params(native, H=H, W=W, cost_stride=H * W, start_stride=H * W, goal_stride=H * W, obst_stride=H * W,
                T=H * W)
    p.workspace_bytes -= 1
    assert no_launch.nastar_b200_forward_coupled(ctypes.byref(p), 0x80000, 0x90000, None) == EWORKSPACE


def test_workspace_query_grows_with_T_and_B(native):
    q = native.lib().nastar_b200_forward_coupled_workspace_bytes
    for H, W in ((32, 32), (64, 64), (100, 72), (144, 136)):
        assert q(100, H, W, 4096) > q(100, H, W, 1024) > 0
        assert q(1000, H, W, 1024) > q(100, H, W, 1024)
        # the per-map at-goal bitmap alone: ceil(T/32) words per map
        assert q(100, H, W, 65536) - q(100, H, W, 32) >= 100 * (65536 // 32 - 2) * 4
    assert q(0, 32, 32, 1024) == 0 and q(4, 32, 32, 0) == 0 and q(4, 100000, 100000, 1024) == 0
