"""CPU-only checks of the search entry points' status codes: rejected arguments return before any launch.

The device addresses below are fake and never dereferenced: every case returns before a kernel, a memset or a stream
call is issued, so the launch counter must not move."""
import ctypes
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EINVAL, EUNSUPPORTED, EWORKSPACE = 1, 2, 4
COST_TAPS = 2


@pytest.fixture(scope="module")
def built_lib():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "neural-astar_b200"), "-s", "all"])
    from neural_astar import _native

    return _native


@pytest.fixture
def no_launch(built_lib):
    L = built_lib.lib()
    before = L.nastar_b200_launch_count()
    yield L
    assert L.nastar_b200_launch_count() == before, "a rejected call launched something"


def _fwd(native, **kw):
    p = native.FwdParams()
    p.cost, p.start, p.goal, p.obst = 0x10000, 0x20000, 0x30000, 0x40000
    p.cost_stride = p.start_stride = p.goal_stride = p.obst_stride = 32 * 32
    p.histories, p.paths = 0x50000, 0x60000
    p.B, p.H, p.W, p.T = 4, 32, 32, 100
    p.g_ratio, p.one_minus_g_ratio = 0.5, 0.5
    for k, v in kw.items():
        setattr(p, k, v)
    return ctypes.byref(p)


def _bwd(native, **kw):
    p = native.BwdParams()
    p.cost, p.start, p.goal, p.obst = 0x10000, 0x20000, 0x30000, 0x40000
    p.cost_stride = p.start_stride = p.goal_stride = p.obst_stride = p.grad_stride = 96 * 64
    p.grad_histories, p.grad_cost, p.T_batch, p.t_solve = 0x50000, 0x60000, 0x70000, 0x80000
    p.B, p.H, p.W = 4, 96, 64
    p.g_ratio, p.one_minus_g_ratio, p.sqrt_w = 0.5, 0.5, 8.0
    for k, v in kw.items():
        setattr(p, k, v)
    return ctypes.byref(p)


@pytest.mark.parametrize("kw,status", [
    (dict(B=0), EINVAL),
    (dict(T=0), EINVAL),
    (dict(cost_kind=3), EINVAL),
    (dict(H=96, W=96, cost_kind=COST_TAPS), EUNSUPPORTED),       # the fused hand-off covers H, W <= 64 only
    (dict(H=100000, W=100000), EUNSUPPORTED),
    (dict(H=0, W=5), EINVAL),                                      # the size check runs before the engine choice
    (dict(H=256, W=256, cost_stride=65536, start_stride=65536, goal_stride=65536, obst_stride=65536), EWORKSPACE),
])
def test_forward_status_codes(built_lib, no_launch, kw, status):
    assert no_launch.nastar_b200_forward(_fwd(built_lib, **kw), None) == status


@pytest.mark.parametrize("kw,status", [
    (dict(T_batch=None), EINVAL),
    (dict(H=100000, W=100000), EUNSUPPORTED),
    (dict(), EWORKSPACE),                                          # 96x64: the generic engine needs its workspace
])
def test_backward_status_codes(built_lib, no_launch, kw, status):
    assert no_launch.nastar_b200_backward(_bwd(built_lib, **kw), None) == status


# (H, W) -> (nastar_b200_engine_for, nastar_b200_bin16_supported) for the shapes the GPU tests choose per engine
# (test_gpu_forward_parity.py, test_gpu_backward_parity.py, test_gpu_engine_schedules.py): a threshold change must not
# move one of them to another engine unnoticed.  1 = warp32, 4 = warp64, 2 / 3 = generic with state in shared memory /
# in the HBM workspace; bin16 = engine 5 takes binary aliased planes of this shape.
ENGINE_TABLE = {
    (32, 32): (1, 0),
    **{hw: (4, 0) for hw in [(33, 33), (1, 64), (64, 1), (2, 64), (64, 2), (32, 33), (33, 32), (40, 20), (20, 40),
                             (63, 64), (47, 61), (64, 64), (48, 64), (50, 47), (48, 40)]},
    **{hw: (2, 1) for hw in [(65, 40), (1, 65), (70, 3), (97, 131), (131, 131), (96, 64), (96, 50), (65, 41),
                             (100, 72)]},
    **{hw: (3, 1) for hw in [(131, 132), (132, 132), (144, 136), (160, 128), (256, 256)]},
    (512, 512): (3, 0),
    (600, 64): (3, 0),
}


def test_engine_table(built_lib):
    L = built_lib.lib()
    got = {hw: (L.nastar_b200_engine_for(*hw), L.nastar_b200_bin16_supported(*hw)) for hw in ENGINE_TABLE}
    assert got == ENGINE_TABLE


def test_glue_entry_points_status_codes(no_launch):
    L = no_launch
    assert L.nastar_b200_batch_steps(0x10000, 0x20000, 4, 0, 0x30000, None) == EINVAL               # T = 0
    assert L.nastar_b200_pack_inputs(0x10000, 3, 32, 32, 0x20000, 1024, 0x30000, 1024, 4, 32, 32,
                                     0x40008, None) == EINVAL                                        # out not 16-B aligned
    assert L.nastar_b200_cost_from_taps(0x10000, 0, 32, 32, 0.0, 1.0, 0x20000, None) == EINVAL       # B = 0
    assert L.nastar_b200_selftest_sqrt(0, 0x10000, None) == EINVAL                                   # n = 0
