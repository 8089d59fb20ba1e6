"""CPU-only checks of the fused last-conv + head entry point: it rejects bad arguments before any launch."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built_lib():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "neural-astar_b200"), "-s", "all"])
    from neural_astar import _native

    return _native


def test_abi_version_is_4_everywhere(built_lib):
    header = open(os.path.join(ROOT, "include", "nastar_b200.h")).read()
    assert re.search(r"#define NASTAR_B200_ABI_VERSION 4\b", header)
    assert built_lib.ABI_VERSION == 4
    assert built_lib.lib().nastar_b200_abi_version() == 4


def test_conv3x3_head_taps_rejects_bad_arguments_without_a_gpu(built_lib):
    L = built_lib.lib()
    f = L.nastar_b200_conv3x3_head_taps
    hw = np.zeros((256, 9), np.float32)
    # fake, 16-B aligned device addresses: validation must fail before anything touches them
    x, w, b, t = 0x10000, 0x20000, 0x30000, 0x40000
    h = hw.ctypes.data
    before = L.nastar_b200_launch_count()
    EINVAL, EUNSUPPORTED = 1, 2
    assert f(None, 1, 32, 32, 128, 256, w, b, h, t, None) == EINVAL            # null input
    assert f(x, 1, 32, 32, 128, 256, None, b, h, t, None) == EINVAL            # null weights
    assert f(x, 1, 32, 32, 128, 256, w, None, h, t, None) == EINVAL            # null bias
    assert f(x, 1, 32, 32, 128, 256, w, b, None, t, None) == EINVAL            # null head weights
    assert f(x, 1, 32, 32, 128, 256, w, b, h, None, None) == EINVAL            # null output
    assert f(x, 0, 32, 32, 128, 256, w, b, h, t, None) == EINVAL               # bad sizes
    assert f(x, 1, -1, 32, 128, 256, w, b, h, t, None) == EINVAL
    assert f(x, 1, 32, 0, 128, 256, w, b, h, t, None) == EINVAL
    assert f(x, 1, 32, 32, 0, 256, w, b, h, t, None) == EINVAL
    assert f(x + 4, 1, 32, 32, 128, 256, w, b, h, t, None) == EINVAL           # misaligned input (TMA needs 16 B)
    assert f(x, 1, 32, 32, 64, 256, w, b, h, t, None) == EUNSUPPORTED          # unsupported channel counts
    assert f(x, 1, 32, 32, 128, 128, w, b, h, t, None) == EUNSUPPORTED
    assert f(x, 1, 65, 32, 128, 256, w, b, h, t, None) == EUNSUPPORTED         # maps beyond 64x64
    assert f(x, 1, 32, 96, 128, 256, w, b, h, t, None) == EUNSUPPORTED
    assert L.nastar_b200_launch_count() == before     # nothing above was launched


def test_conv3x3_head_taps_binding_validates_layouts(built_lib):
    x = torch.zeros(1, 128, 8, 8).contiguous(memory_format=torch.channels_last)
    w = torch.zeros(256, 128, 3, 3).contiguous(memory_format=torch.channels_last)
    b = torch.zeros(256)
    hw = np.zeros((256, 9), np.float32)
    with pytest.raises(ValueError):
        built_lib.conv3x3_head_taps(x, w, b, hw)                               # CPU tensors
    with pytest.raises(ValueError):
        built_lib.conv3x3_head_taps(x, w, b, hw.reshape(9, 256))               # wrong head layout
