"""The step graph runs the search beside the fused 128->256 convolution + head kernel (csrc/nastar_convhead.cuh).  A
warp's registers come from one of an SM's four 16 384-register sub-partition files, and the convolution CTA's 12 warps
take 3 of each, so one search warp must fit next to 3 convolution warps on every sub-partition; shared memory must hold
one CTA of each.  Checked on the built library's resource usage (cuobjdump), without a GPU."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "neural-astar_b200")
CONV = "_ZN6nastar19conv3x3_head_kernelE14CUtensorMap_stS0_NS_12ConvHeadArgsENS_15ConvHeadWeightsE"
# astar_warp32_kernel<kTrace = 0, kBwd = 0, kExit, kFused = 1, kNews>: every variant search_from_taps launches at 32x32
STEP_SEARCH = re.compile(r"_ZN6nastar19astar_warp32_kernelILb0ELb0ELi\d+ELb1ELb[01]EEEvNS_10SearchArgsE")
SUBPARTITION_REGS = 16384
SM_SHARED = 228 * 1024
CONV_WARPS = 12


@pytest.fixture(scope="module")
def lib_path():
    subprocess.check_call(["make", "-C", PKG, "-s", "all"])
    from neural_astar import _native

    return _native.LIB_PATH


def _cuobjdump(*args):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    return subprocess.run([os.path.join(os.path.dirname(nvcc), "cuobjdump"), *args], check=True, capture_output=True,
                          text=True).stdout


@pytest.fixture(scope="module")
def usage(lib_path):
    """{mangled kernel name: {"REG": n, "STACK": n, "SHARED": n, "LOCAL": n, ...}} of every sm_90a kernel."""
    out, name = {}, None
    for line in _cuobjdump("-res-usage", lib_path).splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1)
        elif name and "REG:" in line:
            out[name] = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", line)}
            name = None
    return out


def _warp_regs(regs_per_thread):
    return (regs_per_thread + 7) // 8 * 8 * 32          # allocated per warp in units of 8 registers per thread


def test_conv_kernel_fits_144_registers_without_spills(usage):
    u = usage[CONV]
    assert u["REG"] <= 144, u
    assert u["STACK"] == 0 and u["LOCAL"] == 0, u


def test_setmaxnreg_stays_inside_the_launch_budget(usage, lib_path):
    sass = _cuobjdump("-sass", "-fun", CONV, lib_path)
    inc = [int(v, 16) for v in re.findall(r"USETMAXREG\.TRY_ALLOC\.CTAPOOL \w+, (0x[0-9a-f]+)", sass)]
    dec = [int(v, 16) for v in re.findall(r"USETMAXREG\.DEALLOC\.CTAPOOL (0x[0-9a-f]+)", sass)]
    assert len(inc) == 1 and len(dec) == 1, (inc, dec)
    # one producer warpgroup gives registers back, two consumer warpgroups take them
    assert 128 * dec[0] + 256 * inc[0] <= CONV_WARPS * 32 * usage[CONV]["REG"]


def test_every_step_graph_search_warp_fits_beside_a_conv_cta(usage):
    search = {k: v for k, v in usage.items() if STEP_SEARCH.fullmatch(k)}
    assert len(search) >= 2, "the fused-prologue search kernels are missing from the library"
    conv = CONV_WARPS // 4 * _warp_regs(usage[CONV]["REG"])
    for name, u in search.items():
        assert conv + _warp_regs(u["REG"]) <= SUBPARTITION_REGS, (name, u["REG"], usage[CONV]["REG"])


def test_shared_memory_fits_a_conv_cta_and_a_search_cta(usage):
    # ConvHeadLayout at the widest tile (64-pixel rows, 2 rows per tile: A boxes of 4 rows) + its 1 KB alignment slack:
    # 4 B stages of 32 KB, 2 A stages, bias, head weights, 12 mbarriers
    dynamic = 4 * 32768 + 2 * (4 * 64 * 128) + 256 * 4 + 256 * 9 * 4 + 2 * 6 * 8 + 1024
    conv = dynamic + usage[CONV]["SHARED"]                  # SHARED counts the 1 KB the system reserves per CTA
    for name, u in usage.items():
        if STEP_SEARCH.fullmatch(name):
            assert conv + u["SHARED"] <= SM_SHARED, (name, conv, u["SHARED"])
