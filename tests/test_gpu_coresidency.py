"""The fused 128->256 convolution + head kernel gives the same bits when the search shares its SMs: taps computed
while search CTAs are resident equal taps computed alone, at the flagship batch and at 1000 maps."""
import os

import numpy as np
import pytest
import torch

from golden_util import Golden

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ckpt_planner():
    from neural_astar.planner import NeuralAstar

    state = np.load(os.path.join(ROOT, "tests", "golden", "mazes032_ckpt_planner_state.npz"))
    na = NeuralAstar(encoder_arch="CNN")
    na.load_state_dict({k: torch.from_numpy(state[k]) for k in state.files})
    return na.cuda().eval()


@pytest.mark.parametrize("name,B", [("mazes032_vanilla_test", 100), ("inputs_mazes032_all1000", 1000)])
def test_fused_taps_beside_the_search_equal_taps_alone(name, B):
    from neural_astar import _native
    from neural_astar.planner import encoder as enc_mod

    g = Golden(name)
    maps, start, goal = (torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (g.obst, g.start, g.goal))
    assert maps.shape[0] == B
    na = _ckpt_planner()
    enc = na.encoder
    with torch.no_grad():
        plan = enc._inference_plan(maps.device)
        with enc_mod._conv_flags():
            x = enc_mod._run_layers(plan.body[1:], _native.conv1_marks(maps, start, goal, *plan.conv1))
        x3 = x.contiguous(memory_format=torch.channels_last)
        w, b = plan.last.w, plan.last.b
        alone = _native.conv3x3_head_taps(x3, w, b, plan.head_w)
        search_taps = alone.clone()
        bias, scale = plan.head_b, plan.const
        torch.cuda.synchronize()
        main, side = torch.cuda.current_stream(), torch.cuda.Stream()
        for _ in range(3):
            side.wait_stream(main)
            with torch.cuda.stream(side):          # the search first, so its CTAs are resident when the conv starts
                out = na.astar.search_from_taps(search_taps, bias, scale, start, goal, maps)
            beside = _native.conv3x3_head_taps(x3, w, b, plan.head_w)
            main.wait_stream(side)
            torch.cuda.synchronize()
            assert torch.equal(beside, alone)
    assert float(out.histories.sum()) > 0
