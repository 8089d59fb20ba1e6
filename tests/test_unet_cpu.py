"""The Unet encoder on the CPU: segmentation_models_pytorch 0.3.1's vgg16_bn U-Net layout, its forward restated with
torch.nn.functional, initialisation, validation, and the C ABI's rejections of the upsample-concat entry point."""
import os
import subprocess

import pytest
import torch
import torch.nn.functional as F

from neural_astar.planner import NeuralAstar
from neural_astar.planner.encoder import Unet

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EINVAL = 1

# torchvision's vgg16_bn cfg "D"; module indices of the conv / BatchNorm pairs follow from it
CFG = [64, 64, "M", 128, 128, "M", 256, 256, 256, "M", 512, 512, 512, "M", 512, 512, 512, "M"]
STAGE_OUT = [64, 128, 256, 512, 512, 512]
DEC = [256, 128, 64, 32, 16]


def _bn(t, prefix, c):
    t.update({f"{prefix}.weight": (c,), f"{prefix}.bias": (c,), f"{prefix}.running_mean": (c,),
              f"{prefix}.running_var": (c,), f"{prefix}.num_batches_tracked": ()})


def expected_layout(input_dim, d):
    t, i, cin = {}, 0, input_dim
    for v in CFG:
        if v == "M":
            i += 1
            continue
        t[f"encoder.features.{i}.weight"] = (v, cin, 3, 3)
        t[f"encoder.features.{i}.bias"] = (v,)
        _bn(t, f"encoder.features.{i + 1}", v)
        i, cin = i + 3, v
    head = STAGE_OUT[d]
    for j in range(2):
        t[f"decoder.center.{j}.0.weight"] = (head, head, 3, 3)
        _bn(t, f"decoder.center.{j}.1", head)
    ins = [head] + DEC[:d - 1]
    skips = [STAGE_OUT[k] for k in range(d - 1, 0, -1)] + [0]
    for b, (ci, cs, co) in enumerate(zip(ins, skips, DEC[:d])):
        t[f"decoder.blocks.{b}.conv1.0.weight"] = (co, ci + cs, 3, 3)
        _bn(t, f"decoder.blocks.{b}.conv1.1", co)
        t[f"decoder.blocks.{b}.conv2.0.weight"] = (co, co, 3, 3)
        _bn(t, f"decoder.blocks.{b}.conv2.1", co)
    t["segmentation_head.0.weight"] = (1, DEC[d - 1], 3, 3)
    t["segmentation_head.0.bias"] = (1,)
    return t


@pytest.mark.parametrize("d", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("input_dim", [1, 2, 4])
def test_state_dict_layout(input_dim, d):
    m = Unet(input_dim, d).model
    got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert got == expected_layout(input_dim, d)
    assert [n for n, _ in m.named_children()] == ["encoder", "decoder", "segmentation_head"]
    assert len(m.encoder.features) == 44 and len(m.decoder.blocks) == d


@pytest.mark.parametrize("d,entries,params", [(4, 153, 23_343_777), (1, 117, 15_906_049), (5, 165, 23_756_113)])
def test_counts(d, entries, params):
    m = Unet(2, d).model
    assert len(m.state_dict()) == entries
    assert sum(p.numel() for p in m.parameters()) == params


def functional_unet(x, sd, d, training=False):
    """The U-Net's logits from the state dict alone; train-mode BatchNorm normalises by the batch's statistics."""
    def _cbr(x, conv, bn, bias=True):
        x = F.conv2d(x, sd[conv + ".weight"], sd[conv + ".bias"] if bias else None, padding=1)
        x = F.batch_norm(x, sd[bn + ".running_mean"].clone(), sd[bn + ".running_var"].clone(), sd[bn + ".weight"],
                         sd[bn + ".bias"], training=training, eps=1e-5)
        return F.relu(x)

    feats, i = [], 0
    for v in CFG:
        if v == "M":
            feats.append(x)
            x = F.max_pool2d(x, 2, 2)
            i += 1
        else:
            x = _cbr(x, f"encoder.features.{i}", f"encoder.features.{i + 1}")
            i += 3
    feats.append(x)                   # s0..s5
    feats = feats[1:d + 1][::-1]      # s_d .. s1
    x = feats[0]
    for j in range(2):
        x = _cbr(x, f"decoder.center.{j}.0", f"decoder.center.{j}.1", bias=False)
    skips = feats[1:]
    for b in range(d):
        x = F.interpolate(x, scale_factor=2, mode="nearest")
        if b < len(skips):
            x = torch.cat([x, skips[b]], 1)
        x = _cbr(x, f"decoder.blocks.{b}.conv1.0", f"decoder.blocks.{b}.conv1.1", bias=False)
        x = _cbr(x, f"decoder.blocks.{b}.conv2.0", f"decoder.blocks.{b}.conv2.1", bias=False)
    return F.conv2d(x, sd["segmentation_head.0.weight"], sd["segmentation_head.0.bias"], padding=1)


def _randomise_bn(m, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                c = mod.num_features
                mod.running_mean.copy_(torch.randn(c, generator=g) * 0.1)
                mod.running_var.copy_(torch.rand(c, generator=g) + 0.5)
                mod.weight.copy_(torch.rand(c, generator=g) + 0.5)
                mod.bias.copy_(torch.randn(c, generator=g) * 0.1)


@pytest.mark.parametrize("hw", [(32, 32), (64, 128)])
@pytest.mark.parametrize("d", [1, 4, 5])
@pytest.mark.parametrize("train", [False, True])
def test_forward_matches_functional(d, hw, train):
    torch.manual_seed(d)
    enc = Unet(2, d)
    _randomise_bn(enc.model, d)
    x = torch.rand(2, 2, *hw)
    sd = {k: v.clone() for k, v in enc.model.state_dict().items()}
    enc.train(train)
    with torch.no_grad():
        got = enc(x)
    ref = functional_unet(x, sd, d, training=train)
    torch.testing.assert_close(got, torch.sigmoid(ref), atol=1e-5, rtol=0)


def test_state_dict_round_trip_through_planner():
    torch.manual_seed(0)
    a = NeuralAstar(encoder_arch="Unet", encoder_depth=4)
    torch.manual_seed(1)
    b = NeuralAstar(encoder_arch="Unet", encoder_depth=4)
    b.load_state_dict(a.state_dict(), strict=True)
    for (ka, va), (kb, vb) in zip(a.state_dict().items(), b.state_dict().items()):
        assert ka == kb and torch.equal(va, vb)
    enc_keys = {k[len("encoder.model."):] for k in a.state_dict() if k.startswith("encoder.model.")}
    assert enc_keys == set(expected_layout(2, 4))
    x = torch.rand(1, 2, 32, 32)
    a.eval(), b.eval()
    with torch.no_grad():
        assert torch.equal(a.encoder(x), b.encoder(x))


@pytest.mark.parametrize("d", [0, 6, -1])
def test_bad_depth(d):
    with pytest.raises(ValueError, match="encoder_depth"):
        Unet(2, d)


def test_bad_sides():
    enc = Unet(2, 4).eval()
    with pytest.raises(ValueError, match="divisible by 2\\*\\*4"):
        enc(torch.rand(1, 2, 24, 32))
    with pytest.raises(ValueError, match="divisible"):
        enc.model(torch.rand(1, 2, 32, 40))
    Unet(2, 3).eval()(torch.rand(1, 2, 24, 32))    # 24 is divisible by 2**3


def test_init_rules():
    torch.manual_seed(0)
    m = Unet(2, 5).model
    convs = [(n, c) for n, c in m.named_modules() if isinstance(c, torch.nn.Conv2d)]
    for n, c in convs:
        if n.startswith("decoder."):
            assert c.bias is None, n
        elif n != "encoder.features.0":
            assert torch.count_nonzero(c.bias) == 0, n
    first = m.encoder.features[0]
    assert torch.count_nonzero(first.bias) > 0          # re-created first conv: PyTorch's default init
    for n, bn in m.named_modules():
        if isinstance(bn, torch.nn.BatchNorm2d):
            assert torch.all(bn.weight == 1) and torch.all(bn.bias == 0), n
    # kaiming_normal_(fan_out) on VGG convs: std = sqrt(2 / (9 * out)); kaiming_uniform_(fan_in) on the decoder
    w = m.encoder.features[14].weight.detach()
    assert abs(float(w.std()) - (2 / (9 * 256)) ** 0.5) < 0.1 * (2 / (9 * 256)) ** 0.5
    w = m.decoder.blocks[0].conv1[0].weight.detach()
    bound = (6 / (9 * w.shape[1])) ** 0.5
    assert float(w.abs().max()) <= bound and float(w.abs().max()) > 0.9 * bound
    h = m.segmentation_head[0]
    assert torch.count_nonzero(h.bias) == 0
    assert float(h.weight.detach().abs().max()) <= (6 / (9 * 16 + 9)) ** 0.5


@pytest.mark.parametrize("d", [1, 4, 5])
def test_smp_interchange(d):
    smp = pytest.importorskip("segmentation_models_pytorch")
    torch.manual_seed(0)
    theirs = smp.Unet(encoder_name="vgg16_bn", encoder_weights=None, classes=1, in_channels=2, encoder_depth=d,
                      decoder_channels=DEC[:d]).eval()
    ours = Unet(2, d).eval()
    ours.model.load_state_dict(theirs.state_dict(), strict=True)
    theirs.load_state_dict(ours.model.state_dict(), strict=True)
    x = torch.rand(2, 2, 64, 64)
    with torch.no_grad():
        torch.testing.assert_close(ours(x), torch.sigmoid(theirs(x)), atol=1e-5, rtol=0)


@pytest.fixture
def no_launch():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "neural-astar_b200"), "-s", "all"])
    from neural_astar import _native

    L = _native.lib()
    before = L.nastar_b200_launch_count()
    yield L
    assert L.nastar_b200_launch_count() == before, "a rejected call launched something"


@pytest.mark.parametrize("args", [
    (0, 4, 16, 16, 256, 0x20000, 512, 0x30000),        # dec NULL
    (0x10000, 4, 16, 16, 256, 0x20000, 512, 0),        # out NULL
    (0x10000, 4, 16, 16, 256, 0, 512, 0x30000),        # skip NULL with Cs > 0
    (0x10000, 0, 16, 16, 256, 0x20000, 512, 0x30000),  # B = 0
    (0x10000, 4, 0, 16, 256, 0x20000, 512, 0x30000),   # h = 0
    (0x10000, 4, 16, -1, 256, 0x20000, 512, 0x30000),  # w < 0
    (0x10000, 4, 16, 16, 0, 0x20000, 512, 0x30000),    # Cd = 0
    (0x10000, 4, 16, 16, 256, 0x20000, -4, 0x30000),   # Cs < 0
    (0x10000, 4, 16, 16, 18, 0x20000, 512, 0x30000),   # Cd not a multiple of 4
    (0x10000, 4, 16, 16, 256, 0x20000, 6, 0x30000),    # Cs not a multiple of 4
    (0x10008, 4, 16, 16, 256, 0x20000, 512, 0x30000),  # dec not 16-B aligned
    (0x10000, 4, 16, 16, 256, 0x20004, 512, 0x30000),  # skip not 16-B aligned
    (0x10000, 4, 16, 16, 256, 0x20000, 512, 0x30008),  # out not 16-B aligned
])
def test_upsample_concat_status_codes(no_launch, args):
    assert no_launch.nastar_b200_upsample_concat(*args, None) == EINVAL


def test_head_taps_status_codes(no_launch):
    assert no_launch.nastar_b200_head_taps(0x10008, 64, 16, 0x20000, 0x30000, None) == EINVAL   # x not 16-B aligned
    assert no_launch.nastar_b200_head_taps(0x10000, 0, 16, 0x20000, 0x30000, None) == EINVAL    # P = 0
    assert no_launch.nastar_b200_head_taps(0x10000, 64, 24, 0x20000, 0x30000, None) == 2         # C = 24: unsupported
