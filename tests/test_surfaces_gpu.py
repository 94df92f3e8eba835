"""GPU: refapi surfaces around the hot path against the reference goldens (fp32, TF32 off), the 1-D CTC conv head through
the sm_90a CTC kernels, and the deformable ResNet units through the sm_90a DCN kernels (checked against the CPU oracle
and against the closed form for zero offsets: modulated DCN with offset 0 and mask 1/2 == half a dense conv)."""
import numpy as np
import pytest
import torch

from oracle import capi
from tests import surfaces_common as sc
from tests.weights import fill_state_dict

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _fp32_exact():
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def test_backbones_match_reference_golden():
    sc.check_backbones("cuda", 2e-4)


def test_attention_head_matches_reference_golden():
    sc.check_attention("cuda", 2e-4)


def test_ctc_conv_head_matches_reference_golden():
    sc.check_ctc_head("cuda", 2e-4, train=True)


def _refapi_resnet():
    from megreader_b200 import refapi
    refapi.install()
    import backbones.resnet as res          # resolves to megreader_b200/refapi (the reference is absent on the GPU box)
    assert "refapi" in res.__file__
    return res


def test_deformable_bottleneck_against_oracle():
    res = _refapi_resnet()
    torch.manual_seed(0)
    for modulated in (True, False):
        unit = res.Bottleneck(32, 8, stride=1, dcn=dict(modulated=modulated, deformable_groups=1))
        fill_state_dict(unit, "dcnunit.")
        unit = unit.cuda().eval()
        x = torch.randn(2, 32, 9, 11, device="cuda")
        with torch.no_grad():
            y = unit(x)
            # same unit, conv2 evaluated by the CPU oracle
            a = torch.relu(unit.bn1(unit.conv1(x)))
            field = unit.conv2_offset(a)
            if modulated:
                off, mask = field[:, :18], field[:, -9:].sigmoid()
                mask_np = mask.cpu().numpy().astype(np.float64)
            else:
                off, mask_np = field, None
            c2 = capi.dcn_forward(a.cpu().numpy().astype(np.float64), unit.conv2.weight.cpu().numpy().astype(np.float64),
                                  None, off.cpu().numpy().astype(np.float64), mask_np, stride=1, padding=1)
            b = torch.relu(unit.bn2(torch.from_numpy(np.asarray(c2, np.float32)).cuda()))
            ref = torch.relu(unit.bn3(unit.conv3(b)) + x)
        sc.close(y, ref.cpu().numpy(), "Bottleneck(dcn modulated=%s)" % modulated, 2e-4)


def test_deformable_resnet50_zero_offsets_closed_form():
    res = _refapi_resnet()
    torch.manual_seed(1)
    net = res.deformable_resnet50(pretrained=False)
    plain = res.resnet50(pretrained=False)
    sd = {k: v for k, v in net.state_dict().items() if "conv2_offset" not in k}
    for k in list(sd):
        # offset 0 / mask sigmoid(0) = 1/2 in every unit of layers 2-4 (resnet.py:222-226,161-165)
        if k.endswith("conv2.weight") and k.startswith(("layer2", "layer3", "layer4")):
            sd[k] = sd[k] * 0.5
    plain.load_state_dict(sd)
    net, plain = net.cuda().eval(), plain.cuda().eval()
    x = torch.randn(2, 3, 64, 96, device="cuda")
    with torch.no_grad():
        got, want = net(x), plain(x)
    for i, (g, w) in enumerate(zip(got, want)):
        sc.close(g, w.cpu().numpy(), "deformable_resnet50 stage %d" % i, 2e-4)
    # and it trains: gradients reach the offset branch through the DCN backward kernels
    net.train()
    out = net(x)[-1]
    out.square().mean().backward()
    g = net.layer3[1].conv2_offset.weight.grad
    assert g is not None and torch.isfinite(g).all() and float(g.abs().max()) > 0
