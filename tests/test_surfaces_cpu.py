"""CPU: the ATen-composed surfaces of megreader_b200.refapi (SURVEY.md §8 A9/A10) reproduce the reference goldens and carry the
reference's exact state-dict keys/shapes, deformable trunk included (names, shapes and the EAST head's outputs recorded from the
unmodified reference by oracle/make_ref_golden_cpu.py; compared with it live as well where the reference tree is present)."""
import gzip
import json
import os

import numpy as np
import pytest
import torch

from oracle import ref_loader
from tests import surfaces_common as sc


def test_backbones_reproduce_reference_golden():
    torch.set_num_threads(4)
    sc.check_backbones("cpu", 1e-5)


def test_attention_head_reproduces_reference_golden():
    sc.check_attention("cpu", 2e-5)


def test_ctc_conv_head_eval_reproduces_reference_golden():
    sc.check_ctc_head("cpu", 1e-5, train=False)


def test_ctc_conv_head_train_refuses_cpu():
    with pytest.raises(NotImplementedError):
        sc.check_ctc_head("cpu", 1e-5, train=True)


def _keys(m):
    return [(k, tuple(v.shape)) for k, v in m.state_dict().items()]


GOLD = os.path.join(os.path.dirname(__file__), "golden")


def test_state_dict_keys_equal_stored_reference_keys():
    import sys
    import types
    import megreader_b200.refapi.backbones as mb
    import megreader_b200.refapi.decoders as md
    import megreader_b200.refapi.backbones.resnet as mres
    from megreader_b200 import dcn as mdcn
    from megreader_b200 import deform_pool as mpool
    with gzip.open(os.path.join(GOLD, "ref_state_keys.json.gz"), "rt") as f:
        ref = json.load(f)["modules"]
    stored = lambda name: [(k, tuple(shape)) for k, shape in ref[name]]  # noqa: E731
    shim = types.ModuleType("assets.ops.dcn")
    shim.ModulatedDeformConv, shim.DeformConv = mdcn.ModulatedDeformConv, mdcn.DeformConv
    saved = sys.modules.get("assets.ops.dcn")
    sys.modules["assets.ops.dcn"] = shim
    try:
        mine = mres.deformable_resnet50(pretrained=False)
        mine_v1 = mres.ResNet(mres.BasicBlock, [1, 1, 1, 1], dcn=dict(modulated=False, deformable_groups=2))
    finally:
        if saved is not None:
            sys.modules["assets.ops.dcn"] = saved
        else:
            del sys.modules["assets.ops.dcn"]
    ours = {"resnet34": mb.resnet34(pretrained=False), "resnet101": mb.resnet101(pretrained=False),
            "Resnet34FPN": mb.Resnet34FPN(resnet_pretrained=False), "resnet50dilated_ppm_128": mb.resnet50dilated_ppm(inner_channels=128),
            "AttentionDecoder": md.AttentionDecoder(64, inner_channels=128, max_size=16, height=2),
            "CTCDecoder": md.CTCDecoder(64, inner_channels=96), "EASTDecoder": md.EASTDecoder(channels=64),
            "deformable_resnet50": mine, "resnet_v1_dcn": mine_v1}
    for cls in ("DeformRoIPoolingPack", "ModulatedDeformRoIPoolingPack"):
        ours[cls] = getattr(mpool, cls)(0.5, 3, 8, False, trans_std=0.1, deform_fc_channels=32)
    for name, m in ours.items():
        assert _keys(m) == stored(name), name
    geo = [[n, list(c.stride), list(c.dilation), list(c.padding)] for n, c in mb.resnet50dilated_ppm().named_modules()
           if isinstance(c, torch.nn.Conv2d)]
    assert geo == ref["geo_resnet50dilated_ppm"]


def test_east_decoder_reproduces_stored_reference_outputs():
    """decoders/east.py:7-60 on CPU: the reference's parameters -> its loss, metrics and predictions (train and eval branches)."""
    import megreader_b200.refapi.decoders as md
    from oracle.make_ref_golden_cpu import east_case
    g = np.load(os.path.join(GOLD, "east_ref.npz"))
    m = md.EASTDecoder(channels=32).train()
    m.load_state_dict({k[3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("sd.")})
    x, label = east_case()
    lm, pm, mm = m(x, label, None, True)
    close = lambda a, k: torch.testing.assert_close(a.detach(), torch.from_numpy(g[k]), rtol=1e-4, atol=1e-5)  # noqa: E731
    close(lm, "train.loss")
    for k in pm:
        close(pm[k], "train.pred." + k)
    for k in mm:
        close(mm[k], "train.metric." + k)
    assert {"train.pred." + k for k in pm} | {"train.metric." + k for k in mm} == {k for k in g.files if k.startswith("train.") and k != "train.loss"}
    m.eval()
    pe = m(x, label, None, False)
    for k in pe:
        close(pe[k], "eval.pred." + k)


@pytest.mark.skipif(not ref_loader.available(), reason="reference tree not present (the stored reference data above is compared anywhere)")
def test_state_dict_keys_equal_reference():
    import sys
    import types
    ref_loader.install()
    # the reference's DCN python modules import their compiled extension at import time; a placeholder lets the
    # module *definitions* load so that parameter names can be compared (nothing is executed through it)
    sys.modules.setdefault("assets.ops.dcn.deform_conv_cuda", types.ModuleType("assets.ops.dcn.deform_conv_cuda"))
    sys.modules.setdefault("assets.ops.dcn.deform_pool_cuda", types.ModuleType("assets.ops.dcn.deform_pool_cuda"))
    import backbones as rb
    import decoders as rd
    import megreader_b200.refapi.backbones as mb
    import megreader_b200.refapi.decoders as md
    import megreader_b200.refapi.backbones.resnet as mres
    from megreader_b200 import dcn as mdcn
    pairs = [(rb.resnet34(pretrained=False), mb.resnet34(pretrained=False)),
             (rb.resnet101(pretrained=False), mb.resnet101(pretrained=False)),
             (rb.Resnet34FPN(resnet_pretrained=False), mb.Resnet34FPN(resnet_pretrained=False)),
             (rb.resnet50dilated_ppm(inner_channels=128), mb.resnet50dilated_ppm(inner_channels=128)),
             (rd.AttentionDecoder(64, inner_channels=128, max_size=16, height=2),
              md.AttentionDecoder(64, inner_channels=128, max_size=16, height=2)),
             (rd.CTCDecoder(64, inner_channels=96), md.CTCDecoder(64, inner_channels=96)),
             (rd.EASTDecoder(channels=64), md.EASTDecoder(channels=64))]
    for r, m in pairs:
        assert _keys(r) == _keys(m)
    # deformable trunk: our modules resolve `assets.ops.dcn` lazily; bind it to megreader_b200.dcn for this process
    shim = types.ModuleType("assets.ops.dcn")
    shim.ModulatedDeformConv, shim.DeformConv = mdcn.ModulatedDeformConv, mdcn.DeformConv
    ref_dcn = rb.deformable_resnet50(pretrained=False)
    saved = sys.modules.get("assets.ops.dcn")
    sys.modules["assets.ops.dcn"] = shim
    try:
        mine = mres.deformable_resnet50(pretrained=False)
        mine_v1 = mres.ResNet(mres.BasicBlock, [1, 1, 1, 1], dcn=dict(modulated=False, deformable_groups=2))
    finally:
        if saved is not None:
            sys.modules["assets.ops.dcn"] = saved
    assert _keys(ref_dcn) == _keys(mine)
    ref_v1 = rb.resnet.ResNet(rb.resnet.BasicBlock, [1, 1, 1, 1], dcn=dict(modulated=False, deformable_groups=2))
    assert _keys(ref_v1) == _keys(mine_v1)
    # zero-initialised offset branch (resnet.py:222-226)
    for mod in mine.modules():
        if hasattr(mod, "conv2_offset"):
            assert float(mod.conv2_offset.weight.abs().max()) == 0.0 and float(mod.conv2_offset.bias.abs().max()) == 0.0
    # deformable RoI pooling packs: same fully-connected stacks
    import assets.ops.dcn.modules.deform_pool as rpool
    from megreader_b200 import deform_pool as mpool
    for cls in ("DeformRoIPoolingPack", "ModulatedDeformRoIPoolingPack"):
        r = getattr(rpool, cls)(0.5, 3, 8, False, trans_std=0.1, deform_fc_channels=32)
        m = getattr(mpool, cls)(0.5, 3, 8, False, trans_std=0.1, deform_fc_channels=32)
        assert _keys(r) == _keys(m)
    # dilation surgery moved the same convs (resnet_dilated.py:37-49)
    rp, mp = rb.resnet50dilated_ppm(), mb.resnet50dilated_ppm()
    geo = lambda net: [(n, c.stride, c.dilation, c.padding) for n, c in net.named_modules() if isinstance(c, torch.nn.Conv2d)]
    assert geo(rp) == geo(mp)


@pytest.mark.skipif(not ref_loader.available(), reason="reference tree not present (the stored reference data above is compared anywhere)")
def test_east_decoder_equals_reference_module():
    """decoders/east.py:7-60 on CPU: same parameters -> same loss, metrics and predictions (train and eval branches)."""
    ref_loader.install()
    import decoders as rd
    import megreader_b200.refapi.decoders as md
    torch.manual_seed(0)
    r, m = rd.EASTDecoder(channels=32).train(), md.EASTDecoder(channels=32).train()
    m.load_state_dict(r.state_dict())
    x = torch.randn(2, 32, 6, 10)
    label = {"heatmap": (torch.rand(2, 1, 24, 40) > 0.7).float(), "heatmap_weight": torch.rand(2, 1, 24, 40),
             "densebox": torch.randn(2, 8, 24, 40) * 50, "densebox_weight": torch.rand(2, 8, 24, 40)}
    lr, pr, mr_ = r(x, label, None, True)
    lm, pm, mm = m(x, label, None, True)
    torch.testing.assert_close(lm, lr)
    for k in pr:
        torch.testing.assert_close(pm[k], pr[k])
    for k in mr_:
        torch.testing.assert_close(mm[k], mr_[k])
    r.eval(); m.eval()
    pe_r, pe_m = r(x, label, None, False), m(x, label, None, False)
    for k in pe_r:
        torch.testing.assert_close(pe_m[k], pe_r[k])
