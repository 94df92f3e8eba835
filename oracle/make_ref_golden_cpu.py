"""Record what the CPU tests compare with the UNMODIFIED reference modules (oracle/ref_loader.py) under tests/golden/, so that
those comparisons run where the reference tree is absent.

    python -m oracle.make_ref_golden_cpu        # needs the reference tree (MEGREADER_REFERENCE)

    crnn_ref_b3.npz          reference CRNN backbone + decoder on tests.weights.crnn_batch(3, 2, 100, 8, 26): train loss / log-probs,
                             eval log-probs (tests/test_oracle_crnn.py)
    east_ref.npz             reference EASTDecoder(channels=32): its state dict, inputs, and train / eval outputs
    ref_state_keys.json.gz   state-dict names and shapes of the reference modules tests/test_surfaces_cpu.py compares, conv
                             geometry of the dilated trunk
"""
import gzip
import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")


def keys(m):
    return [[k, list(v.shape)] for k, v in m.state_dict().items()]


def geo(net):
    return [[n, list(c.stride), list(c.dilation), list(c.padding)] for n, c in net.named_modules() if isinstance(c, torch.nn.Conv2d)]


def east_case():
    torch.manual_seed(0)
    x = torch.randn(2, 32, 6, 10)
    label = {"heatmap": (torch.rand(2, 1, 24, 40) > 0.7).float(), "heatmap_weight": torch.rand(2, 1, 24, 40),
             "densebox": torch.randn(2, 8, 24, 40) * 50, "densebox_weight": torch.rand(2, 8, 24, 40)}
    return x, label


def main():
    from oracle import ref_loader
    from tests.weights import crnn_batch, fill_state_dict
    assert ref_loader.install(), "reference tree not present"
    sys.modules.setdefault("assets.ops.dcn.deform_conv_cuda", types.ModuleType("assets.ops.dcn.deform_conv_cuda"))
    sys.modules.setdefault("assets.ops.dcn.deform_pool_cuda", types.ModuleType("assets.ops.dcn.deform_pool_cuda"))
    import backbones as rb
    import decoders as rd
    torch.set_num_threads(1)
    # ---- CRNN
    rbb = fill_state_dict(rb.crnn_backbone(), "bb.")
    rdec = fill_state_dict(rd.CRNNDecoder(in_channels=512, inner_channels=256), "dec.")
    x, labels, lengths = crnn_batch(3, 2, 100, 8, 26)
    tx, tl, tn = torch.from_numpy(x), torch.from_numpy(labels), torch.from_numpy(lengths)
    loss, pred = rdec(rbb.train()(tx), targets=tl, lengths=tn, train=True)
    ev = rdec.eval()(rbb.eval()(tx), train=False)
    np.savez_compressed(os.path.join(GOLD, "crnn_ref_b3.npz"), loss=loss.detach().numpy(), pred=pred.detach().numpy(),
                        eval_pred=ev.detach().numpy())
    state = {"crnn_backbone": keys(rbb), "crnn_decoder": keys(rdec)}
    # ---- EAST decoder
    torch.manual_seed(0)
    r = rd.EASTDecoder(channels=32).train()
    x, label = east_case()
    out = {"sd." + k: v.clone().numpy() for k, v in r.state_dict().items()}   # a copy: the train forward updates BatchNorm statistics in place
    lr, pr, mr_ = r(x, label, None, True)
    out["train.loss"] = lr.detach().numpy()
    out.update({"train.pred." + k: v.detach().numpy() for k, v in pr.items()})
    out.update({"train.metric." + k: v.detach().numpy() for k, v in mr_.items()})
    r.eval()
    out.update({"eval.pred." + k: v.detach().numpy() for k, v in r(x, label, None, False).items()})
    np.savez_compressed(os.path.join(GOLD, "east_ref.npz"), **out)
    # ---- state-dict names / shapes
    import assets.ops.dcn.modules.deform_pool as rpool
    state.update({
        "resnet34": keys(rb.resnet34(pretrained=False)), "resnet101": keys(rb.resnet101(pretrained=False)),
        "Resnet34FPN": keys(rb.Resnet34FPN(resnet_pretrained=False)),
        "resnet50dilated_ppm_128": keys(rb.resnet50dilated_ppm(inner_channels=128)),
        "AttentionDecoder": keys(rd.AttentionDecoder(64, inner_channels=128, max_size=16, height=2)),
        "CTCDecoder": keys(rd.CTCDecoder(64, inner_channels=96)), "EASTDecoder": keys(rd.EASTDecoder(channels=64)),
        "deformable_resnet50": keys(rb.deformable_resnet50(pretrained=False)),
        "resnet_v1_dcn": keys(rb.resnet.ResNet(rb.resnet.BasicBlock, [1, 1, 1, 1], dcn=dict(modulated=False, deformable_groups=2))),
        "geo_resnet50dilated_ppm": geo(rb.resnet50dilated_ppm()),
    })
    for cls in ("DeformRoIPoolingPack", "ModulatedDeformRoIPoolingPack"):
        state[cls] = keys(getattr(rpool, cls)(0.5, 3, 8, False, trans_std=0.1, deform_fc_channels=32))
    with gzip.open(os.path.join(GOLD, "ref_state_keys.json.gz"), "wt") as f:
        json.dump({"modules": state}, f, sort_keys=True)


if __name__ == "__main__":
    main()
