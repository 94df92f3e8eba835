"""Generate tests/golden/*.npz from the UNMODIFIED reference (needs the reference tree).

Run:  python -m oracle.make_golden            (from the repo root; needs /root/reference)

2D-CTC: the reference's CUDA op cannot run here (no GPU, does not build on torch 2.11), so the
golden vectors come from the reference's own pure-Python CTCLoss2D (decoders/ctc_loss2d.py:86-154)
with (mask + classify) == log_probs, on cases where it does not numerically saturate
(SURVEY.md §8c: valid while every per-state height-sum stays above fp32 tiny, i.e. loss <~ 60).
"""
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def ctc2d_case(seed, T, H, N, C, S, Lmax, peak):
    g = torch.Generator().manual_seed(seed)
    tl = torch.randint(1, Lmax + 1, (N,), generator=g)
    targets = torch.zeros(N, S, dtype=torch.long)
    for b in range(N):
        targets[b, :tl[b]] = torch.randint(1, C, (int(tl[b]),), generator=g)
    il = torch.full((N,), T, dtype=torch.long)
    mask_logit = torch.randn(T, H, N, generator=g)
    cls_logit = torch.randn(T, H, N, C, generator=g)
    if peak > 0:
        # push the classifier toward a monotone alignment of the target so the loss stays small
        for b in range(N):
            L = int(tl[b])
            for t in range(T):
                k = min(L - 1, t * L // T)
                cls_logit[t, :, b, targets[b, k]] += peak
    mask = mask_logit.log_softmax(1)
    classify = cls_logit.log_softmax(3)
    return mask, classify, targets, il, tl


def make_ctc2d():
    m = ref_loader.load("decoders.ctc_loss2d")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ref = m.CTCLoss2D(blank=0, reduction="none")
    cases = [  # name, seed, T, H, N, C, S, Lmax, peak
        ("doc", 1, 32, 8, 16, 20, 20, 6, 4.0),      # docstring shape decoders/ctc_loss2d.py:37-45 (short targets)
        ("small", 2, 8, 4, 4, 6, 5, 3, 0.0),
        ("cfg3", 3, 32, 8, 8, 38, 32, 5, 5.0),      # res50-ppm-2d-ctc.yaml shape, peaked
        ("h1", 4, 12, 1, 3, 7, 6, 4, 2.0),          # H=1 degenerates to 1D CTC
        ("rep", 5, 16, 3, 4, 5, 8, 6, 3.0),         # tiny alphabet -> repeated labels (have_three false)
    ]
    for name, seed, T, H, N, C, S, Lmax, peak in cases:
        mask, classify, targets, il, tl = ctc2d_case(seed, T, H, N, C, S, Lmax, peak)
        classify.requires_grad_(True)
        loss = ref(mask, classify, targets, il, tl)
        # autograd of the reference python loss = TRUE derivative -exp(G + nll - lp); the CUDA op's K3
        # returns exp(lp) + that on in-target classes (SURVEY.md App. B1.1), which tests check.
        (ref_grad,) = torch.autograd.grad(loss.sum(), classify)
        classify = classify.detach()
        lp = (mask.unsqueeze(-1) + classify).contiguous()
        np.savez_compressed(
            os.path.join(GOLD, "ctc2d_pyref_%s.npz" % name),
            log_probs=lp.numpy(), targets=targets.numpy(), input_lengths=il.numpy(),
            target_lengths=tl.numpy(), ref_nll=loss.detach().numpy(),
            ref_autograd=ref_grad.numpy())
        print("ctc2d", name, "ref nll", loss.detach().numpy()[:4])


def make_crnn():
    """cfg 1 exactly (crnn.yaml): reference crnn_backbone + CRNNDecoder(nn.CTCLoss), N=4, 3x32x100, fp32, CPU."""
    from tests.weights import crnn_batch, fill_state_dict
    ref_loader.install()
    import backbones as rb
    import decoders as rd
    torch.manual_seed(0)
    bb = fill_state_dict(rb.crnn_backbone(), "bb.")
    dec = fill_state_dict(rd.CRNNDecoder(in_channels=512, inner_channels=256), "dec.")
    for name, (N, W) in {"cfg1": (4, 100), "w128": (3, 128)}.items():
        T = W // 4 + 1
        x, labels, lengths = crnn_batch(0, N, W, 8, T)
        bb.train(); dec.train()
        bb.zero_grad(); dec.zero_grad()
        tx = torch.from_numpy(x)
        feat = bb(tx)
        loss, pred = dec(feat, targets=torch.from_numpy(labels), lengths=torch.from_numpy(lengths), train=True)
        loss.mean().backward()
        grads = {"grad." + k: v.grad.numpy().copy() for k, v in list(bb.named_parameters()) + list(dec.named_parameters())
                 if k in ("cnn.0.0.0.weight", "cnn.2.1.weight", "cnn.6.1.bias", "cnn.6.0.bias",
                          "rnn.1.embedding.weight", "rnn.1.embedding.bias", "rnn.0.rnn.bias_hh_l0_reverse")}
        gnorm = {"gnorm." + k: np.float64(v.grad.double().norm().item())
                 for k, v in list(bb.named_parameters()) + list(dec.named_parameters())}
        bn_after = {"bn." + k: v.numpy().copy() for k, v in bb.state_dict().items() if "running" in k and k.startswith("cnn.2")}
        # eval-mode forward AFTER the training forward (running stats updated once), like eval.py would see
        bb.eval(); dec.eval()
        with torch.no_grad():
            prob = dec(bb(tx), train=False)                       # (N, C, 1, T) softmax
        # re-load pristine weights for the next case (BN running stats were updated)
        np.savez_compressed(os.path.join(GOLD, "crnn_ref_%s.npz" % name), x=x[:, :1], labels=labels, lengths=lengths,
                            feature=feat.detach().numpy(), loss=np.float64(loss.item()), log_probs=pred.detach().numpy(),
                            eval_prob=prob.numpy(), **grads, **gnorm, **bn_after)
        print("crnn", name, "loss", loss.item(), "feat", tuple(feat.shape), "pred", tuple(pred.shape))
        fill_state_dict(bb, "bb."); fill_state_dict(dec, "dec.")


def make_surfaces():
    """Recognition-side surfaces around the hot path (SURVEY.md §8 A9/A10 + the 1-D CTC conv head): outputs of the
    UNMODIFIED reference modules on CPU, fp32, weights from tests.weights.fill_state_dict (name-seeded)."""
    from tests.weights import fill_state_dict, surface_inputs
    ref_loader.install()
    import backbones as rb
    import decoders as rd
    x, x2, feat, tg_pad, ln = surface_inputs()
    tx = torch.from_numpy(x)
    out = {}
    with torch.no_grad():
        m = fill_state_dict(rb.resnet18(pretrained=False), "r18.").eval()
        for i, f in enumerate(m(tx)):
            out["r18.%d" % i] = f.numpy()
        m = fill_state_dict(rb.resnet50dilated_ppm(), "ppm.").eval()
        out["ppm"] = m(tx).numpy()
        m = fill_state_dict(rb.Resnet50FPN(resnet_pretrained=False), "fpn50.").eval()
        out["fpn50"] = m(tx).numpy()
    # training-mode trunk (batch statistics) with a gradient norm per stage
    m = fill_state_dict(rb.Resnet18FPN(resnet_pretrained=False), "fpn18.").train()
    y = m(torch.from_numpy(x2))
    y.square().mean().backward()
    out["fpn18.train"] = y.detach().numpy()
    for k in ("bottom_up.conv1.weight", "bottom_up.layer3.0.downsample.0.weight", "top_down.merge_layer.weight"):
        out["fpn18.gnorm." + k] = np.float64(dict(m.named_parameters())[k].grad.double().norm().item())

    tf, tt, tl = torch.from_numpy(feat), torch.from_numpy(tg_pad), torch.from_numpy(ln)
    att = fill_state_dict(rd.AttentionDecoder(256, gt_as_output=True), "attn.").train()
    loss, amap = att(tf, targets=tt, lengths=tl)
    loss.sum().backward()
    out["attn.loss"] = loss.detach().numpy()
    out["attn.map"] = amap.detach().numpy()
    for k in ("encode.0.0.weight", "decoder.attn.attn.weight", "decoder.attn.v", "decoder.rnn.weight_hh",
              "decoder.embedding.weight", "onehot_embedding_x.weight"):
        out["attn.gnorm." + k] = np.float64(dict(att.named_parameters())[k].grad.double().norm().item())
    with torch.no_grad():
        out["attn.eval"] = att.eval()(tf).numpy()
    ctc = fill_state_dict(rd.CTCDecoder(256), "ctc1d.")
    with torch.no_grad():                                     # eval first: pristine BN running statistics
        out["ctc1d.eval"] = ctc.eval()(tf, train=False).numpy()
    loss, lp = ctc.train()(tf, targets=tt, lengths=tl, train=True)
    loss.backward()
    out["ctc1d.loss"] = np.float64(loss.item())
    out["ctc1d.log_probs"] = lp.detach().numpy()
    for k in ("encode.0.0.weight", "pred_conv.weight", "pred_conv.bias"):
        out["ctc1d.gnorm." + k] = np.float64(dict(ctc.named_parameters())[k].grad.double().norm().item())
    np.savez_compressed(os.path.join(GOLD, "surfaces_ref.npz"), **out)
    print("surfaces", {k: getattr(v, "shape", v) for k, v in out.items()})


def make_head():
    """2D-CTC head epilogue (decoders/ctc_decoder2d.py:37-45): run the UNMODIFIED reference module on CPU with its
    `ctc_loss` replaced by a fixed linear functional of `pred`, capture the two conv branches' raw outputs with
    forward hooks, and record pred plus the gradients that reach those raw outputs."""
    import types
    from tests.weights import fill_state_dict
    ref_loader.install()
    ops_stub = types.ModuleType("ops")
    ops_stub.ctc_loss_2d = None
    saved = sys.modules.get("ops")
    sys.modules["ops"] = ops_stub
    try:
        import decoders as rd
        dec = fill_state_dict(rd.CTCDecoder2D(16, inner_channels=8), "d2.").train()
    finally:
        if saved is not None:
            sys.modules["ops"] = saved
        else:
            del sys.modules["ops"]
    rng = np.random.RandomState(21)
    feat = torch.from_numpy((rng.standard_normal((5, 16, 8, 32)) * 3.0).astype(np.float32))
    weight = torch.from_numpy(rng.standard_normal((32, 8, 5, 38)).astype(np.float32))
    lengths = torch.tensor([3, 1, 4, 2, 5])
    captured = {}

    def grab(name):
        def hook(module, inputs, output):
            output.retain_grad()
            captured[name] = output
        return hook
    dec.pred_mask[2].register_forward_hook(grab("mask_logits"))
    dec.pred_classify[2].register_forward_hook(grab("cls_logits"))
    dec.ctc_loss = lambda pred, *a: (pred * weight).sum(dim=(0, 1, 3))
    out = {}
    # case "a": `saved_tiny` as fill_state_dict left it (a large value: the clamp and its zero gradient hit ~half the
    # entries); "b": the real tiny = finfo(float32).tiny, ordinary logits; "c": real tiny, 1x1 convs scaled x25 so that
    # part of mask*classify underflows below tiny
    real_tiny = float(torch.finfo(torch.float32).tiny)
    for tag, tiny, gain in (("a", None, 1.0), ("b", real_tiny, 1.0), ("c", real_tiny, 25.0)):
        with torch.no_grad():
            if tiny is not None:
                dec.saved_tiny.fill_(tiny)
            dec.pred_mask[2].weight.mul_(gain)
            dec.pred_classify[2].weight.mul_(gain)
        dec.zero_grad()
        loss, pred = dec(feat, targets=torch.zeros(5, 32), lengths=lengths, train=True)
        loss.sum().backward()
        dlp = (weight / lengths.float().view(1, 1, -1, 1)).contiguous()      # the upstream gradient that reached pred
        out.update({tag + ".tiny": np.float32(dec.saved_tiny.item()),
                    tag + ".mask_logits": captured["mask_logits"].detach().numpy(),
                    tag + ".cls_logits": captured["cls_logits"].detach().numpy(), tag + ".pred": pred.detach().numpy(),
                    tag + ".grad_pred": dlp.numpy(), tag + ".grad_mask_logits": captured["mask_logits"].grad.numpy(),
                    tag + ".grad_cls_logits": captured["cls_logits"].grad.numpy()})
        print("head", tag, tuple(pred.shape), "tiny", dec.saved_tiny.item(), "clamped fraction",
              float((pred <= float(np.log(dec.saved_tiny.item())) + 1e-6).float().mean()))
    for tag in sorted({k.split(".")[0] for k in out}):      # one file per case: each stays well under 1 MB
        np.savez_compressed(os.path.join(GOLD, "ctc2d_head_ref_%s.npz" % tag), **{k: v for k, v in out.items() if k.startswith(tag + ".")})


def make_input():
    """Recognition input step (crnn.yaml processes): run the UNMODIFIED reference ResizeImage (modes resize and pad),
    NormalizeImage and MakeRecognitionLabel on CPU (cv2 4.x from this image) and record their outputs."""
    ref_loader.install()
    from data.processes.resize_image import ResizeImage
    from data.processes.normalize_image import NormalizeImage
    from data.processes.make_recognition_label import MakeRecognitionLabel
    from tests.input_cases import MODES, input_cases
    images, texts = input_cases()
    out = {}
    for mode, size in MODES.items():
        rz = ResizeImage(mode=mode, image_size=list(size))
        nm = NormalizeImage()
        batch = []
        for im in images:
            d = {"image": im.astype("float32")}                     # data/lmdb_dataset.py:87
            d = nm.process(rz.process(d))
            batch.append(d["image"].numpy())
        out["image." + mode] = np.stack(batch)
    mk = MakeRecognitionLabel()
    labels, lengths = [], []
    for t in texts:
        d = mk.process({"gt": t})
        labels.append(np.asarray(d["label"], np.int32))
        lengths.append(int(d["length"]))
    out["labels"] = np.stack(labels)
    out["lengths"] = np.asarray(lengths, np.int32)
    np.savez_compressed(os.path.join(GOLD, "input_ref.npz"), **out)
    print("input", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    os.makedirs(GOLD, exist_ok=True)
    which = sys.argv[1:] or ["ctc2d"]
    if "ctc2d" in which:
        make_ctc2d()
    if "crnn" in which:
        make_crnn()
    if "surfaces" in which:
        make_surfaces()
    if "head" in which:
        make_head()
    if "input" in which:
        make_input()
