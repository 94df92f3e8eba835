"""TEST INFRASTRUCTURE ONLY (never imported by the product): CPU restatement of the tail of the reference's 2D-CTC head,
decoders/ctc_decoder2d.py:37-45, on the conv branches' raw outputs.

    mask_logits [N,1,H,W]  -> masking  = Softmax(dim=2)                      (:21, last module of pred_mask)
    cls_logits  [N,C,H,W]  -> classify = softmax(dim=1)                      (:41)
    pred = log(max(mask * classify, tiny)).permute(3,2,0,1).contiguous()     (:43-45)  -> (W,H,N,C)

Pinned by tests/golden/ctc2d_head_ref_*.npz, which oracle/make_golden.py produced by running the UNMODIFIED reference
module's forward (its `ctc_loss` attribute replaced by a fixed linear functional so that an arbitrary upstream
gradient reaches `pred`)."""
import torch


def head_log_probs(mask_logits, cls_logits, tiny=None):
    tiny = torch.tensor(torch.finfo(torch.float32).tiny if tiny is None else tiny, dtype=cls_logits.dtype)
    mask = torch.softmax(mask_logits, dim=2)
    classify = torch.softmax(cls_logits, dim=1)
    pred = torch.log(torch.max(mask * classify, tiny))
    return pred.permute(3, 2, 0, 1).contiguous()


def head_grads(mask_logits, cls_logits, grad_log_probs, tiny=None):
    """autograd of the restatement: -> (grad_mask_logits, grad_cls_logits)"""
    m = mask_logits.detach().clone().requires_grad_(True)
    z = cls_logits.detach().clone().requires_grad_(True)
    head_log_probs(m, z, tiny).backward(grad_log_probs)
    return m.grad, z.grad
