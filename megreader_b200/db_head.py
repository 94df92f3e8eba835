"""DB (Differentiable Binarization) detector tail as two autograd nodes on csrc/db_head.cu:

  StepFunction             the two transposed-convolution logit maps -> (binary, thresh, thresh_binary)
                           (decoders/seg_detector.py:146-147 with the nn.Sigmoid at the end of binarize / thresh)
  L1BalanceCELossFunction  (binary, thresh, thresh_binary) + the DB batch -> (loss, bce_loss, dice_loss, l1_loss)
                           (decoders/seg_detector_loss.py:162-185), hard-negative mining included, without host synchronisation

They are separate nodes because the reference keeps the decoder and the criterion as separate modules.  CUDA only; no CPU
fallback."""
import torch
from torch.autograd import Function

from . import _lib

_DTYPES = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _require_cuda(what, *ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise NotImplementedError("megreader_b200: %s runs on CUDA only (no CPU fallback)" % what)


class StepFunction(Function):
    """(zb [N,1,H,W], zt [N,1,H,W] or None, k) -> (binary, thresh, thresh_binary), fp32 maps; thresh and thresh_binary are
    None when zt is None (adaptive=False).  The logits may be fp32, bf16 or fp16; their gradients come back in that dtype."""

    @staticmethod
    def forward(ctx, zb, zt, k):
        _require_cuda("the DB step function", zb, zt)
        if zb.dtype not in _DTYPES or (zt is not None and (zt.dtype != zb.dtype or zt.shape != zb.shape)):
            raise RuntimeError("StepFunction: expected two logit maps of one shape and dtype (fp32 / bf16 / fp16), got %s %s and %s"
                               % (zb.dtype, tuple(zb.shape), None if zt is None else (zt.dtype, tuple(zt.shape))))
        zb = zb.contiguous()
        zt = zt.contiguous() if zt is not None else None
        f32 = dict(dtype=torch.float32, device=zb.device)
        binary = torch.empty(zb.shape, **f32)
        thresh = torch.empty(zb.shape, **f32) if zt is not None else None
        tb = torch.empty(zb.shape, **f32) if zt is not None else None
        with torch.cuda.device(zb.device):
            _lib.check(_lib.lib().mr_db_step_fwd(zb.data_ptr(), _ptr(zt), _DTYPES[zb.dtype], zb.numel(), float(k),
                                                 binary.data_ptr(), _ptr(thresh), _ptr(tb), _stream()), "db_step_fwd")
        ctx.k, ctx.dtype, ctx.adaptive = float(k), zb.dtype, zt is not None
        ctx.save_for_backward(binary, thresh, tb)
        return binary, thresh, tb

    @staticmethod
    def backward(ctx, g_b, g_t, g_s):
        binary, thresh, tb = ctx.saved_tensors
        c = lambda g: g.contiguous().float() if g is not None else None  # noqa: E731
        g_b, g_t, g_s = c(g_b), c(g_t), c(g_s)
        dzb = torch.empty(binary.shape, dtype=ctx.dtype, device=binary.device)
        dzt = torch.empty(binary.shape, dtype=ctx.dtype, device=binary.device) if ctx.adaptive else None
        with torch.cuda.device(binary.device):
            _lib.check(_lib.lib().mr_db_step_bwd(binary.data_ptr(), _ptr(thresh), _ptr(tb), _ptr(g_b), _ptr(g_t), _ptr(g_s),
                                                 _DTYPES[ctx.dtype], binary.numel(), ctx.k, dzb.data_ptr(), _ptr(dzt),
                                                 _stream()), "db_step_bwd")
        return dzb, dzt, None


def step_function(zb, zt, k):
    return StepFunction.apply(zb, zt, k)


class L1BalanceCELossFunction(Function):
    """(binary, thresh, thresh_binary [N,1,H,W] fp32; gt [N,1,H,W], mask, thresh_map, thresh_mask [N,H,W]) ->
    (loss, bce_loss, dice_loss, l1_loss), four 0-dim fp32 tensors.  Differentiable in the three maps."""

    @staticmethod
    def forward(ctx, binary, thresh, thresh_binary, gt, mask, thresh_map, thresh_mask, eps, l1_scale, bce_scale,
                negative_ratio, bce_eps):
        maps = (binary, thresh, thresh_binary, gt, mask, thresh_map, thresh_mask)
        _require_cuda("L1BalanceCELoss", *maps)
        if binary.dim() != 4 or binary.size(1) != 1:
            raise RuntimeError("L1BalanceCELoss: expected binary [N,1,H,W], got %s" % (tuple(binary.shape),))
        N, _, H, W = binary.shape
        for name, t, shape in (("thresh", thresh, binary.shape), ("thresh_binary", thresh_binary, binary.shape),
                               ("gt", gt, binary.shape), ("mask", mask, (N, H, W)), ("thresh_map", thresh_map, (N, H, W)),
                               ("thresh_mask", thresh_mask, (N, H, W))):
            if tuple(t.shape) != tuple(shape):
                raise RuntimeError("L1BalanceCELoss: %s has shape %s, expected %s" % (name, tuple(t.shape), tuple(shape)))
        maps = tuple(t.contiguous().float() for t in maps)
        dev = binary.device
        L = _lib.lib()
        ws = torch.empty(int(L.mr_db_loss_workspace_bytes(N, H, W)), dtype=torch.uint8, device=dev)
        out = torch.empty(4, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(L.mr_db_loss_fwd_f32(*[t.data_ptr() for t in maps], N, H, W, float(eps), float(bce_eps), float(l1_scale),
                                            float(bce_scale), float(negative_ratio), ws.data_ptr(), out.data_ptr(), _stream()),
                       "db_loss_fwd")
        ctx.save_for_backward(*maps, ws)
        ctx.scales = (float(l1_scale), float(bce_scale))
        return out[0], out[1], out[2], out[3]

    @staticmethod
    def backward(ctx, g_loss, g_bce, g_dice, g_l1):
        *maps, ws = ctx.saved_tensors
        binary = maps[0]
        N, _, H, W = binary.shape
        z = binary.new_zeros(())
        g = torch.stack([(t if t is not None else z).reshape(()).float() for t in (g_loss, g_bce, g_dice, g_l1)])
        d = [torch.empty_like(binary) for _ in range(3)]
        with torch.cuda.device(binary.device):
            _lib.check(_lib.lib().mr_db_loss_bwd_f32(*[t.data_ptr() for t in maps], N, H, W, *ctx.scales, ws.data_ptr(),
                                                     g.data_ptr(), *[t.data_ptr() for t in d], _stream()), "db_loss_bwd")
        return tuple(d) + (None,) * 9


def l1_balance_ce_loss(binary, thresh, thresh_binary, gt, mask, thresh_map, thresh_mask, eps=1e-6, l1_scale=10, bce_scale=5,
                       negative_ratio=3.0, bce_eps=1e-6):
    return L1BalanceCELossFunction.apply(binary, thresh, thresh_binary, gt, mask, thresh_map, thresh_mask, eps, l1_scale,
                                         bce_scale, negative_ratio, bce_eps)
