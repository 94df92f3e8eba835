"""Host side of deformable convolution v1 / v2: same names, argument order and in-place behaviour as the
reference's pybind module `assets.ops.dcn.deform_conv_cuda` (assets/ops/dcn/src/deform_conv_cuda.cpp:681-695), the
autograd Functions (assets/ops/dcn/functions/deform_conv.py:8-181) and the nn.Modules
(assets/ops/dcn/modules/deform_conv.py:10-157).  Arithmetic: megreader_b200/csrc/dcn.cu through the C-ABI.

Dtypes: the dtype of the input `x` is the compute dtype.
  x float32                  weight / bias float32           -> the fp32 kernels, output and gradients float32
  x float16 or bfloat16 (T)  weight / bias T or float32      -> the half-precision fused kernels (csrc/dcn_tcgen05.cu): output,
                                                                grad_input / grad_offset / grad_mask in T, grad_weight /
                                                                grad_bias in the weight's dtype (fp32 accumulation throughout)
  anything else                                              -> RuntimeError naming the dtypes
offset and mask are converted to x's dtype first (under torch.autocast the offset conv returns half precision even for an fp32
x; upcasting is lossless).  Half-precision shapes outside the fused path (groups, deformable groups > 1, C % 64 != 0; C % 128
!= 0 for the data gradient) are rare -- none of the reference's trunks has one -- and run the fp32 kernels on fp32 copies, with
the results converted back.
"""
import math

import torch
import torch.nn as nn
from torch.autograd import Function
from torch.nn.modules.utils import _pair

from . import _lib

WORKSPACE_CAP_BYTES = 2 << 30  # column scratch per call (caller-side allocation, C-ABI takes the pointer)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _out_hw(H, W, kh, kw, sh, sw, ph, pw, dh, dw):
    return (H + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1, (W + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1


def _slab(t):
    """(tensor, batch stride in elements) with every per-sample slab contiguous (deform_conv_cuda.cpp:535-538
    indexes offset[b] / mask[b] per sample)."""
    if t.size(0) > 0 and not t[0].is_contiguous():
        t = t.contiguous()
    return t, (t.stride(0) if t.size(0) > 1 else t[0].numel() if t.size(0) else 0)


def _workspace(x, C, kh, kw, Ho, Wo, Cout=0, backward=False):
    """Scratch for the op: room for the column matrix of nb samples (unfused kernels) and, when Cout is given, for the fused
    forward's NHWC input copy + packed weights (csrc/dcn_tcgen05.cu) -- whichever is larger."""
    per = C * kh * kw * Ho * Wo * 4
    nb = max(1, min(x.size(0), WORKSPACE_CAP_BYTES // max(per, 1)))
    nbytes = nb * per
    if Cout and backward:
        nbytes = max(nbytes, int(_lib.lib().mr_dcn_fused_wgrad_workspace_bytes(x.size(0), C, x.size(2), x.size(3), Cout, Ho, Wo)),
                     int(_lib.lib().mr_dcn_fused_backward_workspace_bytes(x.size(0), C, x.size(2), x.size(3), Cout, Ho, Wo, kh, kw)))
    elif Cout:
        nbytes = max(nbytes, int(_lib.lib().mr_dcn_fused_workspace_bytes(x.size(0), C, x.size(2), x.size(3), Cout, kh, kw)))
    nbytes = (nbytes + 255) // 256 * 256
    return torch.empty(nbytes // 4, dtype=torch.float32, device=x.device), nbytes


_HALF_CODE = {torch.bfloat16: 1, torch.float16: 2}   # dtype codes of the C-ABI (0 = float32)


def _check(x, weight, bias=None):
    if not x.is_cuda:
        raise RuntimeError("Not implemented on the CPU")
    wd = weight.dtype
    ok = wd == torch.float32 if x.dtype == torch.float32 else x.dtype in _HALF_CODE and wd in (x.dtype, torch.float32)
    if not ok or (bias is not None and bias.dtype != wd):
        raise RuntimeError("megreader_b200 dcn: unsupported dtypes: input %s, weight %s%s (a float32 input needs float32 "
                           "weight and bias; a float16 / bfloat16 input needs weight and bias both in its dtype or both "
                           "float32)" % (x.dtype, wd, "" if bias is None else ", bias %s" % bias.dtype))
    if not x.is_contiguous():
        raise RuntimeError("input tensor has to be contiguous")          # deform_conv_cuda.cpp:493
    if not weight.is_contiguous():
        raise RuntimeError("weight tensor has to be contiguous")         # deform_conv_cuda.cpp:494


def _codes(x, weight):
    """(dtype, weight_dtype) codes of the half-precision C entry points."""
    return _HALF_CODE[x.dtype], 0 if weight.dtype == torch.float32 else _HALF_CODE[weight.dtype]


def _half_workspace(x, nbytes):
    return torch.empty(int(nbytes), dtype=torch.uint8, device=x.device)


def _in_dtype(t, dtype):
    """t itself when it has `dtype` (or is None), else a copy in `dtype` that _write_back returns to t."""
    return t if t is None or t.dtype == dtype else t.to(dtype)


def _write_back(pairs):
    for t, tc in pairs:
        if tc is not t:
            t.copy_(tc)


def _float(t):
    return None if t is None else t.float()


def _forward(x, weight, bias, offset, mask, output, kh, kw, sh, sw, ph, pw, dh, dw, group, dg):
    _check(x, weight, bias)
    offset, mask = offset.to(x.dtype), _in_dtype(mask, x.dtype)
    if output.dtype != x.dtype:
        raise RuntimeError("megreader_b200 dcn: output is %s, input %s" % (output.dtype, x.dtype))
    B, C, H, W = x.shape
    Cout = weight.size(0)
    if weight.size(2) != kh or weight.size(3) != kw:
        raise RuntimeError("Input shape and kernel shape wont match: (%d x %d vs %d x %d)."
                           % (kh, kw, weight.size(2), weight.size(3)))           # :506-508
    if C != weight.size(1) * group:
        raise RuntimeError("Input shape and kernel channels wont match: (%d vs %d)." % (C, weight.size(1) * group))
    Ho, Wo = _out_hw(H, W, kh, kw, sh, sw, ph, pw, dh, dw)
    offset_in, mask_in = offset, mask
    offset, obs = _slab(offset)
    mbs = 0
    if mask is not None:
        mask, mbs = _slab(mask)
    assert output.is_contiguous() and output.numel() == B * Cout * Ho * Wo
    if x.dtype != torch.float32:
        code, wcode = _codes(x, weight)
        ws_bytes = _lib.lib().mr_dcn_fused_workspace_bytes_h(B, C, H, W, Cout, kh, kw)
        ws = _half_workspace(x, ws_bytes)
        p = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
        with torch.cuda.device(x.device):
            rc = _lib.lib().mr_dcn_forward_fused_h(
                x.data_ptr(), weight.data_ptr(), p(bias), offset.data_ptr(), obs, p(mask), mbs, output.data_ptr(),
                ws.data_ptr(), ws_bytes, B, C, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, group, dg, code, wcode, _stream())
        if rc != _lib.MR_ERR_UNSUPPORTED:
            _lib.check(rc, "dcn_forward")
            return
        # outside the fused path: the fp32 kernels on fp32 copies
        out32 = torch.empty(output.shape, dtype=torch.float32, device=output.device)
        _forward(x.float(), weight.float(), _float(bias), offset_in.float(), _float(mask_in), out32, kh, kw, sh, sw, ph, pw,
                 dh, dw, group, dg)
        output.copy_(out32)
        return
    ws, ws_bytes = _workspace(x, C, kh, kw, Ho, Wo, Cout)
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().mr_dcn_forward_f32(
            x.data_ptr(), weight.data_ptr(), bias.data_ptr() if bias is not None else None, offset.data_ptr(), obs,
            mask.data_ptr() if mask is not None else None, mbs, output.data_ptr(), ws.data_ptr(), ws_bytes,
            B, C, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, group, dg, _stream()), "dcn_forward")


def _backward(x, weight, offset, mask, grad_output, grad_input, grad_weight, grad_bias, grad_offset, grad_mask,
              scale, kh, kw, sh, sw, ph, pw, dh, dw, group, dg):
    _check(x, weight)
    if grad_input is not None and grad_input.dtype != x.dtype:
        raise RuntimeError("megreader_b200 dcn: grad_input is %s, input %s" % (grad_input.dtype, x.dtype))
    for g in (grad_weight, grad_bias):
        if g is not None and g.dtype != weight.dtype:
            raise RuntimeError("megreader_b200 dcn: weight gradients are %s, weight %s" % (g.dtype, weight.dtype))
    # offset / mask (and their gradients) in x's dtype; gradients allocated in another dtype get the result copied back
    offset, mask, grad_output = offset.to(x.dtype), _in_dtype(mask, x.dtype), grad_output.to(x.dtype)
    goff_c, gmask_c = _in_dtype(grad_offset, x.dtype), _in_dtype(grad_mask, x.dtype)
    _backward_same_dtype(x, weight, offset, mask, grad_output, grad_input, grad_weight, grad_bias, goff_c, gmask_c, scale,
                         kh, kw, sh, sw, ph, pw, dh, dw, group, dg)
    _write_back([(grad_offset, goff_c), (grad_mask, gmask_c)])


def _backward_same_dtype(x, weight, offset, mask, grad_output, grad_input, grad_weight, grad_bias, grad_offset, grad_mask,
                         scale, kh, kw, sh, sw, ph, pw, dh, dw, group, dg):
    B, C, H, W = x.shape
    Cout = weight.size(0)
    Ho, Wo = _out_hw(H, W, kh, kw, sh, sw, ph, pw, dh, dw)
    offset_in, mask_in = offset, mask
    offset, obs = _slab(offset)
    mbs = gobs = gmbs = 0
    if mask is not None:
        mask, mbs = _slab(mask)
    if grad_offset is not None:
        assert grad_offset.size(0) == 0 or grad_offset[0].is_contiguous()
        gobs = _slab(grad_offset)[1]
    if grad_mask is not None:
        assert grad_mask.size(0) == 0 or grad_mask[0].is_contiguous()
        gmbs = _slab(grad_mask)[1]
    grad_output = grad_output.contiguous()
    p = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    if x.dtype != torch.float32:
        code, wcode = _codes(x, weight)
        ws_bytes = _lib.lib().mr_dcn_fused_backward_workspace_bytes_h(B, C, H, W, Cout, Ho, Wo, kh, kw)
        ws = _half_workspace(x, ws_bytes)
        with torch.cuda.device(x.device):
            rc = _lib.lib().mr_dcn_backward_fused_h(
                x.data_ptr(), weight.data_ptr(), offset.data_ptr(), obs, p(mask), mbs, grad_output.data_ptr(),
                p(grad_input), p(grad_weight), p(grad_bias), p(grad_offset), gobs, p(grad_mask), gmbs, float(scale),
                ws.data_ptr(), ws_bytes, B, C, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, group, dg, code, wcode, _stream())
        if rc != _lib.MR_ERR_UNSUPPORTED:
            _lib.check(rc, "dcn_backward")
            return
        # outside the fused path: the fp32 kernels on fp32 copies (the accumulating gradients start from the caller's values)
        grads = (grad_input, grad_weight, grad_bias, grad_offset, grad_mask)
        g32 = [_float(g) for g in grads]
        _backward_same_dtype(x.float(), weight.float(), offset_in.float(), _float(mask_in), grad_output.float(), *g32, scale,
                             kh, kw, sh, sw, ph, pw, dh, dw, group, dg)
        _write_back([(g, gc) for g, gc in zip(grads, g32) if g is not None])
        return
    ws, ws_bytes = _workspace(x, C, kh, kw, Ho, Wo, Cout, backward=True)
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().mr_dcn_backward_f32(
            x.data_ptr(), weight.data_ptr(), offset.data_ptr(), obs, p(mask), mbs, grad_output.data_ptr(),
            p(grad_input), p(grad_weight), p(grad_bias), p(grad_offset), gobs, p(grad_mask), gmbs, float(scale),
            ws.data_ptr(), ws_bytes, B, C, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, group, dg, _stream()),
            "dcn_backward")


# ---- the five functions the reference's extension exports (deform_conv_cuda.cpp:681-695) -------------------------
def modulated_deform_conv_cuda_forward(input, weight, bias, ones, offset, mask, output, columns, kernel_h, kernel_w,
                                       stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w, group,
                                       deformable_group, with_bias):
    """deform_conv_cuda.cpp:486-564.  Writes `output` in place; `ones` / `columns` are ignored scratch handles."""
    _forward(input, weight, bias if with_bias else None, offset, mask, output, kernel_h, kernel_w, stride_h, stride_w,
             pad_h, pad_w, dilation_h, dilation_w, group, deformable_group)


def modulated_deform_conv_cuda_backward(input, weight, bias, ones, offset, mask, columns, grad_input, grad_weight,
                                        grad_bias, grad_offset, grad_mask, grad_output, kernel_h, kernel_w, stride_h,
                                        stride_w, pad_h, pad_w, dilation_h, dilation_w, group, deformable_group,
                                        with_bias):
    """deform_conv_cuda.cpp:566-679.  Accumulates into the caller-zeroed grad_* tensors."""
    _backward(input, weight, offset, mask, grad_output, grad_input, grad_weight, grad_bias if with_bias else None,
              grad_offset, grad_mask, 1.0, kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w, dilation_h,
              dilation_w, group, deformable_group)


def _v1_shape_check(input, offset, weight, kH, kW, dH, dW, padH, padW, dilationH, dilationW, group, dg):
    """shape_check, deform_conv_cuda.cpp:61-149 (the checks that can fire from the python wrappers)."""
    if weight.dim() != 4:
        raise RuntimeError("4D weight tensor (nOutputPlane,nInputPlane,kH,kW) expected, but got: %s" % weight.dim())
    if not (kW > 0 and kH > 0 and dW > 0 and dH > 0 and dilationW > 0 and dilationH > 0):
        raise RuntimeError("kernel size, stride and dilation should be greater than zero")
    if input.dim() != 4:
        raise RuntimeError("3D or 4D input tensor expected but got: %s" % input.dim())
    B, C, H, W = input.shape
    if C != weight.size(1) * group:
        raise RuntimeError("invalid number of input planes, expected: %d, but got: %d" % (weight.size(1) * group, C))
    Ho, Wo = _out_hw(H, W, kH, kW, dH, dW, padH, padW, dilationH, dilationW)
    if Ho < 1 or Wo < 1:
        raise RuntimeError("Given input size: (%d x %d x %d). Calculated output size: (%d x %d x %d). Output size is "
                           "too small" % (C, H, W, weight.size(0), Ho, Wo))
    if offset.size(2) != Ho or offset.size(3) != Wo:
        raise RuntimeError("invalid spatial size of offset, expected height: %d width: %d, but got height: %d width: "
                           "%d" % (Ho, Wo, offset.size(2), offset.size(3)))                       # :129-132
    if offset.size(1) != dg * 2 * kH * kW:
        raise RuntimeError("invalid number of channels of offset")                                # :134-135


def deform_conv_forward_cuda(input, weight, offset, output, columns, ones, kW, kH, dW, dH, padW, padH, dilationW,
                             dilationH, group, deformable_group, im2col_step):
    """deform_conv_cuda.cpp:151-258 (DCNv1)."""
    _v1_shape_check(input, offset, weight, kH, kW, dH, dW, padH, padW, dilationH, dilationW, group, deformable_group)
    _forward(input, weight, None, offset, None, output, kH, kW, dH, dW, padH, padW, dilationH, dilationW, group,
             deformable_group)
    return 1


def deform_conv_backward_input_cuda(input, offset, gradOutput, gradInput, gradOffset, weight, columns, kW, kH, dW, dH,
                                    padW, padH, dilationW, dilationH, group, deformable_group, im2col_step):
    """deform_conv_cuda.cpp:260-371."""
    _v1_shape_check(input, offset, weight, kH, kW, dH, dW, padH, padW, dilationH, dilationW, group, deformable_group)
    _backward(input, weight, offset, None, gradOutput, gradInput, None, None, gradOffset, None, 1.0, kH, kW, dH, dW,
              padH, padW, dilationH, dilationW, group, deformable_group)
    return 1


def deform_conv_backward_parameters_cuda(input, offset, gradOutput, gradWeight, columns, ones, kW, kH, dW, dH, padW,
                                         padH, dilationW, dilationH, group, deformable_group, scale, im2col_step):
    """deform_conv_cuda.cpp:373-484.  gradWeight += scale * dW."""
    _backward(input, gradWeight.new_empty(gradWeight.shape), offset, None, gradOutput, None, gradWeight, None, None,
              None, scale, kH, kW, dH, dW, padH, padW, dilationH, dilationW, group, deformable_group)
    return 1


# ---- autograd Functions (functions/deform_conv.py) ----------------------------------------------------------------
class DeformConvFunction(Function):
    """functions/deform_conv.py:8-105."""

    @staticmethod
    def forward(ctx, input, offset, weight, stride=1, padding=0, dilation=1, groups=1, deformable_groups=1,
                im2col_step=64):
        if input is not None and input.dim() != 4:
            raise ValueError("Expected 4D tensor as input, got {}D tensor instead.".format(input.dim()))
        ctx.stride, ctx.padding, ctx.dilation = _pair(stride), _pair(padding), _pair(dilation)
        ctx.groups, ctx.deformable_groups, ctx.im2col_step = groups, deformable_groups, im2col_step
        ctx.save_for_backward(input, offset, weight)
        output = input.new_empty(DeformConvFunction._output_size(input, weight, ctx.padding, ctx.dilation, ctx.stride))
        if not input.is_cuda:
            raise NotImplementedError
        step = min(im2col_step, input.shape[0])
        assert input.shape[0] % step == 0, 'im2col step must divide batchsize'          # :43-45
        deform_conv_forward_cuda(input, weight, offset, output, None, None, weight.size(3), weight.size(2),
                                 ctx.stride[1], ctx.stride[0], ctx.padding[1], ctx.padding[0], ctx.dilation[1],
                                 ctx.dilation[0], groups, deformable_groups, step)
        return output

    @staticmethod
    def backward(ctx, grad_output):
        input, offset, weight = ctx.saved_tensors
        grad_input = grad_offset = grad_weight = None
        if not grad_output.is_cuda:
            raise NotImplementedError
        step = min(ctx.im2col_step, input.shape[0])
        assert input.shape[0] % step == 0, 'im2col step must divide batchsize'
        args = (weight.size(3), weight.size(2), ctx.stride[1], ctx.stride[0], ctx.padding[1], ctx.padding[0],
                ctx.dilation[1], ctx.dilation[0], ctx.groups, ctx.deformable_groups)
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
            grad_input = torch.zeros_like(input)
            grad_offset = torch.zeros_like(offset)
            deform_conv_backward_input_cuda(input, offset, grad_output, grad_input, grad_offset, weight, None, *args,
                                            step)
        if ctx.needs_input_grad[2]:
            grad_weight = torch.zeros_like(weight)
            _backward(input, weight, offset, None, grad_output, None, grad_weight, None, None, None, 1.0,
                      weight.size(2), weight.size(3), ctx.stride[0], ctx.stride[1], ctx.padding[0], ctx.padding[1],
                      ctx.dilation[0], ctx.dilation[1], ctx.groups, ctx.deformable_groups)
        return grad_input, grad_offset, grad_weight, None, None, None, None, None, None

    @staticmethod
    def _output_size(input, weight, padding, dilation, stride):
        size = (input.size(0), weight.size(0))
        for d in range(input.dim() - 2):
            kernel = dilation[d] * (weight.size(d + 2) - 1) + 1
            size += ((input.size(d + 2) + 2 * padding[d] - kernel) // stride[d] + 1,)
        if not all(s > 0 for s in size):
            raise ValueError("convolution input is too small (output would be {})".format('x'.join(map(str, size))))
        return size


class ModulatedDeformConvFunction(Function):
    """functions/deform_conv.py:108-177: scalar stride / padding / dilation used for both axes (:140-142)."""

    @staticmethod
    def forward(ctx, input, offset, mask, weight, bias=None, stride=1, padding=0, dilation=1, groups=1,
                deformable_groups=1):
        ctx.stride, ctx.padding, ctx.dilation = stride, padding, dilation
        ctx.groups, ctx.deformable_groups = groups, deformable_groups
        ctx.with_bias = bias is not None
        if not input.is_cuda:
            raise NotImplementedError
        ctx.save_for_backward(input, offset, mask, weight, bias if ctx.with_bias else input.new_empty(1))
        output = input.new_empty(ModulatedDeformConvFunction._infer_shape(ctx, input, weight))
        modulated_deform_conv_cuda_forward(input, weight, bias, None, offset, mask, output, None, weight.shape[2],
                                           weight.shape[3], stride, stride, padding, padding, dilation, dilation,
                                           groups, deformable_groups, ctx.with_bias)
        return output

    @staticmethod
    def backward(ctx, grad_output):
        if not grad_output.is_cuda:
            raise NotImplementedError
        input, offset, mask, weight, bias = ctx.saved_tensors
        grad_input = torch.zeros_like(input)
        grad_offset = torch.zeros_like(offset)
        grad_mask = torch.zeros_like(mask)
        grad_weight = torch.zeros_like(weight)
        grad_bias = torch.zeros_like(bias)
        modulated_deform_conv_cuda_backward(input, weight, bias, None, offset, mask, None, grad_input, grad_weight,
                                            grad_bias, grad_offset, grad_mask, grad_output, weight.shape[2],
                                            weight.shape[3], ctx.stride, ctx.stride, ctx.padding, ctx.padding,
                                            ctx.dilation, ctx.dilation, ctx.groups, ctx.deformable_groups,
                                            ctx.with_bias)
        if not ctx.with_bias:
            grad_bias = None
        return grad_input, grad_offset, grad_mask, grad_weight, grad_bias, None, None, None, None, None

    @staticmethod
    def _infer_shape(ctx, input, weight):
        Ho, Wo = _out_hw(input.size(2), input.size(3), weight.size(2), weight.size(3), ctx.stride, ctx.stride,
                         ctx.padding, ctx.padding, ctx.dilation, ctx.dilation)
        return input.size(0), weight.size(0), Ho, Wo


deform_conv = DeformConvFunction.apply
modulated_deform_conv = ModulatedDeformConvFunction.apply


# ---- modules (modules/deform_conv.py): parameter names `weight`, `bias`, `conv_offset`, `conv_offset_mask` ---------
def _uniform_init(weight, in_channels, kernel_size):
    n = in_channels
    for k in kernel_size:
        n *= k
    stdv = 1. / math.sqrt(n)
    weight.data.uniform_(-stdv, stdv)


class DeformConv(nn.Module):
    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 deformable_groups=1, bias=False):
        super().__init__()
        assert not bias
        assert in_channels % groups == 0, 'in_channels {} cannot be divisible by groups {}'.format(in_channels, groups)
        assert out_channels % groups == 0, 'out_channels {} cannot be divisible by groups {}'.format(out_channels, groups)
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size, self.stride = _pair(kernel_size), _pair(stride)
        self.padding, self.dilation = _pair(padding), _pair(dilation)
        self.groups, self.deformable_groups = groups, deformable_groups
        self.weight = nn.Parameter(torch.Tensor(out_channels, in_channels // groups, *self.kernel_size))
        self.reset_parameters()

    def reset_parameters(self):
        _uniform_init(self.weight, self.in_channels, self.kernel_size)

    def forward(self, x, offset):
        return deform_conv(x, offset, self.weight, self.stride, self.padding, self.dilation, self.groups,
                           self.deformable_groups)


class DeformConvPack(DeformConv):
    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.conv_offset = nn.Conv2d(self.in_channels,
                                     self.deformable_groups * 2 * self.kernel_size[0] * self.kernel_size[1],
                                     kernel_size=self.kernel_size, stride=_pair(self.stride),
                                     padding=_pair(self.padding), bias=True)
        self.init_offset()

    def init_offset(self):
        self.conv_offset.weight.data.zero_()
        self.conv_offset.bias.data.zero_()

    def forward(self, x):
        return deform_conv(x, self.conv_offset(x), self.weight, self.stride, self.padding, self.dilation, self.groups,
                           self.deformable_groups)


class ModulatedDeformConv(nn.Module):
    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 deformable_groups=1, bias=True):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size = _pair(kernel_size)
        self.stride, self.padding, self.dilation = stride, padding, dilation
        self.groups, self.deformable_groups = groups, deformable_groups
        self.with_bias = bias
        self.weight = nn.Parameter(torch.Tensor(out_channels, in_channels // groups, *self.kernel_size))
        if bias:
            self.bias = nn.Parameter(torch.Tensor(out_channels))
        else:
            self.register_parameter('bias', None)
        self.reset_parameters()

    def reset_parameters(self):
        _uniform_init(self.weight, self.in_channels, self.kernel_size)
        if self.bias is not None:
            self.bias.data.zero_()

    def forward(self, x, offset, mask):
        return modulated_deform_conv(x, offset, mask, self.weight, self.bias, self.stride, self.padding,
                                     self.dilation, self.groups, self.deformable_groups)


class ModulatedDeformConvPack(ModulatedDeformConv):
    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.conv_offset_mask = nn.Conv2d(self.in_channels,
                                          self.deformable_groups * 3 * self.kernel_size[0] * self.kernel_size[1],
                                          kernel_size=self.kernel_size, stride=_pair(self.stride),
                                          padding=_pair(self.padding), bias=True)
        self.init_offset()

    def init_offset(self):
        self.conv_offset_mask.weight.data.zero_()
        self.conv_offset_mask.bias.data.zero_()

    def forward(self, x):
        out = self.conv_offset_mask(x)
        o1, o2, mask = torch.chunk(out, 3, dim=1)
        offset = torch.cat((o1, o2), dim=1)
        return modulated_deform_conv(x, offset, torch.sigmoid(mask), self.weight, self.bias, self.stride,
                                     self.padding, self.dilation, self.groups, self.deformable_groups)
