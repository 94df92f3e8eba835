"""General 2-D convolution on the wgmma implicit-GEMM kernels (csrc/gemm_tcgen05.cu) as an autograd Function, and the module
swap that puts the reference-named trunks on it.

    conv2d(x, weight, bias, stride, padding, dilation)            x, result: (N, C, H, W) bf16 in channels_last memory
    EngineConv2d                                                   nn.Conv2d subclass (same parameters / state-dict keys)
    EngineBatchNorm2d                                              nn.BatchNorm2d subclass on the NHWC row kernels of the CRNN engine
    use_engine_convs(module)                                       swaps every eligible nn.Conv2d / nn.BatchNorm2d of a trunk in place

Covers what the ResNet-50 / dilated / PPM / FPN trunks and the 2D-CTC head branches use (backbones/resnet.py:110-256,
resnet_dilated.py:50-69, ppm.py:6-44, fpn_top_down.py:6-30, decoders/ctc_decoder2d.py:16-27): 1x1 and 3x3 kernels, stride 1 / 2,
any dilation, groups = 1, C_in % 64 == 0; the stem (C_in = 3, 7x7 stride 2) is an unfold + the same tensor-core GEMM.
bf16 operands, fp32 accumulation, fp32 master weights.  Forward = implicit GEMM; input gradient = implicit GEMM of dz with the
flipped / transposed weights (stride 2: over the zero-upsampled dz); weight gradient = implicit GEMM over pixels (split-K).
CUDA only -- there is no CPU fallback."""
import os

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import nnops as ops


def _pad_to(n, m):
    return -(-n // m) * m


# Weight gradients off the critical path.  A convolution's weight gradient depends only on dz and the saved input, and nothing in
# the backward pass consumes it (the parameter's .grad is read after backward() returns), while the input gradient feeds the next
# layer's BatchNorm / ReLU / convolution chain -- small dependent kernels that leave most SMs idle at the configured batches.  So the
# weight-gradient kernels of leaf parameters whose .grad is still unset run on a side stream (forked from the backward's stream, one
# per device) and are joined by a callback the autograd engine runs at the end of the backward pass: transparent to the caller, and
# captured as a parallel branch when the step is recorded into a CUDA graph.  OFF by default: code that reads a gradient INSIDE the
# backward pass on the backward's stream (parameter hooks, e.g. a bucketing DistributedDataParallel wrapper) would read it before
# the join.  A training loop that only touches gradients after backward() returns switches it on with
# use_engine_convs(model, wgrad_side_stream=True) (bench_trunks.py does) or MR_CONV_WGRAD_SIDE_STREAM=1.
WGRAD_SIDE_STREAM = os.environ.get("MR_CONV_WGRAD_SIDE_STREAM", "0") == "1"
_side_streams = {}
_pending = {}


def _side_stream(device):
    key = device.index if device.index is not None else torch.cuda.current_device()
    if key not in _side_streams:
        _side_streams[key] = torch.cuda.Stream(device=device)
        _pending[key] = []
    return key, _side_streams[key]


def _join_side_streams():
    """end-of-backward callback: the stream that ran backward() waits for every weight gradient still in flight"""
    for key, events in _pending.items():
        if events:
            cur = torch.cuda.current_stream(key)
            for ev in events:
                cur.wait_event(ev)
            events.clear()


class _Conv2dFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, stride, padding, dilation):
        if not x.is_cuda:
            raise NotImplementedError("megreader_b200.conv_engine: CUDA tensors only (no CPU fallback)")
        Cout, Cin, kh, kw = weight.shape
        sh, sw = stride
        ph, pw = padding
        dh, dw = dilation
        N, C, H, W = x.shape
        assert C == Cin and Cin % 64 == 0
        if x.numel() == 0 or (H + 2 * ph - dh * (kh - 1) - 1) // sh + 1 <= 0 or (W + 2 * pw - dw * (kw - 1) - 1) // sw + 1 <= 0:
            raise RuntimeError("megreader_b200.conv_engine: empty convolution problem: input %s, kernel %s, stride %s, padding %s, "
                               "dilation %s" % (tuple(x.shape), (kh, kw), stride, padding, dilation))
        xh = x.to(torch.bfloat16).contiguous(memory_format=torch.channels_last).permute(0, 2, 3, 1).contiguous()   # NHWC
        Cp = _pad_to(Cout, 8)                                   # weight-gradient kernel wants Cout % 8 == 0
        Wm = ops.conv_weight_pack(weight.detach().float().contiguous(), Cin, kh * kw * Cin, torch.bfloat16, 0)   # [Cout, K]
        if Cp != Cout:
            Wm = F.pad(Wm, (0, 0, 0, Cp - Cout))
        bz = None
        if bias is not None:
            bz = bias.detach().float()
            if Cp != Cout:
                bz = F.pad(bz, (0, Cp - Cout))
        y, Ho, Wo = ops.conv2d_fprop_tc(xh, Wm, kh, kw, sh, sw, ph, pw, dh, dw, bias=bz)
        ctx.save_for_backward(xh, weight)
        ctx.geo = (N, H, W, Cin, Cout, Cp, kh, kw, sh, sw, ph, pw, dh, dw, Ho, Wo, bias is not None, x.dtype)
        out = y.view(N, Ho, Wo, Cp)
        if Cp != Cout:
            out = out[..., :Cout]
        return out.permute(0, 3, 1, 2)                          # (N, Cout, Ho, Wo) view, channels_last memory

    @staticmethod
    def backward(ctx, dy):
        xh, weight = ctx.saved_tensors
        N, H, W, Cin, Cout, Cp, kh, kw, sh, sw, ph, pw, dh, dw, Ho, Wo, has_bias, in_dtype = ctx.geo
        dz = dy.permute(0, 2, 3, 1).to(torch.bfloat16)
        if Cp != Cout:
            dz = F.pad(dz, (0, Cp - Cout))
        dz = dz.contiguous()                                    # [N, Ho, Wo, Cp]
        dx = dw_ = db = None
        if ctx.needs_input_grad[1]:
            def wgrad():
                dWm = ops.conv2d_wgrad_tc(dz, xh, kh, kw, sh, sw, ph, pw, dh, dw)           # [Cp, kh*kw*Cin] fp32
                return dWm[:Cout].view(Cout, kh, kw, Cin).permute(0, 3, 1, 2).contiguous().to(weight.dtype)
            if WGRAD_SIDE_STREAM and weight.is_leaf and weight.grad is None and not torch.is_grad_enabled():
                cur = torch.cuda.current_stream(dz.device)
                key, side = _side_stream(dz.device)
                side.wait_stream(cur)                           # dz and the saved input are complete on `cur` here
                with torch.cuda.stream(side):
                    dw_ = wgrad()
                    ev = torch.cuda.Event()
                    ev.record(side)
                for t in (dz, xh):
                    t.record_stream(side)                       # the allocator must not hand their memory out before `side` is done
                dw_.record_stream(cur)                          # allocated on `side`, consumed on `cur` after the join
                _pending[key].append(ev)
                # one callback per weight gradient (the first to run joins them all): nothing is left behind if an earlier backward
                # pass died before its callback ran
                torch.autograd.Variable._execution_engine.queue_callback(_join_side_streams)
            else:
                dw_ = wgrad()
        if has_bias and ctx.needs_input_grad[2]:
            db = dz.view(-1, Cp)[:, :Cout].float().sum(0)
        if ctx.needs_input_grad[0]:
            # dgrad = stride-1 convolution of (zero-upsampled) dz with the flipped, transposed weights, padding d*(k-1) - p
            Kp = _pad_to(Cp, 64)                                # the forward kernel wants its channel count % 64 == 0
            if Kp == Cout:
                # one launch: [Cin][(flipped tap) * Cout + co] bf16 straight from the fp32 master weights
                Wd = ops.conv_weight_pack(weight.detach().float().contiguous(), Cin, kh * kw * Cin, torch.bfloat16, 1)
            else:                                               # few-channel heads (Cout = 1, 38): pad through the framework
                w = weight.detach().float()
                Wd = w.flip(2, 3).permute(1, 2, 3, 0)           # [Cin, kh, kw, Cout]
                Wd = F.pad(Wd, (0, Kp - Cout))
                dz = F.pad(dz, (0, Kp - Cp))
                Wd = Wd.reshape(Cin, kh * kw * Kp).to(torch.bfloat16).contiguous()
            if sh > 1 or sw > 1:
                Hu, Wu = (Ho - 1) * sh + 1, (Wo - 1) * sw + 1
                up = torch.zeros((N, Hu, Wu, Kp), dtype=torch.bfloat16, device=dz.device)
                up[:, ::sh, ::sw] = dz
                dz = up
            qh, qw = dh * (kh - 1) - ph, dw * (kw - 1) - pw
            # output size of the transposed problem must be (H, W): rows lost to the stride's floor come back as extra padding
            Hd, Wd_ = dz.size(1), dz.size(2)
            eh, ew = H - (Hd + 2 * qh - dh * (kh - 1)), W - (Wd_ + 2 * qw - dw * (kw - 1))
            if qh < 0 or qw < 0 or eh or ew:
                # asymmetric / negative padding: materialise it (rare: only when p > d*(k-1) or the stride drops rows)
                dz = F.pad(dz, (0, 0, max(qw, 0), max(qw, 0) + max(ew, 0), max(qh, 0), max(qh, 0) + max(eh, 0)))
                if qh < 0 or qw < 0:
                    dz = dz[:, -qh if qh < 0 else 0:, -qw if qw < 0 else 0:]
                dz = dz.contiguous()
                qh = qw = 0
            g, Hg, Wg = ops.conv2d_fprop_tc(dz.contiguous(), Wd, kh, kw, 1, 1, qh, qw, dh, dw)
            assert (Hg, Wg) == (H, W), ((Hg, Wg), (H, W))
            dx = g.view(N, H, W, Cin).permute(0, 3, 1, 2).to(in_dtype)
        return dx, dw_, db, None, None, None


def conv2d(x, weight, bias=None, stride=(1, 1), padding=(0, 0), dilation=(1, 1)):
    return _Conv2dFn.apply(x, weight, bias, tuple(stride), tuple(padding), tuple(dilation))


class _StemFn(torch.autograd.Function):
    """Convolutions whose input has few channels (the 7x7 stride-2 stem on RGB, backbones/resnet.py:198): unfold + one
    tensor-core GEMM (K = C*kh*kw padded to 64).  The images need no gradient."""

    @staticmethod
    def forward(ctx, x, weight, bias, stride, padding, dilation):
        Cout, Cin, kh, kw = weight.shape
        N, C, H, W = x.shape
        cols = F.unfold(x.float(), (kh, kw), dilation, padding, stride)           # [N, C*kh*kw, L]
        L = cols.size(2)
        K = Cin * kh * kw
        Kp = _pad_to(K, 64)
        A = torch.zeros((N * L, Kp), dtype=torch.bfloat16, device=x.device)
        A[:, :K] = cols.transpose(1, 2).reshape(N * L, K)
        Wm = torch.zeros((Cout, Kp), dtype=torch.bfloat16, device=x.device)
        Wm[:, :K] = weight.detach().reshape(Cout, K)
        y = ops.gemm_tc(A, Wm, transB=True, out_dtype=torch.bfloat16, bias=bias.detach().float() if bias is not None else None)
        Ho = (H + 2 * padding[0] - dilation[0] * (kh - 1) - 1) // stride[0] + 1
        Wo = L // Ho
        ctx.save_for_backward(A)
        ctx.geo = (Cout, Cin, kh, kw, K, bias is not None, weight.dtype)
        return y.view(N, Ho, Wo, Cout).permute(0, 3, 1, 2)

    @staticmethod
    def backward(ctx, dy):
        (A,) = ctx.saved_tensors
        Cout, Cin, kh, kw, K, has_bias, wdtype = ctx.geo
        dz = dy.permute(0, 2, 3, 1).reshape(-1, Cout).to(torch.bfloat16).contiguous()
        # [Cout, Kp] = dz^T A: a tiny output over a reduction as long as the batch has pixels (524,288 rows at 8 x 512 x 512) --
        # split-K over up to 128 CTAs, fp32 atomics into the zero-filled result
        splits = max(1, min(128, dz.size(0) // 4096))
        if splits > 1:
            dWm = torch.zeros((Cout, A.size(1)), dtype=torch.float32, device=dz.device)
            ops.gemm_tc(dz, A, transA=True, transB=False, out=dWm, beta=1.0, splits=splits)
        else:
            dWm = ops.gemm_tc(dz, A, transA=True, transB=False, out_dtype=torch.float32)
        dw_ = dWm[:, :K].reshape(Cout, Cin, kh, kw).to(wdtype)
        db = dz.float().sum(0) if has_bias else None
        return None, dw_, db, None, None, None


class EngineConv2d(nn.Conv2d):
    """nn.Conv2d whose arithmetic runs on megreader_b200's wgmma kernels (same parameters, same state-dict keys)."""

    def forward(self, x):
        if self.groups != 1 or self.padding_mode != "zeros" or isinstance(self.padding, str):
            raise NotImplementedError("EngineConv2d: groups = 1, zero padding only")
        if self.in_channels % 64 == 0:
            return conv2d(x, self.weight, self.bias, self.stride, self.padding, self.dilation)
        return _StemFn.apply(x, self.weight, self.bias, self.stride, self.padding, self.dilation)


class _BatchNormFn(torch.autograd.Function):
    """nn.BatchNorm2d on the NHWC row kernels of csrc/nn_kernels.cu (the CRNN engine's: column statistics through block partials,
    row-tiled normalisation, fused backward): x (N, C, H, W) in channels_last memory, bf16 or fp32, C % 8 == 0."""

    @staticmethod
    def forward(ctx, x, gamma, beta, running_mean, running_var, momentum, eps, batch_stats):
        N, C, H, W = x.shape
        rows = x.contiguous(memory_format=torch.channels_last).permute(0, 2, 3, 1).reshape(N * H * W, C)
        g, b = gamma.detach().float(), beta.detach().float()
        # the result is a fresh channels_last tensor (not a view made inside the Function: an in-place ReLU may follow); the kernels
        # write its NHWC rows
        out = torch.empty((N, C, H, W), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
        out_rows = out.permute(0, 2, 3, 1).reshape(N * H * W, C)
        assert out_rows.data_ptr() == out.data_ptr() and rows.is_contiguous()
        if batch_stats:
            _, mean, invstd = ops.bn_train_fwd(rows, None, g, b, running_mean, running_var, momentum, eps, out=out_rows)
        else:
            mean = running_mean.float()
            invstd = torch.rsqrt(running_var.float() + eps)
            ops.bn_apply(rows, None, mean, invstd, g, b, out=out_rows)
        ctx.save_for_backward(rows, mean, invstd, g)
        ctx.batch_stats = batch_stats
        ctx.shape = (N, C, H, W)
        return out

    @staticmethod
    def backward(ctx, dy):
        rows, mean, invstd, g = ctx.saved_tensors
        N, C, H, W = ctx.shape
        dyr = dy.to(rows.dtype).contiguous(memory_format=torch.channels_last).permute(0, 2, 3, 1).reshape(N * H * W, C)
        dx = torch.empty((N, C, H, W), dtype=rows.dtype, device=rows.device, memory_format=torch.channels_last)
        dx_rows = dx.permute(0, 2, 3, 1).reshape(N * H * W, C)
        if ctx.batch_stats:
            _, dgamma, dbeta, _ = ops.bn_train_bwd(dyr, rows, None, mean, invstd, g, want_dbias=False, out=dx_rows)
        else:                                                   # frozen statistics: an affine map per channel
            d32 = dyr.float()
            dbeta = d32.sum(0)
            dgamma = (d32 * ((rows.float() - mean) * invstd)).sum(0)
            dx_rows.copy_(d32 * (g * invstd))
        return dx, dgamma, dbeta, None, None, None, None, None


class EngineBatchNorm2d(nn.BatchNorm2d):
    """nn.BatchNorm2d whose arithmetic runs on megreader_b200's NHWC kernels (same parameters / buffers / state-dict keys).
    Configurations the kernels do not cover (no affine parameters, no running statistics, cumulative momentum, C % 8 != 0) go
    through the framework's CUDA implementation; CPU tensors raise."""

    def forward(self, x):
        if not x.is_cuda:
            raise NotImplementedError("megreader_b200.conv_engine: CUDA tensors only (no CPU fallback); restore_library_convs() "
                                      "gives the framework modules back")
        if (x.dim() != 4 or not self.affine or not self.track_running_stats or self.momentum is None
                or self.num_features % 8 or x.dtype not in (torch.float32, torch.bfloat16) or x.numel() == 0):
            return super().forward(x)
        if self.training:
            if x.numel() // x.size(1) <= 1:                     # same refusal as torch.nn.functional.batch_norm
                raise ValueError("Expected more than 1 value per channel when training, got input size %s" % (tuple(x.shape),))
            self.num_batches_tracked.add_(1)
        return _BatchNormFn.apply(x, self.weight, self.bias, self.running_mean, self.running_var, float(self.momentum),
                                  float(self.eps), bool(self.training))


class EngineConvTranspose2d(nn.ConvTranspose2d):
    """nn.ConvTranspose2d with kernel = stride = 2 x 2 (the up-sampling layers of decoders/east.py:20-21) on the wgmma convolution
    kernels: such a layer is a 1 x 1 convolution to 4 * C_out channels -- one output channel block per (row, column) offset inside the
    2 x 2 cell -- followed by a depth-to-space rearrangement.  The weight re-layout and the rearrangement are framework views / copies,
    so autograd carries the gradients back to the reference-shaped parameters.  Other geometries use the library implementation."""

    def _engine_ok(self, x):
        if not x.is_cuda:
            raise NotImplementedError("megreader_b200.conv_engine: CUDA tensors only (no CPU fallback); restore_library_convs() "
                                      "gives the framework modules back")
        return (x.dim() == 4 and tuple(self.kernel_size) == (2, 2) and tuple(self.stride) == (2, 2)
                and tuple(self.padding) == (0, 0) and tuple(self.output_padding) == (0, 0) and tuple(self.dilation) == (1, 1)
                and self.groups == 1 and self.in_channels % 64 == 0)

    def forward(self, x, output_size=None):
        if output_size is not None or not self._engine_ok(x):
            return super().forward(x, output_size)
        cin, cout = self.in_channels, self.out_channels
        n, _, h, w = x.shape
        w_eq = self.weight.permute(2, 3, 1, 0).reshape(4 * cout, cin, 1, 1)        # row (a * 2 + b) * C_out + co  <-  W[ci, co, a, b]
        b_eq = self.bias.repeat(4) if self.bias is not None else None
        y = conv2d(x, w_eq, b_eq)                                                    # (N, 4 C_out, H, W), NHWC memory
        yh = y.permute(0, 2, 3, 1).reshape(n, h, w, 2, 2, cout)                      # (N, H, W, a, b, C_out): still a view
        out = yh.permute(0, 1, 3, 2, 4, 5).reshape(n, 2 * h, 2 * w, cout)            # (N, 2H, 2W, C_out): the one copy
        return out.permute(0, 3, 1, 2)                                               # channels_last view


def eligible(m):
    return (type(m) is nn.Conv2d and m.groups == 1 and m.padding_mode == "zeros" and not isinstance(m.padding, str)
            and (m.in_channels % 64 == 0 or m.in_channels <= 4))


def _cast_input_hook(mod, args):
    x = args[0]
    if torch.is_tensor(x) and x.is_floating_point() and x.dtype != mod.weight.dtype:
        return (x.to(mod.weight.dtype),) + tuple(args[1:])
    return None


def use_engine_convs(module, batchnorm=True, wgrad_side_stream=None):
    """Re-class every eligible nn.Conv2d below `module` to EngineConv2d and (batchnorm=True) every nn.BatchNorm2d to
    EngineBatchNorm2d (parameters and buffers stay the same objects).  Returns the number of convolutions switched.
    wgrad_side_stream=True / False sets the process-wide WGRAD_SIDE_STREAM switch (weight gradients off the critical path).  Undo with restore_library_convs().  The layers that stay with the library (transposed and grouped
    convolutions, Linear) get a pre-hook that casts the bf16 activations arriving from engine layers to their weights' dtype."""
    if wgrad_side_stream is not None:                       # process-wide switch, see WGRAD_SIDE_STREAM above
        global WGRAD_SIDE_STREAM
        WGRAD_SIDE_STREAM = bool(wgrad_side_stream)
    n = 0
    for m in module.modules():
        if eligible(m):
            m.__class__ = EngineConv2d
            n += 1
        elif batchnorm and type(m) is nn.BatchNorm2d:
            m.__class__ = EngineBatchNorm2d
        elif type(m) is nn.ConvTranspose2d and tuple(m.kernel_size) == (2, 2) and tuple(m.stride) == (2, 2) and m.in_channels % 64 == 0 \
                and not os.environ.get("MR_NO_ENGINE_CONVT"):
            m.__class__ = EngineConvTranspose2d
        elif isinstance(m, (nn.Conv2d, nn.ConvTranspose2d, nn.Linear)) and type(m) is not EngineConv2d \
                and not hasattr(m, "_mr_cast_hook"):
            m._mr_cast_hook = m.register_forward_pre_hook(_cast_input_hook)
    return n


def restore_library_convs(module):
    n = 0
    for m in module.modules():
        if type(m) is EngineConv2d:
            m.__class__ = nn.Conv2d
            n += 1
        if type(m) is EngineBatchNorm2d:
            m.__class__ = nn.BatchNorm2d
        if type(m) is EngineConvTranspose2d:
            m.__class__ = nn.ConvTranspose2d
        if hasattr(m, "_mr_cast_hook"):
            m._mr_cast_hook.remove()
            del m._mr_cast_hook
    return n
