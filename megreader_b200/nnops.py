"""Thin torch-tensor wrappers over the C-ABI building blocks (include/megreader_b200.h, csrc/nn_kernels.cu,
csrc/gemm.cu).  No arithmetic happens in Python; these only allocate outputs and pass pointers."""
import os

import torch

from . import _lib

F32, BF16 = 0, 1


def code(dtype):
    if dtype == torch.float32:
        return F32
    if dtype == torch.bfloat16:
        return BF16
    raise TypeError("megreader_b200: compute dtype must be float32 or bfloat16, got %s" % dtype)


def _st():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return t.data_ptr() if t is not None else None


def _chk(rc, what):
    _lib.check(rc, what)


def nchw_to_nhwc(x, Cp, dtype):
    N, C, H, W = x.shape
    y = torch.empty((N, H, W, Cp), dtype=dtype, device=x.device)
    _chk(_lib.lib().mr_nchw_to_nhwc(_p(x), N, C, H, W, Cp, code(dtype), _p(y), _st()), "nchw_to_nhwc")
    return y


def nhwc_to_nchw(x, C):
    N, H, W, Cp = x.shape
    y = torch.empty((N, C, H, W), dtype=torch.float32, device=x.device)
    _chk(_lib.lib().mr_nhwc_to_nchw(_p(x), N, C, H, W, Cp, code(x.dtype), _p(y), _st()), "nhwc_to_nchw")
    return y


def im2col(x, kh, kw, ph, pw, Kp):
    N, H, W, C = x.shape
    Ho, Wo = H + 2 * ph - kh + 1, W + 2 * pw - kw + 1
    col = torch.empty((N * Ho * Wo, Kp), dtype=x.dtype, device=x.device)
    _chk(_lib.lib().mr_im2col_nhwc(_p(x), N, H, W, C, kh, kw, ph, pw, Kp, code(x.dtype), _p(col), _st()), "im2col")
    return col, Ho, Wo


def col2im(dcol, N, H, W, C, kh, kw, ph, pw):
    dx = torch.empty((N, H, W, C), dtype=dcol.dtype, device=dcol.device)
    _chk(_lib.lib().mr_col2im_nhwc(_p(dcol), N, H, W, C, kh, kw, ph, pw, dcol.size(1), code(dcol.dtype), _p(dx), _st()),
         "col2im")
    return dx


def pool_out(H, W, k, s, p):
    return (H + 2 * p[0] - k[0]) // s[0] + 1, (W + 2 * p[1] - k[1]) // s[1] + 1


def bias_relu_pool_fwd(z, bias, N, H, W, C, k, s, p):
    Ho, Wo = pool_out(H, W, k, s, p)
    y = torch.empty((N, Ho, Wo, C), dtype=z.dtype, device=z.device)
    idx = torch.empty((N, Ho, Wo, C), dtype=torch.uint8, device=z.device)
    _chk(_lib.lib().mr_bias_relu_pool_fwd(_p(z), _p(bias), N, H, W, C, k[0], k[1], s[0], s[1], p[0], p[1], code(z.dtype),
                                          _p(y), _p(idx), _st()), "bias_relu_pool_fwd")
    return y, idx


def bias_relu_pool_bwd(dy, y, idx, N, H, W, C, k, s, p, want_dbias=True):
    """-> (dz [N*H*W, C], dbias [C] fp32 = column sums of dz, fused)."""
    dz = torch.empty((N * H * W, C), dtype=dy.dtype, device=dy.device)
    dbias = torch.empty((C,), dtype=torch.float32, device=dy.device) if want_dbias else None
    _chk(_lib.lib().mr_bias_relu_pool_bwd(_p(dy), _p(y), _p(idx), N, H, W, C, k[0], k[1], s[0], s[1], p[0], p[1],
                                          code(dy.dtype), _p(dz), _p(dbias), _p(_sums(C, dy.device)), _st()),
         "bias_relu_pool_bwd")
    return dz, dbias


def bias_act(x, bias, relu=False, out=None):
    rows, C = x.shape
    y = out if out is not None else torch.empty_like(x)
    _chk(_lib.lib().mr_bias_act(_p(x), _p(bias), rows, C, int(relu), code(x.dtype), _p(y), _st()), "bias_act")
    return y


def _sums(C, dev):
    return torch.empty((2 * C,), dtype=torch.float64, device=dev)


def bn_train_fwd(z, bias, gamma, beta, running_mean, running_var, momentum, eps, out=None):
    rows, C = z.shape
    y = out if out is not None else torch.empty_like(z)
    mean = torch.empty((C,), dtype=torch.float32, device=z.device)
    invstd = torch.empty_like(mean)
    _chk(_lib.lib().mr_bn_train_fwd(_p(z), _p(bias), _p(gamma), _p(beta), _p(running_mean), _p(running_var),
                                    float(momentum), float(eps), rows, C, code(z.dtype), _p(y), _p(mean), _p(invstd),
                                    _p(_sums(C, z.device)), _st()), "bn_train_fwd")
    return y, mean, invstd


def bn_apply(z, bias, mean, invstd, gamma, beta, out=None):
    rows, C = z.shape
    y = out if out is not None else torch.empty_like(z)
    _chk(_lib.lib().mr_bn_apply(_p(z), _p(bias), _p(mean), _p(invstd), _p(gamma), _p(beta), rows, C, code(z.dtype), _p(y),
                                _st()), "bn_apply")
    return y


def bn_train_bwd(dy, z, bias, mean, invstd, gamma, want_dbias=True, out=None):
    rows, C = z.shape
    dx = out if out is not None else torch.empty_like(z)
    dgamma = torch.empty((C,), dtype=torch.float32, device=z.device)
    dbeta = torch.empty_like(dgamma)
    dbias = torch.empty_like(dgamma) if want_dbias else None
    sums = torch.empty((3 * C,), dtype=torch.float64, device=z.device)
    _chk(_lib.lib().mr_bn_train_bwd(_p(dy), _p(z), _p(bias), _p(mean), _p(invstd), _p(gamma), rows, C, code(z.dtype),
                                    _p(dx), _p(dgamma), _p(dbeta), _p(dbias), _p(sums), _st()), "bn_train_bwd")
    return dx, dgamma, dbeta, dbias


def colsum(a, out=None, accumulate=False):
    rows, C = a.shape
    if out is None:
        out = torch.empty((C,), dtype=torch.float32, device=a.device)
    _chk(_lib.lib().mr_colsum(_p(a), rows, C, code(a.dtype), _p(out), int(accumulate), _p(_sums(C, a.device)), _st()),
         "colsum")
    return out


def cast(x, dtype):
    if x.dtype == dtype and x.is_contiguous():
        return x
    x = x.contiguous()
    y = torch.empty(x.shape, dtype=dtype, device=x.device)
    _chk(_lib.lib().mr_cast(_p(x), code(x.dtype), x.numel(), code(dtype), _p(y), _st()), "cast")
    return y


# bf16 GEMMs of the engine: "tc" = the repo's wgmma kernel (csrc/gemm_tcgen05.cu) wherever it covers the form, "cublas" = library
# Default "cublas" for the LSTM projections / Linear / conv0 / weight gradients; the routing has not been re-measured on H100.
GEMM_BACKEND = __import__("os").environ.get("MEGREADER_B200_GEMM", "cublas")
GEMM_POLICY = __import__("os").environ.get("MEGREADER_B200_GEMM_POLICY", "big")      # "big" | "all"


def _gemm_tc_try(A, B, out, M, N, K, transA, transB, alpha, beta):
    """Route one bf16 GEMM to the hand-written kernel.  Returns True when it ran."""
    if alpha != 1.0 or (transA and transB):
        return False
    if GEMM_POLICY == "big" and (transA or K < 256 or N < 128):
        return False      # the K = 32 conv0 GEMM and the split-K weight-gradient forms stay library GEMMs
    lib = _lib.lib()
    if transA:
        # weight-gradient form dW[M,N] = A^T B over a long K: split-K with fp32 atomic accumulation into a zeroed output
        if out.dtype != torch.float32:
            return False
        if beta == 0.0:
            out.zero_()
        elif beta != 1.0:
            return False
        tiles = ((M + 127) // 128) * ((N + 255) // 256)
        splits = max(1, min(-(-296 // tiles), (K + 63) // 64))
        rc = lib.mr_gemm_tcgen05(_p(A), _p(B), _p(out), M, N, K, A.stride(0), B.stride(0), out.stride(0), 1, 0,
                                 code(out.dtype), None, 0, 1.0, int(splits), _st())
    else:
        if beta != 0.0:
            return False
        rc = lib.mr_gemm_tcgen05(_p(A), _p(B), _p(out), M, N, K, A.stride(0), B.stride(0), out.stride(0), 0, int(transB),
                                 code(out.dtype), None, 0, 0.0, 1, _st())
    if rc == _lib.MR_ERR_UNSUPPORTED:
        return False
    _chk(rc, "gemm_tcgen05")
    return True


def gemm(A, B, transA=False, transB=False, out=None, out_dtype=None, alpha=1.0, beta=0.0):
    """Row-major out[M,N] = alpha * op(A) op(B) + beta * out.  A, B: 2-D, unit inner stride (row stride = ld).  bf16 operands go
    to the wgmma kernel when it covers the form (NT / NN, TN with fp32 output); everything else is a plain library GEMM."""
    assert A.dim() == 2 and B.dim() == 2 and A.stride(1) == 1 and B.stride(1) == 1 and A.dtype == B.dtype
    M, K = (A.size(1), A.size(0)) if transA else (A.size(0), A.size(1))
    Kb, N = (B.size(1), B.size(0)) if transB else (B.size(0), B.size(1))
    assert K == Kb, (A.shape, B.shape, transA, transB)
    if out is None:
        out = torch.empty((M, N), dtype=out_dtype or A.dtype, device=A.device)
    assert out.stride(1) == 1 and out.shape == (M, N)
    if GEMM_BACKEND == "tc" and A.dtype == torch.bfloat16 and _gemm_tc_try(A, B, out, M, N, K, transA, transB, alpha, beta):
        return out
    _chk(_lib.lib().mr_gemm(_p(A), _p(B), _p(out), M, N, K, A.stride(0), B.stride(0), out.stride(0), int(transA),
                            int(transB), code(A.dtype), code(out.dtype), float(alpha), float(beta), _st()), "gemm")
    return out


def gemm_batched_raw(pA, pB, pC, M, N, K, lda, ldb, ldc, sA, sB, sC, batch, transA, transB, in_dtype, out_dtype,
                     alpha=1.0, beta=0.0):
    _chk(_lib.lib().mr_gemm_batched(pA, pB, pC, M, N, K, lda, ldb, ldc, sA, sB, sC, batch, int(transA), int(transB),
                                    code(in_dtype), code(out_dtype), float(alpha), float(beta), _st()), "gemm_batched")


def _ptr_array(tensors):
    import ctypes
    return (ctypes.c_void_p * len(tensors))(*[(t.data_ptr() if t is not None else None) for t in tensors])


def lstm_cell_fwd(gates, b_ih, b_hh, c_prev, c_out, h_out, ldh, h_state):
    """Each argument: list (one entry per direction, 1 or 2) of tensors; c_prev entries may be None."""
    B, H4 = gates[0].shape
    _chk(_lib.lib().mr_lstm_cell_fwd(_ptr_array(gates), _ptr_array(b_ih), _ptr_array(b_hh), _ptr_array(c_prev),
                                     _ptr_array(c_out), _ptr_array(h_out), ldh, _ptr_array(h_state), len(gates), B,
                                     H4 // 4, code(gates[0].dtype), _st()), "lstm_cell_fwd")


def lstm_cell_bwd(gates, c, c_prev, dh_out, ldh, dh_rec, dc, dgates):
    B, H4 = gates[0].shape
    _chk(_lib.lib().mr_lstm_cell_bwd(_ptr_array(gates), _ptr_array(c), _ptr_array(c_prev), _ptr_array(dh_out), ldh,
                                     _ptr_array(dh_rec), _ptr_array(dc), _ptr_array(dgates), len(gates), B, H4 // 4,
                                     code(gates[0].dtype), _st()), "lstm_cell_bwd")


def adam_step(p, g, m, v, lr, beta1, beta2, eps, step, grad_scale=1.0, shadow=None):
    _chk(_lib.lib().mr_adam_step(_p(p), _p(g), _p(m), _p(v), p.numel(), float(lr), float(beta1), float(beta2), float(eps),
                                 int(step), float(grad_scale), _p(shadow), _st()), "adam_step")


def gemm_tc(A, B, transA=False, transB=True, out=None, out_dtype=None, bias=None, relu=False, beta=0.0, splits=1):
    """Hand-written wgmma/TMA bf16 GEMM (csrc/gemm_tcgen05.cu).  Same storage convention as gemm(); forms NT / TN.
    Raises MegReaderB200Error(MR_ERR_UNSUPPORTED) for shapes it does not cover."""
    assert A.dim() == 2 and B.dim() == 2 and A.stride(1) == 1 and B.stride(1) == 1
    assert A.dtype == torch.bfloat16 and B.dtype == torch.bfloat16
    M, K = (A.size(1), A.size(0)) if transA else (A.size(0), A.size(1))
    Kb, N = (B.size(1), B.size(0)) if transB else (B.size(0), B.size(1))
    assert K == Kb, (A.shape, B.shape, transA, transB)
    if out is None:
        out = torch.empty((M, N), dtype=out_dtype or torch.bfloat16, device=A.device)
    assert out.stride(1) == 1 and out.shape == (M, N)
    _chk(_lib.lib().mr_gemm_tcgen05(_p(A), _p(B), _p(out), M, N, K, A.stride(0), B.stride(0), out.stride(0), int(transA),
                                    int(transB), code(out.dtype), _p(bias), int(relu), float(beta), int(splits), _st()),
         "gemm_tcgen05")
    return out


def conv_fprop_tc(x, Wm, kh, kw, ph, pw, out_dtype=torch.bfloat16, bias=None, relu=False):
    """Implicit-GEMM conv (csrc/gemm_tcgen05.cu): x NHWC bf16 [N,H,W,C], Wm [Cout, kh*kw*C] bf16 -> [N*Ho*Wo, Cout]."""
    N, H, W, C = x.shape
    Cout = Wm.size(0)
    assert x.is_contiguous() and Wm.is_contiguous() and Wm.size(1) == kh * kw * C
    Ho, Wo = H + 2 * ph - kh + 1, W + 2 * pw - kw + 1
    y = torch.empty((N * Ho * Wo, Cout), dtype=out_dtype, device=x.device)
    _chk(_lib.lib().mr_conv_fprop_tcgen05(_p(x), _p(Wm), _p(y), N, H, W, C, Cout, kh, kw, ph, pw, code(out_dtype), _p(bias),
                                          int(relu), _st()), "conv_fprop_tcgen05")
    return y, Ho, Wo


def conv_wgrad_tc(dz, x, kh, kw, ph, pw, splits=0, out=None):
    """dWm [Cout, kh*kw*C] fp32 from dz [N,Ho,Wo,Cout] and x [N,H,W,C] (NHWC bf16).  `out`: a ZEROED [Cout, K] fp32
    buffer to accumulate into (lets the caller allocate it on another stream than the one the kernel runs on)."""
    N, H, W, C = x.shape
    Cout = dz.size(-1)
    K = kh * kw * C
    dWm = out if out is not None else torch.zeros((Cout, K), dtype=torch.float32, device=x.device)
    if splits <= 0:
        tiles = ((Cout + 127) // 128) * ((K + 255) // 256)
        splits = max(1, -(-288 // tiles))
    _chk(_lib.lib().mr_conv_wgrad_tcgen05(_p(dz), _p(x), _p(dWm), N, H, W, C, Cout, kh, kw, ph, pw, int(splits), _st()),
         "conv_wgrad_tcgen05")
    return dWm


def conv2d_fprop_tc(x, Wm, kh, kw, sh, sw, ph, pw, dh, dw, out_dtype=torch.bfloat16, bias=None, relu=False):
    """General implicit-GEMM conv (stride, dilation): x NHWC bf16 [N,H,W,C] -> ([N*Ho*Wo, Cout], Ho, Wo)."""
    N, H, W, C = x.shape
    Cout = Wm.size(0)
    assert x.is_contiguous() and Wm.is_contiguous() and Wm.size(1) == kh * kw * C
    Ho, Wo = (H + 2 * ph - dh * (kh - 1) - 1) // sh + 1, (W + 2 * pw - dw * (kw - 1) - 1) // sw + 1
    y = torch.empty((N * Ho * Wo, Cout), dtype=out_dtype, device=x.device)
    _chk(_lib.lib().mr_conv2d_fprop_tcgen05(_p(x), _p(Wm), _p(y), N, H, W, C, Cout, kh, kw, sh, sw, ph, pw, dh, dw,
                                            code(out_dtype), _p(bias), int(relu), _st()), "conv2d_fprop_tcgen05")
    return y, Ho, Wo


# minimum 64-pixel k-blocks per split of conv2d_wgrad_tc (MR_WGRAD_MIN_KB; not re-tuned on H100)
_WGRAD_MIN_KB = max(1, int(os.environ.get("MR_WGRAD_MIN_KB", "16")))


def conv2d_wgrad_tc(dz, x, kh, kw, sh, sw, ph, pw, dh, dw, splits=0, out=None):
    """dWm [Cout, kh*kw*C] fp32 from dz [N,Ho,Wo,Cout] and x [N,H,W,C] (NHWC bf16), stride / dilation as the forward."""
    N, H, W, C = x.shape
    Cout = dz.size(-1)
    K = kh * kw * C
    dWm = out if out is not None else torch.zeros((Cout, K), dtype=torch.float32, device=x.device)
    if splits <= 0:
        tiles = ((Cout + 127) // 128) * ((K + 255) // 256)
        splits = max(1, -(-288 // tiles))
        # a split should own enough 64-pixel k-blocks to amortise its fixed cost (pipeline set-up and the fp32 atomic
        # epilogue of a whole output tile): small weights over many pixels (layer1 of a ResNet) otherwise spend their time in atomics
        kb_total = dz.size(0) * dz.size(1) * -(-dz.size(2) // 64)
        splits = max(1, min(splits, kb_total // _WGRAD_MIN_KB))
    _chk(_lib.lib().mr_conv2d_wgrad_tcgen05(_p(dz), _p(x), _p(dWm), N, H, W, C, Cout, kh, kw, sh, sw, ph, pw, dh, dw,
                                            int(splits), _st()), "conv2d_wgrad_tcgen05")
    return dWm


def lstm_step_fwd_tc(h_prev, Whh, gates, bias, c_prev, c_out, h_out, ldh, h_next, have_h):
    """Fused recurrent GEMM + LSTM cell, both directions (lists of 2 tensors each), unit-major gate layout."""
    B, H4 = gates[0].shape
    _chk(_lib.lib().mr_lstm_step_fwd_tcgen05(_ptr_array(h_prev), _ptr_array(Whh), _ptr_array(gates), _ptr_array(bias),
                                             _ptr_array(c_prev), _ptr_array(c_out), _ptr_array(h_out), ldh,
                                             _ptr_array(h_next), int(have_h), B, H4 // 4, _st()), "lstm_step_fwd_tcgen05")


def lstm_step_bwd_tc(dG_next, Whh, gates, c, c_prev, dh_out, ldh, dc, dgates, have_rec):
    B, H4 = gates[0].shape
    _chk(_lib.lib().mr_lstm_step_bwd_tcgen05(_ptr_array(dG_next), _ptr_array(Whh), _ptr_array(gates), _ptr_array(c),
                                             _ptr_array(c_prev), _ptr_array(dh_out), ldh, _ptr_array(dc),
                                             _ptr_array(dgates), int(have_rec), B, H4 // 4, _st()), "lstm_step_bwd_tcgen05")


def lstm_seq_flags(B, device):
    return torch.empty((2 * ((B + 127) // 128) + 1,), dtype=torch.int32, device=device)


def lstm_seq_fwd_tc(Whh, G, bias, C, Y, flags):
    """Persistent whole-sequence recurrence (both directions).  Returns False when the device cannot hold the grid
    (MR_ERR_UNSUPPORTED): the caller then runs the per-step kernels."""
    _, T, B, H4 = G.shape
    rc = _lib.lib().mr_lstm_seq_fwd_tcgen05(_ptr_array(Whh), G.data_ptr(), _ptr_array(bias), C.data_ptr(), Y.data_ptr(),
                                            flags.data_ptr(), T, B, H4 // 4, _st())
    if rc == _lib.MR_ERR_UNSUPPORTED:
        return False
    _chk(rc, "lstm_seq_fwd_tcgen05")
    return True


def lstm_seq_bwd_tc(WhhT, G, C, dY, dG, flags):
    """WhhT: the two recurrent weight matrices transposed, [H, 4H] bf16 (unit-major gate columns)."""
    _, T, B, H4 = G.shape
    rc = _lib.lib().mr_lstm_seq_bwd_tcgen05(_ptr_array(WhhT), G.data_ptr(), C.data_ptr(), dY.data_ptr(), dG.data_ptr(),
                                            flags.data_ptr(), T, B, H4 // 4, _st())
    if rc == _lib.MR_ERR_UNSUPPORTED:
        return False
    _chk(rc, "lstm_seq_bwd_tcgen05")
    return True


def conv_weight_pack(w, Cp, Kp, dtype, mode):
    """nn.Conv2d weight (fp32) -> GEMM operand: mode 0 [Cout, Kp] forward matrix, mode 1 [Cin, kh*kw*Cout] dgrad matrix."""
    w = w.detach()
    assert w.dtype == torch.float32 and w.is_contiguous()
    Cout, Cin, kh, kw = w.shape
    out = torch.empty((Cout, Kp) if mode == 0 else (Cin, kh * kw * Cout), dtype=dtype, device=w.device)
    _chk(_lib.lib().mr_conv_weight_pack(w.data_ptr(), Cout, Cin, kh, kw, Cp, Kp, mode, code(dtype), out.data_ptr(), _st()),
         "conv_weight_pack")
    return out


def gate_rows_permute(a, H, dtype, b=None, inverse=False):
    """[4H, cols] (or [4H]) fp32 rows: gate-major <-> unit-major (see mr_gate_rows_permute); optional b is added."""
    a = a.detach()
    assert a.dtype == torch.float32 and a.is_contiguous() and a.size(0) == 4 * H
    cols = a.numel() // (4 * H)
    out = torch.empty(a.shape, dtype=dtype, device=a.device)
    _chk(_lib.lib().mr_gate_rows_permute(a.data_ptr(), b.detach().data_ptr() if b is not None else None, H, cols,
                                         int(inverse), code(dtype), out.data_ptr(), _st()), "gate_rows_permute")
    return out
