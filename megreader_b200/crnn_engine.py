"""Execution engine behind the CRNN surfaces (refapi/backbones/crnn.py, refapi/decoders/crnn.py).

The nn.Modules only own parameters (reference names / shapes, SURVEY.md App. C).  The arithmetic of
    backbones/crnn.py:46-59   7 x (conv [+BN | +ReLU] [+MaxPool])
    decoders/crnn.py:8-24     2 x (bidirectional LSTM + Linear)
    decoders/crnn.py:95-99    log_softmax -> CTC (mean, zero_infinity)
runs here as two hand-orchestrated autograd Functions over megreader_b200's CUDA kernels: activations stay NHWC
in the compute dtype (fp32 for parity runs, bf16 for throughput; fp32 accumulation and fp32 master weights in both),
every convolution is im2col (csrc/nn_kernels.cu) + one dense GEMM (csrc/gemm.cu), bias+ReLU+MaxPool and BatchNorm are
single fused passes, the LSTM is one input-projection GEMM per direction plus a per-step recurrent GEMM and a fused
cell kernel, and the loss is the fused log_softmax+CTC of csrc/ctc2d.cu.  CUDA only: there is no CPU path.
"""
import torch
import torch.nn.functional as F

from . import ctc1d
from . import nnops as ops

_COMPUTE_DTYPE = torch.float32
# bf16 mode: convolutions with C % 64 == 0 run as wgmma implicit GEMMs (csrc/gemm_tcgen05.cu); False routes them
# through im2col + cuBLAS (kept for A/B comparison in benchmarks)
USE_TCGEN05 = __import__("os").environ.get("MEGREADER_B200_TCGEN05", "1") != "0"
# Fused wgmma LSTM time steps (recurrent GEMM + cell in one launch).  Correct (tests/test_nn_kernels_gpu.py) but
# the per-launch barrier set-up dominates a 4-k-block GEMM, so it is opt-in.
# BiLSTM recurrence on the bf16 path: "seq" = one persistent wgmma launch per layer and pass (csrc/lstm_seq_tcgen05.cu),
# "step" = one fused wgmma launch per time step, "cublas" = strided-batched cuBLAS GEMM + cell kernel per step.
LSTM_MODE = __import__("os").environ.get("MEGREADER_B200_LSTM", "seq")
if __import__("os").environ.get("MEGREADER_B200_LSTM_FUSED", "0") == "1":     # older switch
    LSTM_MODE = "step"
# conv weight gradients on a side stream, overlapped with the rest of the backward chain (MEGREADER_B200_WGRAD_STREAM=0: off)
WGRAD_SIDE_STREAM = __import__("os").environ.get("MEGREADER_B200_WGRAD_STREAM", "1") == "1"
_SIDE_STREAMS = {}


def _side_stream(dev):
    key = str(dev)
    if key not in _SIDE_STREAMS:
        _SIDE_STREAMS[key] = torch.cuda.Stream(device=dev)
    return _SIDE_STREAMS[key]


LAST_LSTM_FLAGS = None      # scratch of the most recent persistent launch; last word != 0 <=> an inter-CTA wait timed out


def set_compute_dtype(dtype):
    """torch.float32 (default; parity with the reference within 1e-4) or torch.bfloat16 (BASELINE.json cfg 2)."""
    global _COMPUTE_DTYPE
    ops.code(dtype)
    _COMPUTE_DTYPE = dtype


def compute_dtype():
    if torch.is_autocast_enabled() and torch.get_autocast_gpu_dtype() == torch.bfloat16:
        return torch.bfloat16
    return _COMPUTE_DTYPE


def _require_cuda(t, what):
    if not t.is_cuda:
        raise NotImplementedError("megreader_b200.%s: CUDA tensors only (no CPU fallback)" % what)


def _vn(dtype):
    return 4 if dtype == torch.float32 else 8


# ------------------------------------------------------------------------------------------------ backbone
def _conv_layers(module):
    """[(conv, bn|None, pool|None)] in order, read off the reference-shaped Sequential (backbones/crnn.py:15-43)."""
    out = []
    for blk in module.cnn:
        conv = bn = pool = None
        for m in blk.modules():
            if isinstance(m, torch.nn.Conv2d):
                conv = m
            elif isinstance(m, torch.nn.BatchNorm2d):
                bn = m
            elif isinstance(m, torch.nn.MaxPool2d):
                pool = m
        out.append((conv, bn, pool))
    return out


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


def _weight_matrix(w, Cp, Kp, dtype):
    """conv weight [Cout, Cin, kh, kw] fp32 -> GEMM operand [Cout, Kp] in `dtype`, column = (i*kw + j)*Cp + c (one launch)."""
    w = w.detach()
    if w.dtype == torch.float32 and w.is_contiguous():
        return ops.conv_weight_pack(w, Cp, Kp, dtype, 0)
    Cout, Cin, kh, kw = w.shape
    m = w.permute(0, 2, 3, 1)
    if Cp != Cin:
        m = F.pad(m, (0, Cp - Cin))
    m = m.reshape(Cout, kh * kw * Cp)
    if Kp != m.size(1):
        m = F.pad(m, (0, Kp - m.size(1)))
    return ops.cast(m.contiguous(), dtype)


def _weight_grad(dWm, Cin, Cp, kh, kw):
    Cout = dWm.size(0)
    return dWm[:, :kh * kw * Cp].reshape(Cout, kh, kw, Cp)[..., :Cin].permute(0, 3, 1, 2).contiguous()


class _BackboneFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, module, bn_batch_stats, save, dtype, *params):
        # bn_batch_stats = module.training: BatchNorm normalises with batch statistics and updates its running buffers
        #                  (also under torch.no_grad(), exactly like nn.BatchNorm2d);
        # save           = torch.is_grad_enabled(): keep what the backward needs (also in eval() mode: frozen-BN fine-tuning).
        layers = _conv_layers(module)
        vn = _vn(dtype)
        N, Cin, H, W = x.shape
        Cp = -(-Cin // vn) * vn
        a = ops.nchw_to_nhwc(x.contiguous().float(), Cp, dtype)
        ctx.in_nhwc, ctx.in_channels, ctx.in_dtype = tuple(a.shape), Cin, x.dtype
        saved = []
        for (conv, bn, pool) in layers:
            kh, kw = conv.kernel_size
            ph, pw = conv.padding
            assert conv.stride == (1, 1) and conv.dilation == (1, 1) and conv.groups == 1
            C = a.size(3)
            K = kh * kw * C
            Kp = -(-K // vn) * vn
            Wm = _weight_matrix(conv.weight, C, Kp, dtype)
            implicit = USE_TCGEN05 and dtype == torch.bfloat16 and C % 64 == 0
            if implicit:
                # wgmma implicit GEMM: activation tiles are gathered straight into swizzled smem, no im2col in HBM
                z, Ho, Wo = ops.conv_fprop_tc(a, Wm, kh, kw, ph, pw)
                col = None
            else:
                col, Ho, Wo = ops.im2col(a, kh, kw, ph, pw, Kp)
                z = ops.gemm(col, Wm, transB=True)                  # [P, Cout] raw conv output (no bias yet)
            Cout = Wm.size(0)
            rec = {"col": col if save else None, "x": a if (save and implicit) else None, "Wm": Wm,
                   "in_shape": tuple(a.shape), "k": (kh, kw), "p": (ph, pw), "Cin": conv.in_channels, "out_hw": (Ho, Wo)}
            if bn is not None:
                if bn_batch_stats:
                    # momentum=None is PyTorch's cumulative moving average: factor 1 / num_batches_tracked (after the increment)
                    mom = bn.momentum if bn.momentum is not None else 1.0 / (float(bn.num_batches_tracked.item()) + 1.0)
                    y, mean, invstd = ops.bn_train_fwd(z, conv.bias, bn.weight, bn.bias, bn.running_mean, bn.running_var,
                                                       mom, bn.eps)
                    bn.num_batches_tracked += 1
                    rec.update(z=z if save else None, mean=mean, invstd=invstd, kind="bn")
                else:
                    invstd = torch.rsqrt(bn.running_var + bn.eps)
                    y = ops.bn_apply(z, conv.bias, bn.running_mean, invstd, bn.weight, bn.bias)
                    rec.update(z=z if save else None, mean=bn.running_mean.detach().clone(), invstd=invstd, kind="bn_eval")
                a = y.view(N, Ho, Wo, Cout)
            else:
                assert pool is not None, "CRNN: every ReLU block is followed by a MaxPool (backbones/crnn.py:18-35)"
                k, s, p = _pair(pool.kernel_size), _pair(pool.stride), _pair(pool.padding)
                y, idx = ops.bias_relu_pool_fwd(z, conv.bias, N, Ho, Wo, Cout, k, s, p)
                rec.update(y=y, idx=idx, pool=(k, s, p), kind="pool")
                a = y
            saved.append(rec)
        ctx.saved = saved
        ctx.layers = layers
        ctx.dtype = dtype
        ctx.N = N
        feat = a                                                       # [N, Hf, Wf, 512] NHWC
        ctx.feat_shape = tuple(feat.shape)
        return feat.permute(0, 3, 1, 2)                                # (N, 512, Hf, Wf) view, channels-last memory

    @staticmethod
    def backward(ctx, dfeat):
        if ctx.saved is None or not ctx.saved[-1]:
            raise RuntimeError("megreader_b200 CRNN backbone: the saved activations were freed by the first backward() "
                               "(retain_graph is not supported by this engine)")
        N, Hf, Wf, Cf = ctx.feat_shape
        dtype = ctx.dtype
        dy = ops.cast(dfeat.permute(0, 2, 3, 1).contiguous(), dtype).view(N * Hf * Wf, Cf)
        grads = []
        # The weight gradients are off the critical path (dz_L -> dgrad_L -> pool/BN backward_{L-1} -> ...): they run on a
        # side stream and fill the SMs that the HBM-bound elementwise kernels and the tail waves of the dgrad kernels
        # leave idle.  Joined before the gradients are handed back (also inside CUDA-graph capture: fork/join by events).
        main = torch.cuda.current_stream(dfeat.device)
        side = _side_stream(dfeat.device) if WGRAD_SIDE_STREAM else None
        deferred = []                                   # (slot in grads, dWm, Cin, C, kh, kw) finished after the join
        for li in range(len(ctx.layers) - 1, -1, -1):
            conv, bn, pool = ctx.layers[li]
            rec = ctx.saved[li]
            Nn, H, W, C = rec["in_shape"]
            Ho, Wo = rec["out_hw"]
            Cout = rec["Wm"].size(0)
            kh, kw = rec["k"]
            ph, pw = rec["p"]
            if rec["kind"] == "bn":
                dz, dgamma, dbeta, dbias = ops.bn_train_bwd(dy, rec["z"], conv.bias, rec["mean"], rec["invstd"], bn.weight)
            elif rec["kind"] == "bn_eval":
                # eval-mode BatchNorm is a per-channel affine map y = (z + b - mean) * invstd * gamma + beta (rare path:
                # frozen-BN fine-tuning / saliency; plain tensor arithmetic, fp32)
                dyf, zf = dy.float(), rec["z"].float()
                xhat = (zf + conv.bias.detach() - rec["mean"]) * rec["invstd"]
                dgamma, dbeta = (dyf * xhat).sum(0), dyf.sum(0)
                dzf = dyf * (bn.weight.detach() * rec["invstd"])
                dbias = dzf.sum(0)
                dz = ops.cast(dzf.contiguous(), dtype)
            else:
                k, s, p = rec["pool"]
                dz, dbias = ops.bias_relu_pool_bwd(dy, rec["y"], rec["idx"], Nn, Ho, Wo, Cout, k, s, p)
                dgamma = dbeta = None
            dW = None
            if rec["x"] is not None:
                dz4 = dz.view(Nn, Ho, Wo, Cout)
                if side is not None:
                    dWm = torch.zeros((Cout, kh * kw * C), dtype=torch.float32, device=dz.device)
                    side.wait_stream(main)
                    dz.record_stream(side)
                    rec["x"].record_stream(side)
                    with torch.cuda.stream(side):
                        ops.conv_wgrad_tc(dz4, rec["x"], kh, kw, ph, pw, out=dWm)
                    deferred.append((dWm, rec["Cin"], C, kh, kw))
                else:
                    dWm = ops.conv_wgrad_tc(dz4, rec["x"], kh, kw, ph, pw)                 # [Cout, K] fp32
                    dW = _weight_grad(dWm, rec["Cin"], C, kh, kw)
            else:
                dWm = ops.gemm(dz, rec["col"], transA=True, out_dtype=torch.float32)      # [Cout, Kp]
                dW = _weight_grad(dWm, rec["Cin"], C, kh, kw)
            layer_grads = [dW if dW is not None else deferred[-1]] + [dbias] + ([dgamma, dbeta] if bn is not None else [])
            grads = layer_grads + grads
            if li > 0 or ctx.needs_input_grad[0]:
                if rec["x"] is not None and Cout % 64 == 0:
                    # input gradient = convolution of dz with the flipped, transposed weights, padding k-1-p
                    wsrc = conv.weight.detach()
                    if wsrc.dtype == torch.float32 and wsrc.is_contiguous() and wsrc.size(1) == C:
                        Wd = ops.conv_weight_pack(wsrc, C, kh * kw * C, dtype, 1)          # flipped + transposed, one launch
                    else:
                        Wd = ops.cast(wsrc.flip(2, 3).permute(1, 2, 3, 0).reshape(C, kh * kw * Cout).contiguous(), dtype)
                    dy, _, _ = ops.conv_fprop_tc(dz4, Wd, kh, kw, kh - 1 - ph, kw - 1 - pw)
                else:
                    dcol = ops.gemm(dz, rec["Wm"])                                           # [P, Kp]
                    dy = ops.col2im(dcol, Nn, H, W, C, kh, kw, ph, pw).view(Nn * H * W, C)
            rec.clear()
        dx = None
        if ctx.needs_input_grad[0]:
            Nn, H0, W0, C0 = ctx.in_nhwc
            dx = ops.nhwc_to_nchw(dy.view(Nn, H0, W0, C0), ctx.in_channels).to(ctx.in_dtype)
        if deferred:
            main.wait_stream(side)
            grads = [_weight_grad(*g) if isinstance(g, tuple) else g for g in grads]
        return (dx, None, None, None, None) + tuple(grads)


def _backbone_params(module):
    ps = []
    for conv, bn, _ in _conv_layers(module):
        ps += [conv.weight, conv.bias]
        if bn is not None:
            ps += [bn.weight, bn.bias]
    return ps


def backbone_forward(module, x):
    """backbones/crnn.py:57-59."""
    _require_cuda(x, "crnn_backbone")
    return _BackboneFn.apply(x, module, module.training, torch.is_grad_enabled(), compute_dtype(),
                             *_backbone_params(module))


# ------------------------------------------------------------------------------------------------ BiLSTM + Linear
def _lstm_dir_params(rnn, d):
    sfx = "_reverse" if d == 1 else ""
    return [getattr(rnn, n + "_l0" + sfx) for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]


def _bilstm_params(module):
    return _lstm_dir_params(module.rnn, 0) + _lstm_dir_params(module.rnn, 1) + [module.embedding.weight,
                                                                                 module.embedding.bias]


def _bilstm_forward_impl(X, params, dtype, training):
    """X [T, N, I] (compute dtype, contiguous) -> (out [T, N, nOut], saved dict)."""
    T, N, I = X.shape
    w_ih = [params[0], params[4]]
    w_hh = [params[1], params[5]]
    b_ih = [params[2], params[6]]
    b_hh = [params[3], params[7]]
    w_emb, b_emb = params[8], params[9]
    H = w_hh[0].size(1)
    dev = X.device
    if LSTM_MODE != "cublas" and USE_TCGEN05 and dtype == torch.bfloat16 and H % 64 == 0:
        return _bilstm_forward_fused(X, params, training)
    Wih = [ops.cast(w.detach(), dtype) for w in w_ih]
    Whh = torch.stack([ops.cast(w.detach(), dtype) for w in w_hh])                 # [2, 4H, H]
    X2 = X.view(T * N, I)
    G = torch.empty((2, T, N, 4 * H), dtype=dtype, device=dev)
    for d in range(2):
        ops.gemm(X2, Wih[d], transB=True, out=G[d].view(T * N, 4 * H))               # input projection, all steps
    Cst = torch.empty((2, T, N, H), dtype=torch.float32, device=dev)
    Y = torch.empty((T, N, 2 * H), dtype=dtype, device=dev)
    hst = torch.zeros((2, N, H), dtype=dtype, device=dev)
    esz = G.element_size()
    for s in range(T):
        tf, tr = s, T - 1 - s
        if s > 0:
            # both directions in one strided-batched GEMM: G[d][t_d] += h_d W_hh_d^T
            pC = G.data_ptr() + tf * N * 4 * H * esz
            sC = (T + tr - tf) * N * 4 * H
            ops.gemm_batched_raw(hst.data_ptr(), Whh.data_ptr(), pC, N, 4 * H, H, H, H, 4 * H, N * H, 4 * H * H, sC, 2,
                                 False, True, dtype, dtype, 1.0, 1.0)
        ts, tps = (tf, tr), (tf - 1, tr + 1)
        ops.lstm_cell_fwd([G[d, ts[d]] for d in (0, 1)], b_ih, b_hh,
                          [Cst[d, tps[d]] if s > 0 else None for d in (0, 1)], [Cst[d, ts[d]] for d in (0, 1)],
                          [Y[ts[d], :, d * H:(d + 1) * H] for d in (0, 1)], 2 * H, [hst[0], hst[1]])
    Wemb = ops.cast(w_emb.detach(), dtype)
    nOut = Wemb.size(0)
    out_dtype = dtype if nOut % _vn(dtype) == 0 else torch.float32   # the 38-class logits leave in fp32
    E = ops.gemm(Y.view(T * N, 2 * H), Wemb, transB=True, out_dtype=out_dtype)
    ops.bias_act(E, b_emb, relu=False, out=E)
    saved = dict(X=X, G=G, C=Cst, Y=Y, Wih=Wih, Whh=Whh, Wemb=Wemb, H=H) if training else None
    return E.view(T, N, nOut), saved


_PERM_CACHE = {}


def _unit_major_perm(H, dev):
    """perm[4*j + g] = g*H + j : reference gate-major rows (i|f|g|o blocks) -> unit-major rows; inv undoes it."""
    key = (H, str(dev))
    if key not in _PERM_CACHE:
        perm = torch.arange(4 * H, device=dev).view(4, H).t().reshape(-1)
        inv = torch.arange(4 * H, device=dev).view(H, 4).t().reshape(-1)
        _PERM_CACHE[key] = (perm, inv)
    return _PERM_CACHE[key]


def _bilstm_forward_fused(X, params, training):
    """bf16 path: each time step is ONE wgmma launch (recurrent GEMM + cell, both directions), csrc/gemm_tcgen05.cu."""
    dtype = torch.bfloat16
    T, N, I = X.shape
    w_ih, w_hh = [params[0], params[4]], [params[1], params[5]]
    b_ih, b_hh = [params[2], params[6]], [params[3], params[7]]
    w_emb, b_emb = params[8], params[9]
    H = w_hh[0].size(1)
    dev = X.device
    perm, _ = _unit_major_perm(H, dev)
    def _rows(w, b=None, out_dtype=dtype):
        w = w.detach()
        if w.dtype == torch.float32 and w.is_contiguous() and (b is None or b.is_contiguous()):
            return ops.gate_rows_permute(w, H, out_dtype, b=b)                          # permute (+ add) + cast, one launch
        v = w if b is None else w + b.detach()
        return ops.cast(v[perm].contiguous(), out_dtype)
    Wih = [_rows(w) for w in w_ih]
    Whh = [_rows(w) for w in w_hh]
    bias = [_rows(b_ih[d], b_hh[d], torch.float32) for d in (0, 1)]
    X2 = X.view(T * N, I)
    G = torch.empty((2, T, N, 4 * H), dtype=dtype, device=dev)
    for d in range(2):
        ops.gemm(X2, Wih[d], transB=True, out=G[d].view(T * N, 4 * H))               # input projection, all steps
    Cst = torch.empty((2, T, N, H), dtype=torch.float32, device=dev)
    Y = torch.empty((T, N, 2 * H), dtype=dtype, device=dev)
    global LAST_LSTM_FLAGS
    flags = LAST_LSTM_FLAGS = ops.lstm_seq_flags(N, dev).zero_()
    if LSTM_MODE == "seq" and ops.lstm_seq_fwd_tc(Whh, G, bias, Cst, Y, flags):
        steps = ()                                                                     # whole sequence done in one launch
    else:
        steps = range(T)
        hbuf = torch.zeros((2, 2, N, H), dtype=dtype, device=dev)                      # [ping-pong][direction]
    for s in steps:
        ts, tps = (s, T - 1 - s), (s - 1, T - s)
        cur, nxt = s & 1, (s + 1) & 1
        ops.lstm_step_fwd_tc([hbuf[cur, 0], hbuf[cur, 1]], Whh, [G[d, ts[d]] for d in (0, 1)], bias,
                             [Cst[d, tps[d]] if s > 0 else None for d in (0, 1)], [Cst[d, ts[d]] for d in (0, 1)],
                             [Y[ts[d], :, d * H:(d + 1) * H] for d in (0, 1)], 2 * H, [hbuf[nxt, 0], hbuf[nxt, 1]], s > 0)
    Wemb = ops.cast(w_emb.detach(), dtype)
    nOut = Wemb.size(0)
    out_dtype = dtype if nOut % _vn(dtype) == 0 else torch.float32
    E = ops.gemm(Y.view(T * N, 2 * H), Wemb, transB=True, out_dtype=out_dtype)
    ops.bias_act(E, b_emb, relu=False, out=E)
    saved = dict(X=X, G=G, C=Cst, Y=Y, Wih=Wih, Whh=Whh, Wemb=Wemb, H=H, fused=True, perm=perm, flags=flags) if training else None
    return E.view(T, N, nOut), saved


def _bilstm_backward_fused(dE, sv):
    dtype = torch.bfloat16
    X, G, Cst, Y, H, perm = sv["X"], sv["G"], sv["C"], sv["Y"], sv["H"], sv["perm"]
    T, N, I = X.shape
    dev = X.device
    _, inv = _unit_major_perm(H, dev)
    dE2 = ops.cast(dE.reshape(T * N, -1), dtype)
    Y2 = Y.view(T * N, 2 * H)
    dWemb = ops.gemm(dE2, Y2, transA=True, out_dtype=torch.float32)
    dbemb = ops.colsum(dE2)
    dY3 = ops.gemm(dE2, sv["Wemb"]).view(T, N, 2 * H)
    dG = torch.empty((2, T, N, 4 * H), dtype=dtype, device=dev)
    dc = torch.zeros((2, N, H), dtype=torch.float32, device=dev)
    WhhT = [w.t().contiguous() for w in sv["Whh"]]                                   # [H, 4H]: K-major operand of dG W_hh
    if LSTM_MODE == "seq" and ops.lstm_seq_bwd_tc(WhhT, G, Cst, dY3, dG, sv["flags"]):
        steps = ()
    else:
        steps = range(T - 1, -1, -1)
    for s in steps:
        ts, tps, tn = (s, T - 1 - s), (s - 1, T - s), (s + 1, T - 2 - s)
        have_rec = s < T - 1
        ops.lstm_step_bwd_tc([dG[d, tn[d]] if have_rec else dG[d, ts[d]] for d in (0, 1)], sv["Whh"],
                             [G[d, ts[d]] for d in (0, 1)], [Cst[d, ts[d]] for d in (0, 1)],
                             [Cst[d, tps[d]] if s > 0 else None for d in (0, 1)],
                             [dY3[ts[d], :, d * H:(d + 1) * H] for d in (0, 1)], 2 * H, [dc[0], dc[1]],
                             [dG[d, ts[d]] for d in (0, 1)], have_rec)
    X2 = X.view(T * N, I)
    grads = []
    dX = torch.empty((T * N, I), dtype=dtype, device=dev)
    for d in range(2):
        dG2 = dG[d].view(T * N, 4 * H)
        dWih = ops.gemm(dG2, X2, transA=True, out_dtype=torch.float32)[inv]
        if d == 0:
            A = dG[0, 1:].reshape((T - 1) * N, 4 * H)
            Bm = Y[:T - 1].view((T - 1) * N, 2 * H)[:, :H]
        else:
            A = dG[1, :T - 1].reshape((T - 1) * N, 4 * H)
            Bm = Y[1:].view((T - 1) * N, 2 * H)[:, H:]
        dWhh = (ops.gemm(A, Bm, transA=True, out_dtype=torch.float32) if T > 1
                else torch.zeros(4 * H, H, device=dev))[inv]
        db = ops.colsum(dG2)[inv]
        grads += [dWih, dWhh, db, db.clone()]
        if d == 0 or ops.GEMM_BACKEND != "tc":
            ops.gemm(dG2, sv["Wih"][d], out=dX, beta=0.0 if d == 0 else 1.0)
        else:
            dX.add_(ops.gemm(dG2, sv["Wih"][d]))       # wgmma kernel: no bf16 accumulate form -> own GEMM + one add
    return dX.view(T, N, I), grads + [dWemb, dbemb]


def _bilstm_backward_impl(dE, sv, dtype):
    """dE [T, N, nOut] -> (dX [T, N, I], grads for the 10 parameters in _bilstm_params order)."""
    if sv.get("fused"):
        return _bilstm_backward_fused(dE, sv)
    X, G, Cst, Y, H = sv["X"], sv["G"], sv["C"], sv["Y"], sv["H"]
    T, N, I = X.shape
    dev = X.device
    dE2 = ops.cast(dE.reshape(T * N, -1), dtype)
    Y2 = Y.view(T * N, 2 * H)
    dWemb = ops.gemm(dE2, Y2, transA=True, out_dtype=torch.float32)
    dbemb = ops.colsum(dE2)
    dY = ops.gemm(dE2, sv["Wemb"])                                                   # [T*N, 2H]
    dY3 = dY.view(T, N, 2 * H)
    dG = torch.empty((2, T, N, 4 * H), dtype=dtype, device=dev)
    dc = torch.zeros((2, N, H), dtype=torch.float32, device=dev)
    dhr = torch.empty((2, N, H), dtype=dtype, device=dev)
    esz = dG.element_size()
    for s in range(T - 1, -1, -1):
        tf, tr = s, T - 1 - s
        ts, tps = (tf, tr), (tf - 1, tr + 1)
        ops.lstm_cell_bwd([G[d, ts[d]] for d in (0, 1)], [Cst[d, ts[d]] for d in (0, 1)],
                          [Cst[d, tps[d]] if s > 0 else None for d in (0, 1)],
                          [dY3[ts[d], :, d * H:(d + 1) * H] for d in (0, 1)], 2 * H,
                          [dhr[d] if s < T - 1 else None for d in (0, 1)], [dc[0], dc[1]], [dG[d, ts[d]] for d in (0, 1)])
        if s > 0:
            # dh_rec_d = dG_d[t_d] W_hh_d   (both directions, one strided-batched GEMM)
            pA = dG.data_ptr() + tf * N * 4 * H * esz
            sA = (T + tr - tf) * N * 4 * H
            ops.gemm_batched_raw(pA, sv["Whh"].data_ptr(), dhr.data_ptr(), N, H, 4 * H, 4 * H, H, H, sA, 4 * H * H, N * H,
                                 2, False, False, dtype, dtype, 1.0, 0.0)
    X2 = X.view(T * N, I)
    grads = []
    dX = torch.empty((T * N, I), dtype=dtype, device=dev)
    for d in range(2):
        dG2 = dG[d].view(T * N, 4 * H)
        dWih = ops.gemm(dG2, X2, transA=True, out_dtype=torch.float32)
        # dW_hh = sum_t dG[t]^T h_{t_prev}: forward dir pairs dG[1:] with Y[:-1], reverse dir dG[:-1] with Y[1:]
        if d == 0:
            A = dG[0, 1:].reshape((T - 1) * N, 4 * H)
            Bm = Y[:T - 1].view((T - 1) * N, 2 * H)[:, :H]
        else:
            A = dG[1, :T - 1].reshape((T - 1) * N, 4 * H)
            Bm = Y[1:].view((T - 1) * N, 2 * H)[:, H:]
        dWhh = ops.gemm(A, Bm, transA=True, out_dtype=torch.float32) if T > 1 else torch.zeros(4 * H, H, device=dev)
        db = ops.colsum(dG2)
        grads += [dWih, dWhh, db, db.clone()]
        ops.gemm(dG2, sv["Wih"][d], out=dX, beta=0.0 if d == 0 else 1.0)
    return dX.view(T, N, I), grads + [dWemb, dbemb]


class _BiLSTMFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, dtype, training, *params):
        X = ops.cast(x.contiguous(), dtype)
        out, sv = _bilstm_forward_impl(X, params, dtype, training)
        ctx.sv, ctx.dtype, ctx.in_dtype = sv, dtype, x.dtype
        return out

    @staticmethod
    def backward(ctx, dout):
        dX, grads = _bilstm_backward_impl(dout.contiguous(), ctx.sv, ctx.dtype)
        ctx.sv = None
        return (dX.to(ctx.in_dtype), None, None) + tuple(grads)


def bilstm_forward(module, x):
    """decoders/crnn.py:16-24: (T, N, nIn) -> LSTM -> Linear -> (T, N, nOut)."""
    _require_cuda(x, "BidirectionalLSTM")
    return _BiLSTMFn.apply(x, compute_dtype(), torch.is_grad_enabled(), *_bilstm_params(module))


def decoder_forward(module, feature, targets=None, lengths=None, train=False):
    """decoders/crnn.py:80-104."""
    _require_cuda(feature, "CRNNDecoder")
    b, c, h, w = feature.size()
    if h > 1:
        feature = module.fpn2rnn(feature)
        b, c, h, w = feature.size()
    assert h == 1, "the height of conv must be 1"
    seq = feature.squeeze(2).permute(2, 0, 1)          # (W, N, C) view; the BiLSTM entry makes it contiguous
    pred = module.rnn(seq)                             # (T, N, classes)
    if train:
        T = pred.size(0)
        pred_size = torch.full((b,), T, dtype=torch.int64, device=pred.device)
        if module.loss_func == 'pytorch':
            loss, lp = ctc1d.ctc_loss_from_logits(pred.float(), targets, pred_size, lengths, blank=0,
                                                  zero_infinity=True, reduction="mean")
        else:   # decoders/ctc_loss.py:118-121: per-sample nll / target_length, no zero_infinity
            nll, lp = ctc1d.ctc_loss_from_logits(pred.float(), targets, pred_size, lengths, blank=0,
                                                 zero_infinity=False, reduction="none")
            loss = nll / lengths.to(nll.device).to(nll.dtype)
        return loss, lp.to(torch.float64)              # decoders/crnn.py:96 hands float64 log-probs back
    pred = pred.float().permute(1, 2, 0).unsqueeze(2)
    return F.softmax(pred, dim=1)
