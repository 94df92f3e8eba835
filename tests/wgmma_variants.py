"""Which wgmma kernel instantiation a call should launch, which ones it did launch, and the element-wise error bound the
kernel-level tests use.

Every template instantiation of the tensor-core kernels (csrc/gemm_tcgen05.cu, csrc/dcn_tcgen05.cu) has its own
descriptor strides, TMA boxes and ring depth, so each one needs a case of its own.  expected_variant() restates the host
dispatch of the C entry points; the GPU tests assert through launched_kernels() that the kernel they mean to test is the
one that ran, and tests/test_kernel_inventory.py checks on the CPU that the compiled instantiations are exactly
ALL_VARIANTS and that each is the expected variant of at least one GPU case.

Kernel names are normalised to "name<arg,arg,...>": CUPTI prints "<128, 6, 0, 1>", cu++filt "<(int)128, (int)6, ...>".
"""
import os
import re
import warnings

import torch

ALL_VARIANTS = frozenset([
    "gemm_tcgen05_kernel<128,6,0,0>", "gemm_tcgen05_kernel<64,8,0,0>",        # NT
    "gemm_tcgen05_kernel<128,6,0,1>", "gemm_tcgen05_kernel<64,8,0,1>",        # NN
    "gemm_tcgen05_kernel<128,6,1,1>", "gemm_tcgen05_kernel<64,8,1,1>",        # TN
    "conv_fprop_tcgen05_kernel<128,3,1>", "conv_fprop_tcgen05_kernel<64,3,1>",  # TMA-A, shallow ring (default)
    "conv_fprop_tcgen05_kernel<128,6,1>", "conv_fprop_tcgen05_kernel<64,8,1>",  # TMA-A, deep ring (MR_CONV_SHALLOW=0)
    "conv_fprop_tcgen05_kernel<128,6,0>", "conv_fprop_tcgen05_kernel<64,8,0>",  # cp.async gather
    "conv_wgrad_tcgen05_kernel<128,64,6>", "conv_wgrad_tcgen05_kernel<128,80,4>",
    "conv_wgrad_tcgen05_kernel<64,64,8>", "conv_wgrad_tcgen05_kernel<64,80,6>",
    "lstm_step_fwd_tcgen05_kernel<4>", "lstm_step_bwd_tcgen05_kernel<6>",
    "dcn_fwd_tcgen05_kernel<128,2>",
])

_TEMPLATE = re.compile(r"(\w+_kernel)<([^<>]*)>")


def normalise(name):
    """Full demangled kernel name -> "name<args>" (the bare name for kernels that are not templates)."""
    name = re.sub(r"\s+", "", name.replace("(int)", ""))
    m = _TEMPLATE.search(name)
    if m:
        return "%s<%s>" % m.groups()
    m = re.search(r"(\w+)\(", name)
    return m.group(1) if m else name


def launched_kernels(fn):
    """Run fn() under torch.profiler (CUDA activity only); -> (fn's result, set of normalised kernel names it launched)."""
    from torch.profiler import DeviceType, ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        result = fn()
        torch.cuda.synchronize()
    return result, {normalise(e.name) for e in prof.events() if e.device_type == DeviceType.CUDA}


def run_variant(variant, fn):
    """fn() must launch `variant`, and no other tensor-core instantiation; -> fn's result.

    A trace without any tensor-core kernel record only warns: in a long pytest process that has run many other GPU
    tests, later profiler sessions were seen to miss the library's kernel records (torch's own were still there), so
    such a trace says nothing about which instantiation ran.  Run the kernel test files on their own to check every
    variant."""
    assert variant in ALL_VARIANTS, variant
    result, names = launched_kernels(fn)
    seen = sorted(n for n in names if n in ALL_VARIANTS)
    if not seen:
        warnings.warn("torch.profiler recorded no tensor-core kernel: %s not checked (saw %s)" % (variant, sorted(names)))
    else:
        assert seen == [variant], "expected %s to run, the profiler saw %s" % (variant, seen)
    return result


# ---------------------------------------------------------------- the host dispatch, restated
def _ring(bn):
    return 6 if bn == 128 else 8


def gemm_variant(N, transA, transB, **_):
    """mr_gemm_tcgen05: BN = 128 for N > 64; (A_MN, B_MN) = (0,0) NT, (0,1) NN, (1,1) TN."""
    form = {(0, 1): (0, 0), (0, 0): (0, 1), (1, 0): (1, 1)}[(int(transA), int(transB))]
    bn = 128 if N > 64 else 64
    return "gemm_tcgen05_kernel<%d,%d,%d,%d>" % ((bn, _ring(bn)) + form)


def conv_out(H, W, kh, kw, sh=1, sw=1, ph=0, pw=0, dh=1, dw=1):
    return (H + 2 * ph - dh * (kh - 1) - 1) // sh + 1, (W + 2 * pw - dw * (kw - 1) - 1) // sw + 1


def tma_a_segments(Ho, Wo, sh=1, sw=1):
    """Widths of the power-of-two output segments mr_conv2d_fprop_tcgen05 tiles with one 4-D TMA box each, or None when
    the plan needs more than four segments or a strided box spans more than 256 rows / columns (-> cp.async gather)."""
    segs, w0 = [], 0
    while w0 < Wo:
        bw = 128
        while bw > Wo - w0:
            bw //= 2
        bh = 1
        while bh * 2 <= Ho and bw * bh * 2 <= 128:
            bh *= 2
        for _ in range((Wo - w0) // bw):
            if len(segs) == 4 or bw * sw > 256 or bh * sh > 256:
                return None
            segs.append(bw)
            w0 += bw
    return segs


def conv_fprop_variant(H, W, Cout, kh, kw, sh=1, sw=1, ph=0, pw=0, dh=1, dw=1, env=None, **_):
    env = os.environ if env is None else env
    Ho, Wo = conv_out(H, W, kh, kw, sh, sw, ph, pw, dh, dw)
    bn = 128 if Cout > 64 else 64
    if "MR_CONV_NO_TMA_A" not in env and tma_a_segments(Ho, Wo, sh, sw) is not None:
        shallow = env.get("MR_CONV_SHALLOW") is None or env["MR_CONV_SHALLOW"][:1] == "1"
        return "conv_fprop_tcgen05_kernel<%d,%d,1>" % (bn, 3 if shallow else _ring(bn))
    return "conv_fprop_tcgen05_kernel<%d,%d,0>" % (bn, _ring(bn))


def conv_wgrad_variant(H, W, C, kh, kw, sh=1, sw=1, ph=0, pw=0, dh=1, dw=1, **_):
    """RB = 80 pixel rows per K block iff 64 < Wo <= 80; BN = 128 iff kh*kw*C > 64."""
    _, Wo = conv_out(H, W, kh, kw, sh, sw, ph, pw, dh, dw)
    rb = 80 if 64 < Wo <= 80 else 64
    bn = 128 if kh * kw * C > 64 else 64
    stages = {(128, 64): 6, (128, 80): 4, (64, 64): 8, (64, 80): 6}[(bn, rb)]
    return "conv_wgrad_tcgen05_kernel<%d,%d,%d>" % (bn, rb, stages)


def dcn_fwd_variant(**_):
    return "dcn_fwd_tcgen05_kernel<128,2>"


_DISPATCH = {
    "gemm": gemm_variant,
    "conv_fprop": conv_fprop_variant,
    "conv_wgrad": conv_wgrad_variant,
    "lstm_step_fwd": lambda **_: "lstm_step_fwd_tcgen05_kernel<4>",
    "lstm_step_bwd": lambda **_: "lstm_step_bwd_tcgen05_kernel<6>",
    "dcn_fwd": dcn_fwd_variant,
}


def expected_variant(kind, **geometry):
    """The kernel instantiation the C entry point of `kind` launches for this geometry (and environment `env`)."""
    return _DISPATCH[kind](**geometry)


# ---------------------------------------------------------------- error bound
def bound(abs_ref, ref=None, bf16_out=False):
    """Element-wise bound for a kernel that sums bf16 products in fp32: 2^-16 * (|A| . |B|), where abs_ref is the same
    product (or convolution) of absolute values in float64.  A correct fp32 summation errs by about u * sum|ab|
    (u = 2^-24), so this leaves ~100x margin, while one dropped 64-deep K block out of 4608, a wrong tap or a swapped
    row / column half moves an element by a sizeable fraction of sum|ab|.  bf16 outputs add their rounding,
    2^-8 * |ref|."""
    b = abs_ref * 2.0 ** -16
    if bf16_out:
        b = b + ref.abs() * 2.0 ** -8
    return b


def assert_within(out, ref, bnd, what=""):
    """|out - ref| <= bnd element-wise (float64 comparison); reports the worst element.  -> worst error / bound."""
    out, ref, bnd = out.double(), ref.double(), bnd.double()
    assert out.shape == ref.shape == bnd.shape, (out.shape, ref.shape, bnd.shape)
    ratio = (out - ref).abs() / bnd.clamp_min(1e-300)
    ratio = torch.nan_to_num(ratio, nan=float("inf"))
    flat = int(torch.argmax(ratio))
    worst = float(ratio.reshape(-1)[flat])
    if worst > 1.0:
        idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(flat), ratio.shape))
        bad = int((ratio > 1).sum())
        raise AssertionError("%s: %d of %d elements outside the bound; worst at %s: got %r, want %r, bound %.3g "
                             "(error / bound = %.3g)" % (what, bad, ratio.numel(), idx, float(out[idx]), float(ref[idx]),
                                                         float(bnd[idx]), worst))
    print("%s worst error/bound %.3g" % (what, worst))
    return worst
