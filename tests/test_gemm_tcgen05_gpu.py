"""GPU: the hand-written wgmma + TMA GEMM (csrc/gemm_tcgen05.cu) against a plain PyTorch fp32 reference of the same
product on bf16-rounded inputs (fp32 accumulation both sides: tolerance covers summation order only)."""
import zlib

import pytest
import torch

from tests import wgmma_variants as wv

pytestmark = pytest.mark.gpu

SHAPES = [  # M, N, K
    (128, 256, 64), (128, 128, 128), (256, 256, 512), (300, 200, 136), (1000, 512, 4608), (130, 38 * 8, 72),
    (64, 64, 64), (4096, 64, 576),
]


def _ref(A, B):
    return A.float() @ B.float()


@pytest.mark.parametrize("shape", SHAPES, ids=["x".join(map(str, s)) for s in SHAPES])
def test_nt(cuda, shape):
    from megreader_b200 import nnops
    M, N, K = shape
    torch.manual_seed(0)
    A = torch.randn(M, K, device=cuda).bfloat16()
    B = torch.randn(N, K, device=cuda).bfloat16()
    ref = _ref(A, B.t())
    out = nnops.gemm_tc(A, B, out_dtype=torch.float32)
    torch.testing.assert_close(out, ref, rtol=1e-4, atol=1e-3 * (K ** 0.5))
    bias = torch.randn(N, device=cuda)
    out2 = nnops.gemm_tc(A, B, out_dtype=torch.bfloat16, bias=bias, relu=True)
    torch.testing.assert_close(out2.float(), torch.relu(ref + bias), rtol=1e-2, atol=1e-2 * (K ** 0.5))


@pytest.mark.parametrize("shape", [(128, 256, 64), (512, 4608, 4100), (64, 72, 1000), (256, 1152, 333 * 8)],
                         ids=lambda s: "x".join(map(str, s)))
def test_tn_splitk(cuda, shape):
    """weight-gradient form: C[M,N] += A[K,M]^T B[K,N], fp32 atomics, split-K."""
    from megreader_b200 import nnops
    M, N, K = shape
    torch.manual_seed(1)
    A = torch.randn(K, M, device=cuda).bfloat16()
    B = torch.randn(K, N, device=cuda).bfloat16()
    ref = _ref(A.t(), B)
    out = nnops.gemm_tc(A, B, transA=True, transB=False, out_dtype=torch.float32)
    torch.testing.assert_close(out, ref, rtol=1e-4, atol=1e-3 * (K ** 0.5))
    acc = torch.ones(M, N, device=cuda)
    nnops.gemm_tc(A, B, transA=True, transB=False, out=acc, beta=1.0, splits=4)
    torch.testing.assert_close(acc, ref + 1, rtol=1e-4, atol=1e-3 * (K ** 0.5))


def test_strided_operands_and_unsupported(cuda):
    from megreader_b200 import nnops
    from megreader_b200._lib import MegReaderB200Error
    torch.manual_seed(2)
    wide = torch.randn(200, 256, device=cuda).bfloat16()
    B = torch.randn(96, 128, device=cuda).bfloat16()
    out = nnops.gemm_tc(wide[:, 128:], B, out_dtype=torch.float32)          # lda = 256, K = 128
    torch.testing.assert_close(out, _ref(wide[:, 128:], B.t()), rtol=1e-4, atol=2e-2)
    with pytest.raises(MegReaderB200Error):
        nnops.gemm_tc(torch.randn(8, 20, device=cuda).bfloat16()[:, :12], B[:, :12])   # lda % 8 != 0


# ---------------------------------------------------------------- every instantiation, against float64 with an element-wise bound
def G(form, M, N, K, pad_a=0, pad_b=0, off=0, ldc_pad=0, out="f32", bias=False, relu=False, beta=0, splits=1):
    """One case: form NT / NN / TN; pad_a / pad_b: extra row pitch of the operand storage beyond the inner size rounded
    up to 8 (the kernel needs lda, ldb % 8 == 0, so ragged M / N of the TN form and ragged N of the NN form live in
    padded storage); off: column offset of both operands inside that storage (a multiple of 8: 16-byte aligned bases);
    ldc_pad: extra row pitch of C; beta = 1 accumulates onto a non-zero fp32 C."""
    return dict(form=form, M=M, N=N, K=K, pad_a=pad_a, pad_b=pad_b, off=off, ldc_pad=ldc_pad, out=out, bias=bias,
                relu=relu, beta=beta, splits=splits)


_FORMS = {"NT": (False, True), "NN": (False, False), "TN": (True, False)}

CASES = [
    # three forms x both tile widths, ragged M and K
    *[G(f, 300, n, 136) for f in ("NT", "NN", "TN") for n in (38, 200)],
    # one partial K block (K < 64), M = 1 / 129 / 300, N = 1 / 38 / 65 / 200
    G("NT", 1, 1, 8), G("NT", 129, 65, 40), G("NT", 300, 38, 8),
    G("NN", 129, 38, 8), G("NN", 1, 65, 40), G("NN", 300, 1, 136),
    G("TN", 129, 1, 40), G("TN", 1, 200, 8), G("TN", 300, 65, 136),
    # long K: one missing 64-deep block out of 72 is far outside the bound
    G("NT", 256, 200, 4608), G("NN", 129, 38, 4608), G("TN", 65, 200, 4608, beta=1, splits=3),
    # strided operands (lda / ldb > inner size, non-zero 16-byte aligned base offset), strided output
    G("NT", 129, 65, 136, pad_a=24, pad_b=8, off=8, ldc_pad=3), G("NN", 300, 38, 136, pad_a=8, pad_b=16, off=8, ldc_pad=5),
    G("NN", 129, 200, 72, pad_a=64, pad_b=40, off=16), G("TN", 129, 38, 136, pad_a=16, pad_b=8, off=8, ldc_pad=1, beta=1),
    # bf16 output: N % 8 != 0 takes the scalar store, N % 32 == 0 and an aligned pitch the 16-byte store
    G("NT", 300, 38, 136, out="bf16"), G("NN", 129, 65, 40, out="bf16"), G("NT", 129, 128, 136, out="bf16"),
    G("NN", 300, 200, 136, out="bf16", ldc_pad=8),
    # bias + ReLU (fp32 and bf16 out)
    G("NT", 300, 38, 136, bias=True, relu=True), G("NT", 129, 200, 40, bias=True, relu=True, out="bf16"),
    G("NN", 129, 65, 136, bias=True, relu=True), G("NN", 300, 38, 72, bias=True, relu=True, out="bf16"),
    G("NT", 129, 65, 136, bias=True),
    # split-K / accumulation: beta = 1 onto a non-zero C, splits 1, 3 and more than there are K blocks
    G("TN", 300, 200, 1000, beta=1, splits=1), G("TN", 300, 200, 1000, beta=1, splits=3),
    G("TN", 129, 38, 136, beta=1, splits=99), G("TN", 129, 65, 40, beta=1, splits=3),
    G("NT", 129, 200, 1000, beta=1, splits=3), G("NN", 300, 38, 1000, beta=1, splits=7),
    # bias with splits = 1 and beta = 1: C + AB + b
    G("NT", 129, 65, 136, bias=True, beta=1), G("TN", 300, 38, 136, bias=True, beta=1),
]


def _case_id(c):
    s = "%s-%dx%dx%d" % (c["form"], c["M"], c["N"], c["K"])
    for k, default in (("pad_a", 0), ("pad_b", 0), ("off", 0), ("ldc_pad", 0), ("out", "f32"), ("bias", False),
                       ("relu", False), ("beta", 0), ("splits", 1)):
        if c[k] != default:
            s += "-%s%s" % (k, "" if c[k] is True else c[k])
    return s


def case_variant(c):
    transA, transB = _FORMS[c["form"]]
    return wv.expected_variant("gemm", N=c["N"], transA=transA, transB=transB)


VARIANTS = {case_variant(c) for c in CASES}


def _stored(rows, cols, pad, off, dev):
    """[rows, cols] bf16 view with row pitch round_up(cols, 8) + pad + off, starting `off` columns into its storage."""
    ld = -(-cols // 8) * 8 + pad + off
    return torch.randn(rows, ld, device=dev).bfloat16()[:, off:off + cols]


@pytest.mark.parametrize("c", CASES, ids=[_case_id(c) for c in CASES])
def test_variant_vs_float64(cuda, c):
    """C (+)= op(A) op(B) (+ bias, ReLU) on bf16 operands against float64 on the same operands, element-wise within
    wv.bound; the expected instantiation must be the kernel that ran, and C's row padding must stay untouched."""
    from megreader_b200 import nnops
    torch.manual_seed(zlib.crc32(_case_id(c).encode()))
    transA, transB = _FORMS[c["form"]]
    M, N, K = c["M"], c["N"], c["K"]
    A = _stored(K, M, c["pad_a"], c["off"], cuda) if transA else _stored(M, K, c["pad_a"], c["off"], cuda)
    B = _stored(N, K, c["pad_b"], c["off"], cuda) if transB else _stored(K, N, c["pad_b"], c["off"], cuda)
    opA = (A.t() if transA else A).double()
    opB = (B.t() if transB else B).double()
    ref, absref = opA @ opB, opA.abs() @ opB.abs()
    dtype = torch.bfloat16 if c["out"] == "bf16" else torch.float32
    storage = torch.full((M, N + c["ldc_pad"]), 1234.5, device=cuda, dtype=dtype)
    out = storage[:, :N]
    if c["beta"]:
        out.copy_(torch.randn(M, N, device=cuda))
        ref, absref = ref + out.double(), absref + out.double().abs()
    bias = torch.randn(N, device=cuda) if c["bias"] else None
    if bias is not None:
        ref, absref = ref + bias.double(), absref + bias.double().abs()
    if c["relu"]:
        ref = torch.relu(ref)
    wv.run_variant(case_variant(c), lambda: nnops.gemm_tc(A, B, transA=transA, transB=transB, out=out, bias=bias,
                                                        relu=c["relu"], beta=float(c["beta"]), splits=c["splits"]))
    wv.assert_within(out, ref, wv.bound(absref, ref, dtype == torch.bfloat16), case_variant(c) + " " + _case_id(c))
    assert bool((storage[:, N:] == 1234.5).all()), "the epilogue wrote past column N"


def test_unsupported_combinations(cuda):
    """Forms and arguments the kernel does not cover raise MR_ERR_UNSUPPORTED instead of computing something else."""
    from megreader_b200 import nnops
    from megreader_b200._lib import MegReaderB200Error
    A = torch.randn(128, 128, device=cuda).bfloat16()
    B = torch.randn(128, 128, device=cuda).bfloat16()
    f32 = torch.zeros(128, 128, device=cuda)
    bias = torch.randn(128, device=cuda)
    calls = {
        "(1,1) form": lambda: nnops.gemm_tc(A, B, transA=True, transB=True, out=f32),
        "beta 0.5": lambda: nnops.gemm_tc(A, B, out=f32, beta=0.5),
        "bf16 with beta 1": lambda: nnops.gemm_tc(A, B, out=torch.zeros(128, 128, device=cuda).bfloat16(), beta=1.0),
        "lda % 8": lambda: nnops.gemm_tc(torch.randn(128, 140, device=cuda).bfloat16()[:, :128], B, out=f32),
        "unaligned base": lambda: nnops.gemm_tc(torch.randn(128, 136, device=cuda).bfloat16()[:, 4:132], B, out=f32),
        "bias with split-K": lambda: nnops.gemm_tc(A, B, out=f32, bias=bias, beta=1.0, splits=2),
        "ReLU with beta 1": lambda: nnops.gemm_tc(A, B, out=f32, relu=True, beta=1.0),
    }
    for what, call in calls.items():
        try:
            call()
        except MegReaderB200Error as e:
            assert "not supported" in str(e), (what, str(e))
        else:
            pytest.fail("%s was accepted" % what)
    torch.cuda.synchronize()
    assert bool((f32 == 0).all()), "a refused call wrote its output"
