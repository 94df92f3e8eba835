"""GPU: the hand-written wgmma + TMA GEMM (csrc/gemm_tcgen05.cu) against a plain PyTorch fp32 reference of the same
product on bf16-rounded inputs (fp32 accumulation both sides: tolerance covers summation order only)."""
import pytest
import torch

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
