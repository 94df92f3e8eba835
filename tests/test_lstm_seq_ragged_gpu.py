"""GPU: the persistent BiLSTM recurrence (csrc/lstm_seq_tcgen05.cu) at a batch whose last 64-row tile is ragged and
that still fits co-resident (N = 500: 4 x 16 x 2 forward CTAs, 8 x 8 x 2 backward CTAs).  Every test asserts that both
persistent entries accepted the call, so a fall-back to the per-step kernels cannot pass for them."""
import pytest
import torch

from tests.test_nn_kernels_gpu import _bilstm_case, _bilstm_run

pytestmark = pytest.mark.gpu


@pytest.fixture
def accepted(monkeypatch):
    """records the return value of every persistent forward / backward call the engine makes"""
    from megreader_b200 import crnn_engine
    calls = {"fwd": [], "bwd": []}
    fwd, bwd = crnn_engine.ops.lstm_seq_fwd_tc, crnn_engine.ops.lstm_seq_bwd_tc

    def f(*a):
        calls["fwd"].append(fwd(*a))
        return calls["fwd"][-1]

    def b(*a):
        calls["bwd"].append(bwd(*a))
        return calls["bwd"][-1]
    monkeypatch.setattr(crnn_engine.ops, "lstm_seq_fwd_tc", f)
    monkeypatch.setattr(crnn_engine.ops, "lstm_seq_bwd_tc", b)
    return calls


def _check_persistent(calls):
    from megreader_b200 import crnn_engine
    assert calls["fwd"] == [True] and calls["bwd"] == [True], calls
    assert int(crnn_engine.LAST_LSTM_FLAGS[-1]) == 0, "inter-CTA wait timed out"


@pytest.mark.parametrize("shape", [(9, 500, 128, 256, 38), (4, 500, 64, 128, 16)])
def test_bilstm_persistent_ragged_vs_torch(cuda, accepted, shape):
    """The persistent kernels against nn.LSTM + nn.Linear in fp32 (the bounds of test_bilstm_fused_tcgen05_paths)."""
    m, x, dout, ref, ref_dx, ref_grads = _bilstm_case(cuda, *shape, seed=6)
    out, dx, grads = _bilstm_run(m, x, dout, "seq")
    _check_persistent(accepted)
    torch.testing.assert_close(out, ref, rtol=5e-2, atol=5e-2)
    torch.testing.assert_close(dx, ref_dx, rtol=5e-2, atol=0.02 * float(ref_dx.abs().max()) + 5e-2)
    for got, want in zip(grads, ref_grads):
        torch.testing.assert_close(got, want, rtol=5e-2, atol=0.02 * float(want.abs().max()) + 0.05)


@pytest.mark.parametrize("shape", [(26, 500, 256, 256, 38), (5, 1100, 64, 64, 16)])
def test_bilstm_persistent_ragged_equals_stepwise(cuda, accepted, shape):
    """The persistent kernels against the per-step fused kernels (the bounds of test_bilstm_persistent_equals_stepwise).
    N = 1100 at H = 64: 9 forward and 18 backward row tiles, ragged, on 72 CTAs each way."""
    m, x, dout, _, _, _ = _bilstm_case(cuda, *shape, seed=8)
    out_a, dx_a, g_a = _bilstm_run(m, x, dout, "step")
    assert accepted["fwd"] == [] and accepted["bwd"] == []
    out_b, dx_b, g_b = _bilstm_run(m, x, dout, "seq")
    _check_persistent(accepted)
    torch.testing.assert_close(out_b, out_a, rtol=1e-2, atol=1e-2)
    torch.testing.assert_close(dx_b, dx_a, rtol=1e-2, atol=1e-2 * float(dx_a.abs().max()) + 1e-3)
    for got, want in zip(g_b, g_a):
        torch.testing.assert_close(got, want, rtol=1e-2, atol=1e-2 * float(want.abs().max()) + 1e-3)
