"""GPU: the fused per-step LSTM kernels (lstm_step_fwd_tc / lstm_step_bwd_tc, csrc/gemm_tcgen05.cu) for ONE time step of
both directions against a float64 restatement of their contract:

    forward : pre = Gx + h_prev W_hh^T + b   (gate columns unit-major: column 4j + g, g = i, f, g, o)
              i, f, o = sigmoid, g = tanh of pre; written back over Gx (bf16)
              c = f c_prev + i g (fp32);  h = o tanh(c) (bf16, into the [B, 2H] layer output and into h_next)
    backward: dh = dY + dG_next W_hh;  tc = tanh(c);  dct = dc + dh o (1 - tc^2)
              dG = (dct g i(1-i), dct c_prev f(1-f), dct i (1-g^2), dh tc o(1-o)) (bf16);  dc <- dct f (fp32)

The two directions get different data (a mixed-up blockIdx.z fails) and the layer output / dY are the two H-wide
halves of one [B, 2H] tensor (ldh = 2H).  The reference uses the kernel's own bf16 operands; what is left is the
kernel's arithmetic:

  * activations (bf16 stores of values in [-1, 1]): rounding <= 2^-9 = 2e-3, tanh.approx.f32 ~2^-11 ~ 5e-4, fp32
    summation of the recurrent product negligible -> 4e-3 absolute;
  * c (fp32, from unrounded fp32 activations): i g and f c_prev each carry the ~1e-3 relative activation error ->
    3e-3 (1 + |c_prev|);
  * h (bf16): 2e-3 rounding + tanh.approx of c and the o error -> 6e-3;
  * dG (bf16) and dc (fp32): every term is a product of dct or dh with factors <= 1 whose tanh.approx error is
    ~1e-3, plus bf16 rounding (2^-9 relative) for dG -> 8e-3 (dG) and 4e-3 (dc) times the row scale
    max_j (|dh_j| + |dc_j|).
A wrong accumulator row or column, a swapped gate or a missing K block moves elements by O(1) of these scales.
"""
import pytest
import torch

from tests import wgmma_variants as wv

pytestmark = pytest.mark.gpu

VARIANTS = {wv.expected_variant("lstm_step_fwd"), wv.expected_variant("lstm_step_bwd")}

SHAPES = [(B, H) for H in (64, 256) for B in (1, 128, 129, 300)]
FLAGS = [(1, True), (1, False), (0, True), (0, False)]       # (have_h / have_rec, c_prev given)


def _within(got, ref, tol, what):
    """|got - ref| <= tol element-wise; reports the worst element."""
    wv.assert_within(got, ref, torch.broadcast_to(torch.as_tensor(tol, dtype=torch.float64, device=ref.device), ref.shape),
                     what)


def _unit_major_gates(pre):
    """[B, 4H] unit-major -> (i, f, g, o), each [B, H]."""
    p = pre.view(pre.size(0), -1, 4)
    return p[..., 0], p[..., 1], p[..., 2], p[..., 3]


@pytest.mark.parametrize("flags", FLAGS, ids=["rec-cprev", "rec", "first-cprev", "first"])
@pytest.mark.parametrize("shape", SHAPES, ids=["B%d-H%d" % s for s in SHAPES])
def test_lstm_step_fwd(cuda, shape, flags):
    from megreader_b200 import nnops
    B, H = shape
    have_h, with_c = flags
    torch.manual_seed(B * 1000 + H + 7 * have_h + 3 * with_c)
    h_prev = [(torch.randn(B, H, device=cuda) * 0.5).bfloat16() for _ in range(2)]
    Whh = [(torch.randn(4 * H, H, device=cuda) / H ** 0.5).bfloat16() for _ in range(2)]
    Gx = [torch.randn(B, 4 * H, device=cuda).bfloat16() for _ in range(2)]
    bias = [torch.randn(4 * H, device=cuda) * 0.5 for _ in range(2)]
    c_prev = [torch.randn(B, H, device=cuda) * 2 if with_c else None for _ in range(2)]
    gates = [g.clone() for g in Gx]
    c_out = [torch.full((B, H), float("nan"), device=cuda) for _ in range(2)]
    Y = torch.zeros(B, 2 * H, device=cuda).bfloat16()
    h_out = [Y[:, :H], Y[:, H:]]
    h_next = [torch.zeros(B, H, device=cuda).bfloat16() for _ in range(2)]
    wv.run_variant(wv.expected_variant("lstm_step_fwd"),
                   lambda: nnops.lstm_step_fwd_tc(h_prev, Whh, gates, bias, c_prev, c_out, h_out, 2 * H, h_next, have_h))
    for d in range(2):
        pre = Gx[d].double() + bias[d].double()
        if have_h:
            pre = pre + h_prev[d].double() @ Whh[d].double().t()
        i, f, g, o = _unit_major_gates(pre)
        i, f, g, o = torch.sigmoid(i), torch.sigmoid(f), torch.tanh(g), torch.sigmoid(o)
        cp = c_prev[d].double() if with_c else torch.zeros_like(i)
        c = f * cp + i * g
        h = o * torch.tanh(c)
        tag = "lstm fwd B=%d H=%d dir %d" % (B, H, d)
        _within(gates[d], torch.stack([i, f, g, o], -1).view(B, 4 * H), 4e-3, tag + " activations")
        _within(c_out[d], c, 3e-3 * (1 + cp.abs()), tag + " c")
        _within(h_out[d], h, 6e-3, tag + " h (layer output)")
        assert torch.equal(h_next[d], h_out[d]), tag + ": h_next differs from the layer output"


@pytest.mark.parametrize("flags", FLAGS, ids=["rec-cprev", "rec", "first-cprev", "first"])
@pytest.mark.parametrize("shape", SHAPES, ids=["B%d-H%d" % s for s in SHAPES])
def test_lstm_step_bwd(cuda, shape, flags):
    from megreader_b200 import nnops
    B, H = shape
    have_rec, with_c = flags
    torch.manual_seed(B * 1000 + H + 7 * have_rec + 3 * with_c + 1)
    act = lambda t: torch.stack([torch.sigmoid(t[..., 0]), torch.sigmoid(t[..., 1]), torch.tanh(t[..., 2]),  # noqa: E731
                                 torch.sigmoid(t[..., 3])], -1).view(B, 4 * H)
    gates = [act(torch.randn(B, H, 4, device=cuda) * 1.5).bfloat16() for _ in range(2)]
    c = [torch.randn(B, H, device=cuda) * 1.5 for _ in range(2)]
    c_prev = [torch.randn(B, H, device=cuda) * 1.5 if with_c else None for _ in range(2)]
    dY = torch.randn(B, 2 * H, device=cuda).bfloat16()
    dh_out = [dY[:, :H], dY[:, H:]]
    dG_next = [(torch.randn(B, 4 * H, device=cuda) * 0.5).bfloat16() for _ in range(2)]
    Whh = [(torch.randn(4 * H, H, device=cuda) / H ** 0.5).bfloat16() for _ in range(2)]
    dc_in = [torch.randn(B, H, device=cuda) for _ in range(2)]
    dc = [t.clone() for t in dc_in]
    dgates = [torch.full((B, 4 * H), float("nan"), device=cuda).bfloat16() for _ in range(2)]
    wv.run_variant(wv.expected_variant("lstm_step_bwd"),
                   lambda: nnops.lstm_step_bwd_tc(dG_next, Whh, gates, c, c_prev, dh_out, 2 * H, dc, dgates, have_rec))
    for d in range(2):
        i, f, g, o = _unit_major_gates(gates[d].double())
        dh = dh_out[d].double()
        if have_rec:
            dh = dh + dG_next[d].double() @ Whh[d].double()
        tc = torch.tanh(c[d].double())
        cp = c_prev[d].double() if with_c else torch.zeros_like(tc)
        dct = dc_in[d].double() + dh * o * (1 - tc * tc)
        dG = torch.stack([dct * g * i * (1 - i), dct * cp * f * (1 - f), dct * i * (1 - g * g), dh * tc * o * (1 - o)], -1)
        scale = (dh.abs() + dc_in[d].double().abs()).amax(1, keepdim=True)
        tag = "lstm bwd B=%d H=%d dir %d" % (B, H, d)
        _within(dgates[d], dG.view(B, 4 * H), 8e-3 * scale, tag + " dgates")
        _within(dc[d], dct * f, 4e-3 * scale, tag + " dc")
