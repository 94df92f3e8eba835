"""GPU: the cfg-3 / cfg-4 models (BASELINE.json) with EVERY convolution on the repo's wgmma kernels (conv_engine) against the
same modules on the library path in fp32: training loss within bf16 tolerance, finite gradients for every parameter, and the
parameter gradients' direction (cosine) for the layers that see the largest signals."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("cfg", [3, 4])
def test_trunk_step_engine_vs_library(cuda, cfg):
    import bench_trunks
    from megreader_b200 import conv_engine
    torch.manual_seed(0)
    import numpy as np
    np.random.seed(0)
    net, n_engine = bench_trunks.build(cfg, cuda, engine=False)
    # BatchNorm on running statistics for this comparison: with 4 samples the batch statistics of the PPM's 1x1-bin branch are
    # taken over 4 values per channel, which turns bf16 rounding into O(1) changes of the normalised activations (measured:
    # gradient directions decorrelate layer by layer while loss and gradient norms agree) -- a property of the model at this
    # batch size, not of the kernels (tests/test_conv_engine_gpu.py pins every geometry separately)
    for m in net.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.eval()
    x, y, l = [t.to(cuda) for t in bench_trunks.synth(1, 4, bench_trunks.CFG[cfg]["hw"], 8)]
    state = {k: v.clone() for k, v in net.state_dict().items()}

    def run():
        for p in net.parameters():
            p.grad = None
        torch.manual_seed(1); np.random.seed(1)          # the attention decoder draws teacher-forcing coins
        loss, _ = net(x, y, l)
        loss = loss.mean()
        loss.backward()
        g = {n: p.grad.detach().float().clone() for n, p in net.named_parameters() if p.grad is not None}
        net.load_state_dict(state)                        # BatchNorm running statistics
        return float(loss), g
    loss_ref, g_ref = run()
    # weight gradients on the side stream (what bench.py --config 3 / 4 runs; tests/test_conv_engine_gpu.py covers the one-stream path)
    assert conv_engine.use_engine_convs(net, wgrad_side_stream=True) > 40
    try:
        loss_eng, g_eng = run()
    finally:
        conv_engine.WGRAD_SIDE_STREAM = False
    assert abs(loss_eng - loss_ref) / abs(loss_ref) < 5e-2, (loss_eng, loss_ref)
    assert all(torch.isfinite(v).all() for v in g_eng.values())
    assert set(g_eng) == set(g_ref)
    # gradient direction of the big weight tensors (bf16 trunk, 50+ layers deep: cosine, not element-wise)
    checked = 0
    for n, r in g_ref.items():
        if r.numel() >= 64 * 64 and float(r.norm()) > 1e-6:
            cos = float((r * g_eng[n]).sum() / (r.norm() * g_eng[n].norm() + 1e-20))
            assert cos > 0.9, (n, cos)
            checked += 1
    assert checked > 20
