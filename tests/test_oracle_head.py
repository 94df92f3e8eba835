"""CPU: the restatement of the 2D-CTC head epilogue (oracle/head_port.py) against goldens recorded from the UNMODIFIED
reference module (decoders/ctc_decoder2d.py forward, oracle/make_golden.py head): pred and both logits' gradients, with
the max(., tiny) clamp inactive, underflow-active and (through a large saved_tiny) active on most entries."""
import os

import numpy as np
import pytest
import torch
from tests.cases import load_head_golden

from oracle import head_port



@pytest.mark.parametrize("tag", ["a", "b", "c"])
def test_head_port_reproduces_reference(tag):
    g = load_head_golden()
    m, z = torch.from_numpy(g[tag + ".mask_logits"]), torch.from_numpy(g[tag + ".cls_logits"])
    tiny = float(g[tag + ".tiny"])
    pred = head_port.head_log_probs(m, z, tiny)
    np.testing.assert_allclose(pred.numpy(), g[tag + ".pred"], rtol=1e-6, atol=1e-6)
    dm, dz = head_port.head_grads(m, z, torch.from_numpy(g[tag + ".grad_pred"]), tiny)
    np.testing.assert_allclose(dm.numpy(), g[tag + ".grad_mask_logits"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(dz.numpy(), g[tag + ".grad_cls_logits"], rtol=1e-5, atol=1e-5)
