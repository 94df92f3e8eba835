"""CPU: the CRNN oracle port (oracle/crnn_port.py) reproduces what the UNMODIFIED reference modules computed (golden vectors
recorded by oracle/make_golden.py and oracle/make_ref_golden_cpu.py) and carries their state-dict names; where the reference tree
is present it is also compared with them live, bit for bit."""
import gzip
import json
import os

import numpy as np
import pytest
import torch

from oracle import crnn_port, ref_loader
from tests.weights import crnn_batch, fill_state_dict

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _port():
    bb = fill_state_dict(crnn_port.CRNNBackbonePort(), "bb.")
    dec = fill_state_dict(crnn_port.CRNNDecoderPort(), "dec.")
    return bb, dec


def test_port_reproduces_golden():
    g = np.load(os.path.join(GOLD, "crnn_ref_cfg1.npz"))
    bb, dec = _port()
    torch.set_num_threads(1)
    x = torch.from_numpy(np.repeat(g["x"], 3, axis=1))
    loss, pred = dec(bb.train()(x), torch.from_numpy(g["labels"]), torch.from_numpy(g["lengths"]), train=True)
    np.testing.assert_allclose(loss.item(), float(g["loss"]), rtol=1e-5)
    np.testing.assert_allclose(pred.detach().numpy(), g["log_probs"], rtol=1e-4, atol=1e-5)


def test_port_reproduces_reference_outputs_and_state_dict_names():
    """Same weights and batch as test_port_equals_unmodified_reference, against the stored reference outputs."""
    g = np.load(os.path.join(GOLD, "crnn_ref_b3.npz"))
    with gzip.open(os.path.join(GOLD, "ref_state_keys.json.gz"), "rt") as f:
        names = json.load(f)["modules"]
    bb, dec = _port()
    assert [[k, list(v.shape)] for k, v in bb.state_dict().items()] == names["crnn_backbone"]
    assert [[k, list(v.shape)] for k, v in dec.state_dict().items()] == names["crnn_decoder"]
    torch.set_num_threads(1)
    x, labels, lengths = crnn_batch(3, 2, 100, 8, 26)
    tx, tl, tn = torch.from_numpy(x), torch.from_numpy(labels), torch.from_numpy(lengths)
    loss, pred = dec(bb.train()(tx), tl, tn, train=True)
    np.testing.assert_allclose(loss.detach().numpy(), g["loss"], rtol=1e-5)
    np.testing.assert_allclose(pred.detach().numpy(), g["pred"], rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(dec.eval()(bb.eval()(tx), train=False).detach().numpy(), g["eval_pred"], rtol=1e-4, atol=1e-5)


@pytest.mark.skipif(not ref_loader.available(), reason="reference tree not present (the stored outputs above are compared anywhere)")
def test_port_equals_unmodified_reference():
    ref_loader.install()
    import backbones as rb
    import decoders as rd
    rbb = fill_state_dict(rb.crnn_backbone(), "bb.")
    rdec = fill_state_dict(rd.CRNNDecoder(in_channels=512, inner_channels=256), "dec.")
    bb, dec = _port()
    assert list(bb.state_dict()) == list(rbb.state_dict()) and list(dec.state_dict()) == list(rdec.state_dict())
    x, labels, lengths = crnn_batch(3, 2, 100, 8, 26)
    tx, tl, tn = torch.from_numpy(x), torch.from_numpy(labels), torch.from_numpy(lengths)
    a = rdec(rbb.train()(tx), targets=tl, lengths=tn, train=True)
    b = dec(bb.train()(tx), tl, tn, train=True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    pa = rdec.eval()(rbb.eval()(tx), train=False)
    pb = dec.eval()(bb.eval()(tx), train=False)
    assert torch.equal(pa, pb)
