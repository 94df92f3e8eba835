"""CPU, where the reference tree is present: the reference's three recognition yamls build UNCHANGED on megreader_b200's surfaces.

The reference's own structure/model.py (BasicModel :16-24, SequenceRecognitionModel :160-181) and concern/charsets.py are imported
from the reference tree; `getattr(backbones, name)` / `getattr(decoders, name)` (structure/model.py:20-21) then resolve to
megreader_b200/refapi.  The state dict (names and shapes: what checkpoints hold) must equal the one the reference's own modules
produce for the same yaml.  What it exercises is the reference's own builder and yaml files, so it is skipped where the
reference tree is absent; the per-module state dicts are compared anywhere by tests/test_surfaces_cpu.py."""
import json
import os
import subprocess
import sys

import pytest

from oracle import ref_loader

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _probe(mode):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "boundary_probe.py"), mode], capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.skipif(not ref_loader.available(), reason="reference tree not present")
def test_reference_yamls_build_on_refapi_with_identical_state_dicts():
    ours, ref = _probe("refapi"), _probe("reference")
    assert "refapi" in ours["backbones_file"] and "refapi" in ours["decoders_file"]
    assert ref["backbones_file"].startswith(ref_loader.REF)
    assert set(ours["models"]) == {"crnn.yaml", "res50-ppm-2d-ctc.yaml", "fpn50-attention-decoder.yaml"}
    for y, m in ours["models"].items():
        r = ref["models"][y]
        assert (m["model"], m["backbone"], m["decoder"]) == (r["model"], r["backbone"], r["decoder"])
        assert m["n_params"] == r["n_params"], y
        assert m["state"] == r["state"], (y, sorted(set(m["state"]) ^ set(r["state"]))[:10])
