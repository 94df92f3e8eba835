"""Helper of tests/test_seg_detector_cpu.py (run as a subprocess): build the model of the reference's
experiments/seg_detector/seg_detector_db.yaml with the reference's OWN structure/model.py::SegDetectorModel, with `backbones` /
`decoders` / `ops` / `assets` resolved either to the reference (mode "reference") or to megreader_b200/refapi (mode "refapi").
The backbone is built with pretrained=False (its default downloads a checkpoint).  Prints one JSON object."""
import json
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
mode = sys.argv[1]
from oracle import ref_loader  # noqa: E402

assert ref_loader.install()
REF = ref_loader.REF
if mode == "refapi":
    import megreader_b200
    sys.path.insert(0, os.path.join(os.path.dirname(megreader_b200.__file__), "refapi"))
else:
    # the reference's native extensions are not built for CPU: their import sites only need the module objects
    for name in ("ops.ctc_2d.ctc_2d_csrc", "assets.ops.dcn.deform_conv_cuda", "assets.ops.dcn.deform_pool_cuda"):
        sys.modules[name] = types.ModuleType(name)
import torch  # noqa: E402
import yaml  # noqa: E402
import backbones  # noqa: E402
import decoders  # noqa: E402
import structure.model as smodel  # noqa: E402  (always the reference's file)

assert smodel.__file__.startswith(REF)
conf = yaml.safe_load(open(os.path.join(REF, "experiments/seg_detector/seg_detector_db.yaml")))
exp = [d for d in conf["define"] if d["name"] == "Experiment"][0]
builder = exp["structure"]["builder"]
args = json.loads(json.dumps(builder["model_args"]))
args.setdefault("backbone_args", {})["pretrained"] = False
model = getattr(smodel, builder["model"])(args, torch.device("cpu"))
print(json.dumps({"backbones_file": backbones.__file__, "decoders_file": decoders.__file__, "model": builder["model"],
                  "backbone": args["backbone"], "decoder": args["decoder"], "loss_class": args["loss_class"],
                  "criterion": type(model.criterion.module).__module__ + "." + type(model.criterion.module).__name__,
                  "state": [[k, list(v.shape)] for k, v in model.state_dict().items()],
                  "n_params": sum(p.numel() for p in model.parameters())}))
