"""Regenerate reference_state_maps.json: the state-dict key -> shape maps of the reference's networks/ccnet.py Seg_Model
(num_classes=19, recurrence=2, built around this repository's cc_attention package with the inplace_abn stand-in) and of the
reference's own cc_attention CrissCrossAttention(512).  Run from the repository root with the reference checkout as the
argument:  python tests/golden/make_reference_maps.py <path to CCNet checkout>"""
import importlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main(ref):
    sys.path[:0] = [ROOT, os.path.join(ROOT, "harness", "shims"), ref]
    ccnet = importlib.import_module("networks.ccnet")
    with torch.device("meta"):
        seg = ccnet.Seg_Model(num_classes=19, recurrence=2)
    fn = importlib.machinery.SourceFileLoader("ref_functions", os.path.join(ref, "cc_attention", "functions.py")).load_module()
    cca = fn.CrissCrossAttention(512)
    out = {
        "seg_model": {k: list(v.shape) for k, v in seg.state_dict().items()},
        "seg_model_params": sum(p.numel() for p in seg.parameters()),
        "seg_model_recurrence": seg.recurrence,
        "criss_cross_attention_512": {k: list(v.shape) for k, v in cca.state_dict().items()},
    }
    with open(os.path.join(ROOT, "tests", "golden", "reference_state_maps.json"), "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)


if __name__ == "__main__":
    main(sys.argv[1])
