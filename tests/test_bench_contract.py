"""The bench.py JSON contract, checked on the committed H100 bench lines (profiles/) and on the projection autograd node of
the module (CPU, fp64) -- no GPU needed."""
import glob
import json
import os

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALL = sorted(glob.glob(os.path.join(ROOT, "profiles", "h100_bench_line*.json")))
LINES = [p for p in ALL if "reference_arm" not in p]
REF_LINES = [p for p in ALL if "reference_arm" in p]

REQUIRED = ["metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
            "vs_baseline", "dtype", "data", "config", "clocks", "e2e", "gpu_launches", "roofline", "cpu_baseline"]


@pytest.mark.parametrize("path", LINES, ids=[os.path.basename(p) for p in LINES])
def test_committed_bench_line_has_the_contract_fields(path):
    d = json.load(open(path))
    for key in REQUIRED:
        assert key in d, key
    assert d["metric"] == "cca_fwd_bwd_pixels_per_s" and d["unit"] == "pixels/s" and d["higher_is_better"] is True
    assert d["scaling"] == "weak" and d["vs_baseline"] is None and d["data"] == "synthetic" and d["dtype"] == "f32"
    assert "workload" in d["config"] and "model" not in d["config"]
    px = 8 * 97 * 97 * d["n_gpus"]
    assert abs(d["value"] - px / (d["ms_per_step"] * 1e-3)) <= 1e-6 * d["value"]          # value is the whole-job aggregate
    r = d["roofline"]
    assert r["bound"] == "hbm" and r["unit"] == "GB/s" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert r["op_fwd"]["frac"] > 0 and r["op_bwd"]["frac"] > 0 and r["other_dtype"]["dtype"] == "bf16"
    assert "module" in d and 0 < d["module"]["ms_per_step"]
    if "error" not in (d.get("ccnet") or {"error": 1}):
        assert d["ccnet"]["train_images_per_s"] > 0 and d["ccnet"]["per_gpu_batch"] * d["n_gpus"] == 8
    e = d["e2e"]
    assert e["h2d_bytes_per_step"] == 8 * 512 * 97 * 97 * 4 and e["d2h_bytes_per_step"] == 2 * e["h2d_bytes_per_step"]
    assert e["value"] < d["value"]                          # host copies + the module's projections are inside e2e
    assert d["gpu_launches"] > 0
    c = d["clocks"]
    assert not set(c["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    if d["n_gpus"] == 1 and d["cpu_baseline"] is not None:
        b = d["cpu_baseline"]
        assert b["kind"] in ("port", "reference") and b["cores"] >= 1 and b["value"] > 0 and b["sample"]


@pytest.mark.parametrize("path", REF_LINES, ids=[os.path.basename(p) for p in REF_LINES])
def test_committed_reference_arm_line(path):
    """`bench.py --impl reference`: same metric / unit / config as our arm, the CPU reference timed on the host cores."""
    d = json.load(open(path))
    ours = json.load(open(LINES[0]))
    assert d["impl"] == "reference" and d["metric"] == ours["metric"] and d["unit"] == ours["unit"]
    assert d["higher_is_better"] is True and d["config"]["workload"] == ours["config"]["workload"]
    b = d["cpu_baseline"]
    assert b["kind"] in ("port", "reference") and b["cores"] >= 1 and b["sample"] and b["value"] == d["value"]
    e = d["e2e"]
    assert e["value"] == d["value"] and e["h2d_bytes_per_step"] == 0 and e["d2h_bytes_per_step"] == 0
    assert d["value"] < 1e-2 * ours["value"]                # the point of the exercise


def test_qkv_projection_node_matches_the_three_convs():
    """ccnet_b200.module._QKVProject (one autograd node, GEMMs on the [pixels, C] view) == the reference's three
    nn.Conv2d 1x1 projections (functions.py:29,32,35), values and all gradients, in fp64 on the CPU."""
    from ccnet_b200.module import _QKVProject
    torch.manual_seed(0)
    x = torch.randn(2, 64, 5, 7, dtype=torch.float64).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    convs = [torch.nn.Conv2d(64, o, 1).double() for o in (8, 8, 64)]
    args = [t for c in convs for t in (c.weight, c.bias)]
    outs = _QKVProject.apply(x, *args)
    gs = [torch.randn_like(t) for t in outs]
    sum((o * g).sum() for o, g in zip(outs, gs)).backward()
    got = [x.grad.clone()] + [p.grad.clone() for p in args]
    x.grad = None
    for c in convs:
        c.zero_grad()
    refs = [c(x) for c in convs]
    sum((o * g).sum() for o, g in zip(refs, gs)).backward()
    want = [x.grad] + [p.grad for p in args]
    for o, r in zip(outs, refs):
        assert o.shape == r.shape and o.is_contiguous(memory_format=torch.channels_last)
        assert (o - r).abs().max().item() <= 1e-12
    for a, b in zip(got, want):
        assert a.shape == b.shape and (a - b).abs().max().item() <= 1e-10
