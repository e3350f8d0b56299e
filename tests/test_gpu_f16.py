"""GPU tests (H100: ``pytest -m gpu``) of float16 I/O: the f16 tensor-core kernels and the generic kernels' __half path against
the fp64 oracle at the fp16 budget of tests/f16_budget.py, under every launch knob, through torch.ops, and the drop-in module
under torch.autocast(float16) and model.half() against the reference module's own fp16 numerics.

Each comparison prints one ``ERR {json}`` line (run with ``-s`` to see the measured errors next to the budgets)."""
import json
import os
import subprocess
import sys

import pytest
import torch

import f16_budget as fb
import tc_budget as tb
from test_gpu_tc_edges import SWEEP, SWEEP_IDS, _inputs, _small

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H16 = torch.float16
KNOBS = ("CCA_B200_DELTA", "CCA_B200_LAG", "CCA_B200_PDL", "CCA_B200_L2HINT")


def _dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _run(q, k, v, dout, impl):
    """forward + backward (with delta) on the GPU; results on the CPU"""
    from ccnet_b200 import cca_backward, cca_forward
    dev = _dev()
    q, k, v, dout = (t.to(dev) for t in (q, k, v, dout))
    out, lse = cca_forward(q, k, v, impl=impl)
    dq, dk, dv, delta = cca_backward(dout, q, k, v, out, lse, impl=impl, want_delta=True)
    res = dict(out=out, lse=lse, dq=dq, dk=dk, dv=dv, delta=delta)
    return {n: (t.cpu() if t is not None else None) for n, t in res.items()}


def _check(got, ref, budget, what):
    errs = fb.check({n: t for n, t in got.items() if t is not None}, ref, budget, what)
    print("ERR", json.dumps(dict(what=what, err={n: float(f"{e:.2e}") for n, e in errs.items()},
                                 budget={n: budget[n] for n in errs})))
    return errs


# ---------------------------------------------------------------------------------------------------------------------
# 1. tensor-core (and generic) kernels against the oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [s for s, _ in SWEEP], ids=SWEEP_IDS)
def test_f16_edge_sweep_vs_oracle(shape):
    """forward, backward and delta in float16 at every shape of the tensor-core edge sweep (and on the generic kernels where the
    shape is small), against the fp64 oracle on the same f16 inputs.  Lines longer than 112 pixels run, as for bf16, on the
    fp32 kernels and are rounded to f16 once (ccnet_b200/functional.py); they are held to the same budget, except lse: the
    fp32 kernels form S with the bf16x3 split, whose error reaches lse directly (up to 4.8e-5 at these shapes on an H100,
    within the fp32 budget of tests/tc_budget.py, 8e-4), while the f16 kernels' S is exact up to fp32 accumulation."""
    from ccnet_b200.functional import tc_eligible
    assert tc_eligible(*shape, H16), shape
    q, k, v, dout = _inputs(shape, seed=sum(shape), scale=0.7, dtype=H16)
    ref = fb.reference(q, k, v, dout)
    got = _run(q, k, v, dout, "tc")
    assert got["out"].dtype == H16 and got["dq"].dtype == H16 and got["lse"].dtype == torch.float32
    assert got["out"].is_contiguous(memory_format=torch.channels_last)
    tiled = max(shape[3], shape[4]) > 112
    _check(got, ref, dict(fb.F16_BUDGET, lse=tb.FP32_BUDGET["lse"]) if tiled else fb.F16_BUDGET, f"{shape} f16 tc")
    if _small(shape):
        got = _run(q, k, v, dout, "simt")
        assert got.pop("delta") is None and got["out"].dtype == H16
        _check(got, ref, fb.F16_SIMT, f"{shape} f16 simt")


def test_f16_benchmark_shape_vs_oracle_on_samples():
    """B=8, C=512, 97x97 (the benchmark's attention step): the persistent schedule with its cross-CTA hand-offs, checked against
    the oracle on the first, a middle and the last sample."""
    shape = (8, 64, 512, 97, 97)
    q, k, v, dout = _inputs(shape, seed=1234, scale=0.7, dtype=H16)
    got = _run(q, k, v, dout, "tc")
    for b in (0, 3, 7):
        sl = slice(b, b + 1)
        ref = fb.reference(q[sl], k[sl], v[sl], dout[sl])
        _check({n: t[sl] for n, t in got.items()}, ref, fb.F16_BUDGET, f"{shape} f16 tc sample {b}")


def test_f16_long_lines_native_kernels_noise_floor(monkeypatch):
    """f16 I/O with lines longer than one tile on the native f16 kernels (what a C-ABI caller gets, and the Python entry points
    with CCA_B200_BF16_NATIVE=1): every element is the sum of up to 2*ceil(L/112) f16-rounded partials in no fixed order.
    Measured on an H100 80GB HBM3 (700 W) at 1x32x128x113x200 (two tiles per line): out 8.4e-4, lse 4.1e-6, dq 8.4e-4, dk 8.7e-4,
    dv 6.0e-4, delta 3.8e-4 -- inside the one-tile budget.  Held to twice that budget as its noise floor (at most 6e-3, below
    the bf16 budget of 1e-2)."""
    monkeypatch.setenv("CCA_B200_BF16_NATIVE", "1")
    shape = (1, 32, 128, 113, 200)
    q, k, v, dout = _inputs(shape, seed=41 + sum(shape), scale=0.7, dtype=H16)
    floor = {n: 2 * b for n, b in fb.F16_BUDGET.items()}
    assert max(floor.values()) <= 1e-2
    _check(_run(q, k, v, dout, "tc"), fb.reference(q, k, v, dout), floor, f"{shape} f16 native")


# ---------------------------------------------------------------------------------------------------------------------
# 2. launch knobs (read from the environment once per process: one child process per setting)
# ---------------------------------------------------------------------------------------------------------------------
ONE_TILE = (2, 64, 512, 97, 97)
KNOB_SETTINGS = [
    {}, {"CCA_B200_DELTA": "0"}, {"CCA_B200_LAG": "0"}, {"CCA_B200_PDL": "0"}, {"CCA_B200_L2HINT": "0"}, {"CCA_B200_L2HINT": "2"},
]


def _knob_child(path):
    """(child process) f16 tensor-core forward + backward + delta at ONE_TILE -> torch.save(path)"""
    torch.save(_run(*_inputs(ONE_TILE, seed=sum(ONE_TILE), scale=0.7, dtype=H16), "tc"), path)


def test_f16_launch_knobs_are_bit_identical(tmp_path):
    """With one tile per line every f16 output element is one store plus one f16 reduce-add, whatever the knobs change about
    when and where the bytes move: the results are bit-identical, and the defaults are within the budget."""
    _dev()
    res = []
    for setting in KNOB_SETTINGS:
        path = tmp_path / f"knobs_{len(res)}.pt"
        env = {k: v for k, v in os.environ.items() if k not in KNOBS}
        env.update(setting)
        env["PYTHONPATH"] = os.pathsep.join([ROOT, os.path.join(ROOT, "tests")] + ([env["PYTHONPATH"]] if "PYTHONPATH" in env else []))
        cmd = [sys.executable] + ["-s"] * sys.flags.no_user_site + ["-c", "import sys, test_gpu_f16 as t; t._knob_child(sys.argv[1])",
                                                                    str(path)]
        r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, (setting, r.stdout[-2000:], r.stderr[-4000:])
        res.append(torch.load(path))
    _check(res[0], fb.reference(*_inputs(ONE_TILE, seed=sum(ONE_TILE), scale=0.7, dtype=H16)), fb.F16_BUDGET, "f16 default knobs")
    for setting, got in zip(KNOB_SETTINGS[1:], res[1:]):
        for n in fb.TENSORS:
            assert torch.equal(got[n], res[0][n]), (setting, n)


# ---------------------------------------------------------------------------------------------------------------------
# 3. the module under fp16 autocast and model.half(), against the reference module's own fp16 numerics
# ---------------------------------------------------------------------------------------------------------------------
PARAMS = ("gamma", "query_conv.weight", "query_conv.bias", "key_conv.weight", "key_conv.bias", "value_conv.weight",
          "value_conv.bias")


def _module_run(m, x, g, mode):
    """R = 2 forward + backward of `m` on x (CPU fp32 tensors), in fp32 / under fp16 autocast / in half; (y, x.grad, {param: grad})
    on the CPU as fp64"""
    dev = next(m.parameters()).device
    m.zero_grad(set_to_none=True)
    xd = x.to(dev, torch.float16 if mode == "half" else x.dtype).requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.float16, enabled=mode == "autocast"):
        y = m(m(xd))
    (y.to(g.dtype) * g.to(dev)).sum().backward()
    grads = {n: p.grad.detach().cpu().double() for n, p in m.named_parameters()}
    return y.detach().cpu().double(), xd.grad.cpu().double(), grads


def _rel(got, ref, scale=0.0):
    return (got - ref).abs().max().item() / max(1.0, ref.abs().max().item(), scale)


@pytest.mark.parametrize("mode", ["autocast", "half"])
@pytest.mark.parametrize("C", [512, 64], ids=["C512-tc", "C64-generic"])
def test_module_fp16_vs_reference_fp16_numerics(C, mode):
    """RCCA R = 2 under torch.autocast(float16) (the projections run in fp16, the attention on the f16 kernels, the residual in
    fp32) and after model.half(): y, x.grad and all seven parameter gradients against the fp64 oracle module.  Each error is
    at most max(2x the error of the oracle module run the same way on the GPU, the fp16 budget)."""
    import cc_attention
    from oracle import cca_oracle as O
    dev = _dev()
    torch.manual_seed(5 + C)
    B, H, W = 2, 24, 40
    ref = O.CrissCrossAttentionOracle(C)
    with torch.no_grad():
        ref.gamma.fill_(0.7)
    x = torch.randn(B, C, H, W)
    g = torch.randn(B, C, H, W)
    r64 = O.CrissCrossAttentionOracle(C).double()
    r64.load_state_dict(ref.state_dict())
    ref64 = _module_run(r64, x.double(), g.double(), "fp32")
    ours = cc_attention.CrissCrossAttention(C).to(dev)
    ours.load_state_dict(ref.state_dict())
    amp_ref = O.CrissCrossAttentionOracle(C).to(dev)
    amp_ref.load_state_dict(ref.state_dict())
    if mode == "half":
        ours, amp_ref = ours.half(), amp_ref.half()
    got = _module_run(ours, x, g, mode)
    base = _module_run(amp_ref, x, g, mode)
    names = ["y", "x.grad"] + list(PARAMS)
    flat = lambda r: [r[0], r[1]] + [r[2][n] for n in PARAMS]
    errs = {}
    for n, a, b, r in zip(names, flat(got), flat(base), flat(ref64)):
        # a bias gradient is a sum over every pixel: measured against its weight's gradient, as in test_gpu_parity.py
        scale = ref64[2][n.replace(".bias", ".weight")].abs().max().item() if n.endswith(".bias") else 0.0
        e, eb = _rel(a, r, scale), _rel(b, r, scale)
        bound = max(2 * eb, fb.F16_BUDGET["out"] if n == "y" else fb.F16_BUDGET["dq"])
        errs[n] = (float(f"{e:.2e}"), float(f"{eb:.2e}"))
        assert torch.isfinite(a).all() and e <= bound, (C, mode, n, e, eb)
    print("ERR", json.dumps(dict(what=f"module C={C} {mode}", err_ours_vs_reference_amp=errs)))


def test_grad_scaler_step_and_inf_propagation():
    """One GradScaler step under fp16 autocast at C = 512: finite gradients at the default scale, no skipped step.  And an inf in
    dout makes dq, dk, dv non-finite -- what the scaler's inf check relies on to skip a step."""
    import cc_attention
    from ccnet_b200 import cca_backward, cca_forward
    dev = _dev()
    torch.manual_seed(11)
    m = cc_attention.CrissCrossAttention(512).to(dev)
    with torch.no_grad():
        m.gamma.fill_(0.5)
    opt = torch.optim.SGD(m.parameters(), lr=1e-3)
    scaler = torch.amp.GradScaler("cuda")
    x = torch.randn(2, 512, 24, 40, device=dev)
    with torch.autocast("cuda", dtype=torch.float16):
        loss = m(m(x)).float().square().mean()
    scaler.scale(loss).backward()
    scaler.unscale_(opt)
    for n, p in m.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), n
    scale0 = scaler.get_scale()
    scaler.step(opt)
    scaler.update()
    assert scaler.get_scale() == scale0                         # no inf found: the step ran, the scale did not back off

    q, k, v, dout = (t.to(dev) for t in _inputs((1, 64, 512, 20, 30), seed=2, scale=0.7, dtype=H16))
    out, lse = cca_forward(q, k, v, impl="tc")
    dout[0, 3, 5, 7] = float("inf")
    for g in cca_backward(dout, q, k, v, out, lse, impl="tc"):
        assert not torch.isfinite(g).all()


# ---------------------------------------------------------------------------------------------------------------------
# 4. torch.ops
# ---------------------------------------------------------------------------------------------------------------------
def test_torch_ops_f16_match_the_functional_path():
    """torch.ops.cca.forward / backward in float16 are bit-equal to ccnet_b200.functional (and channels-last on the tensor-core
    path, as their fake implementations say); opcheck validates the registration on real f16 tensors."""
    from ccnet_b200 import cca_backward, cca_forward
    dev = _dev()
    q, k, v, do = (t.to(dev) for t in _inputs((2, 64, 512, 20, 30), seed=4, scale=0.7, dtype=H16))
    out, lse = torch.ops.cca.forward(q, k, v)
    ro, rl = cca_forward(q, k, v)
    assert torch.equal(out, ro) and torch.equal(lse, rl) and out.dtype == H16
    assert out.is_contiguous(memory_format=torch.channels_last)
    dq, dk, dv = torch.ops.cca.backward(do, q, k, v, out, lse)
    rq, rk, rv = cca_backward(do, q, k, v, ro, rl)
    assert torch.equal(dq, rq) and torch.equal(dk, rk) and torch.equal(dv, rv)
    qg, kg, vg = (t.clone().requires_grad_(True) for t in (q, k, v))
    o2, _ = torch.ops.cca.forward(qg, kg, vg)
    o2.backward(do)
    assert torch.equal(qg.grad, rq) and torch.equal(kg.grad, rk) and torch.equal(vg.grad, rv)
    torch.library.opcheck(torch.ops.cca.forward.default, (q, k, v), test_utils=("test_schema", "test_faketensor"))
    torch.library.opcheck(torch.ops.cca.backward.default, (do, q, k, v, out, lse), test_utils=("test_schema", "test_faketensor"))
