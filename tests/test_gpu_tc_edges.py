"""GPU tests (H100: ``pytest -m gpu``): the wgmma kernels at the edges of their work decomposition and under every launch knob,
against the fp64 oracle at the bf16x3 error budget of tests/tc_budget.py.

cca_items.cuh cuts a line of L pixels into nt = ceil(L/112) tiles of tl = ceil(L/nt) pixels; the longest tile picks the LK = 80
or LK = 112 kernels, and the statistics pass leaves row.nt + col.nt partial log-sum-exp planes per pixel.  The sweep covers
each side of those cuts, up to nt = 8 per direction (16 planes), and the fp32 backward's 32-channel ring at C up to 2048.

Each comparison prints one ``ERR {json}`` line (run with ``-s`` to see the measured errors next to the budgets)."""
import json
import os
import subprocess
import sys

import pytest
import torch

import tc_budget as tb

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF16_TOL = 1e-2
BF16_BUDGET = {n: BF16_TOL for n in tb.TENSORS}
KNOBS = ("CCA_B200_DELTA", "CCA_B200_LAG", "CCA_B200_PDL", "CCA_B200_L2HINT")


def _dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _inputs(shape, seed, scale, dtype):
    """seeded CPU q, k, v, dout, rounded to dtype"""
    B, Cq, C, H, W = shape
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, Cq, H, W, generator=g) * scale
    k = torch.randn(B, Cq, H, W, generator=g) * scale
    v = torch.randn(B, C, H, W, generator=g)
    dout = torch.randn(B, C, H, W, generator=g)
    return tuple(t.to(dtype) for t in (q, k, v, dout))


def _run(q, k, v, dout, impl):
    """forward + backward (with delta) on the GPU; results on the CPU"""
    from ccnet_b200 import cca_backward, cca_forward
    dev = _dev()
    q, k, v, dout = (t.to(dev) for t in (q, k, v, dout))
    out, lse = cca_forward(q, k, v, impl=impl)
    dq, dk, dv, delta = cca_backward(dout, q, k, v, out, lse, impl=impl, want_delta=True)
    res = dict(out=out, lse=lse, dq=dq, dk=dk, dv=dv, delta=delta)
    return {n: (t.cpu() if t is not None else None) for n, t in res.items()}


def _budget(dtype, impl="tc", peaked=False):
    if dtype == torch.bfloat16:
        # the generic kernels' bf16 backward rounds P and dS to bf16 per line (held to 3x in test_gpu_parity.py too)
        return dict(BF16_BUDGET, dq=3 * BF16_TOL, dk=3 * BF16_TOL, dv=3 * BF16_TOL) if impl == "simt" else BF16_BUDGET
    if impl == "simt":
        return tb.FP32_SIMT
    return tb.FP32_PEAKED_BUDGET if peaked else tb.FP32_BUDGET


def _check(got, ref, budget, what):
    errs = tb.check({n: t for n, t in got.items() if t is not None}, ref, budget, what)
    print("ERR", json.dumps(dict(what=what, err={n: float(f"{e:.2e}") for n, e in errs.items()},
                                 budget={n: budget[n] for n in errs})))
    return errs


# ---------------------------------------------------------------------------------------------------------------------
# 1. edge sweep
# ---------------------------------------------------------------------------------------------------------------------
F32, BF = torch.float32, torch.bfloat16
SWEEP = [
    # (B, Cq, C, H, W), dtypes
    ((1, 16, 64, 80, 80), (F32, BF)),        # tl = 80: the longest LK = 80 tile, one per line
    ((1, 32, 128, 81, 9), (F32, BF)),        # the shortest line on LK = 112
    ((1, 48, 192, 112, 112), (F32, BF)),     # a full LK = 112 tile, Cq = 48
    ((2, 16, 64, 113, 3), (F32, BF)),        # the first tiled length: tiles of 57 + 56
    ((1, 64, 256, 160, 5), (F32, BF)),       # LK = 80, tiled: two full 80-pixel tiles
    ((1, 64, 256, 161, 5), (F32, BF)),       # LK = 112, tiled
    ((1, 16, 128, 7, 224), (F32, BF)),       # two full 112-pixel tiles
    ((1, 16, 128, 7, 225), (F32, BF)),       # three tiles
    ((1, 32, 64, 449, 6), (F32, BF)),        # nt = 5
    ((2, 16, 64, 896, 9), (F32, BF)),        # nt = 8 along columns
    ((1, 16, 64, 9, 896), (F32, BF)),        # nt = 8 along rows
    ((1, 16, 64, 896, 896), (F32,)),         # 16 partial lse planes (the fp64 oracle alone takes ~40 s)
    ((1, 64, 1024, 97, 97), (F32, BF)),      # long ring runs: 32 (fp32) / 16 (bf16) chunks per item
    ((1, 64, 2048, 33, 47), (F32, BF)),
    ((2, 16, 64, 97, 97), (BF,)),            # Cq = 16 at LK = 112 in bf16
]
SWEEP_IDS = ["x".join(map(str, s)) for s, _ in SWEEP]


def _small(shape):
    B, _, _, H, W = shape
    return B * H * W * (H + W) <= 4_000_000


@pytest.mark.parametrize("shape,dtypes", SWEEP, ids=SWEEP_IDS)
def test_edge_sweep_vs_oracle(shape, dtypes):
    """forward, backward and delta of the tensor-core kernels (and the generic kernels where the shape is small) against the
    fp64 oracle evaluated on the same (dtype-rounded) inputs.  bf16 with a line longer than 112 pixels is what a user of
    ccnet_b200.functional gets: the fp32 kernels on the bf16 values, rounded once.  So at the tiled shapes the bf16 half checks
    that path; the native bf16 kernels with more than one tile per line are only reached through the C ABI
    (test_gpu_parity.py::test_bf16_long_lines_native_kernels_noise_floor)."""
    from ccnet_b200.functional import tc_eligible
    for dt in dtypes:
        assert tc_eligible(shape[0], shape[1], shape[2], shape[3], shape[4], dt), (shape, dt)
        q, k, v, dout = _inputs(shape, seed=sum(shape), scale=0.7, dtype=dt)
        ref = tb.reference(q, k, v, dout)
        got = _run(q, k, v, dout, "tc")
        assert got["out"].dtype == dt and got["lse"].dtype == torch.float32 and got["delta"].dtype == torch.float32
        _check(got, ref, _budget(dt), f"{shape} {dt} tc")
        if _small(shape):
            got = _run(q, k, v, dout, "simt")
            assert got.pop("delta") is None
            _check(got, ref, _budget(dt, "simt"), f"{shape} {dt} simt")


# ---------------------------------------------------------------------------------------------------------------------
# 2. the boundary between the tensor-core kernels and the generic fallback
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,W", [(897, 3), (3, 897)])
def test_line_of_897_falls_back_to_the_generic_kernels(H, W):
    """Lines up to 896 pixels (8 tiles) are the tensor-core kernels'; longer ones go to the generic kernels, whose forward takes
    lines up to 1412 pixels and whose backward (two [L x 33] fp32 tiles in shared memory) lines up to 710.  So a line of 897 has a
    forward but no backward: that call must fail with an error, not fall back to anything else."""
    from ccnet_b200 import capi, cca_backward, cca_forward
    dev = _dev()
    lib = capi.load()
    for which in (capi.CCA_WS_FORWARD, capi.CCA_WS_BACKWARD):
        for dt in (capi.CCA_F32, capi.CCA_BF16):
            assert lib.cca_b200_tc_supported(which, 1, 16, 64, H, W, dt) == 0
            assert lib.cca_b200_tc_supported(which, 1, 16, 64, min(H, 896), min(W, 896), dt) == 1
    shape = (1, 16, 64, H, W)
    q, k, v, dout = _inputs(shape, seed=sum(shape), scale=0.7, dtype=torch.float32)
    qd, kd, vd, dd = (t.to(dev) for t in (q, k, v, dout))
    with pytest.raises(RuntimeError, match="do not cover"):
        cca_forward(qd, kd, vd, impl="tc")
    out, lse = cca_forward(qd, kd, vd, impl="auto")
    assert out.is_contiguous()                                    # the generic kernels ran (NCHW)
    from oracle import cca_oracle as O
    ro, rl = O.cca_forward(q.double(), k.double(), v.double())
    _check(dict(out=out, lse=lse), dict(out=ro, lse=rl), tb.FP32_SIMT, f"{shape} auto")
    with pytest.raises(RuntimeError, match="do not cover"):
        cca_backward(dd, qd, kd, vd, out, lse, impl="tc")
    with pytest.raises(RuntimeError, match="too large for the generic kernels"):
        cca_backward(dd, qd, kd, vd, out, lse, impl="auto")
    # 896 is still the tensor-core kernels' (nt = 8)
    shape = (1, 16, 64, min(H, 896), min(W, 896))
    q, k, v, dout = _inputs(shape, seed=sum(shape), scale=0.7, dtype=torch.float32)
    _check(_run(q, k, v, dout, "tc"), tb.reference(q, k, v, dout), tb.FP32_BUDGET, f"{shape} tc")


def test_generic_backward_line_limit():
    """Shapes the tensor-core kernels do not take (here Cq = 8) run on the generic kernels, whose backward holds two [L x 33]
    fp32 tiles of a line in shared memory: lines up to 710 pixels work, 711 fails with an error."""
    from ccnet_b200 import cca_backward, cca_forward
    dev = _dev()
    for L, ok in ((710, True), (711, False)):
        shape = (1, 8, 64, L, 3)
        q, k, v, dout = _inputs(shape, seed=sum(shape), scale=0.7, dtype=torch.float32)
        qd, kd, vd, dd = (t.to(dev) for t in (q, k, v, dout))
        out, lse = cca_forward(qd, kd, vd)
        if not ok:
            with pytest.raises(RuntimeError, match="too large for the generic kernels"):
                cca_backward(dd, qd, kd, vd, out, lse)
            continue
        dq, dk, dv = cca_backward(dd, qd, kd, vd, out, lse)
        _check(dict(out=out, lse=lse, dq=dq, dk=dk, dv=dv), tb.reference(q, k, v, dout), tb.FP32_SIMT, f"{shape} simt")


# ---------------------------------------------------------------------------------------------------------------------
# 3./4. launch knobs of release builds (read from the environment once per process: one child process per setting) and delta
# ---------------------------------------------------------------------------------------------------------------------
ONE_TILE = (2, 64, 512, 97, 97)
TILED = (1, 32, 128, 113, 200)
KNOB_SETTINGS = [
    {"CCA_B200_DELTA": "0"}, {"CCA_B200_LAG": "0"}, {"CCA_B200_PDL": "0"}, {"CCA_B200_L2HINT": "0"}, {"CCA_B200_L2HINT": "2"},
    {"CCA_B200_DELTA": "0", "CCA_B200_LAG": "0", "CCA_B200_PDL": "0"},
]


def _knob_child(path):
    """(child process) tensor-core forward + backward + delta at ONE_TILE and TILED in both dtypes -> torch.save(path)"""
    res = {}
    for shape in (ONE_TILE, TILED):
        for dt in (F32, BF):
            res[(shape, str(dt))] = _run(*_inputs(shape, seed=sum(shape), scale=0.7, dtype=dt), "tc")
    torch.save(res, path)


def _spawn(tmp_path, setting):
    path = tmp_path / ("knobs_" + "_".join(f"{k[9:]}{v}" for k, v in sorted(setting.items())) + ".pt")
    env = {k: v for k, v in os.environ.items() if k not in KNOBS}
    env.update(setting)
    env["PYTHONPATH"] = os.pathsep.join([ROOT, os.path.join(ROOT, "tests")] + ([env["PYTHONPATH"]] if "PYTHONPATH" in env else []))
    cmd = [sys.executable] + ["-s"] * sys.flags.no_user_site + ["-c", "import sys, test_gpu_tc_edges as t; t._knob_child(sys.argv[1])", str(path)]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (setting, r.stdout[-2000:], r.stderr[-4000:])
    return torch.load(path)


@pytest.fixture(scope="module")
def default_knobs(tmp_path_factory):
    _dev()
    return _spawn(tmp_path_factory.mktemp("default"), {})


@pytest.fixture(scope="module")
def knob_refs():
    out = {}
    for shape in (ONE_TILE, TILED):
        for dt in (F32, BF):
            out[(shape, str(dt))] = tb.reference(*_inputs(shape, seed=sum(shape), scale=0.7, dtype=dt))
    return out


def test_default_knobs_vs_oracle(default_knobs, knob_refs):
    for key, got in default_knobs.items():
        _check(got, knob_refs[key], _budget(torch.float32 if key[1] == str(F32) else torch.bfloat16), f"{key} default knobs")


@pytest.mark.parametrize("setting", KNOB_SETTINGS, ids=[",".join(f"{k[9:]}={v}" for k, v in s.items()) for s in KNOB_SETTINGS])
def test_launch_knob_in_release_build(tmp_path, setting, default_knobs, knob_refs):
    """The knobs only change when and where bytes move (and, DELTA=0, which items compute delta): with one tile per line every
    element is one store plus one add, so the results are bit-identical to the defaults; with tiled lines the adds onto an
    element come in another order (1e-5 relative).  bf16 with tiled lines runs on the fp32 kernels and rounds once
    (ccnet_b200/functional.py): an element of out, dq, dk, dv may then land on the neighbouring bf16 value, and delta, which the
    fp32 backward computes from dout and that bf16 out, moves by exactly sum_c |dout| |out - out_default| at most."""
    got = _spawn(tmp_path, setting)
    for (shape, dt), res in got.items():
        base = default_knobs[(shape, dt)]
        if shape == ONE_TILE:
            for n in tb.TENSORS:
                assert torch.equal(res[n], base[n]), (setting, shape, dt, n)
        else:
            bf = dt == str(BF)
            _check(res, knob_refs[(shape, dt)], _budget(BF if bf else F32), f"{(shape, dt)} {setting}")
            for n in ("lse",) if bf else tb.TENSORS:
                assert tb.error(n, res[n], base[n].double()) <= 1e-5, (setting, shape, dt, n)
            if bf:
                slack = {n: 1e-5 * max(1.0, base[n].abs().max().item()) for n in tb.TENSORS}     # the fp32 reordering
                for n in ("out", "dq", "dk", "dv"):
                    a, b = res[n].double(), base[n].double()
                    assert ((a - b).abs() <= 2.0 ** -7 * torch.maximum(a.abs(), b.abs()) + slack[n]).all(), (setting, n)
                dout = _inputs(shape, seed=sum(shape), scale=0.7, dtype=BF)[3].double()
                bound = (dout.abs() * (res["out"].double() - base["out"].double()).abs()).sum(1) + slack["delta"]
                assert ((res["delta"].double() - base["delta"].double()).abs() <= bound).all(), setting


# ---------------------------------------------------------------------------------------------------------------------
# 5. peaked softmax, backward included
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F32, BF], ids=["fp32", "bf16"])
@pytest.mark.parametrize("shape", [(1, 64, 128, 97, 97), (1, 32, 128, 193, 193)], ids=["1x64x128x97x97", "1x32x128x193x193"])
def test_peaked_softmax_forward_backward(shape, dt):
    """q, k ~ N(0, 1.5^2): logits of std up to ~18, near one-hot attention rows"""
    q, k, v, dout = _inputs(shape, seed=77 + sum(shape), scale=1.5, dtype=dt)
    _check(_run(q, k, v, dout, "tc"), tb.reference(q, k, v, dout), _budget(dt, peaked=True), f"{shape} {dt} peaked")
