"""GPU tests (H100: ``pytest -m gpu``) of the deterministic mode (torch.use_deterministic_algorithms / CCA_FLAG_DETERMINISTIC).

On tiled lines (longer than 112 pixels) the default kernels reduce-add an output element's shares in no fixed order; the planes
mode stores every share into its own partial plane and adds the planes in a fixed order.  Checked here: the same bits from
call to call, under every launch knob (one child process per setting, as in test_gpu_tc_edges.py), whatever the batch and
however it is split into sample groups; accuracy at the budgets of the default kernels; no read of unwritten memory (torch's
deterministic mode fills torch.empty with NaN, and the library's workspaces, which it allocates unfilled, are filled with 0xFF
bytes here); the deterministic weight gradient against fp64; and the module step with its weight gradients, fp32 and under
fp16 autocast, reproducible and close to the default mode."""
import contextlib
import os
import subprocess
import sys

import pytest
import torch

import f16_budget as fb
import tc_budget as tb

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32, BF, F16 = torch.float32, torch.bfloat16, torch.float16
TILED = [(2, 32, 128, 113, 200), (1, 16, 64, 7, 225), (1, 64, 128, 129, 257)]
# 16-bit I/O on tiled lines runs on the fp32 kernels and rounds once (ccnet_b200.functional._upcast)
BUDGET = {F32: tb.FP32_BUDGET, BF: {n: 1e-2 for n in tb.TENSORS},
          F16: {n: max(fb.F16_BUDGET[n], tb.FP32_BUDGET[n]) for n in tb.TENSORS}}
KNOBS = ("CCA_B200_DELTA", "CCA_B200_LAG", "CCA_B200_PDL", "CCA_B200_L2HINT", "CCA_B200_BF16_NATIVE", "CUBLAS_WORKSPACE_CONFIG")


def _inputs(shape, dtype, seed=0):
    B, Cq, C, H, W = shape
    g = torch.Generator().manual_seed(seed + sum(shape))
    q, k = (torch.randn(B, Cq, H, W, generator=g) * 0.7 for _ in range(2))
    v, dout = (torch.randn(B, C, H, W, generator=g) for _ in range(2))
    return tuple(t.to(dtype) for t in (q, k, v, dout))


def _run(q, k, v, dout, deterministic=None):
    """forward + backward (with delta) of the tensor-core kernels on the GPU; results on the CPU"""
    from ccnet_b200 import cca_backward, cca_forward
    q, k, v, dout = (t.cuda() for t in (q, k, v, dout))
    out, lse = cca_forward(q, k, v, impl="tc", deterministic=deterministic)
    dq, dk, dv, delta = cca_backward(dout, q, k, v, out, lse, impl="tc", want_delta=True, deterministic=deterministic)
    return {n: t.cpu() for n, t in dict(out=out, lse=lse, dq=dq, dk=dk, dv=dv, delta=delta).items()}


def _same(a, b, what):
    for n in a:
        assert a[n].dtype == b[n].dtype and a[n].shape == b[n].shape, (what, n)
        assert torch.equal(a[n].contiguous().view(torch.uint8), b[n].contiguous().view(torch.uint8)), f"{what}: {n} differs"


class _DeterministicAlgorithms:
    def __enter__(self):
        self.prev = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(True)

    def __exit__(self, *exc):
        torch.use_deterministic_algorithms(self.prev)


@contextlib.contextmanager
def _poisoned_workspaces():
    """the library's scratch buffers start as 0xFF bytes (NaN as fp32): a read of a byte no kernel wrote shows up as a NaN"""
    from ccnet_b200 import functional as F_
    alloc = F_._workspace
    F_._workspace = lambda nbytes, device: torch.full((max(nbytes, 16),), 255, dtype=torch.uint8, device=device)
    try:
        yield
    finally:
        F_._workspace = alloc


def _all_tiled():
    # deterministic=None follows the flag; torch.empty -> NaN
    with _DeterministicAlgorithms(), _poisoned_workspaces():
        return {(s, str(dt)): _run(*_inputs(s, dt)) for s in TILED for dt in (F32, BF, F16)}


def _knob_child(path):
    torch.save(_all_tiled(), path)


def _module_child(path):
    """(child process) two fwd + bwd steps of the module under fp16 autocast at a tiled shape"""
    torch.save([_module_step((1, 512, 64, 128), autocast=True) for _ in range(2)], path)


def _spawn(tmp_path, fn, setting, name):
    path = tmp_path / f"{name}.pt"
    env = {k: v for k, v in os.environ.items() if k not in KNOBS}
    env.update(setting)
    env["PYTHONPATH"] = os.pathsep.join([ROOT, os.path.join(ROOT, "tests")] + ([env["PYTHONPATH"]] if "PYTHONPATH" in env else []))
    cmd = [sys.executable] + ["-s"] * sys.flags.no_user_site + [
        "-c", f"import sys, test_gpu_deterministic as t; t.{fn}(sys.argv[1])", str(path)]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return torch.load(path)


def test_tiled_lines_are_reproducible_accurate_and_knob_independent(tmp_path):
    first, second = _all_tiled(), _all_tiled()
    for key, got in first.items():
        shape, dt = key
        _same(got, second[key], f"{key} second call")
        for n, t in got.items():
            assert not torch.isnan(t).any(), f"{key}: NaN in {n}"
        q, k, v, dout = _inputs(shape, {"torch.float32": F32, "torch.bfloat16": BF, "torch.float16": F16}[dt])
        tb.check(got, tb.reference(q, k, v, dout), BUDGET[got["out"].dtype], f"{key} deterministic")
    # knobs of the launch (read once per process) and the native 16-bit switch change nothing in this mode
    for setting in ({"CCA_B200_LAG": "0"}, {"CCA_B200_LAG": "1", "CCA_B200_PDL": "0"}, {"CCA_B200_L2HINT": "0"},
                    {"CCA_B200_L2HINT": "2", "CCA_B200_DELTA": "0"}, {"CCA_B200_BF16_NATIVE": "1"}):
        name = "_".join(f"{k[9:]}{v}" for k, v in sorted(setting.items()))
        other = _spawn(tmp_path, "_knob_child", setting, name)
        for key, got in first.items():
            _same(got, other[key], f"{key} {setting}")


def test_batch_and_sample_groups_do_not_change_the_bits():
    from ccnet_b200 import functional as F_
    shape = (4, 32, 128, 113, 200)
    q, k, v, dout = _inputs(shape, F32)
    with _poisoned_workspaces():
        whole = _run(q, k, v, dout, deterministic=True)
    assert not any(torch.isnan(t).any() for t in whole.values())
    for b in range(4):
        one = _run(q[b:b + 1], k[b:b + 1], v[b:b + 1], dout[b:b + 1], deterministic=True)
        _same({n: t[b:b + 1] for n, t in whole.items()}, one, f"sample {b} alone")
    cap = F_.deterministic_workspace_cap
    try:
        F_.deterministic_workspace_cap = 100 << 20      # groups of 1 (backward) / 2 (forward) samples at this shape
        _same(whole, _run(q, k, v, dout, deterministic=True), "split into sample groups")
    finally:
        F_.deterministic_workspace_cap = cap


def test_one_tile_shapes_give_the_default_bits():
    for dt in (F32, BF, F16):
        args = _inputs((2, 64, 256, 97, 97), dt)
        _same(_run(*args, deterministic=True), _run(*args, deterministic=False), f"one tile {dt}")


def test_c_abi_refuses_16_bit_tiled_deterministic():
    from ccnet_b200 import capi
    lib = capi.load()
    B, Cq, C, H, W = 1, 16, 64, 7, 225
    for dt, cdt in ((BF, capi.CCA_BF16), (F16, capi.CCA_F16)):
        q = torch.zeros(B, H, W, Cq, dtype=dt, device="cuda")
        v = torch.zeros(B, H, W, C, dtype=dt, device="cuda")
        out, lse = torch.empty_like(v), torch.empty(B, H, W, device="cuda")
        flags = capi.CCA_FLAG_NHWC | capi.CCA_FLAG_DETERMINISTIC
        nws = lib.cca_b200_workspace_bytes_ex(capi.CCA_WS_FORWARD, B, Cq, C, H, W, cdt, flags)
        ws = torch.empty(nws, dtype=torch.uint8, device="cuda")
        rc = lib.cca_b200_forward(q.data_ptr(), q.data_ptr(), v.data_ptr(), out.data_ptr(), lse.data_ptr(), ws.data_ptr(), nws,
                                  B, Cq, C, H, W, cdt, flags, None)
        assert rc == -2 and b"CCA_F32" in lib.cca_b200_last_error()
        rc = lib.cca_b200_backward(v.data_ptr(), q.data_ptr(), q.data_ptr(), v.data_ptr(), v.data_ptr(), lse.data_ptr(),
                                   q.data_ptr(), q.data_ptr(), out.data_ptr(), ws.data_ptr(), nws, B, Cq, C, H, W, cdt, flags, None)
        assert rc == -2 and b"CCA_F32" in lib.cca_b200_last_error()
        torch.cuda.synchronize()


def _module_step(shape, autocast=False, deterministic=True):
    """y, x.grad and the 7 parameter gradients of one fwd + bwd step of a seeded module, under the deterministic flag (or not)"""
    from ccnet_b200 import CrissCrossAttention
    B, C, H, W = shape
    torch.manual_seed(0)
    m = CrissCrossAttention(C).cuda()
    with torch.no_grad():
        m.gamma.fill_(0.5)
    x = torch.randn(B, C, H, W, device="cuda").contiguous(memory_format=torch.channels_last).requires_grad_(True)
    dy = torch.randn(B, C, H, W, device="cuda")
    with _DeterministicAlgorithms() if deterministic else contextlib.nullcontext():
        with torch.autocast("cuda", dtype=torch.float16, enabled=autocast):
            y = m(x)
        y.backward(dy.to(y.dtype))
    grads = {n: p.grad.cpu() for n, p in m.named_parameters()}
    assert len(grads) == 7
    return dict(y=y.detach().cpu(), dx=x.grad.cpu(), **grads)


@pytest.mark.parametrize("shape", [(2, 512, 97, 97), (1, 512, 64, 128)], ids=["97x97", "64x128"])
def test_fused_module_step_is_reproducible_and_matches_the_default_mode(shape):
    """two steps under the flag give the same bits; y, x.grad and the 7 parameter gradients (the ordered weight-gradient
    sum included) agree with the default mode's to fp32 accuracy.  A bias gradient is a sum over every pixel of a gradient
    whose terms mostly cancel, so its error is measured against the scale of its conv's weight gradient (a sum of the same
    terms times x), as test_gpu_parity.py's weight-gradient check does."""
    a, b = _module_step(shape), _module_step(shape)
    for n, t in a.items():
        assert not torch.isnan(t).any(), n
    _same(a, b, f"module {shape}")
    ref = _module_step(shape, deterministic=False)
    for n, t in a.items():
        err = (t.double() - ref[n].double()).abs().max().item()
        scale = max(1.0, ref[n].abs().max().item())
        if n.endswith(".bias"):
            scale = max(scale, ref[n[:-len("bias")] + "weight"].abs().max().item())
        print(f"ERR module {shape} {n}: {err:.2e} (scale {scale:.2e})")
        assert err <= 1e-4 * scale, (n, err, scale)


@pytest.mark.parametrize("shape", [(1, 512, 97, 97), (3, 512, 20, 31), (1, 512, 1, 5)])
def test_deterministic_weight_gradient_vs_fp64(shape):
    """qkv_project_wgrad's deterministic variant (per-split partials summed in split order) against fp64, at the budget of
    test_gpu_parity.py's default-kernel check: many splits (97x97), a few, and 5 pixels (all but one split without pixels,
    which must still write zero partials).  Under the torch flag with deterministic=None, workspace poisoned."""
    from ccnet_b200.functional import qkv_project_wgrad
    B, C, H, W = shape
    g = torch.Generator().manual_seed(11)
    x = torch.randn(B, C, H, W, generator=g)
    gs = [torch.randn(B, c, H, W, generator=g) for c in (C // 8, C // 8, C)]
    dev = lambda t: t.cuda().contiguous(memory_format=torch.channels_last)
    scale = torch.tensor([0.75], device="cuda")
    with _DeterministicAlgorithms(), _poisoned_workspaces():
        outs = qkv_project_wgrad(dev(x), *(dev(t) for t in gs), scale=scale)
        again = qkv_project_wgrad(dev(x), *(dev(t) for t in gs), scale=scale)
    xm = x.double().permute(0, 2, 3, 1).reshape(-1, C)
    for i, gt in enumerate(gs):
        gm = gt.double().permute(0, 2, 3, 1).reshape(-1, gt.shape[1])
        rw, rb = 0.75 * (gm.t() @ xm), 0.75 * gm.sum(0)
        ew = (outs[2 * i].cpu().double() - rw).abs().max().item()
        eb = (outs[2 * i + 1].cpu().double() - rb).abs().max().item()
        assert ew <= 1e-4 * max(1.0, rw.abs().max().item()), (i, ew)
        assert eb <= 1e-4 * max(1.0, rb.abs().max().item(), rw.abs().max().item()), (i, eb)
    _same({str(i): t.cpu() for i, t in enumerate(outs)}, {str(i): t.cpu() for i, t in enumerate(again)}, f"wgrad {shape}")


def test_module_under_fp16_autocast_is_reproducible(tmp_path):
    a, b = _spawn(tmp_path, "_module_child", {"CUBLAS_WORKSPACE_CONFIG": ":4096:8"}, "autocast")
    _same(a, b, "module under fp16 autocast")
