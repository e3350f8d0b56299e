"""GPU parity tests (H100: ``pytest -m gpu``).  Every call goes through the C ABI
(ccnet_b200.functional -> ctypes -> libcca_b200.so); the oracle is only the checker.

Tolerances (BASELINE.json north_star): fp32 max-abs <= 1e-3 on identical Q/K/V; bf16 <= 1e-2
against the fp32 oracle evaluated on the bf16-rounded Q/K/V (SURVEY.md 8c)."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

FP32_TOL = 1e-3
BF16_TOL = 1e-2

IMPLS = ["simt", "auto"]


def _dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _oracle():
    from oracle import cca_oracle
    return cca_oracle


def _rand_qkv(B, Cq, C, H, W, seed, scale=1.0, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    q = (torch.randn(B, Cq, H, W, generator=g) * scale).to(dtype)
    k = (torch.randn(B, Cq, H, W, generator=g) * scale).to(dtype)
    v = torch.randn(B, C, H, W, generator=g).to(dtype)
    return q, k, v


@pytest.mark.parametrize("impl", IMPLS)
def test_forward_vs_golden_reference_outputs(golden, impl):
    """Identical Q/K/V as the reference module produced; compare with the reference's own O."""
    from ccnet_b200 import cca_forward
    dev = _dev()
    q, k, v = (torch.from_numpy(golden[n]).to(dev) for n in "qkv")
    out, lse = cca_forward(q, k, v, impl=impl)
    ref = torch.from_numpy(golden["o64"]).to(dev)
    assert torch.isfinite(out).all() and torch.isfinite(lse).all()
    err = (out.double() - ref).abs().max().item()
    assert err <= FP32_TOL, (golden["name"], err)
    assert err <= 1e-4 * max(1.0, ref.abs().max().item()), (golden["name"], err)   # SIMT / 3xbf16 are ~fp32 exact


SHAPES = [
    # B, Cq, C, H, W
    (2, 8, 64, 5, 6), (1, 8, 64, 32, 32), (2, 4, 32, 9, 7), (1, 2, 16, 1, 11), (1, 2, 16, 13, 1),
    (1, 1, 8, 1, 1), (1, 16, 128, 17, 33), (1, 64, 512, 97, 97), (2, 64, 512, 65, 65), (1, 7, 19, 40, 70),
    (1, 8, 48, 130, 150),
]


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("shape", SHAPES)
def test_forward_fp32_vs_oracle(shape, impl):
    from ccnet_b200 import cca_forward
    O = _oracle()
    dev = _dev()
    q, k, v = _rand_qkv(*shape, seed=sum(shape))
    out, lse = cca_forward(q.to(dev), k.to(dev), v.to(dev), impl=impl)
    ro, rl = O.cca_forward(q.double(), k.double(), v.double())
    assert (out.cpu().double() - ro).abs().max().item() <= FP32_TOL
    assert (lse.cpu().double() - rl).abs().max().item() <= FP32_TOL


TC_SHAPES = [
    (2, 32, 256, 20, 97), (1, 64, 64, 112, 80), (3, 16, 64, 1, 5), (2, 16, 64, 5, 1), (1, 48, 192, 81, 112),
    (1, 16, 128, 1, 1), (2, 64, 512, 33, 47), (8, 64, 512, 97, 97),
    # lines longer than one tile (key-block tiling, cca_items.cuh): BASELINE configs[4] sweep points and ragged ones
    (1, 64, 512, 129, 129), (1, 64, 512, 193, 193), (1, 32, 128, 113, 200), (2, 16, 64, 230, 7), (1, 16, 64, 1, 300),
]


@pytest.mark.parametrize("shape", TC_SHAPES)
def test_forward_tensor_core_vs_oracle_and_simt(shape):
    """wgmma path (channels-last, bf16x3 split) against the fp64 oracle and the generic kernels."""
    from ccnet_b200 import cca_forward
    O = _oracle()
    dev = _dev()
    q, k, v = _rand_qkv(*shape, seed=3 + sum(shape))
    qd, kd, vd = q.to(dev), k.to(dev), v.to(dev)
    out, lse = cca_forward(qd, kd, vd, impl="tc")
    assert out.shape == v.shape and out.is_contiguous(memory_format=torch.channels_last)
    so, sl = cca_forward(qd, kd, vd, impl="simt")
    assert (out - so).abs().max().item() <= 5e-4 and (lse - sl).abs().max().item() <= 5e-4
    if shape[0] * shape[3] * shape[4] <= 4 * 97 * 97 or shape[0] == 1:
        ro, rl = O.cca_forward(q.double(), k.double(), v.double())
        assert (out.cpu().double() - ro).abs().max().item() <= 5e-4
        assert (lse.cpu().double() - rl).abs().max().item() <= 5e-4
    # channels-last inputs give the same result (no hidden layout dependence): bit-identical with one tile per line (one
    # store + one add per element); with tiled lines an element is the sum of 2*nt-1 adds whose order is not fixed
    out2, _ = cca_forward(qd.contiguous(memory_format=torch.channels_last), kd, vd.contiguous(memory_format=torch.channels_last), impl="tc")
    if max(shape[3], shape[4]) <= 112:
        assert torch.equal(out, out2)
    else:
        assert (out - out2).abs().max().item() <= 1e-5 * max(1.0, out.abs().max().item())


@pytest.mark.parametrize("shape", [(2, 32, 256, 20, 97), (1, 64, 64, 112, 80), (3, 16, 64, 1, 5), (2, 16, 64, 5, 1),
                                   (1, 48, 192, 81, 112), (1, 16, 128, 1, 1), (2, 64, 512, 33, 47), (1, 64, 512, 97, 97),
                                   (1, 64, 512, 129, 129), (1, 64, 512, 193, 193), (1, 32, 128, 113, 200), (2, 16, 64, 230, 7)])
def test_backward_tensor_core_vs_oracle(shape):
    """wgmma backward (channels-last, bf16x3 split, P recomputed from lse) against the fp64 closed form."""
    from ccnet_b200 import cca_backward, cca_forward
    O = _oracle()
    dev = _dev()
    q, k, v = _rand_qkv(*shape, seed=21 + sum(shape), scale=0.7)
    dout = torch.randn(v.shape, generator=torch.Generator().manual_seed(5))
    qd, kd, vd, dd = q.to(dev), k.to(dev), v.to(dev), dout.to(dev)
    out, lse = cca_forward(qd, kd, vd, impl="tc")
    dq, dk, dv = cca_backward(dd, qd, kd, vd, out, lse, impl="tc")
    assert dv.shape == v.shape and dv.is_contiguous(memory_format=torch.channels_last)
    rq, rk, rv = O.cca_backward(dout.double(), q.double(), k.double(), v.double())
    for got, ref, name in ((dq, rq, "dq"), (dk, rk, "dk"), (dv, rv, "dv")):
        tol = FP32_TOL * max(1.0, ref.abs().max().item())
        err = (got.cpu().double() - ref).abs().max().item()
        assert err <= tol, (name, err, tol)
    # and against the generic kernels
    sq, sk, sv = cca_backward(dd, qd, kd, vd, out, lse, impl="simt")
    for got, ref in ((dq, sq), (dk, sk), (dv, sv)):
        assert (got - ref).abs().max().item() <= FP32_TOL * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("shape", [(2, 32, 256, 20, 97), (1, 64, 64, 112, 80), (3, 16, 64, 1, 5), (2, 64, 512, 33, 47), (2, 64, 512, 97, 97),
                                   (1, 64, 512, 129, 129), (1, 64, 512, 193, 193), (1, 32, 128, 113, 200)])
def test_bf16_tensor_core_forward_backward_vs_oracle(shape):
    """bf16 I/O on the wgmma kernels (single-term MMAs, bf16 stores / vector adds): against the fp64 oracle
    evaluated on the bf16-rounded inputs (SURVEY.md 8c), tolerance 1e-2 relative to max|ref| (north_star), forward and gradients."""
    from ccnet_b200 import cca_backward, cca_forward
    O = _oracle()
    dev = _dev()
    q, k, v = _rand_qkv(*shape, seed=41 + sum(shape), scale=0.6, dtype=torch.bfloat16)
    dout = torch.randn(v.shape, generator=torch.Generator().manual_seed(9)).to(torch.bfloat16)
    qd, kd, vd, dd = q.to(dev), k.to(dev), v.to(dev), dout.to(dev)
    out, lse = cca_forward(qd, kd, vd, impl="tc")
    assert out.dtype == torch.bfloat16 and lse.dtype == torch.float32
    ro, rl = O.cca_forward(q.double(), k.double(), v.double())
    assert (out.cpu().double() - ro).abs().max().item() <= BF16_TOL * max(1.0, ro.abs().max().item())
    assert (lse.cpu().double() - rl).abs().max().item() <= BF16_TOL
    dq, dk, dv = cca_backward(dd, qd, kd, vd, out, lse, impl="tc")
    rq, rk, rv = O.cca_backward(dout.double(), q.double(), k.double(), v.double())
    for got, ref, name in ((dq, rq, "dq"), (dk, rk, "dk"), (dv, rv, "dv")):
        assert got.dtype == torch.bfloat16
        err = (got.cpu().double() - ref).abs().max().item()
        assert err <= BF16_TOL * max(1.0, ref.abs().max().item()), (name, err)


def _debug_hook(lib, name, argtypes):
    """A/B hooks exist in debug builds only (python -m ccnet_b200.build --debug)."""
    try:
        fn = getattr(lib, name)
    except AttributeError:
        return None
    fn.argtypes, fn.restype = argtypes, None
    return fn


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_launch_knobs_are_bit_identical(dtype):
    """Programmatic dependent launch (off / on), the item order (lagged or not), the L2 eviction hints and the backward's delta
    mode only change WHEN and WHERE bytes move, never the arithmetic: with one tile per line every output element is one
    store plus one add, so forward and backward must be bit-identical across knobs and repetitions.
    Repeated at the BASELINE shape (every SM busy) to give an ordering bug a chance to show."""
    import ctypes
    from ccnet_b200 import capi, cca_backward, cca_forward
    dev = _dev()
    lib = capi.load()
    pdl = _debug_hook(lib, "cca_b200__set_pdl", [ctypes.c_int])
    ahead = _debug_hook(lib, "cca_b200__set_zero_ahead", [ctypes.c_int])
    dmode = _debug_hook(lib, "cca_b200__set_delta_mode", [ctypes.c_int])
    lag = _debug_hook(lib, "cca_b200__set_lag", [ctypes.c_int])
    hint = _debug_hook(lib, "cca_b200__set_l2_hints", [ctypes.c_int])
    dt = torch.float32 if dtype == "fp32" else torch.bfloat16
    cl = torch.channels_last
    # (pdl, delta mode, lag, hints)
    combos = [(1, -1, -1, 1)] if pdl is None else [(1, -1, -1, 1), (0, -1, -1, 1), (1, 0, 0, 1), (1, 1, 1, 0), (0, 0, 1, 2), (1, 1, 0, 0)]
    for shape in [(8, 64, 512, 97, 97), (2, 32, 256, 20, 97), (5, 16, 64, 7, 3)]:
        q, k, v = _rand_qkv(*shape, seed=5 + sum(shape))
        q, k, v = (t.to(dev).to(dt).contiguous(memory_format=cl) for t in (q, k, v))
        do = torch.randn(v.shape, device=dev).to(dt).contiguous(memory_format=cl)
        ro = rl = rg = None
        try:
            for (lv, dm, lg, hn) in combos:
                if pdl is not None:
                    pdl(lv); dmode(dm); lag(lg); hint(hn)
                for _ in range(4):
                    o, l = cca_forward(q, k, v, impl="tc")
                    g = cca_backward(do, q, k, v, o, l, impl="tc")
                    if ro is None:
                        ro, rl, rg = o, l, g
                    assert torch.equal(o, ro) and torch.equal(l, rl), (shape, lv, dm, lg, hn)
                    # delta computed per item or fetched from the producers is the same number either way
                    assert all(torch.equal(a, b) for a, b in zip(g, rg)), (shape, lv, dm, lg, hn)
        finally:
            if pdl is not None:
                pdl(1); dmode(-1); lag(-1); hint(1)


@pytest.mark.parametrize("dtype,tol", [("fp32", FP32_TOL), ("bf16", BF16_TOL)])
def test_backward_full_batch_c2_vs_oracle(dtype, tol):
    """BASELINE config 2 (B=8, C=512, 97x97): forward AND backward of the persistent single-launch schedule (776 lines per
    direction over one persistent CTA per SM, delta hand-off between CTAs) against the fp64 oracle on the first, a middle and
    the last sample."""
    from ccnet_b200 import cca_backward, cca_forward
    O = _oracle()
    dev = _dev()
    dt = torch.float32 if dtype == "fp32" else torch.bfloat16
    shape = (8, 64, 512, 97, 97)
    q, k, v = _rand_qkv(*shape, seed=1234, scale=0.6, dtype=dt)
    dout = torch.randn(v.shape, generator=torch.Generator().manual_seed(8)).to(dt)
    qd, kd, vd, dd = q.to(dev), k.to(dev), v.to(dev), dout.to(dev)
    out, lse = cca_forward(qd, kd, vd, impl="tc")
    dq, dk, dv = cca_backward(dd, qd, kd, vd, out, lse, impl="tc")
    for b in (0, 3, 7):
        sl = slice(b, b + 1)
        ro, rl = O.cca_forward(q[sl].double(), k[sl].double(), v[sl].double())
        rq, rk, rv = O.cca_backward(dout[sl].double(), q[sl].double(), k[sl].double(), v[sl].double())
        assert (out[sl].cpu().double() - ro).abs().max().item() <= tol * max(1.0, ro.abs().max().item()), b
        assert (lse[sl].cpu().double() - rl).abs().max().item() <= tol, b
        for got, ref, name in ((dq, rq, "dq"), (dk, rk, "dk"), (dv, rv, "dv")):
            err = (got[sl].cpu().double() - ref).abs().max().item()
            assert err <= tol * max(1.0, ref.abs().max().item()), (b, name, err)


def test_tensor_core_peaky_softmax_stress():
    """q,k ~ N(0,1)*1.5: logits std ~18, near one-hot attention; error budget still 1e-3."""
    from ccnet_b200 import cca_forward
    O = _oracle()
    dev = _dev()
    q, k, v = _rand_qkv(1, 64, 128, 97, 97, seed=77, scale=1.5)
    out, lse = cca_forward(q.to(dev), k.to(dev), v.to(dev), impl="tc")
    ro, rl = O.cca_forward(q.double(), k.double(), v.double())
    assert (out.cpu().double() - ro).abs().max().item() <= FP32_TOL
    assert (lse.cpu().double() - rl).abs().max().item() <= FP32_TOL


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("shape", [(2, 8, 64, 5, 6), (1, 16, 128, 17, 33), (1, 64, 512, 97, 97), (1, 2, 16, 1, 11)])
def test_forward_bf16_vs_oracle_on_rounded_inputs(shape, impl):
    from ccnet_b200 import cca_forward
    O = _oracle()
    dev = _dev()
    q, k, v = _rand_qkv(*shape, seed=7 + sum(shape), scale=0.6, dtype=torch.bfloat16)
    out, lse = cca_forward(q.to(dev), k.to(dev), v.to(dev), impl=impl)
    assert out.dtype == torch.bfloat16 and lse.dtype == torch.float32
    ro, rl = O.cca_forward(q.double(), k.double(), v.double())
    scale = max(1.0, ro.abs().max().item())
    assert (out.cpu().double() - ro).abs().max().item() <= BF16_TOL * scale
    assert (lse.cpu().double() - rl).abs().max().item() <= BF16_TOL


@pytest.mark.parametrize("shape", [(2, 8, 64, 5, 6), (2, 4, 32, 9, 7), (1, 2, 16, 1, 11), (1, 2, 16, 13, 1), (1, 1, 8, 1, 1),
                                   (1, 16, 128, 17, 33), (1, 64, 512, 65, 65), (1, 8, 48, 130, 150)])
def test_backward_fp32_vs_oracle(shape):
    from ccnet_b200 import cca_backward, cca_forward
    O = _oracle()
    dev = _dev()
    q, k, v = _rand_qkv(*shape, seed=11 + sum(shape), scale=0.7)
    g = torch.Generator().manual_seed(99)
    dout = torch.randn(v.shape, generator=g)
    out, lse = cca_forward(q.to(dev), k.to(dev), v.to(dev))
    dq, dk, dv = cca_backward(dout.to(dev), q.to(dev), k.to(dev), v.to(dev), out, lse)
    rq, rk, rv = O.cca_backward(dout.double(), q.double(), k.double(), v.double())
    for got, ref, name in ((dq, rq, "dq"), (dk, rk, "dk"), (dv, rv, "dv")):
        tol = FP32_TOL * max(1.0, ref.abs().max().item())
        assert (got.cpu().double() - ref).abs().max().item() <= tol, name


def test_backward_bf16_vs_oracle():
    from ccnet_b200 import cca_backward, cca_forward
    O = _oracle()
    dev = _dev()
    q, k, v = _rand_qkv(2, 8, 64, 12, 10, seed=5, scale=0.6, dtype=torch.bfloat16)
    dout = torch.randn(v.shape, generator=torch.Generator().manual_seed(3)).to(torch.bfloat16)
    out, lse = cca_forward(q.to(dev), k.to(dev), v.to(dev))
    dq, dk, dv = cca_backward(dout.to(dev), q.to(dev), k.to(dev), v.to(dev), out, lse)
    rq, rk, rv = O.cca_backward(dout.double(), q.double(), k.double(), v.double())
    for got, ref in ((dq, rq), (dk, rk), (dv, rv)):
        assert (got.cpu().double() - ref).abs().max().item() <= 3 * BF16_TOL * max(1.0, ref.abs().max().item())


def test_module_vs_golden_fwd_bwd(golden):
    """x -> y through the drop-in nn.Module, R recurrences, with the reference's parameters."""
    import cc_attention
    dev = _dev()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    x = torch.from_numpy(golden["x"]).to(dev).requires_grad_(True)
    m = cc_attention.CrissCrossAttention(x.shape[1]).to(dev)
    m.load_state_dict({n[2:]: torch.from_numpy(a) for n, a in golden.items() if n.startswith("p_")})
    y = x
    for _ in range(int(golden["R"])):
        y = m(y)
    (y * torch.from_numpy(golden["g"]).to(dev)).sum().backward()
    assert (y.detach().cpu() - torch.from_numpy(golden["y"])).abs().max().item() <= FP32_TOL
    assert (x.grad.cpu() - torch.from_numpy(golden["dx"])).abs().max().item() <= FP32_TOL * max(
        1.0, float(np.abs(golden["dx"]).max()))
    for n, p in m.named_parameters():
        ref = torch.from_numpy(golden["d_" + n])
        # a conv's bias gradient is the plain sum of the same per-pixel gradients its weight gradient weighs by x, so both
        # carry the same absolute rounding error; key_conv.bias in particular cancels to exactly 0 in exact arithmetic
        # (softmax shift invariance), so its own magnitude (~1e-5) says nothing about the scale of the summands (~1e3).
        scale = torch.from_numpy(golden["d_" + n.replace(".bias", ".weight")]).abs().max().item()
        tol = 2e-3 * max(1.0, ref.abs().max().item()) if not n.endswith(".bias") else max(2e-3, 1e-5 * scale)
        assert (p.grad.cpu() - ref).abs().max().item() <= tol, n


def test_full_size_properties_and_oracle_c2():
    """BASELINE config 2 (B=8, C=512, 97x97): size-independent properties + oracle on 2 samples."""
    from ccnet_b200 import cca_forward
    O = _oracle()
    dev = _dev()
    torch.manual_seed(0)
    B, Cq, C, H, W = 8, 64, 512, 97, 97
    q = torch.randn(B, Cq, H, W, device=dev) * 0.58
    k = torch.randn(B, Cq, H, W, device=dev) * 0.58
    v1 = torch.randn(B, C, H, W, device=dev)
    v2 = torch.randn(B, C, H, W, device=dev)
    o1, lse = cca_forward(q, k, v1)
    o2, _ = cca_forward(q, k, v2)
    o12, _ = cca_forward(q, k, v1 + 2.0 * v2)
    assert (o12 - (o1 + 2.0 * o2)).abs().max().item() <= 2e-4            # linear in v (|o| ~ 4: 5e-5 relative, the bf16x3 floor)
    ones, _ = cca_forward(q, k, torch.ones_like(v1))
    assert (ones - 1.0).abs().max().item() <= 1e-5                       # attention rows sum to 1
    # oracle on samples 0 and 7
    for b in (0, 7):
        ro, rl = O.cca_forward(q[b:b + 1].cpu().double(), k[b:b + 1].cpu().double(), v1[b:b + 1].cpu().double())
        assert (o1[b:b + 1].cpu().double() - ro).abs().max().item() <= FP32_TOL
        assert (lse[b:b + 1].cpu().double() - rl).abs().max().item() <= FP32_TOL
    # per-sample independence: permuting the batch permutes the output
    perm = torch.tensor([3, 0, 7, 1, 2, 6, 5, 4], device=dev)
    op, _ = cca_forward(q[perm], k[perm], v1[perm])
    assert torch.equal(op, o1[perm])


def test_host_buffer_entry_point():
    """cca_b200_forward_host / backward_host: plain host pointers through the C ABI."""
    from ccnet_b200 import capi
    O = _oracle()
    _dev()
    lib = capi.load()
    B, Cq, C, H, W = 2, 4, 24, 7, 9
    q, k, v = _rand_qkv(B, Cq, C, H, W, seed=42)
    qn, kn, vn = (np.ascontiguousarray(t.numpy()) for t in (q, k, v))
    out = np.empty((B, C, H, W), np.float32)
    lse = np.empty((B, H, W), np.float32)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    rc = lib.cca_b200_forward_host(p(qn), p(kn), p(vn), p(out), p(lse), B, Cq, C, H, W, capi.CCA_F32, 0)
    capi.check(rc, "forward_host")
    ro, rl = O.cca_forward(q.double(), k.double(), v.double())
    assert np.abs(out - ro.numpy()).max() <= FP32_TOL and np.abs(lse - rl.numpy()).max() <= FP32_TOL
    dout = np.random.default_rng(0).standard_normal((B, C, H, W)).astype(np.float32)
    dq, dk, dv = np.empty_like(qn), np.empty_like(kn), np.empty_like(vn)
    rc = lib.cca_b200_backward_host(p(dout), p(qn), p(kn), p(vn), p(out), p(lse), p(dq), p(dk), p(dv),
                                    B, Cq, C, H, W, capi.CCA_F32, 0)
    capi.check(rc, "backward_host")
    rq, rk, rv = O.cca_backward(torch.from_numpy(dout).double(), q.double(), k.double(), v.double())
    for got, ref in ((dq, rq), (dk, rk), (dv, rv)):
        assert np.abs(got - ref.numpy()).max() <= FP32_TOL * max(1.0, ref.abs().max().item())


def test_error_behaviour_on_gpu():
    from ccnet_b200 import cca_forward
    dev = _dev()
    q = torch.randn(1, 4, 5, 5, device=dev)
    with pytest.raises(RuntimeError):
        cca_forward(q, q[:, :, :4], torch.randn(1, 8, 5, 5, device=dev))           # shape mismatch
    with pytest.raises(RuntimeError):
        cca_forward(q, q, torch.randn(1, 8, 5, 5, device=dev, dtype=torch.float16).float().half())  # dtype
    with pytest.raises(RuntimeError, match="unsupported|too large"):
        big = torch.zeros(1, 1, 1, 5000, device=dev)
        cca_forward(big, big, big)


def test_noncontiguous_inputs_and_fresh_output():
    from ccnet_b200 import cca_forward
    O = _oracle()
    dev = _dev()
    q, k, v = _rand_qkv(1, 4, 16, 6, 8, seed=1)
    qd = q.to(dev).permute(0, 1, 3, 2).contiguous().permute(0, 1, 3, 2)     # channels/space strided view
    vd = v.to(dev).to(memory_format=torch.channels_last)
    out, _ = cca_forward(qd, k.to(dev), vd)
    ro, _ = O.cca_forward(q.double(), k.double(), v.double())
    assert (out.cpu().double() - ro).abs().max().item() <= FP32_TOL
    assert out.data_ptr() != vd.data_ptr()


# ---------------------------------------------------------------------------------------------------------------------
# hand-written projection GEMMs (functions.py:29,32,35) and the fused module step around the operator
# ---------------------------------------------------------------------------------------------------------------------
def _proj_params(C, seed):
    g = torch.Generator().manual_seed(seed)
    Cq = C // 8
    bound = 1.0 / (C ** 0.5)
    mk = lambda *s: (torch.rand(*s, generator=g) * 2 - 1) * bound
    return mk(Cq, C), mk(Cq), mk(Cq, C), mk(Cq), mk(C, C), mk(C)


@pytest.mark.parametrize("shape", [(1, 512, 97, 97), (3, 512, 20, 31), (1, 512, 1, 5)])
def test_qkv_projection_gemm_vs_fp64(shape):
    """wgmma bf16x3 GEMM of the three 1x1 convs against fp64 matmul: fp32-level accuracy (north_star 1e-3, typical 1e-5)."""
    from ccnet_b200.functional import qkv_gemm_eligible, qkv_project, qkv_project_dgrad
    dev = _dev()
    B, C, H, W = shape
    wq, bq, wk, bk, wv, bv = _proj_params(C, 5)
    x = torch.randn(B, C, H, W, generator=torch.Generator().manual_seed(1))
    xd = x.to(dev).contiguous(memory_format=torch.channels_last)
    assert qkv_gemm_eligible(xd, C // 8)
    q, k, v = qkv_project(xd, wq.to(dev), bq.to(dev), wk.to(dev), bk.to(dev), wv.to(dev), bv.to(dev))
    xm = x.double().permute(0, 2, 3, 1).reshape(-1, C)
    for got, w, b in ((q, wq, bq), (k, wk, bk), (v, wv, bv)):
        ref = xm @ w.double().t() + b.double()
        assert got.is_contiguous(memory_format=torch.channels_last) and got.shape[1] == w.shape[0]
        err = (got.cpu().double().permute(0, 2, 3, 1).reshape(-1, w.shape[0]) - ref).abs().max().item()
        assert err <= 1e-4 * max(1.0, ref.abs().max().item()), err
    # input gradient
    gq, gk, gv = (torch.randn(t.shape, generator=torch.Generator().manual_seed(7 + i)) for i, t in enumerate((q, k, v)))
    dx = qkv_project_dgrad(*(g.to(dev).contiguous(memory_format=torch.channels_last) for g in (gq, gk, gv)),
                           wq.to(dev), wk.to(dev), wv.to(dev))
    ref = sum(g.double().permute(0, 2, 3, 1).reshape(-1, w.shape[0]) @ w.double() for g, w in ((gq, wq), (gk, wk), (gv, wv)))
    err = (dx.cpu().double().permute(0, 2, 3, 1).reshape(-1, C) - ref).abs().max().item()
    assert err <= 1e-4 * max(1.0, ref.abs().max().item()), err
    # parameter gradients (split-K over the pixels, gamma folded in as a device scalar)
    from ccnet_b200.functional import qkv_project_wgrad, qkv_wgrad_eligible
    assert qkv_wgrad_eligible(C, C // 8)
    scale = torch.tensor([0.75], device=dev)
    outs = qkv_project_wgrad(xd, *(g.to(dev).contiguous(memory_format=torch.channels_last) for g in (gq, gk, gv)), scale=scale)
    for i, g in enumerate((gq, gk, gv)):
        gm = g.double().permute(0, 2, 3, 1).reshape(-1, g.shape[1])
        rw, rb = 0.75 * (gm.t() @ xm), 0.75 * gm.sum(0)
        ew = (outs[2 * i].cpu().double() - rw).abs().max().item()
        eb = (outs[2 * i + 1].cpu().double() - rb).abs().max().item()
        assert ew <= 1e-4 * max(1.0, rw.abs().max().item()), (i, ew)
        assert eb <= 1e-4 * max(1.0, rb.abs().max().item(), rw.abs().max().item()), (i, eb)


def test_fused_module_step_c512_vs_oracle_module():
    """The user-facing module at C=512 (every kernel of the step is this repo's: projection GEMMs, attention, backward) against
    the oracle module on the CPU, recurrence 2, all seven parameter gradients."""
    import cc_attention
    from ccnet_b200.module import _FusedCCAStep  # noqa: F401  (the path under test)
    O = _oracle()
    dev = _dev()
    torch.manual_seed(3)
    C, H, W = 512, 24, 40
    ref = O.CrissCrossAttentionOracle(C)
    with torch.no_grad():
        ref.gamma.fill_(0.7)
    m = cc_attention.CrissCrossAttention(C).to(dev)
    m.load_state_dict(ref.state_dict())
    x = torch.randn(2, C, H, W)
    g = torch.randn(2, C, H, W)
    xd = x.to(dev).requires_grad_(True)
    y = m(m(xd))
    (y * g.to(dev)).sum().backward()
    xr = x.clone().requires_grad_(True)
    yr = ref(ref(xr))
    (yr * g).sum().backward()
    assert (y.detach().cpu() - yr.detach()).abs().max().item() <= FP32_TOL
    assert (xd.grad.cpu() - xr.grad).abs().max().item() <= FP32_TOL * max(1.0, xr.grad.abs().max().item())
    rp = dict(ref.named_parameters())
    for n, p in m.named_parameters():
        r = rp[n].grad
        scale = rp[n.replace(".bias", ".weight")].grad.abs().max().item() if n.endswith(".bias") else r.abs().max().item()
        assert (p.grad.cpu() - r).abs().max().item() <= 2e-3 * max(1.0, scale), n


def test_torch_ops_match_the_functional_path_and_differentiate():
    """torch.ops.cca.forward / backward / forward_residual (SURVEY 8b) give the same bits as ccnet_b200.functional and carry
    autograd; opcheck validates the registration (schema, fake tensor, autograd) on real tensors."""
    from ccnet_b200 import cca_backward, cca_forward
    dev = _dev()
    q, k, v = (t.to(dev) for t in _rand_qkv(2, 16, 64, 9, 11, seed=4))
    out, lse = torch.ops.cca.forward(q, k, v)
    ro, rl = cca_forward(q, k, v)
    assert torch.equal(out, ro) and torch.equal(lse, rl)
    qg, kg, vg = (t.clone().requires_grad_(True) for t in (q, k, v))
    o2, _ = torch.ops.cca.forward(qg, kg, vg)
    do = torch.randn_like(o2)
    o2.backward(do)
    rq, rk, rv = cca_backward(do, q, k, v, ro, rl)
    assert torch.equal(qg.grad, rq) and torch.equal(kg.grad, rk) and torch.equal(vg.grad, rv)
    x = torch.randn_like(v).requires_grad_(True)
    gamma = torch.tensor([0.3], device=dev, requires_grad=True)
    y, _, _ = torch.ops.cca.forward_residual(q, k, v, x, gamma)
    assert torch.allclose(y, 0.3 * ro + x.detach(), atol=1e-6)
    y.backward(do)
    assert torch.allclose(x.grad, do) and torch.allclose(gamma.grad, (do * ro).sum().reshape(1), rtol=1e-4)
    torch.library.opcheck(torch.ops.cca.forward.default, (q, k, v), test_utils=("test_schema", "test_faketensor"))


def test_bf16_long_lines_native_kernels_noise_floor(monkeypatch):
    """bf16 I/O with lines longer than one tile: the native bf16 kernels (what a direct C-ABI caller gets) add up to 2*ceil(L/112)
    bf16-rounded partial results per element in no fixed order; their error sits at the 1e-2 budget (one bf16 rounding of the
    exact gradient alone is 0.3e-2 of max|ref| here), so the Python entry points run such calls on the fp32 kernels and round
    once (ccnet_b200/functional.py).  This test keeps the native kernels covered, at twice the budget."""
    from ccnet_b200 import cca_backward, cca_forward
    O = _oracle()
    dev = _dev()
    monkeypatch.setenv("CCA_B200_BF16_NATIVE", "1")
    shape = (1, 32, 128, 113, 200)
    q, k, v = _rand_qkv(*shape, seed=41 + sum(shape), scale=0.6, dtype=torch.bfloat16)
    dout = torch.randn(v.shape, generator=torch.Generator().manual_seed(9)).to(torch.bfloat16)
    qd, kd, vd, dd = q.to(dev), k.to(dev), v.to(dev), dout.to(dev)
    out, lse = cca_forward(qd, kd, vd, impl="tc")
    dq, dk, dv = cca_backward(dd, qd, kd, vd, out, lse, impl="tc")
    ro, rl = O.cca_forward(q.double(), k.double(), v.double())
    rq, rk, rv = O.cca_backward(dout.double(), q.double(), k.double(), v.double())
    assert (out.cpu().double() - ro).abs().max().item() <= 2 * BF16_TOL * max(1.0, ro.abs().max().item())
    for got, ref, name in ((dq, rq, "dq"), (dk, rk, "dk"), (dv, rv, "dv")):
        assert got.dtype == torch.bfloat16
        err = (got.cpu().double() - ref).abs().max().item()
        assert err <= 2 * BF16_TOL * max(1.0, ref.abs().max().item()), (name, err)
