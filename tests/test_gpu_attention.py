"""H100 tests of the attention map (cc_attention/functions.py:40, `concate`): the tensor-core and generic kernels against the
fp64 oracle within budgets derived by emulation (tests/attn_budget.py), the module surface against the reference's fixtures,
determinism, the C ABI's refusals, a map past 2^31 elements, and the torch.ops registration."""
import glob
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import attn_budget as AB
import ccnet_b200
from ccnet_b200 import capi, cca_attention, cca_forward
from ccnet_b200.functional import cca_attention_backward, cca_attention_forward

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
DTYPES = [torch.float32, torch.bfloat16, torch.float16]
# golden-like, H = 1, W = 1, ragged, and the tiling edges of tests/test_gpu_tc_edges.py (80/81, 112/113, 224/225, 896)
SHAPES = [(2, 16, 5, 6), (1, 16, 1, 11), (1, 32, 13, 1), (2, 48, 37, 29), (1, 64, 40, 72), (1, 64, 80, 81),
          (1, 32, 112, 113), (1, 16, 224, 225), (1, 16, 896, 20)]


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _inputs(shape, dtype, seed, scale=0.7):
    B, Cq, H, W = shape
    g = torch.Generator().manual_seed(seed)
    q, k = ((torch.randn(B, Cq, H, W, generator=g) * scale).to(dtype) for _ in range(2))
    da = torch.randn(B, H, W, H + W, generator=g)
    return q, k, da


@pytest.mark.parametrize("impl", ["tc", "simt"])
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d).split(".")[-1])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_map_and_gradients_match_the_oracle(shape, dtype, impl):
    dev = _dev()
    B, Cq, H, W = shape
    if impl == "simt" and H * W > 30000:
        pytest.skip("the generic kernels are a fallback: checked on the smaller shapes")
    q, k, da = _inputs(shape, dtype, seed=hash(shape) % 1000)
    ref, emu = AB.reference(q, k, da), AB.emulate(q, k, da, dtype)
    bud = AB.budget(emu, ref, dtype)
    qd, kd = q.to(dev), k.to(dev)
    attn = cca_attention_forward(qd, kd, impl)
    assert attn.dtype == torch.float32 and attn.is_contiguous() and tuple(attn.shape) == (B, H, W, H + W)
    dq, dk = cca_attention_backward(da.to(dev), attn, qd, kd, impl)
    assert dq.dtype == dtype and dk.dtype == dtype
    AB.check(dict(attn=attn, dq=dq, dk=dk), ref, bud, (shape, dtype, impl))
    # rows sum to 1, entries >= 0, self entries exactly 0
    assert attn.min().item() >= 0
    assert (attn.sum(-1) - 1).abs().max().item() < 1e-5 * (H + W) ** 0.5 + 1e-5
    assert attn[..., :H].diagonal(dim1=1, dim2=3).abs().max().item() == 0


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d).split(".")[-1])
@pytest.mark.parametrize("shape", [(2, 64, 9, 11), (1, 16, 113, 130)], ids=lambda s: "x".join(map(str, s)))
def test_map_times_v_is_the_forward_output(shape, dtype):
    dev = _dev()
    B, Cq, H, W = shape
    q, k, _ = _inputs(shape, dtype, seed=5)
    v = torch.randn(B, 64, H, W).to(dtype).to(dev)
    qd, kd = q.to(dev), k.to(dev)
    attn = cca_attention_forward(qd, kd)
    out, _ = cca_forward(qd, kd, v)
    vf = v.double()
    o = torch.einsum("bhwg,bcgw->bchw", attn[..., :H].double(), vf) + torch.einsum("bhwg,bchg->bchw", attn[..., H:].double(), vf)
    tol = 2e-4 if dtype == torch.float32 else 4 * 2.0 ** (-8 if dtype == torch.bfloat16 else -11)
    assert (out.double() - o).abs().max().item() <= tol * max(1.0, o.abs().max().item())


FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "attn_*.npz")))


@pytest.mark.parametrize("path", FIXTURES, ids=[os.path.basename(p) for p in FIXTURES])
def test_module_maps_and_gradients_match_the_reference(path):
    dev = _dev()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    f = np.load(path)
    m = ccnet_b200.RCCA(f["x"].shape[1], recurrence=int(f["R"])).to(dev)
    m.cca.load_state_dict({n[2:]: torch.from_numpy(f[n]) for n in f.files if n.startswith("p_")})
    x = torch.from_numpy(f["x"]).to(dev).requires_grad_(True)
    _, maps = m(x, return_attention=True)
    loss = 0
    for i, a in enumerate(maps):
        ref = torch.from_numpy(f[f"A_{i}"])
        assert (a.detach().cpu() - ref).abs().max().item() < 1e-5
        loss = loss + (a * torch.from_numpy(f[f"R_{i}"]).to(dev)).sum()
    loss.backward()
    tol = lambda r: 1e-4 * max(1.0, np.abs(r).max())
    assert np.abs(x.grad.cpu().numpy() - f["dx"]).max() < tol(f["dx"])
    for n, p in m.cca.named_parameters():
        g = p.grad.cpu().numpy() if p.grad is not None else np.zeros(p.shape, np.float32)
        assert np.abs(g - f["d_" + n]).max() < tol(f["d_" + n]), n


def test_module_map_under_f16_autocast_matches_the_oracle_module():
    from oracle.cca_oracle import CrissCrossAttentionOracle
    dev = _dev()
    torch.manual_seed(3)
    ref = CrissCrossAttentionOracle(256)
    m = ccnet_b200.CrissCrossAttention(256).to(dev)
    m.load_state_dict(ref.state_dict())
    x = torch.randn(2, 256, 20, 30)
    xd = x.to(dev).requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.float16):
        _, a = m(xd, return_attention=True)
    assert a.dtype == torch.float32
    r = torch.randn(a.shape)
    (a * r.to(dev)).sum().backward()
    xr = x.double().requires_grad_(True)
    r64 = ref.double()
    ar = AB.attention_map(r64.query_conv(xr), r64.key_conv(xr))
    (ar * r.double()).sum().backward()
    assert (a.detach().cpu().double() - ar.detach()).abs().max().item() < 2e-2
    assert (xd.grad.cpu().double() - xr.grad).abs().max().item() < 5e-2 * max(1.0, xr.grad.abs().max().item())


@pytest.mark.parametrize("C", [64, 512])
def test_return_attention_leaves_y_and_its_gradients_unchanged(C):
    """(deterministic mode: the default mode's weight gradient of the fused C = 512 step adds split-K partials in no fixed
    order, so two runs of the same code need not agree to the bit)"""
    dev = _dev()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        _y_and_grads_unchanged(C, dev)
    finally:
        torch.use_deterministic_algorithms(False)


def _y_and_grads_unchanged(C, dev):
    torch.manual_seed(4)
    m = ccnet_b200.CrissCrossAttention(C).to(dev)
    with torch.no_grad():
        m.gamma.fill_(0.7)
    x = torch.randn(2, C, 17, 19, device=dev)
    y0 = m(x)
    y0.square().sum().backward()
    g0 = [p.grad.clone() for p in m.parameters()]
    m.zero_grad()
    y1, a = m(x, return_attention=True)
    assert torch.equal(y0, y1)
    y1.square().sum().backward()
    assert all(torch.equal(p.grad, g) for p, g in zip(m.parameters(), g0))


@pytest.mark.parametrize("shape", [(2, 32, 129, 129), (1, 64, 193, 193), (2, 16, 113, 200)], ids=lambda s: "x".join(map(str, s)))
def test_deterministic_mode_is_bit_reproducible(shape, monkeypatch):
    dev = _dev()
    q, k, da = (t.to(dev) for t in _inputs(shape, torch.float32, seed=6))
    torch.use_deterministic_algorithms(True)
    try:
        runs = []
        for _ in range(3):
            a = cca_attention_forward(q, k)
            runs.append((a,) + cca_attention_backward(da, a, q, k))
        from ccnet_b200 import functional
        monkeypatch.setattr(functional, "deterministic_workspace_cap", 1)      # one sample per call
        a = cca_attention_forward(q, k)
        runs.append((a,) + cca_attention_backward(da, a, q, k))
    finally:
        torch.use_deterministic_algorithms(False)
    for r in runs[1:]:
        assert all(torch.equal(x, y) for x, y in zip(runs[0], r))
    # the same bits without programmatic dependent launch, in a child process
    path = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"attn_det_{os.getpid()}.pt")
    torch.save(dict(q=q.cpu(), k=k.cpu(), da=da.cpu()), path)
    code = ("import sys, torch; sys.path.insert(0, %r); from ccnet_b200.functional import cca_attention_forward as f, "
            "cca_attention_backward as b; t = torch.load(%r); q, k, da = (t[n].cuda() for n in ('q', 'k', 'da')); "
            "a = f(q, k, deterministic=True); dq, dk = b(da, a, q, k, deterministic=True); "
            "torch.save(dict(a=a.cpu(), dq=dq.cpu(), dk=dk.cpu()), %r)") % (os.path.dirname(HERE), path, path + ".out")
    subprocess.run([sys.executable, "-c", code], check=True, env=dict(os.environ, CCA_B200_PDL="0"))
    got = torch.load(path + ".out")
    os.remove(path)
    os.remove(path + ".out")
    assert torch.equal(got["a"], runs[0][0].cpu())
    assert torch.equal(got["dq"], runs[0][1].cpu()) and torch.equal(got["dk"], runs[0][2].cpu())


@pytest.mark.parametrize("dtype", [capi.CCA_BF16, capi.CCA_F16])
def test_16bit_deterministic_tiled_backward_is_refused(dtype):
    dev = _dev()
    lib = capi.load()
    B, Cq, H, W = 1, 16, 129, 129
    q = torch.zeros(B, Cq, H, W, dtype=torch.bfloat16, device=dev).contiguous(memory_format=torch.channels_last)
    a = torch.zeros(B, H, W, H + W, device=dev)
    flags = capi.CCA_FLAG_NHWC | capi.CCA_FLAG_DETERMINISTIC
    ws = torch.empty(lib.cca_b200_attention_workspace_bytes(1, B, Cq, H, W, dtype, flags), dtype=torch.uint8, device=dev)
    rc = lib.cca_b200_attention_backward(a.data_ptr(), a.data_ptr(), q.data_ptr(), q.data_ptr(), q.data_ptr(), q.data_ptr(),
                                         ws.data_ptr(), ws.numel(), B, Cq, H, W, dtype, flags, None)
    assert rc == -2 and b"DETERMINISTIC" in lib.cca_b200_last_error()


def test_map_past_2_31_elements_matches_the_oracle_on_sampled_pixels():
    """forward and backward with every index into the map past 2^31: rows of the map, dq of query pixels and dk of key
    pixels, each against fp64 from the map the kernel wrote (the forward rows are checked against q, k first)"""
    dev = _dev()
    B, Cq, H, W = 2, 16, 896, 896
    assert B * H * W * (H + W) > 2 ** 31
    g = torch.Generator(device=dev).manual_seed(7)
    q, k = (torch.randn(B, Cq, H, W, device=dev, generator=g) * 0.5 for _ in range(2))
    attn = cca_attention_forward(q, k)
    pix = ((1, 895, 895), (1, 700, 3), (0, 0, 0), (1, 448, 600))
    qd, kd = q.double(), k.double()
    for b, h, w in pix:
        col = qd[b, :, h, w] @ kd[b, :, :, w]
        col[h] = float("-inf")
        ref = torch.softmax(torch.cat([col, qd[b, :, h, w] @ kd[b, :, h, :]]), 0)
        assert (attn[b, h, w].double() - ref).abs().max().item() < 1e-5
    dattn = torch.randn(attn.shape, device=dev, generator=g)
    dq, dk = cca_attention_backward(dattn, attn, q, k)
    ds = lambda a, d: a.double() * (d.double() - (a.double() * d.double()).sum(-1, keepdim=True))   # rows of dS
    for b, h, w in pix:
        s = ds(attn[b, h, w], dattn[b, h, w])
        s[h] = 0
        ref = kd[b, :, :, w] @ s[:H] + kd[b, :, h, :] @ s[H:]
        assert (dq[b, :, h, w].double() - ref).abs().max().item() <= 1e-4 * max(1.0, ref.abs().max().item())
        y, x = h, w                                    # the same pixels as keys: column queries (i, x), row queries (y, j)
        sc = ds(attn[b, :, x], dattn[b, :, x])[:, y]
        sc[y] = 0
        sr = ds(attn[b, y], dattn[b, y])[:, H + x]
        ref = qd[b, :, :, x] @ sc + qd[b, :, y, :] @ sr
        assert (dk[b, :, y, x].double() - ref).abs().max().item() <= 1e-4 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("impl", ["tc", "simt"])
def test_backward_takes_attn_and_dattn_at_any_float_offset(impl):
    """attn and dattn are caller tensors: views at an odd element offset (e.g. from the backward of torch.cat) give the
    bits of aligned copies"""
    dev = _dev()
    shape = (2, 32, 37, 30)                            # H + W odd: rows alternate between 8-byte aligned and not
    q, k, da = (t.to(dev) for t in _inputs(shape, torch.float32, seed=9))
    attn = cca_attention_forward(q, k, impl)
    ref = cca_attention_backward(da, attn, q, k, impl)
    odd = lambda t: torch.empty(t.numel() + 1, device=dev)[1:].view(t.shape).copy_(t)
    for a, d in ((attn, odd(da)), (odd(attn), da), (odd(attn), odd(da))):
        assert (a.data_ptr() | d.data_ptr()) % 8 == 4
        got = cca_attention_backward(d, a, q, k, impl)
        assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])
    torch.cuda.synchronize()


def test_tensor_core_module_map_and_gradients_match_the_oracle_module():
    """the module on the tensor-core map kernels (C = 128: Cq = 16), fp32 with TF32 off, against fp64 autograd of the
    oracle module's convs and the oracle map: RCCA with two steps, a loss on both maps"""
    from oracle.cca_oracle import CrissCrossAttentionOracle
    dev = _dev()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.manual_seed(10)
    ref = CrissCrossAttentionOracle(128)
    with torch.no_grad():
        ref.gamma.fill_(0.6)
    m = ccnet_b200.RCCA(128, recurrence=2).to(dev)
    m.cca.load_state_dict(ref.state_dict())
    B, H, W = 2, 21, 18
    assert ccnet_b200.functional.attention_tc_eligible(B, 16, H, W, torch.float32)
    x = torch.randn(B, 128, H, W)
    rs = [torch.randn(B, H, W, H + W) for _ in range(2)]
    xd = x.to(dev).requires_grad_(True)
    _, maps = m(xd, return_attention=True)
    sum((a * r.to(dev)).sum() for a, r in zip(maps, rs)).backward()
    r64 = ref.double()
    xr = x.double().requires_grad_(True)
    y, loss, refs = xr, 0, []
    for r in rs:
        a = AB.attention_map(r64.query_conv(y), r64.key_conv(y))
        refs.append(a.detach())
        loss = loss + (a * r.double()).sum()
        y = r64(y)
    loss.backward()
    for a, ra in zip(maps, refs):
        assert (a.detach().cpu().double() - ra).abs().max().item() < 1e-5
    rel = lambda got, want: (got.cpu().double() - want).abs().max().item() / max(1.0, want.abs().max().item())
    assert rel(xd.grad, xr.grad) < 1e-4
    for n, p in m.cca.named_parameters():
        want = dict(r64.named_parameters())[n].grad
        if want is not None:
            assert rel(p.grad, want) < 1e-4, n


def test_torch_ops_opcheck_and_compile_without_graph_break():
    """opcheck on both ops, with the autograd registration of cca::attention.  torch.compile(fullgraph=True) covers what
    return_attention adds to a step -- the convs and the map op; the module picks its y path with a ctypes coverage query
    that dynamo does not trace (INTEGRATION.md section 3), so the module as a whole is not compiled fullgraph here."""
    dev = _dev()
    q, k, da = (t.to(dev) for t in _inputs((2, 16, 9, 11), torch.float32, seed=8))
    torch.library.opcheck(torch.ops.cca.attention.default, (q, k), test_utils=("test_schema", "test_faketensor"))
    torch.library.opcheck(torch.ops.cca.attention.default, (q.clone().requires_grad_(True), k.clone().requires_grad_(True)),
                          test_utils=("test_autograd_registration",))
    a = torch.ops.cca.attention(q, k)
    torch.library.opcheck(torch.ops.cca.attention_backward.default, (da, a, q, k), test_utils=("test_schema", "test_faketensor"))
    assert torch.equal(a, cca_attention(q, k))
    m = ccnet_b200.CrissCrossAttention(128).to(dev)
    x = torch.randn(2, 128, 9, 11, device=dev)
    y0, a0 = m(x, return_attention=True)

    def step_map(x):                         # what return_attention adds to the step: the convs and the map op
        return torch.ops.cca.attention(m.query_conv(x), m.key_conv(x), m.impl)
    a1 = torch.compile(step_map, fullgraph=True)(x)             # fullgraph: a graph break raises
    assert torch.allclose(a0, a1, atol=1e-6)
