"""H100 tests (``pytest -m gpu``): the fake implementation of every ``torch.ops.cca`` op gives its results the shapes, dtypes
and memory formats of the real call, for channels-last and NCHW-contiguous inputs, on a shape the tensor-core kernels cover
and one they do not, with each ``impl``.  ``torch.compile`` and ``torch.export`` trace with the fakes, so a mismatch would
give a graph strides the real tensors do not have."""
import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

import ccnet_b200  # noqa: F401  (registers torch.ops.cca)
from ccnet_b200.functional import cca3d_attention_forward, cca3d_forward, cca_attention_forward, cca_forward

pytestmark = pytest.mark.gpu
# (B, Cq, C, H, W): the tensor-core kernels cover Cq = 16, C = 64 (op and map), not Cq = 8, C = 24; clips have T = 3 frames
SHAPES = {"covered": (2, 16, 64, 9, 11), "uncovered": (2, 8, 24, 9, 11)}
T = 3
LAYOUTS = ("channels_last", "contiguous")


def _mode3d(impl):                 # forward3d / backward3d: causal and window come before impl
    return () if impl == "auto" else (False, 0, impl)


def _mode(impl):                   # the 2D ops and both maps: impl comes first ("auto" is left to the schema default)
    return () if impl == "auto" else (impl,)


OPS = {
    "forward": lambda t, i: torch.ops.cca.forward(t["q"], t["k"], t["v"], *_mode(i)),
    "backward": lambda t, i: torch.ops.cca.backward(t["do"], t["q"], t["k"], t["v"], t["out"], t["lse"], *_mode(i)),
    "forward_residual": lambda t, i: torch.ops.cca.forward_residual(t["q"], t["k"], t["v"], t["do"], t["gamma"]),
    "attention": lambda t, i: torch.ops.cca.attention(t["q"], t["k"], *_mode(i)),
    "attention_backward": lambda t, i: torch.ops.cca.attention_backward(t["attn"], t["attn"], t["q"], t["k"], *_mode(i)),
    "forward3d": lambda t, i: torch.ops.cca.forward3d(t["q"], t["k"], t["v"], *_mode3d(i)),
    "backward3d": lambda t, i: torch.ops.cca.backward3d(t["do"], t["q"], t["k"], t["v"], t["out"], t["lse"], *_mode3d(i)),
    "attention3d": lambda t, i: torch.ops.cca.attention3d(t["q"], t["k"], *_mode(i)),
    "attention3d_backward": lambda t, i: torch.ops.cca.attention3d_backward(t["attn"], t["attn"], t["q"], t["k"],
                                                                            *_mode(i)),
    # the last frame of the clip, stepped from the caches of the frames before it
    "forward3d_step": lambda t, i: torch.ops.cca.forward3d_step(t["q"][:, :, -1], t["k"][:, :, -1], t["v"][:, :, -1],
                                                                t["k"][:, :, :-1], t["v"][:, :, :-1]),
}
CASES = [(op, impl) for op in OPS for impl in ("auto", "tc", "simt")
         if impl == "auto" or op not in ("forward_residual", "forward3d_step")]     # (these two take no impl)


def _tensors(op, shape, dtype, layout):
    """the op's inputs on the GPU, q, k, v, do and out in ``layout``; out, lse and attn from the forward on the same inputs"""
    B, Cq, C, H, W = shape
    dims = (T, H, W) if "3d" in op else (H, W)
    g = torch.Generator().manual_seed(0)
    t = {n: (torch.randn(B, c, *dims, generator=g) * 0.6).to(dtype).cuda()
         for n, c in (("q", Cq), ("k", Cq), ("v", C), ("do", C))}
    values, attention = (cca3d_forward, cca3d_attention_forward) if "3d" in op else (cca_forward, cca_attention_forward)
    t["out"], t["lse"] = values(t["q"], t["k"], t["v"])
    t["attn"] = attention(t["q"], t["k"])
    t["gamma"] = torch.full((1,), 0.5, device="cuda", dtype=dtype)
    fmt = torch.contiguous_format
    if layout == "channels_last":
        fmt = torch.channels_last_3d if "3d" in op else torch.channels_last
    for n in ("q", "k", "v", "do", "out"):
        t[n] = t[n].contiguous(memory_format=fmt)
    return t


def _results(r):
    return r if isinstance(r, tuple) else (r,)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("op,impl", CASES)
def test_fake_results_have_the_memory_format_of_the_real_ones(op, impl, layout, shape, dtype):
    t = _tensors(op, SHAPES[shape], dtype, layout)
    mode = FakeTensorMode()
    ft = {n: mode.from_tensor(x) for n, x in t.items()}
    if impl == "tc" and shape == "uncovered":            # both refuse the shape
        with pytest.raises(RuntimeError, match="do not cover"):
            OPS[op](t, impl)
        with mode, pytest.raises(RuntimeError, match="do not cover"):
            OPS[op](ft, impl)
        return
    real = _results(OPS[op](t, impl))
    with mode:
        fake = _results(OPS[op](ft, impl))
    assert len(real) == len(fake)
    for i, (r, f) in enumerate(zip(real, fake)):
        assert (f.shape, f.dtype) == (r.shape, r.dtype), i
        fmts = [torch.contiguous_format] + {4: [torch.channels_last], 5: [torch.channels_last_3d]}.get(r.dim(), [])
        assert ([f.is_contiguous(memory_format=m) for m in fmts] == [r.is_contiguous(memory_format=m) for m in fmts]
                and f.stride() == r.stride()), (i, f.stride(), r.stride())


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_differentiable_entry_points_compile_as_one_graph(dtype):
    """cca, cca_attention, cca3d and cca3d_attention are their ops plus traceable checks: torch.compile(fullgraph=True)
    runs forward and backward with the eager bits"""
    from ccnet_b200 import cca, cca3d, cca3d_attention, cca_attention
    t2 = _tensors("forward", SHAPES["covered"], dtype, "channels_last")
    t3 = _tensors("forward3d", SHAPES["covered"], dtype, "contiguous")
    for fn, args in ((cca, (t2["q"], t2["k"], t2["v"])), (cca_attention, (t2["q"], t2["k"])),
                     (lambda q, k, v: cca3d(q, k, v, causal=True, window=1), (t3["q"], t3["k"], t3["v"])),
                     (cca3d_attention, (t3["q"], t3["k"]))):
        torch._dynamo.reset()
        runs = []
        for f in (torch.compile(fn, fullgraph=True), fn):
            xs = [a.clone().requires_grad_(True) for a in args]
            y = f(*xs)
            y.float().sum().backward()
            runs.append([y] + [x.grad for x in xs])
        assert all(torch.equal(a, b) for a, b in zip(*runs))
