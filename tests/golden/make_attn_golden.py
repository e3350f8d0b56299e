"""Generate the attention-map golden vectors by running the UNMODIFIED reference module on CPU.

Run in the build container only (``/root/reference`` does not exist on the GPU box):

    python tests/golden/make_attn_golden.py

Same loading and ``INF`` instance override as ``make_golden.py``.  The map is the reference's softmax output ``concate``
(functions.py:40), captured with a forward hook on ``m.softmax``; it is contiguous [B,H,W,H+W] with the self entry exactly 0.

Each fixture ``attn_<name>.npz`` (NOT ``cca_*``: the ``golden`` fixture of tests/conftest.py globs those) holds, for one seeded
case run R times: x, the 7 reference parameters (p_*), an upstream R_<i> per recurrence step, the maps A_<i>, and dx plus the
7 parameter grads (d_*) of  sum_i sum(A_i * R_i).
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import HERE, REF, cpu_inf, load_reference  # noqa: E402

CASES = [
    # name, B, in_dim, H, W, R, gamma, seed, input scale       (a subset of make_golden.py's cases)
    ("smoke_2x64x5x6", 2, 64, 5, 6, 1, 1.0, 10, 1.0),
    ("r2_2x32x9x7", 2, 32, 9, 7, 2, 0.75, 12, 1.5),
    ("h1_1x16x1x11", 1, 16, 1, 11, 1, 1.0, 13, 1.0),
    ("w1_1x16x13x1", 1, 16, 13, 1, 1, 1.0, 14, 1.0),
]


def run_case(ref, name, B, C, H, W, R, gamma, seed, scale):
    torch.manual_seed(seed)
    m = ref.CrissCrossAttention(C)
    m.INF = cpu_inf(torch.float32)
    with torch.no_grad():
        m.gamma.fill_(gamma)
    maps = []
    m.softmax.register_forward_hook(lambda mod, inp, out: maps.append(out))
    x = (torch.randn(B, C, H, W) * scale).requires_grad_(True)
    y = x
    for _ in range(R):                      # networks/ccnet.py:118-119
        y = m(y)
    ups = [torch.randn_like(a) for a in maps]
    sum((a * u).sum() for a, u in zip(maps, ups)).backward()
    out = {"x": x.detach().numpy(), "R": np.int64(R), "gamma": np.float32(gamma), "dx": x.grad.numpy()}
    for i, (a, u) in enumerate(zip(maps, ups)):
        assert a.is_contiguous() and tuple(a.shape) == (B, H, W, H + W)
        out[f"A_{i}"] = a.detach().numpy()
        out[f"R_{i}"] = u.numpy()
    for n, p in m.named_parameters():
        out["p_" + n] = p.detach().numpy()
        out["d_" + n] = p.grad.numpy() if p.grad is not None else np.zeros_like(p.detach().numpy())
    np.savez_compressed(os.path.join(HERE, f"attn_{name}.npz"), **out)
    print(name, {k_: v_.shape for k_, v_ in out.items() if hasattr(v_, "shape") and v_.ndim})


if __name__ == "__main__":
    if not os.path.isdir(REF):
        sys.exit("reference tree not present; fixtures can only be regenerated in the build container")
    torch.set_num_threads(1)
    ref = load_reference()
    for case in CASES:
        run_case(ref, *case)
