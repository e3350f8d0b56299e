"""What causal criss-cross attention over clips costs, and what its streaming step saves.

At the clip shapes of tools/cca3d_cost.py (tensor-core kernels, C = 512 or 256, Cq = C / 8; fp32 and bf16): the causal and
the bidirectional ``cca3d_forward`` / ``cca3d_backward``, alternated in one run.  Then ``cca3d_step`` with S = 7 and S = 31
cached frames against ``cca3d_forward(causal=True)`` on S + 1 frames, the recompute-the-window alternative that produces the
same new frame.  Last, the module: ``CrissCrossAttention3D(C, causal=True).step`` (projections, the step, the cache
update) against the module's forward on the S + 1 frames (fp32, no grad).  CUDA events, the L2 flushed before every call,
mean and min over ``--iters`` calls after warm-up.  The card's
name and power limit are in every line.

    python tools/cca3d_causal_cost.py --out profiles/h100_cca3d_causal.jsonl
"""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

from cca3d_cost import SHAPES  # noqa: E402
from deterministic_cost import card, events  # noqa: E402

# (B, C, H, W) of the step; S cached frames
STEP_SHAPES = [(1, 512, 97, 97), (2, 512, 65, 65), (1, 256, 129, 129)]
STEP_S = (7, 31)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_cca3d_causal.jsonl")
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    from ccnet_b200.functional import cca3d_backward, cca3d_forward, cca3d_step
    dev = torch.device("cuda:0")
    info = card()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    lines = []

    def emit(rec):
        rec = dict(info, **rec)
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    def clip(B, Cq, C, T, H, W, dtype):
        g = torch.Generator(device=dev).manual_seed(0)
        mk = lambda c, s=1.0: (torch.randn(B, c, T, H, W, device=dev, generator=g).mul_(s).to(dtype)
                               .contiguous(memory_format=torch.channels_last_3d))
        return mk(Cq, 0.5), mk(Cq, 0.5), mk(C), mk(C)

    for B, C, T, H, W in SHAPES:
        Cq = C // 8
        for dtype in (torch.float32, torch.bfloat16):
            q, k, v, dout = clip(B, Cq, C, T, H, W, dtype)
            shape = dict(shape=[B, C, T, H, W], dtype=str(dtype).split(".")[-1])
            saved = {c: cca3d_forward(q, k, v, "tc", causal=c) for c in (False, True)}
            for causal in (False, True, False, True):            # alternated: the spread of one mode shows in its repeat
                out, lse = saved[causal]
                for what, fn in (("forward3d", lambda: cca3d_forward(q, k, v, "tc", causal=causal)),
                                 ("backward3d", lambda: cca3d_backward(dout, q, k, v, out, lse, "tc", causal=causal))):
                    mean, best = events(fn, args.iters, flush)
                    emit(dict(shape, what=what, causal=causal, ms_mean=round(mean, 4), ms_min=round(best, 4)))
            del q, k, v, dout, saved

    for B, C, H, W in STEP_SHAPES:
        Cq = C // 8
        for dtype in (torch.float32, torch.bfloat16):
            for S in STEP_S:
                q, k, v, _ = clip(B, Cq, C, S + 1, H, W, dtype)
                frame = lambda t: t[:, :, S].contiguous(memory_format=torch.channels_last)
                qf, kf, vf = frame(q), frame(k), frame(v)
                kc, vc = (t[:, :, :S].contiguous(memory_format=torch.channels_last_3d) for t in (k, v))
                shape = dict(shape=[B, C, H, W], S=S, dtype=str(dtype).split(".")[-1])
                for what, fn in (("step", lambda: cca3d_step(qf, kf, vf, kc, vc, "tc")),
                                 ("window_forward3d", lambda: cca3d_forward(q, k, v, "tc", causal=True)),
                                 ("step", lambda: cca3d_step(qf, kf, vf, kc, vc, "tc")),
                                 ("window_forward3d", lambda: cca3d_forward(q, k, v, "tc", causal=True))):
                    mean, best = events(fn, args.iters, flush)
                    emit(dict(shape, what=what, ms_mean=round(mean, 4), ms_min=round(best, 4)))
                del q, k, v, qf, kf, vf, kc, vc

    from ccnet_b200 import CrissCrossAttention3D
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    for B, C, H, W in STEP_SHAPES:
        m = CrissCrossAttention3D(C, causal=True).to(dev).eval()
        for S in STEP_S:
            g = torch.Generator(device=dev).manual_seed(0)
            x = torch.randn(B, C, S + 1, H, W, device=dev, generator=g).contiguous(memory_format=torch.channels_last_3d)
            frames = [x[:, :, t].contiguous(memory_format=torch.channels_last) for t in range(S + 1)]
            with torch.no_grad():
                state = None
                for t in range(S):
                    _, state = m.step(frames[t], state)
                shape = dict(shape=[B, C, H, W], S=S, dtype="float32")
                for what, fn in (("module_step", lambda: m.step(frames[S], state)), ("module_window_forward", lambda: m(x)),
                                 ("module_step", lambda: m.step(frames[S], state)), ("module_window_forward", lambda: m(x))):
                    mean, best = events(fn, args.iters, flush)
                    emit(dict(shape, what=what, ms_mean=round(mean, 4), ms_min=round(best, 4)))
            del x, frames, state
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        for r in lines:
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
