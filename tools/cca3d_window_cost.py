"""What a time window costs in causal criss-cross attention over clips, and what the module's ring-buffer step saves.

(a) At the clip shapes of tools/cca3d_cost.py (tensor-core kernels, C = 512 or 256, Cq = C / 8; fp32 and bf16): the
    windowed (W = 3) and the unwindowed causal ``cca3d_forward`` / ``cca3d_backward``, alternated in one run.
(b) ``CrissCrossAttention3D(512, causal=True, window=W).step`` (projections, the step on a ring of W frames, the write of
    one frame into it) against ``CrissCrossAttention3D(512, causal=True).step(..., max_frames=W)`` (the same step on a cache
    that each call rewrites), both with full caches, at W = 7 and 31, 1x512x97x97 fp32, no grad, alternated.
(c) The generic kernels' windowed forward and backward on one long clip (1x64x2048x8x8, W = 16), which has no unwindowed
    counterpart there (H + W + T - 2 > 2048).
CUDA events, the L2 flushed before every call, mean and min over ``--iters`` calls after warm-up.  The card's name and
power limit are in every line.

    python tools/cca3d_window_cost.py --out profiles/h100_cca3d_window.jsonl
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

CLIP_WINDOW = 3
RING_SHAPE, RING_WINDOWS = (1, 512, 97, 97), (7, 31)
LONG_CLIP, LONG_WINDOW = (1, 64, 2048, 8, 8), 16


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_cca3d_window.jsonl")
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    from ccnet_b200 import CrissCrossAttention3D
    from ccnet_b200.functional import cca3d_backward, cca3d_forward
    dev = torch.device("cuda:0")
    info = card()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    lines = []

    def emit(rec):
        rec = dict(info, **rec)
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    def clip(B, Cq, C, T, H, W, dtype, fmt=torch.channels_last_3d):
        g = torch.Generator(device=dev).manual_seed(0)
        mk = lambda c, s=1.0: torch.randn(B, c, T, H, W, device=dev, generator=g).mul_(s).to(dtype).contiguous(memory_format=fmt)
        return mk(Cq, 0.5), mk(Cq, 0.5), mk(C), mk(C)

    # (a) the windowed against the unwindowed causal op on the tensor cores
    for B, C, T, H, W in SHAPES:
        Cq = C // 8
        for dtype in (torch.float32, torch.bfloat16):
            q, k, v, dout = clip(B, Cq, C, T, H, W, dtype)
            shape = dict(shape=[B, C, T, H, W], dtype=str(dtype).split(".")[-1])
            saved = {w: cca3d_forward(q, k, v, "tc", causal=True, window=w) for w in (None, CLIP_WINDOW)}
            for window in (None, CLIP_WINDOW, None, CLIP_WINDOW):          # alternated
                out, lse = saved[window]
                for what, fn in (("forward3d", lambda: cca3d_forward(q, k, v, "tc", causal=True, window=window)),
                                 ("backward3d", lambda: cca3d_backward(dout, q, k, v, out, lse, "tc", causal=True, window=window))):
                    mean, best = events(fn, args.iters, flush)
                    emit(dict(shape, what=what, window=window or 0, ms_mean=round(mean, 4), ms_min=round(best, 4)))
            del q, k, v, dout, saved

    # (b) the module's ring step against its copying step, both with W frames cached
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    B, C, H, W = RING_SHAPE
    for window in RING_WINDOWS:
        torch.manual_seed(0)
        copy = CrissCrossAttention3D(C, causal=True).to(dev).eval()
        ring = CrissCrossAttention3D(C, causal=True, window=window).to(dev).eval()
        ring.load_state_dict(copy.state_dict())
        g = torch.Generator(device=dev).manual_seed(0)
        frames = [torch.randn(B, C, H, W, device=dev, generator=g).contiguous(memory_format=torch.channels_last)
                  for _ in range(window + 1)]
        with torch.no_grad():
            sc = sr = None
            for t in range(window):
                _, sc = copy.step(frames[t], sc, max_frames=window)
                _, sr = ring.step(frames[t], sr)
            yc, _ = copy.step(frames[window], sc, max_frames=window)
            yr, _ = ring.step(frames[window], sr)          # (writes one slot in place: the timed calls rewrite that slot)
            diff = (yc - yr).abs().max().item()
            shape = dict(shape=[B, C, H, W], window=window, dtype="float32")
            for what, fn in (("module_step_copy", lambda: copy.step(frames[window], sc, max_frames=window)),
                             ("module_step_ring", lambda: ring.step(frames[window], sr)),
                             ("module_step_copy", lambda: copy.step(frames[window], sc, max_frames=window)),
                             ("module_step_ring", lambda: ring.step(frames[window], sr))):
                mean, best = events(fn, args.iters, flush)
                emit(dict(shape, what=what, max_abs_diff=diff, ms_mean=round(mean, 4), ms_min=round(best, 4)))
        del copy, ring, frames, sc, sr

    # (c) the generic windowed op on a clip the unwindowed generic kernels do not take
    B, C, T, H, W = LONG_CLIP
    q, k, v, dout = clip(B, C // 8, C, T, H, W, torch.float32, torch.contiguous_format)
    out, lse = cca3d_forward(q, k, v, "simt", causal=True, window=LONG_WINDOW)
    shape = dict(shape=[B, C, T, H, W], window=LONG_WINDOW, dtype="float32")
    for what, fn in (("simt_forward3d", lambda: cca3d_forward(q, k, v, "simt", causal=True, window=LONG_WINDOW)),
                     ("simt_backward3d", lambda: cca3d_backward(dout, q, k, v, out, lse, "simt", causal=True, window=LONG_WINDOW))) * 2:
        mean, best = events(fn, args.iters, flush)
        emit(dict(shape, what=what, ms_mean=round(mean, 4), ms_min=round(best, 4)))

    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        for r in lines:
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
