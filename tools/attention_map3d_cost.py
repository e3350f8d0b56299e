"""What the attention map of criss-cross attention over clips (CrissCrossAttention3D(..., return_attention=True),
ccnet_b200.cca3d_attention) costs, per shape.

Times the map forward (2D statistics + time statistics + map kernel + time map kernel) and backward (rho pass + map item
kernel + time map backward) on the tensor-core path, fp32 / bf16 / fp16 q, k with Cq = C / 8, CUDA events with the L2
flushed between iterations.  Shapes B x C x T x H x W: 1x512x8x97x97, 2x512x4x97x97, 1x256x32x65x65, 1x512x4x129x257.
Next to each time: the bytes the op must move (computed from the shape: forward reads q, k and writes the map; backward
reads the map and dattn twice -- rho pass and the item / time kernels -- reads q, k and writes dq, dk) and their share of
the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s), with the card's name and power limit.  bf16 with T > 1 runs its
backward on the fp32 kernels (functional._upcast), which the time includes.

    python tools/attention_map3d_cost.py --out profiles/h100_attention_map3d.jsonl
"""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

from deterministic_cost import card, events  # noqa: E402

SHAPES = [(1, 512, 8, 97, 97), (2, 512, 4, 97, 97), (1, 256, 32, 65, 65), (1, 512, 4, 129, 257)]
HBM = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_attention_map3d.jsonl")
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    from ccnet_b200.functional import cca3d_attention_backward, cca3d_attention_forward
    dev = torch.device("cuda:0")
    info = card()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    lines = []
    for B, C, T, H, W in SHAPES:
        Cq = C // 8
        for dtype in (torch.float32, torch.bfloat16, torch.float16):
            g = torch.Generator(device=dev).manual_seed(0)
            q, k = (torch.randn(B, Cq, T, H, W, device=dev, generator=g).mul_(0.5).to(dtype)
                    .contiguous(memory_format=torch.channels_last_3d) for _ in range(2))
            attn = cca3d_attention_forward(q, k, "tc")
            dattn = torch.randn_like(attn)
            es = torch.finfo(dtype).bits // 8
            map_bytes = B * T * H * W * (H + W + T) * 4
            qk_bytes = 2 * B * Cq * T * H * W * es
            for what, fn, nbytes in (
                    ("forward", lambda: cca3d_attention_forward(q, k, "tc"), qk_bytes + map_bytes),
                    ("backward", lambda: cca3d_attention_backward(dattn, attn, q, k, "tc"), 4 * map_bytes + 2 * qk_bytes)):
                mean, best = events(fn, args.iters, flush)
                rec = dict(info, shape=[B, C, T, H, W], dtype=str(dtype).split(".")[-1], what=what, ms_mean=round(mean, 4),
                           ms_min=round(best, 4), bytes=nbytes, hbm_floor_ms=round(nbytes / HBM * 1e3, 4),
                           roofline_fraction=round(nbytes / HBM * 1e3 / mean, 3))
                print(json.dumps(rec))
                lines.append(rec)
            del attn, dattn
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        for r in lines:
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
