"""What the attention map (CrissCrossAttention(..., return_attention=True), ccnet_b200.cca_attention) costs, per shape.

Times the map forward (statistics pre-pass + map kernel) and backward (rho pass + item kernel) on the tensor-core kernels,
fp32 / bf16 / fp16 q, k with C = 512 (Cq = 64), CUDA events with the L2 flushed between iterations.  Shapes: B=8 at 97x97
(the benchmark's), B=8 at 128x128, B=1 at 129x257.  Next to each time: the bytes the op must move (computed from the shape:
forward reads q, k and writes the map; backward reads the map and dattn twice -- rho pass and item kernel -- reads q, k and
writes dq, dk) and their share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s), with the card's name and power limit.

    python tools/attention_map_cost.py --out profiles/h100_attention_map.jsonl
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

SHAPES = [(8, 512, 97, 97), (8, 512, 128, 128), (1, 512, 129, 257)]
HBM = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_attention_map.jsonl")
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    from ccnet_b200.functional import cca_attention_backward, cca_attention_forward
    dev = torch.device("cuda:0")
    info = card()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    lines = []
    for B, C, H, W in SHAPES:
        Cq = C // 8
        for dtype in (torch.float32, torch.bfloat16, torch.float16):
            g = torch.Generator(device=dev).manual_seed(0)
            q, k = (torch.randn(B, Cq, H, W, device=dev, generator=g).mul_(0.5).to(dtype)
                    .contiguous(memory_format=torch.channels_last) for _ in range(2))
            attn = cca_attention_forward(q, k, "tc")
            dattn = torch.randn_like(attn)
            es = torch.finfo(dtype).bits // 8
            map_bytes = B * H * W * (H + W) * 4
            qk_bytes = 2 * B * Cq * H * W * es
            for what, fn, nbytes in (
                    ("forward", lambda: cca_attention_forward(q, k, "tc"), qk_bytes + map_bytes),
                    ("backward", lambda: cca_attention_backward(dattn, attn, q, k, "tc"), 4 * map_bytes + 2 * qk_bytes)):
                mean, best = events(fn, args.iters, flush)
                rec = dict(info, shape=[B, C, H, W], dtype=str(dtype).split(".")[-1], what=what, ms_mean=round(mean, 4),
                           ms_min=round(best, 4), bytes=nbytes, hbm_floor_ms=round(nbytes / HBM * 1e3, 4),
                           roofline_fraction=round(nbytes / HBM * 1e3 / mean, 3))
                print(json.dumps(rec))
                lines.append(rec)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        for r in lines:
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
