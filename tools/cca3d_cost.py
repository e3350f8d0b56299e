"""What criss-cross attention over clips (ccnet_b200.cca3d, the 3D op) costs next to the 2D op on the same frames.

At each shape and dtype (fp32 / bf16 / fp16, tensor-core kernels, C = 512 or 256, Cq = C / 8): the 3D op's forward and
backward, and the 2D op's forward and backward on the same B*T frames, with CUDA events and the L2 flushed between iterations;
their difference is what the time branch costs.  Then, in a profiled run of its own, the time-pass kernels' own times
(cca_time_stats / values / bwd) from torch.profiler, next to the bytes the time pass must move (computed from the shape:
forward (2 Cq + 3 C) elements per pixel -- q, k, v read, out read and written --, backward (6 Cq + 4 C) -- q, k, v, dout read,
dq, dk, dv read and written) and their floor at the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s).  The card's name and
power limit are in every line.

    python tools/cca3d_cost.py --out profiles/h100_cca3d.jsonl
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

# (B, C, T, H, W)
SHAPES = [(1, 512, 8, 97, 97), (2, 512, 4, 97, 97), (1, 256, 32, 65, 65), (1, 512, 4, 129, 257)]
HBM = 3.35e12


def _time_kernels(fn, reps=5):
    """{kernel name: mean us per launch} of the cca_time_* kernels over `reps` calls of fn, from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    res = {}
    for e in prof.key_averages():
        if "cca_time_" in e.key:
            name = e.key.split("cca_time_")[1].split("<")[0].split("(")[0]
            total = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            res[name] = res.get(name, 0.0) + total / reps
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_cca3d.jsonl")
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    from ccnet_b200.functional import cca3d_backward, cca3d_forward, cca_backward, cca_forward
    dev = torch.device("cuda:0")
    info = card()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    lines = []

    def emit(rec):
        rec = dict(info, **rec)
        print(json.dumps(rec))
        lines.append(rec)

    for B, C, T, H, W in SHAPES:
        Cq = C // 8
        for dtype in (torch.float32, torch.bfloat16, torch.float16):
            g = torch.Generator(device=dev).manual_seed(0)
            mk = lambda c, s=1.0: (torch.randn(B, c, T, H, W, device=dev, generator=g).mul_(s).to(dtype)
                                   .contiguous(memory_format=torch.channels_last_3d))
            q, k, v, dout = mk(Cq, 0.5), mk(Cq, 0.5), mk(C), mk(C)
            frames = lambda t: t.transpose(1, 2).reshape(B * T, t.shape[1], H, W)      # channels-last views
            q2, k2, v2, d2 = (frames(t) for t in (q, k, v, dout))
            out, lse = cca3d_forward(q, k, v, "tc")
            out2, lse2 = cca_forward(q2, k2, v2, "tc")
            es = torch.finfo(dtype).bits // 8
            npix = B * T * H * W
            shape = dict(shape=[B, C, T, H, W], dtype=str(dtype).split(".")[-1])
            for what, fn in (("forward3d", lambda: cca3d_forward(q, k, v, "tc")),
                             ("backward3d", lambda: cca3d_backward(dout, q, k, v, out, lse, "tc")),
                             ("forward2d_frames", lambda: cca_forward(q2, k2, v2, "tc")),
                             ("backward2d_frames", lambda: cca_backward(d2, q2, k2, v2, out2, lse2, "tc"))):
                mean, best = events(fn, args.iters, flush)
                emit(dict(shape, what=what, ms_mean=round(mean, 4), ms_min=round(best, 4)))
            kf = _time_kernels(lambda: cca3d_forward(q, k, v, "tc"))
            kb = _time_kernels(lambda: cca3d_backward(dout, q, k, v, out, lse, "tc"))
            fwd_bytes, bwd_bytes = (2 * Cq + 3 * C) * es * npix, (6 * Cq + 4 * C) * es * npix
            emit(dict(shape, what="time_pass_forward", us_stats=round(kf.get("stats_kernel", 0.0), 2),
                      us_values=round(kf.get("values_kernel", 0.0), 2), bytes=fwd_bytes,
                      hbm_floor_us=round(fwd_bytes / HBM * 1e6, 2), kernels=sorted(kf)))
            emit(dict(shape, what="time_pass_backward", us_bwd=round(kb.get("bwd_kernel", 0.0), 2), bytes=bwd_bytes,
                      hbm_floor_us=round(bwd_bytes / HBM * 1e6, 2), kernels=sorted(kb)))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        for r in lines:
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
