"""What the deterministic mode (torch.use_deterministic_algorithms / CCA_FLAG_DETERMINISTIC) costs, per shape.

Times, in the default and in the deterministic mode:
  - the op forward and backward (fp32, tensor-core kernels), CUDA events with the L2 flushed between iterations, as bench.py's
    op_time does;
  - the module's fwd + bwd step (CrissCrossAttention, fp32 and under fp16 autocast), CUDA events around whole steps.
Shapes: B=8, C=512 at 97x97 (one tile per line: the mode changes nothing there but the weight gradient), 64x128 and 128x128;
B=1, C=512 at 129x257.  One JSON line per (shape, what) goes to --out, with the card's name and power limit.

    python tools/deterministic_cost.py --out profiles/h100_deterministic.jsonl

cuBLAS (the autocast step's projections) only runs deterministically with CUBLAS_WORKSPACE_CONFIG set, so this script sets
:4096:8 for both modes unless the environment already has a value.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

SHAPES = [(8, 512, 97, 97), (8, 512, 64, 128), (8, 512, 128, 128), (1, 512, 129, 257)]


def card():
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit",
                        "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (q.stdout.strip().split(", ") + ["?", "?"])[:2] if q.returncode == 0 else (torch.cuda.get_device_name(), "?")
    return {"gpu": name, "power_limit": power}


def events(fn, iters, flush=None):
    """mean and min ms of fn() over iters timed calls, after 3 warm-up calls"""
    for _ in range(3):
        fn()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.zero_()
            torch.cuda._sleep(300000)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sum(ts) / len(ts), min(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_deterministic.jsonl")
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    from ccnet_b200 import CrissCrossAttention, cca_backward, cca_forward
    assert torch.cuda.is_available(), "needs an H100"
    dev = torch.device("cuda")
    meta = card()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)       # > the 50 MB L2
    lines = []
    for B, C, H, W in SHAPES:
        g = torch.Generator(device=dev).manual_seed(0)
        cl = torch.channels_last
        q, k = (torch.randn(B, C // 8, H, W, device=dev, generator=g).contiguous(memory_format=cl) * 0.7 for _ in range(2))
        v, do = (torch.randn(B, C, H, W, device=dev, generator=g).contiguous(memory_format=cl) for _ in range(2))
        row = {"shape": [B, C, H, W], **meta}
        out, lse = cca_forward(q, k, v, impl="tc")
        for det in (False, True):
            tag = "deterministic" if det else "default"
            f = events(lambda: cca_forward(q, k, v, impl="tc", deterministic=det), args.iters, flush)
            b = events(lambda: cca_backward(do, q, k, v, out, lse, impl="tc", deterministic=det), args.iters, flush)
            row[f"op_fwd_ms_{tag}"], row[f"op_bwd_ms_{tag}"] = round(f[0], 4), round(b[0], 4)
        line = dict(row, what="op fp32 (L2 flushed)")
        for amp in (False, True):
            torch.manual_seed(0)
            m = CrissCrossAttention(C).to(dev)
            with torch.no_grad():
                m.gamma.fill_(0.5)
            x = torch.randn(B, C, H, W, device=dev).contiguous(memory_format=cl).requires_grad_(True)
            dy = torch.randn(B, C, H, W, device=dev)

            def step():
                with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
                    y = m(x)
                y.backward(dy.to(y.dtype))
            key = "module_fp16_autocast" if amp else "module_fp32"
            for det in (False, True):
                torch.use_deterministic_algorithms(det)
                try:
                    line[f"{key}_step_ms_{'deterministic' if det else 'default'}"] = round(events(step, args.iters)[0], 4)
                finally:
                    torch.use_deterministic_algorithms(False)
        for k_ in [k_ for k_ in line if k_.endswith("_default")]:
            base = k_[:-len("_default")]
            line[base + "_ratio"] = round(line[base + "_deterministic"] / line[k_], 3)
        lines.append(line)
        print(json.dumps(line), flush=True)
        del q, k, v, do, out, lse
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        for line in lines:
            fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
