"""Op forward / backward time per I/O dtype (fp32, bf16, fp16) at the benchmark's attention step (B=8, C=512, 97x97, Cq=64),
and the nn.Module R=2 fwd+bwd step in fp32 and under torch.autocast(float16).

The dtypes alternate inside one process (one timed call of each per round), so clocks and neighbours on a shared machine weigh
on all of them alike.  Every shape is warmed first; the op timings flush the L2 (256 MB) before each call and bracket it with
CUDA events, as bench.py's per-op timings do.  Writes one JSON line per measurement, with the card's name and power limit.
  python tools/op_dtypes.py [--rounds N] [--steps N]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import bench
from ccnet_b200 import RCCA, cca_backward, cca_forward

B, C, Cq, H, W, R = 8, 512, 64, 97, 97, 2
DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}


def card():
    """name and power limit of GPU 0 (read-only query)"""
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, sm = ([c.strip() for c in r.stdout.strip().split(",")] + ["?", "?", "?"])[:3]
    return {"gpu": name, "power_limit": power, "sm_max_clock": sm}


def events(fn, flush=None):
    if flush is not None:
        flush.zero_()
        torch.cuda._sleep(300000)          # the host enqueues the op's launches while the GPU spins: events bracket the kernels
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def stats(ts):
    return {"ms_mean": statistics.mean(ts), "ms_median": statistics.median(ts), "ms_min": min(ts), "n": len(ts)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20, help="timed op calls per dtype and direction")
    ap.add_argument("--steps", type=int, default=10, help="timed module steps per mode")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "op_dtypes.py needs a CUDA device"
    dev = torch.device("cuda:0")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    meta = card()
    peak, peak_src = bench.measured_peaks()
    torch.manual_seed(0)
    cl = torch.channels_last
    base = [torch.randn(B, c, H, W, device=dev) * s for c, s in ((Cq, 0.58), (Cq, 0.58), (C, 0.58), (C, 1.0))]
    ops = {}
    for name, dt in DTYPES.items():
        q, k, v, do = (t.to(dt).contiguous(memory_format=cl) for t in base)
        out, lse = cca_forward(q, k, v)
        ops[name] = (lambda q=q, k=k, v=v: cca_forward(q, k, v),
                     lambda q=q, k=k, v=v, do=do, out=out, lse=lse: cca_backward(do, q, k, v, out, lse))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    for fwd, bwd in ops.values():                  # warm every shape and dtype
        for _ in range(3):
            fwd()
            bwd()
    torch.cuda.synchronize()
    ts = {(n, d): [] for n in DTYPES for d in ("fwd", "bwd")}
    for _ in range(args.rounds):
        for name, (fwd, bwd) in ops.items():
            ts[(name, "fwd")].append(events(fwd, flush))
            ts[(name, "bwd")].append(events(bwd, flush))
    for name, dt in DTYPES.items():
        es = torch.finfo(dt).bits // 8
        for d in ("fwd", "bwd"):
            s = stats(ts[(name, d)])
            nbytes = bench.alg_bytes(B, C, H, W, es, d == "fwd", d == "bwd")
            print(json.dumps(dict(meta, what=f"op_{d}", dtype=name, B=B, C=C, Cq=Cq, H=H, W=W, **s, alg_bytes=nbytes,
                                  frac_of_hbm_peak=nbytes / s["ms_mean"] / 1e6 / peak, hbm_peak_gbs=peak, peak_source=peak_src,
                                  timing="CUDA events, L2 flushed, dtypes alternating")))
    del ops, base, flush
    torch.cuda.empty_cache()

    # ---- the module: R = 2 fwd + bwd in fp32 (the fused path) and under fp16 autocast (projections in fp16, f16 attention)
    model = RCCA(C, recurrence=R).to(dev)
    with torch.no_grad():
        model.cca.gamma.fill_(1.0)
    x = torch.randn(B, C, H, W, device=dev).contiguous(memory_format=cl).requires_grad_(True)
    g = torch.randn(B, C, H, W, device=dev)

    def step(amp):
        with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
            y = model(x)
        (y.float() * g).sum().backward()
        x.grad = None
        model.zero_grad(set_to_none=True)

    for amp in (False, True, False, True):
        step(amp)
    mts = {False: [], True: []}
    for _ in range(args.steps):
        for amp in (False, True):
            mts[amp].append(events(lambda: step(amp)))
    for amp in (False, True):
        s = stats(mts[amp])
        print(json.dumps(dict(meta, what="module_R2_fwd_bwd_step", mode="fp16 autocast" if amp else "fp32", B=B, C=C, H=H, W=W,
                              R=R, **s, pixels_per_s=B * H * W / (s["ms_mean"] * 1e-3),
                              timing="CUDA events around a whole step, modes alternating")))


if __name__ == "__main__":
    main()
