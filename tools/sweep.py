"""BASELINE config 5: resolution sweep H=W in {65,97,129,193}, C=512, R=2 -- op forward / backward time, % of the measured
HBM roofline, and the CPU reference (oracle module port, B=1) beside it.  Writes one JSON line per size.
All four sizes run on the wgmma kernels (channels-last); lines longer than 112 pixels are tiled (csrc/cca_items.cuh)."""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from ccnet_b200 import cca_backward, cca_forward
from ccnet_b200.functional import tc_eligible
import bench

dev = torch.device("cuda:0")
B, C, Cq, R = 8, 512, 64, 2
peak, src = bench.measured_peaks()
cpu = "--no-cpu" not in sys.argv
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
for HW in (65, 97, 129, 193):
    q = torch.randn(B, Cq, HW, HW, device=dev) * 0.58
    k = torch.randn(B, Cq, HW, HW, device=dev) * 0.58
    v = torch.randn(B, C, HW, HW, device=dev) * 0.58
    do = torch.randn(B, C, HW, HW, device=dev)
    tc = tc_eligible(B, Cq, C, HW, HW, torch.float32)
    if tc:
        q, k, v, do = (t.contiguous(memory_format=torch.channels_last) for t in (q, k, v, do))
    out, lse = cca_forward(q, k, v)
    def t_of(fn, n=5):
        for _ in range(2): fn()
        ts = []
        for _ in range(n):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); fn(); e1.record(); torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        return sum(ts) / len(ts)
    tf = t_of(lambda: cca_forward(q, k, v))
    tb = t_of(lambda: cca_backward(do, q, k, v, out, lse))
    bf, bb = bench.alg_bytes(B, C, HW, HW, 4, True, False), bench.alg_bytes(B, C, HW, HW, 4, False, True)
    rec = {"H": HW, "W": HW, "B": B, "C": C, "R": R, "kernels": "wgmma (channels-last)" if tc else "generic (NCHW)",
           "fwd_ms": tf, "bwd_ms": tb, "fwd_frac_of_hbm_peak": bf / tf / 1e6 / peak, "bwd_frac_of_hbm_peak": bb / tb / 1e6 / peak,
           "op_fwd_bwd_pixels_per_s_R2": B * HW * HW / (R * (tf + tb) * 1e-3), "hbm_peak_gbs": peak, "peak_source": src}
    if cpu:
        from oracle.cca_oracle import CrissCrossAttentionOracle, rcca_forward
        torch.set_num_threads(min(16, os.cpu_count() or 1))
        m = CrissCrossAttentionOracle(C)
        with torch.no_grad(): m.gamma.fill_(1.0)
        x = torch.randn(1, C, HW, HW, requires_grad=True)
        best = 1e9
        for _ in range(2):
            t0 = time.perf_counter(); rcca_forward(m, x, R).sum().backward(); best = min(best, time.perf_counter() - t0)
        rec["cpu_module_fwd_bwd_pixels_per_s_R2"] = HW * HW / best
        rec["cpu_threads"] = torch.get_num_threads()
    print(json.dumps(rec))
    del q, k, v, do, out, lse
