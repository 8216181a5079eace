"""Classifier-head cost: dfd_head_fwd (with the fused loss) + dfd_head_bwd, and the whole B0 train step at K = 2 vs K = 1000.

    python tools/head_time.py [--iters 200] [--steps 20] [--rounds 3]

1. The head alone at N = 256 for (F, K) in {(1280, 2), (1280, 5), (1280, 1000), (2048, 1000)}: CUDA events around
   `--iters` launches of forward + backward after a warm-up; prints us per head step and the achieved fp32 rate of the
   three GEMMs (2 N F K flops each) against the H100 SXM data-sheet 67 TFLOP/s (dense fp32).  K = 2 runs the
   one-CTA-per-image kernels, every other K the tiled GEMMs + the log-sum-exp pass.
2. The graph-replayed Trainer step of EfficientNet-B0, batch 256, 224x224, bf16, at K = 2 and K = 1000, alternated in
   one process (`--rounds` windows of `--steps` steps each): ms per step and the difference.
The GPU name and power limit are read in the same run.  Needs a GPU; there is no fallback.
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FP32_PEAK = 67e12        # H100 SXM data sheet, dense fp32


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        power, clk = [s.strip() for s in q.split(",")]
    except Exception as ex:          # the timings stand without it; say so instead of guessing
        power, clk = "unknown (%s)" % ex, "unknown"
    return dict(gpu=name, power_limit_w=power, max_sm_clock_mhz=clk)


def time_head(N, F, K, iters):
    from deepfake_detection_b200 import _lib
    P = lambda t: t.data_ptr()  # noqa: E731
    g = torch.Generator(device="cuda").manual_seed(0)
    pooled = torch.randn(N, F, device="cuda", generator=g).abs()
    W = torch.randn(K, F, device="cuda", generator=g) / math.sqrt(F)
    b = torch.zeros(K, device="cuda")
    y = torch.randint(0, K, (N,), device="cuda", generator=g)
    logits, dlog = torch.zeros(N, K, device="cuda"), torch.zeros(N, K, device="cuda")
    dW, db, dpooled = torch.zeros(K, F, device="cuda"), torch.zeros(K, device="cuda"), torch.zeros(N, F, device="cuda")
    acc = torch.zeros(2, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def step():
        _lib.call("dfd_head_fwd", P(pooled), P(W), P(b), P(logits), N, F, K, P(y), None, 0.0, 1.0, None, P(acc), P(acc) + 4,
                  P(dlog), st)
        _lib.call("dfd_head_bwd", P(dlog), P(pooled), P(W), P(dW), P(db), P(dpooled), N, F, K, st)

    for _ in range(20):
        step()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        step()
    t1.record()
    torch.cuda.synchronize()
    us = t0.elapsed_time(t1) * 1e3 / iters
    flops = 3 * 2.0 * N * F * K
    return dict(N=N, F=F, K=K, us=round(us, 2), tflops=round(flops / us * 1e-6, 3),
                pct_fp32_peak=round(100.0 * flops / (us * 1e-6) / FP32_PEAK, 2))


def time_steps(steps, rounds, batch=256, res=224):
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.models import init_state_dict
    from deepfake_detection_b200.trainer import Trainer
    trs = {}
    for K in (2, 1000):
        tr = Trainer("efficientnet_b0", batch, res, res, dtype="bf16", lr=0.00256, num_classes=K)
        tr.load_state_dict(init_state_dict(get_spec("efficientnet_b0", num_classes=K), seed=42))
        g = torch.Generator(device="cuda").manual_seed(1234)
        tr.engine.set_input(torch.randn(batch, 3, res, res, device="cuda", generator=g))
        tr.engine.set_target(torch.randint(0, K, (batch,), device="cuda", generator=g))
        for _ in range(5):
            tr.step_resident()
        trs[K] = tr
    torch.cuda.synchronize()
    ms = {2: [], 1000: []}
    for _ in range(rounds):
        for K, tr in trs.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(steps):
                tr.step_resident()
            t1.record()
            torch.cuda.synchronize()
            ms[K].append(t0.elapsed_time(t1) / steps)
    med = {K: sorted(v)[len(v) // 2] for K, v in ms.items()}
    out = dict(batch=batch, res=res, dtype="bf16", ms_per_step_k2=[round(v, 3) for v in ms[2]],
               ms_per_step_k1000=[round(v, 3) for v in ms[1000]], median_k2=round(med[2], 3), median_k1000=round(med[1000], 3),
               added_pct=round(100.0 * (med[1000] - med[2]) / med[2], 3))
    # the two step times also differ by what the data does to the clock of a power-capped card; the head's own share of
    # the K = 1000 step comes from the kernel records of a separate profiled window (head_* kernels / all kernels)
    from torch.profiler import ProfilerActivity, profile
    per = {}
    for K, tr in trs.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                tr.step_resident()
            torch.cuda.synchronize()
        per[K] = {ev.key: ev.device_time_total / steps for ev in prof.key_averages() if ev.device_time_total > 0}
    tot = {K: sum(v.values()) for K, v in per.items()}
    head = sum(t for k, t in per[1000].items() if "head_" in k)
    diff = sorted(((per[1000].get(k, 0.0) - per[2].get(k, 0.0), k) for k in set(per[2]) | set(per[1000])), reverse=True)[:6]
    out.update(profiled_kernel_ms_per_step_k2=round(tot[2] / 1e3, 3), profiled_kernel_ms_per_step_k1000=round(tot[1000] / 1e3, 3),
               profiled_head_us_per_step_k1000=round(head, 1), head_share_pct_k1000=round(100.0 * head / tot[1000], 3),
               largest_kernel_increases_us=[[k[:90], round(d, 1)] for d, k in diff])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("head_time.py needs a CUDA GPU")
    torch.cuda.set_device(0)
    out = dict(info=gpu_info(), head=[time_head(256, F, K, a.iters) for F, K in ((1280, 2), (1280, 5), (1280, 1000), (2048, 1000))])
    for h in out["head"]:
        print("head N=%d F=%d K=%d: %.2f us  %.3f TFLOP/s fp32 (%.2f %% of 67)" % (h["N"], h["F"], h["K"], h["us"], h["tflops"], h["pct_fp32_peak"]))
    out["step"] = time_steps(a.steps, a.rounds)
    s = out["step"]
    print("B0 b256 bf16 step: K=2 %.3f ms  K=1000 %.3f ms  (+%.3f %%); K=1000 head kernels %.1f us/step = %.3f %% of kernel time"
          % (s["median_k2"], s["median_k1000"], s["added_pct"], s["profiled_head_us_per_step_k1000"], s["head_share_pct_k1000"]))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
