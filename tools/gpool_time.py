"""Global-pool cost: forward + backward of every pool type, and the whole B0 train step at avg vs catavgmax.

    python tools/gpool_time.py [--iters 200] [--steps 20] [--rounds 3] [--out FILE]

1. The pool alone, forward + backward, for each type at EfficientNet-B0 b256 (7x7x1280, Swish on load; backward with the
   BatchNorm sums: dfd_pool + dfd_act_bwd for avg, dfd_global_pool + dfd_act_bwd_gpool otherwise), ResNet-50 b256 (7x7x2048;
   dfd_pool + dfd_pool_bwd / dfd_global_pool + dfd_gpool_bwd) and deepfake_v4 b3 (19x19x256, the chunked small-batch path):
   CUDA events around `--iters` launches after a warm-up; us per forward + backward and the HBM rate of the bytes the pair
   must move (16-bit tensor read twice, gradient written once) against the H100 SXM data-sheet 3.35 TB/s.
2. The graph-replayed Trainer step of EfficientNet-B0, batch 256, 224x224, bf16, K = 2, at avg and catavgmax, alternated
   in one process (`--rounds` windows of `--steps` steps each): ms per step and the difference.
The GPU name, power limit and max SM clock are read in the same run.  Needs a GPU; there is no fallback.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from head_time import gpu_info  # noqa: E402

HBM_PEAK = 3.35e12       # H100 SXM data sheet
CASES = (("efficientnet_b0", 256, 49, 1280, True), ("resnet50", 256, 49, 2048, False), ("efficientnet_deepfake_v4", 3, 361, 256, True))


def time_pool(arch, N, hw, C, swish, pool_type, iters):
    from deepfake_detection_b200 import _lib
    P = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    g = torch.Generator(device="cuda").manual_seed(0)
    y = torch.randn(N, hw, C, device="cuda", generator=g).to(torch.bfloat16)
    scale = 0.5 + torch.rand(C, device="cuda", generator=g) if swish else None
    shift = 0.1 * torch.randn(C, device="cuda", generator=g) if swish else None
    mean, rstd = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
    Pw = 2 * C if pool_type == "catavgmax" else C
    pooled, dpooled = torch.zeros(N, Pw, device="cuda"), torch.randn(N, Pw, device="cuda", generator=g)
    am = torch.zeros(N, C, dtype=torch.int32, device="cuda")
    gout = torch.empty_like(y)
    s1, s2 = torch.zeros(8 * C, dtype=torch.float64, device="cuda"), torch.zeros(8 * C, dtype=torch.float64, device="cuda")
    act = _lib.ACT_SWISH if swish else _lib.ACT_NONE
    pt = _lib.POOL_TYPES[pool_type]
    st = torch.cuda.current_stream().cuda_stream

    def step():
        if pool_type == "avg":
            _lib.call("dfd_pool", P(y), P(scale), P(shift), P(pooled), N, hw, C, act, _lib.DT_BF16, None, 8, st)
        else:
            _lib.call("dfd_global_pool", P(y), P(scale), P(shift), P(pooled), P(am), N, hw, C, act, pt, _lib.DT_BF16, 8, st)
        if swish and pool_type == "avg":
            _lib.call("dfd_act_bwd", None, P(y), P(scale), P(shift), P(mean), P(rstd), None, P(dpooled), P(gout), N, hw, C,
                      act, _lib.DT_BF16, P(s1), P(s2), None, st)
        elif swish:
            _lib.call("dfd_act_bwd_gpool", P(y), P(scale), P(shift), P(mean), P(rstd), P(dpooled), P(am), P(gout), N, hw, C,
                      act, pt, _lib.DT_BF16, P(s1), P(s2), None, st)
        elif pool_type == "avg":
            _lib.call("dfd_pool_bwd", P(dpooled), P(gout), N, hw, C, _lib.DT_BF16, st)
        else:
            _lib.call("dfd_gpool_bwd", P(dpooled), P(am), P(gout), N, hw, C, pt, _lib.DT_BF16, st)

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
    # swish: y read by the pool and by the backward, gu written; none: y read by the pool, gradient written
    nbytes = N * hw * C * 2 * (3 if swish else 2)
    return dict(arch=arch, N=N, hw=hw, C=C, pool=pool_type, us=round(us, 2),
                hbm_pct=round(100.0 * nbytes / (us * 1e-6) / HBM_PEAK, 1))


def time_steps(steps, rounds, batch=256, res=224):
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.models import init_state_dict
    from deepfake_detection_b200.trainer import Trainer
    trs = {}
    for gp in ("avg", "catavgmax"):
        tr = Trainer("efficientnet_b0", batch, res, res, dtype="bf16", lr=0.00256, num_classes=2, global_pool=gp)
        tr.load_state_dict(init_state_dict(get_spec("efficientnet_b0", num_classes=2, global_pool=gp), seed=42))
        g = torch.Generator(device="cuda").manual_seed(1234)
        tr.engine.set_input(torch.randn(batch, 3, res, res, device="cuda", generator=g))
        tr.engine.set_target(torch.randint(0, 2, (batch,), device="cuda", generator=g))
        for _ in range(5):
            tr.step_resident()
        trs[gp] = tr
    torch.cuda.synchronize()
    ms = {gp: [] for gp in trs}
    for _ in range(rounds):
        for gp, tr in trs.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(steps):
                tr.step_resident()
            t1.record()
            torch.cuda.synchronize()
            ms[gp].append(t0.elapsed_time(t1) / steps)
    med = {gp: sorted(v)[len(v) // 2] for gp, v in ms.items()}
    return dict(batch=batch, res=res, dtype="bf16", ms_per_step_avg=[round(v, 3) for v in ms["avg"]],
                ms_per_step_catavgmax=[round(v, 3) for v in ms["catavgmax"]], median_avg=round(med["avg"], 3),
                median_catavgmax=round(med["catavgmax"], 3),
                added_pct=round(100.0 * (med["catavgmax"] - med["avg"]) / med["avg"], 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gpool_time.py needs a CUDA GPU")
    torch.cuda.set_device(0)
    out = dict(info=gpu_info(), pool=[])
    for arch, N, hw, C, swish in CASES:
        for gp in ("avg", "max", "avgmax", "catavgmax"):
            r = time_pool(arch, N, hw, C, swish, gp, a.iters)
            out["pool"].append(r)
            print("%s N=%d hw=%d C=%d %-9s fwd+bwd %8.2f us  %5.1f %% of 3.35 TB/s" % (arch, N, hw, C, gp, r["us"], r["hbm_pct"]))
    out["step"] = time_steps(a.steps, a.rounds)
    s = out["step"]
    print("B0 b256 bf16 step: avg %.3f ms  catavgmax %.3f ms  (%+.3f %%)" % (s["median_avg"], s["median_catavgmax"], s["added_pct"]))
    print(json.dumps(out))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f)


if __name__ == "__main__":
    main()
