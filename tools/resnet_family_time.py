"""Train-step time of the dense ResNet family against ResNet-50, and the ResNet-D shortcut's average-pool kernels.

    python tools/resnet_family_time.py [--archs resnet101,resnet50d,...] [--batch 256] [--steps 10] [--rounds 3]
                                       [--iters 200] [--out FILE]

1. For each arch: the graph-replayed Trainer step (bf16, 224x224, SGD) at `--batch`, or at the largest of batch, batch/2,
   ... that fits (the batch used is reported), alternated with a ResNet-50 Trainer at the same batch in one process
   (`--rounds` windows of `--steps` steps each). Only one pair of trainers is alive at a time.
2. dfd_avgpool2_fwd / dfd_avgpool2_bwd_add at the three shortcut shapes of ResNet-50-D b256 at 224x224 (56x56x256,
   28x28x512, 14x14x1024, bf16): CUDA events around `--iters` launches after a warm-up; ms per launch and the algorithmic HBM
   rate (fwd 2*NHWC + 2*N*Ho*Wo*C bytes, bwd with a second source 2*N*Ho*Wo*C + 4*NHWC) against the H100 SXM data-sheet
   3.35 TB/s.
The GPU name, power limit and max SM clock are read in the same run. Needs a GPU; there is no fallback.
"""
import argparse
import gc
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from head_time import gpu_info  # noqa: E402

HBM_PEAK = 3.35e12       # H100 SXM data sheet
POOL_SHAPES = [(56, 56, 256), (28, 28, 512), (14, 14, 1024)]


def _trainer(arch, batch, res):
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.models import init_state_dict
    from deepfake_detection_b200.trainer import Trainer
    tr = Trainer(arch, batch, res, res, dtype="bf16", lr=0.00256, num_classes=2)
    tr.load_state_dict(init_state_dict(get_spec(arch, num_classes=2), seed=42))
    g = torch.Generator(device="cuda").manual_seed(1234)
    tr.engine.set_input(torch.randn(batch, 3, res, res, device="cuda", generator=g))
    tr.engine.set_target(torch.randint(0, 2, (batch,), device="cuda", generator=g))
    for _ in range(3):
        tr.step_resident()
    torch.cuda.synchronize()
    return tr


def _pair(arch, batch, res):
    """(trainers, batch) at the largest batch <= `batch` (halving) at which both fit"""
    while batch >= 1:
        trs = None
        try:
            trs = {arch: _trainer(arch, batch, res), "resnet50": _trainer("resnet50", batch, res)}
            return trs, batch
        except torch.cuda.OutOfMemoryError:
            trs = None
            gc.collect()
            torch.cuda.empty_cache()
            batch //= 2
    raise RuntimeError("%s does not fit at batch 1" % arch)


def time_steps(trs, steps, rounds):
    ms = {k: [] for k in trs}
    for _ in range(rounds):
        for k, tr in trs.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(steps):
                tr.step_resident()
            t1.record()
            torch.cuda.synchronize()
            ms[k].append(t0.elapsed_time(t1) / steps)
    return {k: dict(ms=[round(v, 3) for v in vs], median=round(sorted(vs)[len(vs) // 2], 3)) for k, vs in ms.items()}


def time_pool(batch, iters):
    from deepfake_detection_b200 import _lib
    st = torch.cuda.current_stream().cuda_stream
    out = []
    for H, W, C in POOL_SHAPES:
        Ho, Wo = (H + 1) // 2, (W + 1) // 2
        x = torch.randn(batch, H, W, C, device="cuda").to(torch.bfloat16)
        add = torch.randn_like(x)
        dx = torch.empty_like(x)
        y = torch.empty(batch, Ho, Wo, C, device="cuda", dtype=torch.bfloat16)
        calls = {
            "dfd_avgpool2_fwd": (lambda: _lib.call("dfd_avgpool2_fwd", x.data_ptr(), y.data_ptr(), batch, H, W, C, 0, st),
                                 2 * x.numel() + 2 * y.numel()),
            "dfd_avgpool2_bwd_add": (lambda: _lib.call("dfd_avgpool2_bwd_add", y.data_ptr(), add.data_ptr(), dx.data_ptr(), batch,
                                                       H, W, C, 0, st), 2 * y.numel() + 4 * x.numel()),
        }
        for name, (fn, nbytes) in calls.items():
            for _ in range(10):
                fn()
            torch.cuda.synchronize()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(iters):
                fn()
            t1.record()
            torch.cuda.synchronize()
            ms = t0.elapsed_time(t1) / iters
            out.append(dict(kernel=name, N=batch, H=H, W=W, C=C, ms=round(ms, 4), bytes=nbytes,
                            hbm_pct=round(100.0 * nbytes / (ms * 1e-3) / HBM_PEAK, 1)))
            print("%-22s %dx%dx%dx%d bf16: %.4f ms, %.1f %% of 3.35 TB/s" % (name, batch, H, W, C, ms, out[-1]["hbm_pct"]), flush=True)
        del x, add, dx, y
    return out


def main():
    from deepfake_detection_b200.arch import RESNET_ARCHS
    ap = argparse.ArgumentParser()
    ap.add_argument("--archs", default=",".join(RESNET_ARCHS))
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--res", type=int, default=224)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("resnet_family_time.py needs a CUDA GPU")
    torch.cuda.set_device(0)
    out = dict(info=gpu_info(), res=a.res, dtype="bf16", steps=[])
    print(json.dumps(out["info"]), flush=True)
    out["pool"] = time_pool(a.batch, a.iters)
    for arch in a.archs.split(","):
        trs, batch = _pair(arch, a.batch, a.res)
        r = time_steps(trs, a.steps, a.rounds)
        rec = dict(arch=arch, batch=batch, ms_per_step=r[arch]["median"], resnet50_ms_per_step=r["resnet50"]["median"],
                   img_per_s=round(batch / r[arch]["median"] * 1e3, 1), windows=r)
        out["steps"].append(rec)
        print("%-17s b%d bf16 %d^2: %.3f ms/step (%.0f img/s); resnet50 alternated %.3f ms/step"
              % (arch, batch, a.res, rec["ms_per_step"], rec["img_per_s"], rec["resnet50_ms_per_step"]), flush=True)
        del trs
        gc.collect()
        torch.cuda.empty_cache()
    print(json.dumps(out))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f)


if __name__ == "__main__":
    main()
