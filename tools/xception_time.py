"""Train-step time of Xception against ResNet-50, and the kernels Xception adds.

    python tools/xception_time.py [--batch 64] [--r50-batch 256] [--steps 10] [--rounds 3] [--iters 100] [--out FILE]

1. The graph-replayed Trainer step of xception (bf16, 299x299, SGD) at `--batch`, alternated in one process with a resnet50
   Trainer at `--r50-batch`, 224x224 (`--rounds` windows of `--steps` steps each).
2. CUDA events around `--iters` launches (after a warm-up) of the new kernels at Xception's b`--batch` shapes, bf16: the
   depthwise forward with a BN + ReLU input and the fused depthwise backward in its BN + ReLU mode (147x147x128, 74x74x256,
   37x37x728, 19x19x728), the strided block tail dfd_bn_maxpool_add and dfd_maxpool_bn_bwd_reduce (147->74 x128, 74->37 x256,
   37->19 x728, 19->10 x1024). Algorithmic HBM bytes (each tensor read or written once) over the time, against the H100 SXM
   data-sheet 3.35 TB/s.
The GPU name, power limit and max SM clock are read in the same run. Needs a GPU; there is no fallback.
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
from resnet_family_time import _trainer, time_steps  # noqa: E402

HBM_PEAK = 3.35e12       # H100 SXM data sheet
DW_SHAPES = [(147, 128), (74, 256), (37, 728), (19, 728)]
POOL_SHAPES = [(147, 128), (74, 256), (37, 728), (19, 1024)]


def _time(fn, iters):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def time_kernels(N, iters):
    from deepfake_detection_b200 import _lib
    st = torch.cuda.current_stream().cuda_stream
    L = _lib.lib()
    S = L.stat_slots
    out = []

    def rec(name, shape, ms, nbytes):
        out.append(dict(kernel=name, shape=shape, ms=round(ms, 4), bytes=nbytes,
                        hbm_pct=round(100.0 * nbytes / (ms * 1e-3) / HBM_PEAK, 1)))
        print("%-26s %-18s %.4f ms, %.1f %% of 3.35 TB/s" % (name, shape, ms, out[-1]["hbm_pct"]), flush=True)

    for H, C in DW_SHAPES:
        x = torch.randn(N, H, H, C, device="cuda").to(torch.bfloat16)
        y, gy, gx = torch.empty_like(x), torch.randn_like(x), torch.empty_like(x)
        w = torch.randn(C, 9, device="cuda")
        dW = torch.zeros_like(w)
        v = [torch.rand(C, device="cuda") + 0.5 for _ in range(4)]
        s = torch.zeros(2 * S * C, dtype=torch.float64, device="cuda")
        parts = L.cdll.dfd_dwconv_bwd_parts(N, H, H, C, 3, 1)
        cw = L.cdll.dfd_dwconv_block_channels(C)
        ws = torch.empty((C + cw - 1) // cw * parts * cw * 9, device="cuda")
        shape = "%dx%dx%dx%d" % (N, H, H, C)
        ms = _time(lambda: _lib.call("dfd_dwconv_fwd", x.data_ptr(), v[0].data_ptr(), v[1].data_ptr(), w.data_ptr(), y.data_ptr(),
                                     N, H, H, C, 3, 1, 2, 0, None, None, None, st), iters)
        rec("dfd_dwconv_fwd (BN+ReLU)", shape, ms, 4 * x.numel())
        ms = _time(lambda: _lib.call("dfd_dwconv_bwd_relu", gy.data_ptr(), None, None, None, None, w.data_ptr(), x.data_ptr(),
                                     v[0].data_ptr(), v[1].data_ptr(), v[2].data_ptr(), v[3].data_ptr(), None, gx.data_ptr(),
                                     dW.data_ptr(), N, H, H, C, 3, 1, 0, s.data_ptr(), s[S * C:].data_ptr(), ws.data_ptr(),
                                     ws.numel() * 4, None, st), iters)
        rec("dfd_dwconv_bwd_relu (BN)", shape, ms, 6 * x.numel())
        del x, y, gy, gx, ws
    for H, C in POOL_SHAPES:
        Ho = (H - 1) // 2 + 1
        y = torch.randn(N, H, H, C, device="cuda").to(torch.bfloat16)
        gx = torch.empty_like(y)
        ys = torch.randn(N, Ho, Ho, C, device="cuda").to(torch.bfloat16)
        o, gy = torch.empty_like(ys), torch.randn_like(ys)
        idx = torch.empty(ys.shape, dtype=torch.uint8, device="cuda")
        v = [torch.rand(C, device="cuda") + 0.5 for _ in range(4)]
        s = torch.zeros(2 * S * C, dtype=torch.float64, device="cuda")
        shape = "%dx%dx%dx%d" % (N, H, H, C)
        ms = _time(lambda: _lib.call("dfd_bn_maxpool_add", y.data_ptr(), v[0].data_ptr(), v[1].data_ptr(), ys.data_ptr(),
                                     v[2].data_ptr(), v[3].data_ptr(), o.data_ptr(), idx.data_ptr(), N, H, H, C, 0, st), iters)
        rec("dfd_bn_maxpool_add", shape, ms, 2 * y.numel() + 5 * ys.numel())
        ms = _time(lambda: _lib.call("dfd_maxpool_bn_bwd_reduce", gy.data_ptr(), idx.data_ptr(), y.data_ptr(), v[0].data_ptr(),
                                     v[1].data_ptr(), gx.data_ptr(), N, H, H, C, 0, s.data_ptr(), s[S * C:].data_ptr(), st), iters)
        rec("dfd_maxpool_bn_bwd_reduce", shape, ms, 4 * y.numel() + 3 * ys.numel())
        del y, gx, ys, o, gy, idx
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--r50-batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("xception_time.py needs a CUDA GPU")
    torch.cuda.set_device(0)
    out = dict(info=gpu_info(), dtype="bf16")
    print(json.dumps(out["info"]), flush=True)
    out["kernels"] = time_kernels(a.batch, a.iters)
    trs = {"xception": _trainer("xception", a.batch, 299), "resnet50": _trainer("resnet50", a.r50_batch, 224)}
    r = time_steps(trs, a.steps, a.rounds)
    out["steps"] = dict(xception=dict(batch=a.batch, res=299, **r["xception"]),
                        resnet50=dict(batch=a.r50_batch, res=224, **r["resnet50"]))
    for k, b in (("xception", a.batch), ("resnet50", a.r50_batch)):
        print("%-9s b%d: %.3f ms/step (%.0f img/s)" % (k, b, r[k]["median"], b / r[k]["median"] * 1e3), flush=True)
    print(json.dumps(out))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f)


if __name__ == "__main__":
    main()
