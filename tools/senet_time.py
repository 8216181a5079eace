"""Train-step time of SE-ResNet-50 against ResNet-50, and the kernels the SE-ResNets add.

    python tools/senet_time.py [--batch 256] [--steps 10] [--rounds 3] [--iters 100] [--out FILE]

1. The graph-replayed Trainer step of seresnet50 (bf16, 224x224, SGD) at `--batch`, alternated in one process with a resnet50
   Trainer at the same batch (`--rounds` windows of `--steps` steps each).
2. CUDA events around `--iters` launches (after a warm-up) of the new kernels at seresnet50's b`--batch` shapes, bf16: the stem
   pool dfd_maxpool_ceil_fwd / _bwd (112x112x64 -> 56x56), and per stage dfd_pool_se_relu and dfd_relu_se_bwd_reduce at the
   block output (56x56x256, 28x28x512, 14x14x1024, 7x7x2048). Algorithmic HBM bytes (each tensor read or written once) over
   the time, against the H100 SXM data-sheet 3.35 TB/s.
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
from xception_time import HBM_PEAK, _time  # noqa: E402

SE_SHAPES = [(56, 256, 16), (28, 512, 32), (14, 1024, 64), (7, 2048, 128)]


def time_kernels(N, iters):
    from deepfake_detection_b200 import _lib
    st = torch.cuda.current_stream().cuda_stream
    out = []

    def rec(name, shape, ms, nbytes):
        out.append(dict(kernel=name, shape=shape, ms=round(ms, 4), bytes=nbytes,
                        hbm_pct=round(100.0 * nbytes / (ms * 1e-3) / HBM_PEAK, 1)))
        print("%-24s %-18s %.4f ms, %.1f %% of 3.35 TB/s" % (name, shape, ms, out[-1]["hbm_pct"]), flush=True)

    x = torch.rand(N, 112, 112, 64, device="cuda").to(torch.bfloat16)
    y = torch.empty(N, 56, 56, 64, device="cuda", dtype=torch.bfloat16)
    idx = torch.empty(y.shape, dtype=torch.uint8, device="cuda")
    gx = torch.empty_like(x)
    ms = _time(lambda: _lib.call("dfd_maxpool_ceil_fwd", x.data_ptr(), y.data_ptr(), idx.data_ptr(), N, 112, 112, 64, 0, st), iters)
    rec("dfd_maxpool_ceil_fwd", "%dx112x112x64" % N, ms, 2 * x.numel() + 3 * y.numel())
    ms = _time(lambda: _lib.call("dfd_maxpool_ceil_bwd", y.data_ptr(), idx.data_ptr(), gx.data_ptr(), N, 112, 112, 64, 0, st), iters)
    rec("dfd_maxpool_ceil_bwd", "%dx112x112x64" % N, ms, 2 * x.numel() + 3 * y.numel())
    del x, y, idx, gx
    for H, C, Cse in SE_SHAPES:
        HW = H * H
        y = torch.randn(N, HW, C, device="cuda").to(torch.bfloat16)
        g, out_t, gm = torch.randn_like(y), torch.randn_like(y), torch.empty_like(y)
        sc, sh = torch.rand(C, device="cuda") + 0.5, torch.randn(C, device="cuda")
        Wr, br = torch.randn(Cse, C, device="cuda") * 0.05, torch.zeros(Cse, device="cuda")
        We, be = torch.randn(C, Cse, device="cuda") * 0.1, torch.zeros(C, device="cuda")
        pooled, gate, draw, d_e, dpool = (torch.zeros(N, C, device="cuda") for _ in range(5))
        r, d_rpre = torch.zeros(N, Cse, device="cuda"), torch.zeros(N, Cse, device="cuda")
        shape = "%dx%dx%dx%d" % (N, H, H, C)
        ms = _time(lambda: _lib.call("dfd_pool_se_relu", y.data_ptr(), sc.data_ptr(), sh.data_ptr(), pooled.data_ptr(),
                                     Wr.data_ptr(), br.data_ptr(), We.data_ptr(), be.data_ptr(), gate.data_ptr(), N, HW, C, Cse,
                                     0, 0, 8, st), iters)
        rec("dfd_pool_se_relu", shape, ms, 2 * y.numel())
        ms = _time(lambda: _lib.call("dfd_relu_se_bwd_reduce", g.data_ptr(), None, y.data_ptr(), out_t.data_ptr(), sc.data_ptr(),
                                     sh.data_ptr(), gm.data_ptr(), draw.data_ptr(), pooled.data_ptr(), Wr.data_ptr(),
                                     br.data_ptr(), We.data_ptr(), be.data_ptr(), d_e.data_ptr(), r.data_ptr(), d_rpre.data_ptr(),
                                     dpool.data_ptr(), N, HW, C, Cse, 0, 0, st), iters)
        rec("dfd_relu_se_bwd_reduce", shape, ms, 8 * y.numel())
        del y, g, out_t, gm
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("senet_time.py needs a CUDA GPU")
    torch.cuda.set_device(0)
    out = dict(info=gpu_info(), dtype="bf16")
    print(json.dumps(out["info"]), flush=True)
    out["kernels"] = time_kernels(a.batch, a.iters)
    trs = {"seresnet50": _trainer("seresnet50", a.batch, 224), "resnet50": _trainer("resnet50", a.batch, 224)}
    r = time_steps(trs, a.steps, a.rounds)
    out["steps"] = {k: dict(batch=a.batch, res=224, **r[k]) for k in trs}
    for k in trs:
        print("%-10s b%d: %.3f ms/step (%.0f img/s)" % (k, a.batch, r[k]["median"], a.batch / r[k]["median"] * 1e3), flush=True)
    print(json.dumps(out))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f)


if __name__ == "__main__":
    main()
