"""Cost of TF "SAME" padding: the graph-replayed train step of tf_efficientnet_b0 against efficientnet_b0 (same layers, same
BatchNorm eps 1e-3; the tf plan runs its stem im2col and the stride-2 depthwise convs of stages 1, 2, 3 and 5 through the
`_pad` kernels), batch 256, 3x224x224, bf16, SGD, alternated in one process.

    python tools/tf_same_time.py [--batch 256] [--steps 20] [--rounds 5] [--out FILE]

`--rounds` windows of `--steps` Trainer.step_resident calls each, CUDA events around every window, after 5 warm-up steps of
each trainer; medians and the difference. The GPU name, power limit and max SM clock are read in the same run. Needs a GPU.
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

ARCHS = ("efficientnet_b0", "tf_efficientnet_b0")


def _trainer(arch, batch, res):
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.models import init_state_dict
    from deepfake_detection_b200.trainer import Trainer
    tr = Trainer(arch, batch, res, res, dtype="bf16", opt="sgd", lr=1e-4, num_classes=2, bn_eps=1e-3)
    tr.load_state_dict(init_state_dict(get_spec(arch, num_classes=2), seed=42))
    g = torch.Generator(device="cuda").manual_seed(1234)
    tr.engine.set_input(torch.randn(batch, 3, res, res, device="cuda", generator=g))
    tr.engine.set_target(torch.randint(0, 2, (batch,), device="cuda", generator=g))
    return tr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tf_same_time.py needs a CUDA GPU")
    torch.cuda.set_device(0)
    trs = {arch: _trainer(arch, a.batch, 224) for arch in ARCHS}
    launches = {arch: len(tr.engine.fwd_ops) + len(tr.engine.bwd_ops) for arch, tr in trs.items()}
    for tr in trs.values():
        for _ in range(5):
            tr.step_resident()
    torch.cuda.synchronize()
    ms = {k: [] for k in trs}
    for _ in range(a.rounds):
        for k, tr in trs.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(a.steps):
                tr.step_resident()
            t1.record()
            torch.cuda.synchronize()
            ms[k].append(t0.elapsed_time(t1) / a.steps)
    med = {k: sorted(v)[len(v) // 2] for k, v in ms.items()}
    out = dict(info=gpu_info(), batch=a.batch, res=224, dtype="bf16", planned_ops=launches,
               windows_ms={k: [round(v, 3) for v in vs] for k, vs in ms.items()},
               median_ms={k: round(v, 3) for k, v in med.items()},
               tf_minus_symmetric_ms=round(med["tf_efficientnet_b0"] - med["efficientnet_b0"], 3),
               images_per_sec={k: round(a.batch / (v / 1e3), 1) for k, v in med.items()})
    print("b%d bf16 224 step: efficientnet_b0 %.3f ms, tf_efficientnet_b0 %.3f ms (%+.3f ms)" %
          (a.batch, med["efficientnet_b0"], med["tf_efficientnet_b0"], out["tf_minus_symmetric_ms"]))
    print(json.dumps(out))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f)


if __name__ == "__main__":
    main()
