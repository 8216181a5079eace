"""ResNet DropBlock / drop path / dropout cost: the mask generator alone, and the whole ResNet-50 train step with and
without the three rates.

    python tools/resnet_drop_time.py [--iters 50] [--steps 20] [--rounds 3] [--out FILE]

1. dfd_drop_block_masks over the 27 DropBlock sites of ResNet-50 b256 at 224x224 (one launch, the plan's own table): CUDA
   events around `--iters` launches after a warm-up; ms per launch and the HBM rate of the uint8 masks it writes against the
   H100 SXM data-sheet 3.35 TB/s.
2. The graph-replayed Trainer step of ResNet-50, batch 256, 224x224, bf16, with (drop_rate, drop_path_rate, drop_block_rate)
   = (0.2, 0.05, 0.1) against all rates 0, alternated in one process (`--rounds` windows of `--steps` steps each).
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
RATES = dict(drop_rate=0.2, drop_path_rate=0.05, drop_block_rate=0.1)


def _trainer(rates, batch, res):
    from deepfake_detection_b200.arch import get_spec
    from deepfake_detection_b200.models import init_state_dict
    from deepfake_detection_b200.trainer import Trainer
    tr = Trainer("resnet50", batch, res, res, dtype="bf16", lr=0.00256, num_classes=2, **rates)
    tr.load_state_dict(init_state_dict(get_spec("resnet50", num_classes=2), seed=42))
    g = torch.Generator(device="cuda").manual_seed(1234)
    tr.engine.set_input(torch.randn(batch, 3, res, res, device="cuda", generator=g))
    tr.engine.set_target(torch.randint(0, 2, (batch,), device="cuda", generator=g))
    return tr


def time_generator(e, iters):
    from deepfake_detection_b200 import _lib
    st = torch.cuda.current_stream().cuda_stream
    n = len(e.drop_block_sites)

    def launch():
        _lib.call("dfd_memset_async", e.drop_block_kept.data_ptr(), 0, 8 * n, st)
        _lib.call("dfd_drop_block_masks", e._drop_block_table.data_ptr(), n, e.rng_state.data_ptr(), st)

    for _ in range(5):
        launch()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        launch()
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / iters
    nbytes = sum(m.numel() for m, _ in e.drop_block_masks.values())
    return dict(sites=n, mask_bytes=nbytes, ms_per_launch=round(ms, 4),
                hbm_pct=round(100.0 * nbytes / (ms * 1e-3) / HBM_PEAK, 1))


def time_steps(trs, steps, rounds):
    for tr in trs.values():
        for _ in range(5):
            tr.step_resident()
    torch.cuda.synchronize()
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
    med = {k: sorted(v)[len(v) // 2] for k, v in ms.items()}
    return dict(ms_per_step_off=[round(v, 3) for v in ms["off"]], ms_per_step_drop=[round(v, 3) for v in ms["drop"]],
                median_off=round(med["off"], 3), median_drop=round(med["drop"], 3),
                added_pct=round(100.0 * (med["drop"] - med["off"]) / med["off"], 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("resnet_drop_time.py needs a CUDA GPU")
    torch.cuda.set_device(0)
    trs = {"off": _trainer({}, a.batch, 224), "drop": _trainer(RATES, a.batch, 224)}
    out = dict(info=gpu_info(), rates=RATES, batch=a.batch)
    out["generator"] = time_generator(trs["drop"].engine, a.iters)
    g = out["generator"]
    print("dfd_drop_block_masks, %d sites, %.1f MB of masks: %.4f ms (%.1f %% of 3.35 TB/s)"
          % (g["sites"], g["mask_bytes"] / 1e6, g["ms_per_launch"], g["hbm_pct"]))
    out["step"] = time_steps(trs, a.steps, a.rounds)
    s = out["step"]
    print("R50 b%d bf16 224 step: rates 0 %.3f ms, rates %s %.3f ms (%+.2f %%)"
          % (a.batch, s["median_off"], tuple(RATES.values()), s["median_drop"], s["added_pct"]))
    print(json.dumps(out))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f)


if __name__ == "__main__":
    main()
