"""Runs every GPU parity check without stopping at the first failure and writes gpurun_out/diag.json + .txt.
Development aid for the (expensive) GPU round trips; the same checks are asserted by tests/test_*_gpu.py.

    python tools/gpu_diag.py [--skip-tc] [--only kernels|engine|tc]
"""
import argparse
import json
import os
import sys
import time
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="")
    ap.add_argument("--gemm", default="tc")
    ap.add_argument("--out", default=os.path.join(ROOT, "gpurun_out", "diag"))
    a = ap.parse_args()
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    import engine_checks as EC
    import gpu_checks as GC
    results = {}

    def run(name, fn, *args, **kw):
        t0 = time.time()
        try:
            r = fn(*args, **kw)
            torch.cuda.synchronize()
            results[name] = dict(ok=True, result=r, sec=round(time.time() - t0, 2))
        except Exception as e:  # noqa: BLE001
            results[name] = dict(ok=False, error=repr(e), tb=traceback.format_exc()[-1500:])
            try:
                torch.cuda.synchronize()
            except Exception as e2:  # noqa: BLE001
                results[name]["sync_error"] = repr(e2)
        print(name, json.dumps(results[name], default=str)[:600], flush=True)
        with open(a.out + ".json", "w") as f:
            json.dump(results, f, indent=1, default=str)

    only = set(a.only.split(",")) if a.only else set()

    def want(g):
        return not only or g in only or ("kernels" in only and g in ("mma", "wgrad", "dwconv", "stem", "bn", "small"))

    if want("tc"):
        for M, K, N in [(1000, 16, 96), (4096 + 37, 24, 144), (777, 1152, 320), (5000, 320, 1280), (130, 40, 24),
                        (50176, 80, 480), (300, 64, 64), (128, 64, 16), (256 * 49, 672, 192)]:
            run("gemm_tc_%d_%d_%d" % (M, K, N), GC.check_gemm, "tc", M, K, N)
        run("gemm_tc_fp16", GC.check_gemm, "tc", 3000, 144, 40, dtype=torch.float16)
    if want("mma"):
        for M, K, N in [(1000, 16, 96), (4096 + 37, 24, 144), (777, 1152, 320), (5000, 320, 1280), (130, 40, 24)]:
            run("gemm_mma_%d_%d_%d" % (M, K, N), GC.check_gemm, "mma", M, K, N, with_add=(N == 24))
    if want("wgrad"):
        for M, Nw, Kw in [(5000, 96, 16), (12345, 144, 24), (3000, 1152, 192), (777, 320, 1280), (64, 24, 144)]:
            run("wgrad_%d_%d_%d" % (M, Nw, Kw), GC.check_wgrad, M, Nw, Kw)
    if want("dwconv"):
        for (N, H, W, C, k, s, aff) in [(2, 16, 16, 32, 3, 1, True), (2, 17, 19, 96, 3, 2, True), (2, 14, 14, 144, 5, 1, True),
                                        (2, 15, 15, 240, 5, 2, True), (3, 7, 7, 1152, 5, 1, True), (2, 40, 40, 32, 3, 1, False),
                                        (1, 33, 33, 24, 3, 1, False), (2, 56, 56, 144, 5, 2, True)]:
            run("dwconv_%d_%d_%d_%d_k%d_s%d_%s" % (N, H, W, C, k, s, aff), GC.check_dwconv, N, H, W, C, k, s, affine=aff)
        run("dwconv_fp16", GC.check_dwconv, 2, 14, 14, 80, 3, 1, dtype=torch.float16)
    if want("stem"):
        run("stem_3", GC.check_stem_gemm, 2, 3, 32, 32, 32, 3, 2, 1)
        run("stem_3_odd", GC.check_stem_gemm, 2, 3, 38, 38, 48, 3, 2, 1)
        run("stem_12", GC.check_stem_gemm, 1, 12, 20, 20, 256, 3, 2, 1)
        run("stem_7", GC.check_stem_gemm, 2, 3, 32, 32, 64, 7, 2, 3)
    if want("bn"):
        for (N, HW, C) in [(3, 64, 32), (2, 49, 1152), (4, 200, 144), (2, 1000, 16)]:
            run("bn_chain_%d_%d_%d" % (N, HW, C), GC.check_bn_chain, N, HW, C)
        run("bn_chain_fp16", GC.check_bn_chain, 2, 100, 40, dtype=torch.float16)
    if want("small"):
        run("se_fc", GC.check_se_fc, 5, 144, 6)
        run("se_fc_big", GC.check_se_fc, 3, 1152, 48)
        run("head_hard", GC.check_head, 16, 1280)
        run("head_ls", GC.check_head, 16, 1280, smoothing=0.1)
        run("head_soft", GC.check_head, 16, 512, soft=True)
        for k in ("sgd", "adam", "adamw", "rmsproptf"):
            run("opt_" + k, GC.check_optimizer, k)
        run("transpose", GC.check_transpose)
    if want("resnet"):
        run("conv_dense_3x3", GC.check_conv_dense, 2, 14, 14, 64, 64, 3, 1)
        run("conv_dense_3x3_s2", GC.check_conv_dense, 2, 15, 17, 64, 128, 3, 2)
        run("conv_dense_1x1_s2", GC.check_conv_dense, 2, 12, 12, 64, 256, 1, 2)
        run("maxpool", GC.check_maxpool_relu_pool, 2, 16, 16, 64)
        run("maxpool_odd", GC.check_maxpool_relu_pool, 3, 15, 13, 64)
        run("engine_r18_fp16", EC.run_parity, "resnet18", 8, 96, 96, dtype="fp16", gemm_impl=a.gemm, verbose=True, tame=True, steps=1)
        run("engine_r50_fp16", EC.run_parity, "resnet50", 8, 96, 96, dtype="fp16", gemm_impl=a.gemm, tame=True, steps=1)
        run("engine_r18_bf16", EC.run_parity, "resnet18", 8, 96, 96, dtype="bf16", gemm_impl=a.gemm, tame=True, steps=1)
    if want("engine"):
        run("engine_b0_fp16_%s" % a.gemm, EC.run_parity, "efficientnet_b0", 16, 96, 96, dtype="fp16", gemm_impl=a.gemm, verbose=True)
        run("engine_b0_bf16_%s" % a.gemm, EC.run_parity, "efficientnet_b0", 16, 96, 96, dtype="bf16", gemm_impl=a.gemm)
        run("engine_b4_fp16_%s" % a.gemm, EC.run_parity, "efficientnet_b4", 4, 76, 76, dtype="fp16", gemm_impl=a.gemm)
    ok = sum(1 for v in results.values() if v["ok"])
    print("DIAG DONE: %d/%d checks ran without exception" % (ok, len(results)))


if __name__ == "__main__":
    main()
