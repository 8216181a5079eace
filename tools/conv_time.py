"""3x3 stride-1 convolution on the resnet50 layer shapes (batch 256): materialised im2col + tensor-core GEMM vs the implicit GEMM
(dfd_conv_tc), forward (+statistics) and input gradient (GEMM + col2im vs implicit on dY)."""
import os, struct, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepfake_detection_b200 import _lib

N = int(os.environ.get("CT_N", 256))
st = lambda: torch.cuda.current_stream().cuda_stream
P = lambda t: t.data_ptr()


def timeit(fn, reps=10):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


for (H, C) in [(56, 64), (28, 128), (14, 256), (7, 512)]:
    x = torch.randn(N, H, H, C, device="cuda").bfloat16()
    w = (torch.randn(C, C, 3, 3, device="cuda") / (3 * C ** 0.5)).bfloat16()
    wp = torch.zeros(C * 9 * C, device="cuda", dtype=torch.bfloat16)
    wpT, wpD = torch.zeros_like(wp), torch.zeros_like(wp)
    table = torch.frombuffer(bytearray(struct.pack("<QQQQiiii", P(w), P(wp), P(wpT), P(wpD), C, C, 3, 0)), dtype=torch.uint8).cuda()
    _lib.call("dfd_repack_weights", P(table), 1, 0, st())
    M = N * H * H
    cols = torch.zeros(M, 9 * C, device="cuda", dtype=torch.bfloat16)
    y = torch.zeros(M, C, device="cuda", dtype=torch.bfloat16)
    dx = torch.zeros(M, C, device="cuda", dtype=torch.bfloat16)
    s1 = torch.zeros(_lib.lib().stat_slots, C, dtype=torch.float64, device="cuda")
    s2 = torch.zeros_like(s1)

    def fwd_old():
        _lib.call("dfd_im2col", P(x), P(cols), N, H, H, C, 3, 1, 1, 0, st())
        _lib.call("dfd_gemm_tn", P(cols), P(wp), P(y), M, C, 9 * C, 0, P(s1), P(s2), None, st())

    def fwd_new():
        _lib.call("dfd_conv_tc", P(x), P(wp), P(y), N, H, H, C, C, 3, 1, 0, P(s1), P(s2), None, st())

    def dg_old():
        _lib.call("dfd_gemm_tn", P(y), P(wpT), P(cols), M, 9 * C, C, 0, None, None, None, st())
        _lib.call("dfd_col2im", P(cols), None, P(dx), N, H, H, C, 3, 1, 1, 0, st())

    def dg_new():
        _lib.call("dfd_conv_tc", P(y), P(wpD), P(dx), N, H, H, C, C, 3, 1, 0, None, None, None, st())

    gperm = torch.zeros(C, 9 * C, device="cuda")
    sp_o = _lib.lib().cdll.dfd_gemm_wgrad_splits(M, C, 9 * C)
    sp_n = _lib.lib().cdll.dfd_conv_wgrad_splits(N, H, H, C, C, 3, 1)
    ws = torch.zeros(max(sp_o, sp_n) * C * 9 * C, device="cuda")

    def wg_old():
        _lib.call("dfd_im2col", P(x), P(cols), N, H, H, C, 3, 1, 1, 0, st())
        _lib.call("dfd_gemm_wgrad", P(y), P(cols), P(gperm), M, C, 9 * C, 0, P(ws), ws.numel() * 4, st())

    def wg_new():
        _lib.call("dfd_conv_wgrad_tc", P(y), P(x), P(gperm), N, H, H, C, C, 3, 1, 0, P(ws), ws.numel() * 4, st())

    a, b, c, d = timeit(fwd_old), timeit(fwd_new), timeit(dg_old), timeit(dg_new)
    e_, f_ = timeit(wg_old), timeit(wg_new)
    print("H=%d C=%d  wgrad im2col+gemm %.3f ms (splits %d)  implicit %.3f ms (splits %d, %.0f TFLOP/s)"
          % (H, C, e_, sp_o, f_, sp_n, 2.0 * M * C * 9 * C / f_ / 1e9), flush=True)
    fl = 2.0 * M * C * 9 * C
    print("H=%d C=%d  fwd im2col+gemm %.3f ms  implicit %.3f ms (%.0f TFLOP/s)   dgrad gemm+col2im %.3f ms  implicit %.3f ms (%.0f TFLOP/s)"
          % (H, C, a, b, fl / b / 1e9, c, d, fl / d / 1e9), flush=True)
