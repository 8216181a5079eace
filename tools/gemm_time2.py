"""Diagnostics: plain vs row-packed tensor-core GEMM on the small-K shapes of EfficientNet-B0 (batch 256)."""
import os, sys, struct, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepfake_detection_b200 import _lib
def t(M, N, K, pack, stats=True, reps=20):
    A = torch.randn(M, K, device='cuda').bfloat16(); B = torch.randn(N, K, device='cuda').bfloat16()
    C = torch.empty(M, N, device='cuda', dtype=torch.bfloat16)
    s1 = torch.zeros(8, N, dtype=torch.float64, device='cuda'); s2 = torch.zeros_like(s1)
    st = torch.cuda.current_stream().cuda_stream
    sp = (s1.data_ptr(), s2.data_ptr()) if stats else (None, None)
    if pack > 1:
        Bd = torch.empty(pack * N, pack * K, device='cuda', dtype=torch.bfloat16)
        tb = torch.frombuffer(bytearray(struct.pack("<QQiiii", B.data_ptr(), Bd.data_ptr(), N, K, pack, 0)), dtype=torch.uint8).cuda()
        _lib.call("dfd_blockdiag_weights", tb.data_ptr(), 1, 0, st)
        f = lambda: _lib.call("dfd_gemm_tn_rowpack", A.data_ptr(), Bd.data_ptr(), C.data_ptr(), M, N, K, pack, 0, *sp, None, st)
    else:
        f = lambda: _lib.call("dfd_gemm_tn", A.data_ptr(), B.data_ptr(), C.data_ptr(), M, N, K, 0, *sp, None, st)
    for _ in range(3): f()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): f()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    print("M=%d N=%d K=%d pack=%d stats=%s ms=%.3f GB/s=%.0f" % (M, N, K, pack, stats, ms, 2 * (M * K + M * N) / ms / 1e6))
for (M, N, K, packs) in [(802816, 144, 24, (2, 4, 8)), (802816, 96, 24, (2, 4, 8)), (802816, 24, 144, (1,)), (3211264, 96, 16, (4, 8)),
                         (3211264, 32, 32, (2, 4)), (200704, 240, 40, (1, 2, 4, 8)), (200704, 144, 40, (1, 2, 4, 8)),
                         (50176, 480, 80, (1, 2, 4)), (50176, 672, 112, (1, 2, 4)), (12544, 1152, 192, (1, 2))]:
    for pack in packs:
        t(M, N, K, pack)
