"""mma.sync vs wgmma 1x1 weight gradient on the EfficientNet-B0 layer shapes (batch 256)."""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepfake_detection_b200 import _lib
def t(impl, M, Nw, Kw, reps=10):
    G = torch.randn(M, Nw, device="cuda").bfloat16(); X = torch.randn(M, Kw, device="cuda").bfloat16()
    dW = torch.zeros(Nw, Kw, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    name = impl.replace("+det", "")
    extra = ()
    det = impl.endswith("+det")
    if name == "dfd_gemm_wgrad":
        import struct
        splits = _lib.lib().cdll.dfd_gemm_wgrad_splits(M, Nw, Kw)
        ws = torch.empty(splits * Nw * Kw, device="cuda")
        extra = (ws.data_ptr(), ws.numel() * 4) if det else (None, 0)
        table = torch.frombuffer(bytearray(struct.pack("<QQqqii", ws.data_ptr(), dW.data_ptr(), Nw * Kw, Nw * Kw, splits, 0)), dtype=torch.uint8).cuda()
    def f():
        _lib.call(name, G.data_ptr(), X.data_ptr(), dW.data_ptr(), M, Nw, Kw, 0, *extra, st)
        if det:
            _lib.call("dfd_ordered_reduce", table.data_ptr(), 1, dW.data_ptr(), min(1024, (Nw * Kw // 4 + 255) // 256), st)
    for _ in range(3): f()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): f()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    ref = (G.double().t() @ X.double()) * (reps + 3)
    rel = float((dW.double() - ref).norm() / ref.norm())
    print("%-20s M=%d Nw=%d Kw=%d ms=%.3f GB/s=%.0f rel=%.1e" % (impl, M, Nw, Kw, ms, 2 * M * (Nw + Kw) / ms / 1e6, rel), flush=True)
    return ms
tot = {"dfd_gemm_wgrad_mma": 0.0, "dfd_gemm_wgrad": 0.0, "dfd_gemm_wgrad+det": 0.0}
for shp in [(3211264, 96, 16), (3211264, 32, 32), (3211264, 16, 32), (802816, 144, 24), (802816, 24, 144), (802816, 24, 96), (200704, 240, 40),
            (200704, 40, 240), (50176, 672, 112), (50176, 112, 672), (50176, 480, 80), (50176, 80, 480), (12544, 1152, 192), (12544, 192, 1152),
            (12544, 1280, 320), (12544, 320, 1152)]:
    for impl in tot:
        try: tot[impl] += t(impl, *shp)
        except Exception as e: print("FAIL", impl, shp, repr(e)[:200]); torch.cuda.synchronize()
print(tot)
