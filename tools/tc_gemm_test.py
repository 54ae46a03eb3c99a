"""wgmma 3xTF32 GEMM vs fp64 torch and vs the FP32 SIMT kernel."""
import ctypes, os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from glamr_b200 import lib as L
lib = L.load()
lib.glamr_linear_forward.argtypes = [ctypes.c_int] * 3 + [ctypes.c_void_p] * 3 + [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
g = torch.Generator().manual_seed(0)
for (M, N, K, relu) in [(50, 256, 69, 0), (128, 128, 32, 0), (3200, 768, 256, 0), (100, 69, 256, 0), (1500, 512, 384, 1), (64, 11, 256, 0), (7, 5, 3, 1)]:
    X = torch.randn(M, K, generator=g).cuda(); W = (torch.randn(N, K, generator=g) / K ** 0.5).cuda(); b = torch.randn(N, generator=g).cuda()
    ref = X.double() @ W.double().T + b.double()
    if relu: ref = ref.clamp_min(0)
    out = {}
    for mode in (1, 0):
        Y = torch.full((M, N), float('nan'), device='cuda')
        rc = lib.glamr_linear_forward(M, N, K, X.data_ptr(), W.data_ptr(), b.data_ptr(), relu, Y.data_ptr(), mode, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        out[mode] = (rc, float((Y.double() - ref).abs().max()))
    print(f'M={M} N={N} K={K} relu={relu}: wgmma rc/err {out[1]}  simt rc/err {out[0]}  ref scale {float(ref.abs().max()):.2f}', flush=True)

# latency of the shapes the prior networks launch at B = 1 (one 120-frame window): back-to-back launches on one stream
for (M, N, K) in [(120, 256, 256), (120, 512, 256), (120, 256, 512), (300, 512, 256), (7680, 256, 256), (7680, 512, 256)]:
    X = torch.randn(M, K, generator=g).cuda(); W = (torch.randn(N, K, generator=g) / K ** 0.5).cuda(); b = torch.randn(N, generator=g).cuda()
    Y = torch.empty(M, N, device='cuda')
    line = f'M={M} N={N} K={K}:'
    for mode in (1, 0):
        st = torch.cuda.current_stream().cuda_stream
        for _ in range(20): lib.glamr_linear_forward(M, N, K, X.data_ptr(), W.data_ptr(), b.data_ptr(), 0, Y.data_ptr(), mode, st)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(200): lib.glamr_linear_forward(M, N, K, X.data_ptr(), W.data_ptr(), b.data_ptr(), 0, Y.data_ptr(), mode, st)
        e1.record(); torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / 200
        line += f"  {'wgmma' if mode else 'simt'} {us:.2f} us ({2.0 * M * N * K / us * 1e-6:.2f} TFLOP/s)"
    print(line, flush=True)
