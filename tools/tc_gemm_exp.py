"""Latency experiments on the wgmma GEMM (GLAMR_TC_DEBUG bits: 1 no MMA, 2 no split/store, 4 no epilogue, 8 no loads)."""
import ctypes, os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from glamr_b200 import lib as L
lib = L.load()
lib.glamr_linear_forward.argtypes = [ctypes.c_int] * 3 + [ctypes.c_void_p] * 3 + [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
g = torch.Generator().manual_seed(0)
for (M, N, K) in [(120, 256, 256), (120, 256, 512), (7680, 512, 256)]:
    X = torch.randn(M, K, generator=g).cuda(); W = (torch.randn(N, K, generator=g) / K ** 0.5).cuda(); b = torch.randn(N, generator=g).cuda()
    Y = torch.empty(M, N, device='cuda')
    st = torch.cuda.current_stream().cuda_stream
    for _ in range(20): lib.glamr_linear_forward(M, N, K, X.data_ptr(), W.data_ptr(), b.data_ptr(), 0, Y.data_ptr(), 1, st)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(200): lib.glamr_linear_forward(M, N, K, X.data_ptr(), W.data_ptr(), b.data_ptr(), 0, Y.data_ptr(), 1, st)
    e1.record(); torch.cuda.synchronize()
    print(f"dbg={os.environ.get('GLAMR_TC_DEBUG', '0')} M={M} N={N} K={K}: {e0.elapsed_time(e1) * 1e3 / 200:.2f} us", flush=True)
