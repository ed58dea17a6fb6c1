"""Fixed cost of one wgmma GEMM launch (tiny shapes) and of the narrow strip-convolution tiles."""
import sys, os, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rainbow_iqn_apex_b200._lib import call, ptr
dev = torch.device("cuda")
def bf(*s): return torch.randn(*s, device=dev).to(torch.bfloat16)
def run(M, N, K, reps=50):
    a, b = bf(M, K), bf(N, K)
    c = torch.zeros(M, N, device=dev)
    go = lambda: call("riqn_gemm_bf16_tc", M, N, K, ptr(a), None, ptr(b), None, ptr(c), N, 0, None, None, None, 1, None, None, 0)
    for _ in range(5): go()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        go()
        torch.cuda.synchronize()
        with torch.cuda.graph(g):
            for _ in range(reps): go()
    torch.cuda.synchronize()
    g.replay(); torch.cuda.synchronize()
    e0.record(); g.replay(); e1.record(); torch.cuda.synchronize()
    print(f"M={M} N={N} K={K}: {e0.elapsed_time(e1) * 1e3 / reps:7.2f} us per launch (graph of {reps})")
run(128, 64, 64); run(128, 256, 64); run(128 * 132, 256, 64); run(128 * 132, 256, 512); run(128 * 132 * 3, 64, 512); run(41472, 64, 576)
