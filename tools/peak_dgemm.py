"""Measure the cuBLAS DGEMM peak on this GPU (roofline denominator for the fp64 contraction)."""
import json, sys, torch
n = int(sys.argv[1]) if len(sys.argv) > 1 else 8192
a = torch.randn(n, n, dtype=torch.float64, device='cuda'); b = torch.randn(n, n, dtype=torch.float64, device='cuda')
for _ in range(3): c = a @ b
torch.cuda.synchronize()
best = 1e9; tot = 0.0; reps = 10
for _ in range(reps):
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record(); c = a @ b; e1.record(); torch.cuda.synchronize()
    t = e0.elapsed_time(e1); best = min(best, t); tot += t
print(json.dumps({"dgemm_n": n, "fp64_tflops_burst": 2*n**3/best*1e-9, "fp64_tflops_mean": 2*n**3/(tot/reps)*1e-9}))
