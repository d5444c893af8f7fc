# cuBLAS / cuSOLVER FP64 ceilings on the box (context only; product path is hand-written)
import json, os, time
import torch
torch.backends.cuda.matmul.allow_tf32 = False
dev = torch.device("cuda:0")
res = {}
def ev(fn, n=3):
    fn(); torch.cuda.synchronize()
    best = 1e9
    for _ in range(n):
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    return best
for n in (4096, 8192, 16384):
    a = torch.randn(n, n, dtype=torch.float64, device=dev); b = torch.randn(n, n, dtype=torch.float64, device=dev)
    ms = ev(lambda: torch.matmul(a.t(), b))
    res[f"dgemm_tn_{n}"] = 2*n**3/ms/1e9
    print(f"cuBLAS DGEMM TN n={n}: {ms:.2f} ms {2*n**3/ms/1e9:.2f} TF/s", flush=True)
    del a, b
n = 8192
a = torch.randn(n, n, dtype=torch.float64, device=dev); b = torch.randn(n, n, dtype=torch.float64, device=dev)
t0=time.time(); k=0
e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(60): torch.matmul(a.t(), b); k+=1
e1.record(); torch.cuda.synchronize()
ms = e0.elapsed_time(e1)/k
res["dgemm_tn_8192_sustained"] = 2*n**3/ms/1e9
print(f"cuBLAS DGEMM sustained n=8192 x{k}: {2*n**3/ms/1e9:.2f} TF/s")
for n in (8192, 16384):
    x = torch.rand(n, n, dtype=torch.float64, device=dev); spd = (x + x.t())/2 + n*torch.eye(n, dtype=torch.float64, device=dev)
    ms = ev(lambda: torch.linalg.cholesky(spd, upper=True), n=2)
    res[f"cusolver_potrf_{n}"] = n**3/3/ms/1e9
    print(f"cuSOLVER potrf n={n}: {ms:.2f} ms {n**3/3/ms/1e9:.2f} TF/s (n^3/3)")
    del x, spd
json.dump(res, open(os.path.join(os.environ.get("CAPITAL_OUT_DIR", "."), "probe_cublas.json"), "w"), indent=1)
