"""FC-layer GEMMs of the box / cube heads (configs/Base.yaml:67-70, cube_head.py:63-73): c3d_linear_fwd/_dgrad/_wgrad
(wgmma, our kernels) next to the cuBLAS kernels torch picks for the same bf16 GEMMs (the library bar to match)."""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from omni3d_b200 import conv as K

flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")


def timeit(fn, iters=7):
    for _ in range(2):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


out = []
for name, rows, Kd, N in [("box_fc1", 16384, 12544, 1024), ("cube_fc1", 4096, 12544, 1024), ("box_fc2", 16384, 1024, 1024),
                          ("cube_fc2", 4096, 1024, 1024), ("box_pred", 16384, 1024, 256), ("cube_pred", 4096, 1024, 768)]:
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(rows, Kd, device="cuda", generator=g).bfloat16()
    w = (torch.randn(N, Kd, device="cuda", generator=g) * 0.02).bfloat16()
    wt = w.t().contiguous()
    b = torch.zeros(N, device="cuda")
    dy = torch.randn(rows, N, device="cuda", generator=g).bfloat16()
    dw = torch.zeros(N, Kd, device="cuda")
    fl = 2.0 * rows * Kd * N
    rec = {"layer": name, "rows": rows, "K": Kd, "N": N, "gflop": fl / 1e9}
    for tag, ours, lib in (("fwd", lambda: K.linear_fwd(x, w, b, relu=True), lambda: torch.relu_(torch.nn.functional.linear(x, w, b.bfloat16()))),
                           ("dgrad", lambda: K.linear_dgrad(dy, wt), lambda: dy @ w),
                           ("wgrad", lambda: K.linear_wgrad(x, dy, dw=dw), lambda: dy.t() @ x)):
        t1, t2 = timeit(ours), timeit(lib)
        rec[tag] = {"ours_ms": t1, "ours_tflops": fl / t1 / 1e9, "cublas_ms": t2, "cublas_tflops": fl / t2 / 1e9}
    out.append(rec)
    print(json.dumps(rec), flush=True)
os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
json.dump(out, open(os.path.join(ROOT, "gpurun_out", "linear_bench.json"), "w"), indent=1)
